"""Times the demodulator banks on the GPU.

1. fmdemod_atan_cf, fmdemod_quadri_novect_cf, amdemod_estimator_cf and dcblock_ff at 1024 channels x 480 000 samples, CUDA events after a
   warm-up, each timed over at least 0.5 s.  Reports algorithmic bytes per second (12 B per sample for the three cf32 -> f32 banks, 8 B for
   dcblock) and their share of the H100's 3.35 TB/s HBM3.  For the atan bank it also sets the time against two floors: HBM (12 B per sample)
   and FP64 issue (the FP64 instructions of one inlined double atan2, counted in the kernel's SASS with cuobjdump when it is on the PATH, at
   64 per SM per clock), and reports the larger floor and the share of it the bank reaches.
2. The whole-band WFM geometry of csdr-bankd (20 Msps, --decimation 80 --bw 0.004, 100 channels): the fused DDC bank giving the complex baseband
   (as it does under --fm-demod atan) and the atan bank on its output, each per second of input -- the cost that --fm-demod atan adds.
Prints one JSON line with the card's name and power limit, read in the same run."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import csdr_b200 as cb  # noqa: E402

CH, N, HBM, MIN_SECONDS = 1024, 480_000, 3.35e12, 0.5
FP64_PER_SM_CLK = 64                       # H100 SXM: 64 FP64 lanes per SM per clock (half the FP32 rate)


def timed(fn):
    """seconds per call: two warm-up calls, then enough calls for at least MIN_SECONDS"""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 2
    while True:
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        t = a.elapsed_time(b) / 1e3
        if t >= MIN_SECONDS:
            return t / reps
        reps *= 2


def fp64_per_sample():
    """FP64 instructions of one atan2 in the kernel's SASS, or None.  The kernel inlines atan2 once per call site (the four samples of the
    vector path, the four of the scalar path, the tile's extra sample), each copy with one DSETP.MAX; one sample runs one copy."""
    tool = shutil.which("cuobjdump") or ("/usr/local/cuda/bin/cuobjdump" if os.path.exists("/usr/local/cuda/bin/cuobjdump") else None)
    if not tool:
        return None
    so = Path(cb.__file__).parent / "libcsdr_b200.so"
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([tool, "-sass", str(so)], capture_output=True, text=True, cwd=tmp)
    funcs = [f for f in r.stdout.split("Function : ")[1:] if f.startswith("_ZN5csdrb24fmdemod_atan_bank_kernel")]
    if r.returncode != 0 or not funcs:
        return None
    ops = re.findall(r"^\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", funcs[0], re.M)
    fp64 = sum(1 for o in ops if o.startswith(("DFMA", "DADD", "DMUL", "DSETP", "DMNMX")))
    copies = sum(1 for o in ops if o.startswith("DSETP.MAX"))
    return fp64 / copies if fp64 and copies else None    # includes the shared division slow path once: slightly above the issued work


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    props = torch.cuda.get_device_properties(0)
    res = {"gpu": q.splitlines()[0] if q else torch.cuda.get_device_name(), "channels": CH, "samples": N, "banks": {}}
    L = cb.lib()
    x = (torch.randn((CH, N), dtype=torch.complex64, device="cuda") * 0.5)
    r = torch.randn((CH, N), device="cuda")
    y = torch.empty((CH, N), device="cuda")
    yq = torch.empty((CH, N + (N & 1)), device="cuda")
    ph = [torch.zeros(CH, device="cuda"), torch.zeros(CH, device="cuda")]
    st = torch.zeros((CH, 2), device="cuda")
    s = cb._stream()

    def record(name, fn, bytes_per_sample):
        t = timed(fn)
        res["banks"][name] = {"ms": round(t * 1e3, 3), "GBps": round(CH * N * bytes_per_sample / t / 1e9, 1),
                              "share_of_hbm": round(CH * N * bytes_per_sample / t / HBM, 3)}
        return t

    t_atan = record("fmdemod_atan", lambda: L.csdrb_fmdemod_atan_bank_cf(x.data_ptr(), N, y.data_ptr(), N, CH, N, ph[0].data_ptr(), ph[1].data_ptr(), s), 12)
    record("fmdemod_quadri_novect", lambda: L.csdrb_fmdemod_quadri_novect_bank_cf(x.data_ptr(), N, yq.data_ptr(), yq.stride(0), CH, N, None, None, s), 12)
    record("amdemod_estimator", lambda: L.csdrb_amdemod_estimator_bank_cf(x.data_ptr(), N, y.data_ptr(), N, CH, N, 0.0, 0.0, s), 12)
    record("dcblock", lambda: L.csdrb_dcblock_bank_ff(r.data_ptr(), N, y.data_ptr(), N, CH, N, 0.0, st.data_ptr(), s), 8)

    # the atan bank against its floors: HBM (12 B per sample at 3.35 TB/s) and FP64 issue (instructions per sample at 64 per SM per clock)
    per = fp64_per_sample()
    clock = None
    try:
        clock = float(q.split(",")[2].strip().split()[0]) * 1e6
    except (IndexError, ValueError):
        pass
    hbm_floor = CH * N * 12 / HBM
    bound = {"hbm_floor_ms": round(hbm_floor * 1e3, 3), "fp64_per_sample": per}
    if per and clock:
        fp64_floor = CH * N * per / (FP64_PER_SM_CLK * props.multi_processor_count * clock)
        bound["fp64_floor_ms"] = round(fp64_floor * 1e3, 3)
        bound["larger_floor"] = "fp64" if fp64_floor > hbm_floor else "hbm"
        bound["share_of_larger_floor"] = round(max(fp64_floor, hbm_floor) / t_atan, 3)
    else:
        bound["fp64_floor_ms"] = "not measured"
    res["atan_bound"] = bound

    # the whole-band WFM geometry: the fused DDC bank (complex baseband) and the atan bank, per second of input
    fs, D, bw, C100 = 20_000_000, 80, 0.004, 100
    T = cb.firdes_filter_len(bw)
    taps = cb.firdes_lowpass_f(T, 0.5 / D)
    rates = np.linspace(-0.45, 0.45, C100).astype(np.float32)
    bank = L.csdrb_ddc_bank_create(C100, rates.ctypes.data_as(C.POINTER(C.c_float)), D, taps.ctypes.data_as(C.POINTER(C.c_float)), T, 0, 1024)
    assert bank, L.csdrb_last_error()
    block = 1 << 18
    n_out = (block - T) // D + 1
    pitch = (n_out + 3) & ~3
    wide = (torch.randn(block, dtype=torch.complex64, device="cuda") * 0.3)
    bb = torch.empty((C100, pitch), dtype=torch.complex64, device="cuda")
    disc = torch.empty((C100, pitch), device="cuda")
    blocks_per_s = fs / (n_out * D)                                    # every call after the first consumes n_out * D new samples

    def ddc():
        assert L.csdrb_ddc_bank_process(bank, wide.data_ptr(), block, bb.data_ptr(), pitch, s) == n_out

    t_ddc = timed(ddc)
    t_at = timed(lambda: L.csdrb_fmdemod_atan_bank_cf(bb.data_ptr(), pitch, disc.data_ptr(), pitch, C100, n_out, ph[0].data_ptr(), ph[1].data_ptr(), s))
    L.csdrb_ddc_bank_destroy(bank)
    res["wfm_whole_band"] = {"wideband_sps": fs, "decimation": D, "taps": T, "channels": C100, "block": block,
                             "ddc_ms_per_s_of_input": round(t_ddc * blocks_per_s * 1e3, 3),
                             "atan_ms_per_s_of_input": round(t_at * blocks_per_s * 1e3, 3),
                             "atan_share_of_ddc": round(t_at / t_ddc, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
