"""Time the streaming DDC/NFM bank (DdcBank.process) at several decimations: config 4's shape -- 128 channels of one 2^21-sample wideband block,
shift | fir_decimate_cc D | fmdemod_quadri_cf -- with T = firdes_filter_len(0.25 / D) taps, so every geometry has M = ceil(T / D) = 16 or 17 tap
blocks and the same FP32 work per channel-sample.  D = 50 runs ddc_bank_fused2_kernel<50, 17>, the others ddc_bank_generic_kernel (D = 48 and
52 are config 4's work on the generic kernel).

Prints one JSON line per geometry: card and power limit (read in the same run), ms per block (CUDA events, after warm-up, over >= 1 s), wideband
Msamples/s, and FP32 TFLOP/s from C * N * (10 + 4M) with its fraction of the H100 SXM data-sheet 67 TFLOP/s.

usage: python tools/bench_ddc_geometries.py [--decimations 50,48,52,40,12,100,200,400] [--seconds 1.0]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import csdr_b200 as cb  # noqa: E402

C, N, FP32_PEAK = 128, 1 << 21, 67e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    name, power, clock = ([s.strip() for s in q.stdout.strip().split(",")] + ["?", "?", "?"])[:3]
    return {"card": name or torch.cuda.get_device_name(), "power_limit": power, "max_sm_clock": clock}


def measure(D, seconds, info):
    T = cb.firdes_filter_len(0.25 / D)
    taps = cb.firdes_lowpass_f(T, 0.5 / D)
    M = -(-T // D)
    n_out = cb.fir_out_len(N, D, T)
    gen = torch.Generator(device="cuda").manual_seed(4)
    wide = torch.view_as_complex(torch.rand((N, 2), generator=gen, device="cuda") * 2 - 1)
    bank = cb.DdcBank(np.linspace(-0.45, 0.45, C).astype(np.float32), D, taps, demod=True, chunk=1024)
    out = torch.empty((C, n_out + (n_out & 1)), dtype=torch.float32, device="cuda")
    try:
        for _ in range(5):
            bank.process(wide, out)                                 # every block presents N samples, as bench.py's config 4 leg does
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); bank.process(wide, out); b.record(); b.synchronize()
        reps = max(20, int(seconds * 1e3 / max(a.elapsed_time(b), 1e-3)))
        a.record()
        for _ in range(reps):
            bank.process(wide, out)
        b.record(); b.synchronize()
        ms = a.elapsed_time(b) / reps
    finally:
        bank.close()
    flops = C * N * (10.0 + 4.0 * M)
    kernel = "fused2" if (D == 50 and T <= 850) or (D == 10 and T <= 200) else "generic"
    return dict(info, decimation=D, taps=T, M=M, kernel=kernel, channels=C, block_samples=N, reps=reps, ms_per_block=round(ms, 4),
                wideband_msps=round(N / ms / 1e3, 1), fp32_tflops=round(flops / ms / 1e9, 2), fp32_fraction_of_67=round(flops / ms / 1e9 / 67.0, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--decimations", default="50,48,52,40,12,100,200,400")
    ap.add_argument("--seconds", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = card()
    for D in (int(d) for d in args.decimations.split(",")):
        print(json.dumps(measure(D, args.seconds, info)), flush=True)


if __name__ == "__main__":
    main()
