"""GPU time of the four-step transform csdrb_fft_c2c_large_batch (2^15, 2^16, 2^18, 2^20 points) beside the single-CTA csdrb_fft_c2c_batch at
2^14 for scale, and of the fastddc chain with a long filter (fastddc_init(0.0005, 256): 65536-point forward blocks, 64 channels through the
inverse plan).  Every timed size is first checked against numpy's float64 FFT.  CUDA events around repeated calls after a warm-up, at least
0.5 s per measurement, three measurements each (median and the spread between the fastest and slowest).  Prints one JSON line with the card name
and power limit read in the same run.  `algorithmic_hbm_share` is 16 bytes per point (read once, write once) over the time per transform as a
share of 3.35 TB/s; the four-step transform moves every point through memory twice, so half of that figure is its ceiling."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import csdr_b200 as cb  # noqa: E402

HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn, min_s=0.5, runs=3):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    out = []
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(runs):
        reps, total = 0, 0.0
        while total < min_s * 1e3:
            t0.record()
            for _ in range(4):
                fn()
            t1.record()
            torch.cuda.synchronize()
            total += t0.elapsed_time(t1); reps += 4
        out.append(total / reps)
    return sorted(out)


def rel_rms(a, b):
    return float(np.sqrt(np.sum(np.abs(a - b) ** 2) / np.sum(np.abs(b) ** 2)))


def transform(lg):
    n = 1 << lg
    batch = max(4, (1 << 26) // n)                                       # 2^26 points = 512 MiB in, 512 MiB out per call
    x = torch.randn((batch, n), dtype=torch.complex64, device="cuda") * 0.3
    y = cb.fft_c2c(x[:2])
    err = rel_rms(y.cpu().numpy(), np.fft.fft(x[:2].cpu().numpy().astype(np.complex128), axis=1))
    assert err < 1e-6, (lg, err)
    ms = timed(lambda: cb.fft_c2c(x))
    per = ms[1] / batch
    return {"n": n, "batch": batch, "rel_rms_vs_float64": err, "us_per_transform": round(per * 1e3, 3), "call_ms_min_median_max": [round(m, 4) for m in ms],
            "algorithmic_hbm_share": round(16.0 * n / (per * 1e-3) / HBM, 4)}


def fastddc(bw=0.0005, dec=256, channels=64, nblocks=16):
    ddc = cb.fastddc_init(bw, dec, 0.0)
    x = torch.randn(nblocks * ddc.input_size, dtype=torch.complex64, device="cuda") * 0.3
    shifts = [float(s) for s in np.linspace(-0.45, 0.45, channels)]
    sp, _ = cb.fastddc_fwd_cc(x, ddc)
    pad = torch.cat([torch.zeros(ddc.overlap_length, dtype=torch.complex64, device="cuda"), x]).cpu().numpy().astype(np.complex128)
    want = np.stack([np.fft.fft(pad[b * ddc.input_size:b * ddc.input_size + ddc.fft_size]) for b in range(2)])
    err = rel_rms(sp[:2].cpu().numpy(), want)
    assert err < 1e-6, err
    plan = cb.FastddcInvPlan(shifts, dec, bw, nblocks)
    overlap = torch.zeros(ddc.overlap_length, dtype=torch.complex64, device="cuda")
    _, counts = plan.run(sp)

    def run():
        s, _ = cb.fastddc_fwd_cc(x, ddc, overlap)
        plan.run(s)

    def run_fwd():
        cb.fastddc_fwd_cc(x, ddc)

    ms, ms_fwd = timed(run), timed(run_fwd)
    torch.cuda.synchronize()
    per_channel = int(counts[0])
    plan.close()
    return {"transition_bw": bw, "decimation": dec, "channels": channels, "fft_size": ddc.fft_size, "fft_inv_size": ddc.fft_inv_size, "taps_length": ddc.taps_length,
            "blocks_per_call": nblocks, "forward_rel_rms_vs_float64": err, "outputs_per_channel_per_call": per_channel,
            "forward_ms_min_median_max": [round(m, 4) for m in ms_fwd], "chain_ms_min_median_max": [round(m, 4) for m in ms],
            "forward_msamples_per_s": round(x.numel() / ms_fwd[1] / 1e3, 1), "chain_wideband_msamples_per_s": round(x.numel() / ms[1] / 1e3, 1)}


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {"device": card(), "hbm_peak_bytes_per_s": HBM, "transforms": [transform(lg) for lg in (14, 15, 16, 18, 20)], "fastddc": fastddc()}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
