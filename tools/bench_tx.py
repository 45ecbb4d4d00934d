"""Times the transmit banks on one GPU and prints one JSON line: fir_interpolate_bank (1024 channels, 48 kHz -> 2.4 Msps at I = 50, and 256 channels
at I = 256) and fmmod_bank (1024 channels).  CUDA events around `--iters` launches after a warm-up; the card's name and power limit go with the
numbers.  FP32 work is counted as the multiplies and adds the sums need (4 per tap term)."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import csdr_b200 as cb  # noqa: E402


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tx needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu}
    rng = np.random.default_rng(0)
    for ch, I, T, n in ((1024, 50, 8 * 50 + 1, 48000), (256, 256, 8 * 256 + 1, 48000)):
        x = torch.from_numpy((rng.standard_normal((ch, n)) + 1j * rng.standard_normal((ch, n))).astype(np.complex64)).cuda()
        taps = torch.from_numpy(cb.firdes_lowpass_f(T, 0.5 / I)).cuda()
        ms = timed(lambda: cb.fir_interpolate_bank(x, I, taps), args.iters)
        outs = ch * (n - (T - 1 + I - 1) // I) * I
        flops = 4.0 * ch * (n - (T - 1 + I - 1) // I) * (T - 1)
        res[f"interp_{ch}ch_I{I}_T{T}"] = {"ms": round(ms, 4), "Msamples_out_per_s": round(outs / ms / 1e3, 1), "fp32_TFLOPs": round(flops / ms / 1e9, 2)}
    ch, n = 1024, 48000
    x = torch.from_numpy(rng.uniform(-1, 1, (ch, n)).astype(np.float32)).cuda()
    ph = torch.zeros(ch, dtype=torch.float32, device="cuda")
    ms = timed(lambda: cb.fmmod_bank(x, ph), args.iters)
    res[f"fmmod_{ch}ch"] = {"ms": round(ms, 4), "Msamples_per_s": round(ch * n / ms / 1e3, 1)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
