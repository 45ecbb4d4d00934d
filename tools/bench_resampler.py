"""Time the rational_resampler_ff bank on cuda:0 and print one JSON line: 1024 channels x one second at 64 kHz (64000 samples per row) resampled
by 3/4 (79 taps, what the CLI's default bandwidth 0.05 gives) and by 24/25 (1001 taps).  Per case: kernel milliseconds (CUDA events over 50
calls after warm-up; the call's stream-ordered tap upload is inside the window), input Msamples/s, the algorithmic bytes (4 B in and 4*I/D B out
per input sample) over kernel time, and that as a share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The card's name and power limit
are read in the same run."""
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

HBM_PEAK = 3.35e12
CHANNELS, N = 1024, 64_000
CASES = (("3_4", 3, 4, 79), ("24_25", 24, 25, 1001))                # name, I, D, taps


def power_limit_w():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def time_ms(fn, reps=50, warm=5):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record(); b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    import torch
    import csdr_b200
    if not torch.cuda.is_available():
        raise SystemExit("bench_resampler needs a CUDA device")
    torch.cuda.set_device(0)
    res = {"metric": "rational_resampler_bank", "channels": CHANNELS, "samples_per_channel": N, "device": torch.cuda.get_device_name(0),
           "power_limit_w": power_limit_w()}
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((CHANNELS, N), dtype=torch.float32, device="cuda", generator=g)
    for name, I, D, T in CASES:
        taps = csdr_b200.rational_resampler_get_lowpass_f(T, I, D)
        out = torch.empty((CHANNELS, N * I // D), dtype=torch.float32, device="cuda")
        y, st = csdr_b200.rational_resampler_bank_ff(x, I, D, taps, out=out)
        ms = time_ms(lambda: csdr_b200.rational_resampler_bank_ff(x, I, D, taps, out=out))
        n_out = st[1]
        nbytes = 4.0 * CHANNELS * (N + n_out)
        res[f"r{name}"] = {"taps": T, "outputs_per_channel": n_out, "kernel_ms": round(ms, 4),
                           "msamples_per_s_in": round(CHANNELS * N / (ms * 1e-3) / 1e6, 1),
                           "algorithmic_gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
                           "share_of_hbm_peak": round(nbytes / (ms * 1e-3) / HBM_PEAK, 4)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
