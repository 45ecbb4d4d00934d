"""GPU time of the tone filter banks (csdr_b200/csrc/tone.cu): bfsk_demod_cf and apply_fir_cc (peaks_fir_cc's kernel) for 128 and 1024
channels x 1 s of 2 kHz baseband, at L = 44 (one bit of 45.45 Bd RTTY) and L = 255.  Each row holds 2000 new samples behind the L - 1 carried
ones, as csdr-bankd feeds the bank, and gives 2000 outputs.  CUDA events around 200 launches after warm-up.  FP32 work counted from the
algorithm: 16 L flop per bfsk output (two complex multiply-adds of 8 flop per tap), 8 L per apply_fir_cc output; the squares at the end are
left out.  Prints one JSON line with the kernel times, Msamples/s, achieved flop/s and the card's name and power limit read in this run."""
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import csdr_b200 as cb  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    name, limit = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return name, limit


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    L_ = cb.lib()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rate, warm, reps = 2000, 5, 200
    rng = np.random.default_rng(0)
    results = []
    for ch in (128, 1024):
        for L in (44, 255):
            n = rate + L - 1
            x = torch.from_numpy(((rng.standard_normal((ch, n)) + 1j * rng.standard_normal((ch, n))) * 0.3).astype(np.complex64)).cuda()
            mark = torch.from_numpy(cb.firdes_peak_c(0.0425, L)).cuda()
            space = torch.from_numpy(cb.firdes_peak_c(-0.0425, L)).cuda()
            yf = torch.empty((ch, rate), dtype=torch.float32, device="cuda")
            yc = torch.empty((ch, rate), dtype=torch.complex64, device="cuda")
            calls = {
                "bfsk_demod_cf": (lambda: L_.csdrb_bfsk_demod_bank_cf(x.data_ptr(), n, yf.data_ptr(), rate, ch, n, mark.data_ptr(), space.data_ptr(),
                                                                      L, stream), 16 * L),
                "peaks_fir_cc": (lambda: L_.csdrb_apply_fir_bank_cc(x.data_ptr(), n, yc.data_ptr(), rate, ch, n, mark.data_ptr(), L, stream), 8 * L),
            }
            for name, (call, flop) in calls.items():
                for _ in range(warm):
                    assert call() == rate
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(reps):
                    call()
                t1.record()
                torch.cuda.synchronize()
                ms = t0.elapsed_time(t1) / reps
                outs = ch * rate
                results.append({"kernel": name, "channels": ch, "taps": L, "kernel_ms": round(ms, 4), "msamples_per_s": round(outs / ms / 1e3, 1),
                                "fp32_tflops": round(outs * flop / ms / 1e9, 2)})
    name, limit = card()
    print(json.dumps({"tool": "bench_bfsk", "seconds_of_signal": 1.0, "baseband_hz": rate, "gpu": name, "power_limit": limit, "results": results}))


if __name__ == "__main__":
    main()
