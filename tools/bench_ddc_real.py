"""GPU throughput of the real-input fused DDC bank (csdrb_ddc_bank_f: shift_addition_fc | fir_decimate_cc, generic kernel) against the complex
bank (csdrb_ddc_bank) fed the same samples as x + 0j, in wideband Msamples/s: 128 and 1024 channels at D = 50 (801 taps, 2.4 Msps -> 48 kHz)
and at a direct-sampling geometry, D = 1350 with bw 0.0008 (5001 taps: 64.8 Msps -> 48 kHz).  Both banks without the discriminator, chunk 1024,
one block of 2^21 (D = 50) or 2^23 (D = 1350) samples per call; CUDA events around repeated calls after warm-up, at least 1 s per measurement.
The two outputs are checked to be equal as float values first.  Prints one JSON line with the card name and power limit."""
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
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn, min_s=1.0):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    reps, total = 0, 0.0
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    while total < min_s * 1e3:
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
        total += t0.elapsed_time(t1); reps += 1
    return total / reps


def case(channels, D, bw, n):
    T = cb.firdes_filter_len(bw)
    taps = cb.firdes_lowpass_f(T, 0.5 / D)
    rates = np.linspace(-0.45, 0.45, channels).astype(np.float32)
    g = torch.Generator(device="cuda").manual_seed(channels + D)
    x = torch.rand(n, generator=g, device="cuda") * 2 - 1
    xc = x.to(torch.complex64)
    a = cb.ddc_bank(x, rates, D, taps, demod=False)[0]
    b = cb.ddc_bank(xc, rates, D, taps, demod=False)[0]
    av, bv = torch.view_as_real(a), torch.view_as_real(b)
    assert bool(((av == bv) | (torch.isnan(av) & torch.isnan(bv))).all()), "real and complex banks differ"
    ms_r = timed(lambda: cb.ddc_bank(x, rates, D, taps, demod=False))
    ms_c = timed(lambda: cb.ddc_bank(xc, rates, D, taps, demod=False))
    return {"channels": channels, "D": D, "taps": T, "samples": n, "real_msps": round(n / ms_r / 1e3, 2), "complex_msps": round(n / ms_c / 1e3, 2),
            "real_over_complex": round(ms_c / ms_r, 3)}


def main():
    torch.cuda.set_device(0)
    rows = [case(c, D, bw, n) for D, bw, n in ((50, 0.005, 1 << 21), (1350, 0.0008, 1 << 23)) for c in (128, 1024)]
    print(json.dumps({"bench": "ddc_real", "card": card(), "cases": rows}))


if __name__ == "__main__":
    main()
