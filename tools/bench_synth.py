"""Times the synthesis bank on one GPU against the composition it replaces and prints one JSON line.  Two workloads: 1024 channels x 48 000
inputs at I = 50, T = 401 (48 kHz channels into 2.4 Msps), and 128 channels x 48 000 inputs at I = 256, T = 2049.  The composition is
fir_interpolate_bank, shift_addition_bank_cc (chunk 1024) and torch.sum(dim=0); it is checked against the fused bank within the float64 bound of
tests/synth/synth.py's kind (torch's summation order is not the tree's), not bit for bit.  CUDA events around `--iters` launches after a warm-up;
the card's name and power limit (read-only nvidia-smi query) go with the numbers.  Work is counted from the shapes with every operation its own
instruction (no FMA): per channel and output 4 per tap term actually used, 6 for the phasor step and 6 for the rotation, plus 2 (C - 1) per output
for the tree, and set against the 33.5 T separate-instruction FP32 rate of an H100 SXM."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import csdr_b200 as cb  # noqa: E402

FP32_RATE = 33.5e12


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


def terms_used(I, T):
    """tap terms summed over the I phases of one group: (I - ip) + si*I < T, the reference's count"""
    return sum(len(range(I - ip, T, I)) for ip in range(I))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_synth needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu}
    rng = np.random.default_rng(0)
    for ch, I, T, n in ((1024, 50, 401, 48_000), (128, 256, 2049, 48_000)):
        x = torch.from_numpy((rng.uniform(-1, 1, (ch, n)) + 1j * rng.uniform(-1, 1, (ch, n))).astype(np.complex64)).cuda()
        rates = rng.uniform(-0.49, 0.49, ch).astype(np.float32)
        taps = cb.firdes_lowpass_f(T, 0.5 / I)
        G = n - (T - 1 + I - 1) // I
        nout = G * I
        params = torch.from_numpy(np.array([cb.shift_addition_init(float(r)) for r in rates], np.float32)).cuda()
        d_taps = torch.from_numpy(taps).cuda()
        phase = torch.zeros(ch, dtype=torch.float32, device="cuda")
        y = torch.empty(nout, dtype=torch.complex64, device="cuda")
        sb = cb.lib().csdrb_synth_bank_scratch_bytes(ch, n, I, T, 1024, 0)
        scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")

        def fused():
            cb._check(cb.lib().csdrb_synth_bank_cc(x.data_ptr(), x.stride(0), ch, n, I, d_taps.data_ptr(), T, params.data_ptr(), phase.data_ptr(),
                                                   1024, 0, y.data_ptr(), scratch.data_ptr(), sb, cb._stream()), "synth_bank")

        def composition():
            W = cb.fir_interpolate_bank(x, I, d_taps)
            Y, _ = cb.shift_addition_bank_cc(W, rates, chunk=1024)
            return Y.sum(dim=0)

        ms_fused = timed(fused, args.iters)
        ms_comp = timed(composition, max(2, args.iters // 4))
        # agreement: the fused bank from phase 0 against the composition, within the tree's and torch's summation bounds
        yf, _ = cb.synth_bank(x, rates, I, taps)
        yc = composition()
        Y, _ = cb.shift_addition_bank_cc(cb.fir_interpolate_bank(x, I, d_taps), rates, chunk=1024)
        mag = (Y.real.abs() + Y.imag.abs()).sum(dim=0)
        err = (yf - yc).abs()
        gam = (ch * 2.0 ** -24) / (1 - ch * 2.0 ** -24)                  # any summation order of C terms: gamma(C - 1) <= gamma(C), each side
        ok = bool((err <= 2 * 1.4143 * gam * mag + 1e-30).all())
        del Y, yc, mag, err
        torch.cuda.empty_cache()
        ops = float(ch) * (G * 4 * terms_used(I, T) + nout * 12) + 2.0 * (ch - 1) * nout
        res[f"synth_{ch}ch_I{I}_T{T}"] = {
            "ms_fused": round(ms_fused, 3), "ms_composition": round(ms_comp, 3), "speedup": round(ms_comp / ms_fused, 2),
            "G_channel_samples_per_s": round(ch * nout / ms_fused / 1e6, 1), "fp32_T_ops_per_s": round(ops / ms_fused / 1e9, 2),
            "fraction_of_33_5T": round(ops / ms_fused / 1e-3 / FP32_RATE, 3), "composition_within_bound": ok}
        del x, y, scratch
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
