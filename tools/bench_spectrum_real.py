"""GPU time of the real-input waterfall bank csdrb_spectrum_bank_f (fft_fc N 2N | logaveragepower_cf -70 N A), after checking its bits against
the composition of the existing calls on the same input (frames gathered by torch, the window product, csdrb_fft_r2c_batch ->
csdrb_accumulate_power_cf x A on bins 0..N-1 -> csdrb_log_ff).  Beside it, the only way to this waterfall before the real bank: the complex bank
csdrb_spectrum_bank_cf on the same samples as x + 0j at 2N points (fft_cc 2N 2N | logaveragepower_cf -70 2N A, twice the bins, half of them the
mirror image).  Workloads:
  (a) one real row of 2^25 samples (about 0.5 s of a 64.8 Msps RX888 stream), N = 16384 bins, E = 2N, A = 8
  (b) 1024 rows of 2^17 real samples, N = 1024 bins, E = 2N, A = 8
CUDA events around repeated calls after warm-up, at least 1 s per measurement.  Prints one JSON line with the card name and power limit,
Msamples/s in for both banks and the real bank's HBM share: 4 bytes per input sample read once over 3.35 TB/s (the complex bank reads 8).  The
complex bank serves at most 16384 points, so (a), at 2N = 32768, has no complex-bank column: there x + 0j is the CLI pipe only."""
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

HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn, min_s=1.0):
    for _ in range(2):
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


def bank_runner(L, s, x, rows, n, N, E, A, real):
    """one whole-stream call of the real bank (x float32) or the complex bank (x complex64, fft_size N)"""
    frame = 2 * N if real else N
    w = torch.from_numpy(cb.libcsdr.precalculate_window(frame, "HAMMING")).cuda()
    p = cb.SpectrumParams(N, E, A, 0, -70.0)
    lines_f, scratch_f, bank = ((L.csdrb_spectrum_bank_lines_f, L.csdrb_spectrum_bank_scratch_bytes_f, L.csdrb_spectrum_bank_f) if real else
                                (L.csdrb_spectrum_bank_lines, L.csdrb_spectrum_bank_scratch_bytes, L.csdrb_spectrum_bank_cf))
    lines = lines_f(C.byref(p), C.byref(cb.SpectrumState(0, 0)), n)
    hist = torch.zeros((rows, frame), dtype=torch.float32 if real else torch.complex64, device="cuda")
    acc = torch.zeros((rows, N), dtype=torch.float32, device="cuda")
    out = torch.empty((rows, lines, N), dtype=torch.float32, device="cuda")
    sb = scratch_f(rows, n, C.byref(p))
    scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")

    def run():
        state = cb.SpectrumState(0, 0)
        hist.zero_(); acc.zero_()
        rc = bank(x.data_ptr(), n, rows, n, w.data_ptr(), C.byref(p), hist.data_ptr(), acc.data_ptr(), C.byref(state), out.data_ptr(), lines * N * 4,
                  scratch.data_ptr(), sb, s)
        assert rc == lines, L.csdrb_last_error()
    return run, out, w, lines


def workload(rows, n, N, A):
    L, st = cb.lib(), torch.cuda.current_stream()
    s = C.c_void_p(st.cuda_stream)
    E = 2 * N
    x = torch.randn((rows, n), dtype=torch.float32, device="cuda") * 0.3
    run_real, out, w, lines = bank_runner(L, s, x, rows, n, N, E, A, True)
    run_real()
    # the composition: E = 2N, so frame k is x[:, 2Nk : 2N(k+1)]
    m = rows * lines * A
    frames = (x[:, :lines * A * 2 * N].reshape(rows, lines * A, 2 * N) * w).contiguous()
    spec = torch.empty((rows, lines * A, N + 1), dtype=torch.complex64, device="cuda")
    assert L.csdrb_fft_r2c_batch(frames.data_ptr(), 2 * N, spec.data_ptr(), N + 1, 2 * N, m, s) == 0, L.csdrb_last_error()
    bins = spec[:, :, :N].reshape(rows, lines, A, N).permute(2, 0, 1, 3).contiguous()                # [A][rows][lines][N]
    pw = torch.zeros((rows * lines * N,), dtype=torch.float32, device="cuda"); db = torch.empty_like(pw)
    for f in range(A):
        assert L.csdrb_accumulate_power_cf(bins[f].data_ptr(), pw.data_ptr(), rows * lines * N, s) >= 0
    add = float(np.float32(np.float64(np.float32(-70.0)) - 10.0 * np.log10(A)))
    assert L.csdrb_log_ff(pw.data_ptr(), db.data_ptr(), rows * lines * N, add, s) >= 0
    same = torch.equal(out.view(torch.int32), db.view(rows, lines, N).view(torch.int32))
    assert same, "the real bank and the composition differ"
    del frames, spec, bins, pw, db
    t_real = timed(run_real)
    samples = rows * n
    res = {"rows": rows, "samples_per_row": n, "bins": N, "every": E, "averages": A, "lines_per_row": lines, "bits_equal": same,
           "real_bank_ms": round(t_real, 4), "real_bank_msamples_per_s": round(samples / t_real / 1e3, 1),
           "real_bank_hbm_share_input_once": round(4.0 * samples / (t_real * 1e-3) / HBM, 4)}
    if 2 * N > 16384:                                                   # the complex bank stops at 16384 points: x + 0j at 2N is a CLI pipe only
        res["complex_bank_x_plus_0j_ms"] = None
        res["complex_note"] = f"2N = {2 * N} points is above the complex bank's 16384"
        return res
    xc = torch.complex(x, torch.zeros_like(x))
    run_cplx, _, _, _ = bank_runner(L, s, xc, rows, n, 2 * N, E, A, False)
    t_cplx = timed(run_cplx)
    res.update({"complex_bank_x_plus_0j_ms": round(t_cplx, 4), "complex_bank_msamples_per_s": round(samples / t_cplx / 1e3, 1),
                "speedup": round(t_cplx / t_real, 2)})
    return res


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {"device": card(), "a": workload(1, 1 << 25, 16384, 8), "b": workload(1024, 1 << 17, 1024, 8)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
