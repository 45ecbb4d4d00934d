"""GPU time of the waterfall bank csdrb_spectrum_bank_cf against the composition of the existing per-block calls on the same input
(frames gathered by torch, csdrb_apply_window_rows_c -> csdrb_fft_c2c_batch -> csdrb_accumulate_power_cf x A -> csdrb_log_ff -> halves swapped),
after checking that both give the same bits.  Workloads:
  (a) one row of 2^24 samples, N = 16384, E = 4096, A = 16 (a wide SDR with overlapped frames)
  (b) 1024 rows of 2^17 samples, N = 2048, E = N, A = 8
CUDA events around repeated calls after warm-up, at least 1 s per measurement.  Prints one JSON line with the card name and power limit, Msamples/s
in, both times and the bank's HBM share: 8 bytes per input sample read once over 3.35 TB/s (for E < N the overlapping frames read each sample N/E
times, the repeats from L2)."""
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


def workload(rows, n, N, E, A):
    L, st = cb.lib(), torch.cuda.current_stream()
    s = C.c_void_p(st.cuda_stream)
    x = (torch.randn((rows, n), dtype=torch.complex64, device="cuda") * 0.3)
    w = torch.from_numpy(cb.libcsdr.precalculate_window(N, "HAMMING")).cuda()
    p = cb.SpectrumParams(N, E, A, 0, -70.0)
    lines = L.csdrb_spectrum_bank_lines(C.byref(p), C.byref(cb.SpectrumState(0, 0)), n)
    hist = torch.zeros((rows, N), dtype=torch.complex64, device="cuda"); acc = torch.zeros((rows, N), dtype=torch.float32, device="cuda")
    out = torch.empty((rows, lines, N), dtype=torch.float32, device="cuda")
    sb = L.csdrb_spectrum_bank_scratch_bytes(rows, n, C.byref(p))
    scratch = torch.empty(sb, dtype=torch.uint8, device="cuda")

    def run_bank():
        state = cb.SpectrumState(0, 0)
        rc = L.csdrb_spectrum_bank_cf(x.data_ptr(), n, rows, n, w.data_ptr(), C.byref(p), hist.data_ptr(), acc.data_ptr(), C.byref(state),
                                      out.data_ptr(), lines * N * 4, scratch.data_ptr(), sb, s)
        assert rc == lines, L.csdrb_last_error()

    # the composition: frame f of every line gathered into plane f ([A][rows*lines][N]), then the existing calls
    k = torch.arange(lines * A, device="cuda")
    start = (k + 1) * E - N if E <= N else k * E
    idx = (start[:, None] + torch.arange(N, device="cuda")[None, :]).view(lines, A, N).permute(1, 0, 2)       # [A][lines][N]
    frames = torch.empty((A, rows, lines, N), dtype=torch.complex64, device="cuda")
    win = torch.empty_like(frames); spec = torch.empty_like(frames)
    pw = torch.empty((rows * lines * N,), dtype=torch.float32, device="cuda")
    db = torch.empty_like(pw)
    add = float(np.float32(np.float64(np.float32(-70.0)) - 10.0 * np.log10(A)))
    xp = torch.cat([torch.zeros((rows, N), dtype=torch.complex64, device="cuda"), x], dim=1)                    # zeros before the stream

    def run_composition():
        frames.copy_(xp[:, (idx + N)].permute(1, 0, 2, 3))
        m = A * rows * lines
        assert L.csdrb_apply_window_rows_c(frames.data_ptr(), win.data_ptr(), w.data_ptr(), N, m, s) >= 0
        assert L.csdrb_fft_c2c_batch(win.data_ptr(), N, spec.data_ptr(), N, N, m, 0, s) >= 0
        pw.zero_()
        for f in range(A):
            assert L.csdrb_accumulate_power_cf(spec[f].data_ptr(), pw.data_ptr(), rows * lines * N, s) >= 0
        assert L.csdrb_log_ff(pw.data_ptr(), db.data_ptr(), rows * lines * N, add, s) >= 0
        return torch.cat([db.view(rows, lines, N)[:, :, N // 2:], db.view(rows, lines, N)[:, :, :N // 2]], dim=2)

    hist.zero_(); acc.zero_()
    run_bank()
    same = torch.equal(out.view(torch.int32), run_composition().contiguous().view(torch.int32))
    assert same, "the bank and the composition differ"
    t_bank, t_comp = timed(run_bank), timed(run_composition)
    samples = rows * n
    return {"rows": rows, "samples_per_row": n, "fft_size": N, "every": E, "averages": A, "lines_per_row": lines, "bits_equal": same,
            "bank_ms": round(t_bank, 4), "composition_ms": round(t_comp, 4), "bank_msamples_per_s": round(samples / t_bank / 1e3, 1),
            "composition_msamples_per_s": round(samples / t_comp / 1e3, 1), "speedup": round(t_comp / t_bank, 2),
            "bank_hbm_share_input_once": round(8.0 * samples / (t_bank * 1e-3) / HBM, 4), "input_reads_per_sample": max(1.0, N / E)}


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {"device": card(), "a": workload(1, 1 << 24, 16384, 4096, 16), "b": workload(1024, 1 << 17, 2048, 2048, 8)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
