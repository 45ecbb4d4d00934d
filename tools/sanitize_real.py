"""Every real-input kernel once on small, awkward sizes -- meant to run under `compute-sanitizer --tool memcheck`: the shift_addition_fc bank (shared
and per-row, odd chunks, a sliced chain), its drop-in, and the real fused DDC bank at every generic bucket with both DEMOD values, with d_wide 8 bytes
off a 16-byte boundary, ragged channel counts, a streaming object whose blocks leave keep % 4 == 2 and a retune."""
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import csdr_b200 as cb  # noqa: E402

rng = np.random.default_rng(0)
r = lambda *shape: torch.rand(shape, device="cuda") * 2 - 1
cb.shift_addition_bank_fc(r(16384 + 777), [0.1, -0.3, 0.45], chunk=1024); cb.shift_addition_bank_fc(r(3, 1001), [0.1, -0.3, 0.45], chunk=37)
cb.shift_addition_bank_fc(r(2, 600 * 64 + 13), [0.31, -0.07], chunk=64); cb.shift_addition_bank_fc(r(1100 * 1024 + 1), [0.2], chunk=1024)
cb.libcsdr.shift_addition_fc(rng.normal(size=1021).astype(np.float32), 0.2, 0.3, 1024)
for D, T in ((2, 7), (6, 37), (12, 97), (48, 769), (52, 833), (126, 2395), (400, 8000), (50, 801), (10, 79), (10, 199), (1350, 5001)):
    taps = cb.firdes_lowpass_f(T, 0.5 / D)
    buf = r(T + 37 * D + 11 + 2)
    for demod in (True, False):
        for ch in (1, 37, 65):
            cb.ddc_bank(buf[2:], np.linspace(-0.4, 0.4, ch), D, taps, demod=demod, chunk=1024, offset=100)   # 8 bytes past a 16-byte boundary
D, T = 50, 801
taps = cb.firdes_lowpass_f(T, 0.5 / D)
bank = cb.DdcBank(np.linspace(-0.4, 0.4, 37), D, taps, demod=True, chunk=1024)
w = r(300_000)
N = 65536                                                        # 64 750 consumed per block: the second block starts 8 bytes off a 16-byte boundary
start = 0
for k in range(3):
    if k == 2:
        bank.set_rate(3, 0.11)
    o = bank.process(w[start:start + N])
    start += o.shape[1] * D
bank.close()
torch.cuda.synchronize(); print("sanitize_real: all real-input kernels ran")
