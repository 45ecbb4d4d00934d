"""GPU test (-m gpu) of csdr-synth, the real binary: its stdout equals SynthBank on the streams cut to the shortest source, byte for byte, for
two --block sizes, with sources of unequal lengths, one of them stdin."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("block", [1000, 16384])
def test_csdr_synth_equals_synth_bank(tmp_path, block):
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200 as cb
    rng = np.random.default_rng(block)
    lengths = [30_000, 21_111, 25_000]
    rates = [-0.2, 0.0, 0.15]
    srcs = [(rng.uniform(-1, 1, m) + 1j * rng.uniform(-1, 1, m)).astype(np.complex64) for m in lengths]
    for k in (0, 2):
        srcs[k].tofile(tmp_path / f"s{k}.cf32")
    args = [str(ROOT / "csdr_b200" / "csdr-synth"), "--interpolation", "50", "--block", str(block),
            f"{rates[0]}:{tmp_path / 's0.cf32'}", f"{rates[1]}:-", f"{rates[2]}:{tmp_path / 's2.cf32'}"]
    r = subprocess.run(args, input=srcs[1].tobytes(), capture_output=True, timeout=600)
    assert r.returncode == 0, r.stderr.decode()
    L = min(lengths)
    taps = cb.firdes_lowpass_f(cb.firdes_filter_len(0.05), 0.5 / 50)
    bank = cb.SynthBank(rates, 50, taps)
    try:
        want = bank.process(torch.from_numpy(np.stack([s[:L] for s in srcs])).cuda()).cpu().numpy()
    finally:
        bank.close()
    assert len(r.stdout) == want.nbytes and r.stdout == want.tobytes()
