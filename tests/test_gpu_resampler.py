"""GPU tests (-m gpu) of rational_resampler_ff: the bank (csdrb_rational_resampler_bank_ff), the libcsdr drop-in and the `csdr rational_resampler_ff`
command against the golden vectors of the compiled reference (tests/golden/resampler_golden.npz), the strict restatement
tests/resampler/resampler_oracle.c (bit for bit) and the reference CLI.  The drop-in and CLI bodies also run on the emulated library
(tests/test_resampler_emulated.py)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "resampler"))
sys.path.insert(0, str(ROOT / "tests"))
import resampler as R  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
GOLD = np.load(ROOT / "tests" / "golden" / "resampler_golden.npz")
CASES = sorted({k[:-5] for k in GOLD.files if k.endswith("_geom")})


def _rel(y, ref):
    from oracle.pyoracle import rel_rms
    return rel_rms(y, ref)


def _case(name):
    I, D, T, block = (int(v) for v in GOLD[f"{name}_geom"])
    return I, D, T, block, GOLD[f"{name}_x"], GOLD[f"{name}_taps"], GOLD[f"{name}_y"], tuple(int(v) for v in GOLD[f"{name}_state"])


@pytest.fixture(scope="module")
def gpu():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    csdr_b200.lib()
    return csdr_b200


@pytest.fixture(scope="module")
def clis():
    import test_gpu_cli as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    if not g.REF.exists():
        pytest.skip("oracle/_ref/csdr_ref not built")
    from csdr_b200.build import build
    build()
    return str(g.OURS), str(g.REF)


def test_lowpass_design_matches_the_oracle(gpu, oracle):
    for I, D, T in ((3, 4, 79), (24, 25, 201), (147, 160, 79), (1, 100, 79), (5, 2, 8001)):
        ours = gpu.rational_resampler_get_lowpass_f(T, I, D)
        assert np.array_equal(ours, R.lowpass(oracle, T, I, D)), (I, D, T)
    for name in CASES:                                                  # the reference's -ffast-math build differs in the last ulps
        I, D, T, _, _, taps, _, _ = _case(name)
        assert np.abs(gpu.rational_resampler_get_lowpass_f(T, I, D) - taps).max() <= 1e-6 * np.abs(taps).max(), name


def test_rational_resampler_dropin_golden_and_oracle(gpu):
    ro = R.Oracle()
    for name in CASES:
        I, D, T, block, x, taps, y_ref, st_ref = _case(name)
        if block:
            y = gpu.libcsdr.rational_resampler_ff(x, I, D, taps, block=block)
            assert y.size == y_ref.size and np.array_equal(y, ro.stream(x, I, D, taps, block)), name
        else:
            y, st = gpu.libcsdr.rational_resampler_ff(x, I, D, taps)
            assert st == st_ref and y.size == y_ref.size, (name, st, st_ref)
            yo, so = ro.rational_resampler_ff(x, I, D, taps)
            assert so == st and np.array_equal(y, yo), name
        if np.any(y_ref):
            assert _rel(y, y_ref) <= 1e-5, (name, _rel(y, y_ref))
        else:
            assert not np.any(y), name                                  # T < I: every output is 0 (147/160 with 79 taps)
    # no output possible: the fields the reference leaves uninitialised are {0, 0, last_taps_delay}
    x, taps = GOLD["r3_4_x"], GOLD["r3_4_taps"]
    assert gpu.libcsdr.rational_resampler_ff(x[:20], 3, 4, taps, last_taps_delay=2)[1] == (0, 0, 2)
    assert gpu.libcsdr.rational_resampler_ff(x[:1], 1, 4, taps)[1] == (0, 0, 0)


def test_rational_resampler_bank_golden_oracle_and_lockstep_rows(gpu):
    """three rows (one golden, two others) in one call with padded strides; each row bit for bit the oracle's single call"""
    ro = R.Oracle()
    for name in CASES:
        I, D, T, block, x, taps, y_ref, st_ref = _case(name)
        if block:
            continue
        n = x.size
        rows = np.zeros((3, n + 13), np.float32)
        rows[0, :n] = x; rows[1, :n] = x[::-1]; rows[2, :n] = np.roll(x, 77)
        xd = torch.from_numpy(rows).cuda()[:, :n]
        out = torch.full((3, n * I // D + 7), 1234.5, device="cuda")
        y, st = gpu.rational_resampler_bank_ff(xd, I, D, taps, out=out)
        torch.cuda.synchronize()
        assert st == st_ref and y.shape[1] == y_ref.size, (name, st)
        got = out.cpu().numpy()
        assert np.all(got[:, y_ref.size:] == np.float32(1234.5)), name
        for c in range(3):
            assert np.array_equal(got[c, :y_ref.size], ro.rational_resampler_ff(rows[c, :n], I, D, taps)[0]), (name, c)
        if np.any(y_ref):
            assert _rel(got[0, :y_ref.size], y_ref) <= 1e-5, name
    # a stream cut into bank calls that end on input, carrying the unconsumed tail and last_taps_delay: one call's output on the whole row
    I, D, T, _, x, taps, _, _ = _case("r24_25")
    whole, _ = ro.rational_resampler_ff(x, I, D, taps)
    xd = torch.from_numpy(x).cuda()
    pos, ltd, parts = 0, 0, []
    for cut in (300, 800, 1400, x.size):
        y, (ip, n_out, ltd) = gpu.rational_resampler_bank_ff(xd[pos:cut].unsqueeze(0).contiguous(), I, D, taps, ltd)
        parts.append(y[0].cpu().numpy()); pos += ip
    got = np.concatenate(parts)
    assert np.array_equal(got, whole)


def test_rational_resampler_bank_refusals(gpu):
    x = torch.zeros((2, 1000), device="cuda")
    with pytest.raises(gpu.CsdrB200Error, match="taps"):
        gpu.rational_resampler_bank_ff(x, 3, 4, np.ones(16385, np.float32))
    with pytest.raises(gpu.CsdrB200Error, match="last_taps_delay"):
        gpu.rational_resampler_bank_ff(x, 3, 4, np.ones(79, np.float32), last_taps_delay=3)
    y, st = gpu.rational_resampler_bank_ff(torch.zeros((1, 100_000), device="cuda"), 1, 1, np.ones(8001, np.float32) / 8001)
    torch.cuda.synchronize()
    assert st[1] == y.shape[1] > 0 and float(y.abs().max()) == 0.0


def test_rational_resampler_command(clis):
    """`csdr rational_resampler_ff 3 4` and `5 2 0.02` against the reference CLI: same framing (first call on the whole block, later calls on the
    unconsumed tail plus input_processed new samples, short last read processed), same byte count, outputs within 1e-5"""
    from test_gpu_cli import run_graph
    ours, ref = clis
    for n in (50_000, 4096, 3000):
        rng = np.random.default_rng(n)
        t = np.arange(n)
        x = (0.5 * np.sin(2 * np.pi * 0.02 * t) + 0.1 * rng.standard_normal(n)).astype(np.float32).tobytes()
        for args in ("3 4", "5 2 0.02", "24 25 0.02 BLACKMAN"):
            a = np.frombuffer(run_graph(ours, [f"rational_resampler_ff {args}"], x), np.float32)
            b = np.frombuffer(run_graph(ref, [f"rational_resampler_ff {args}"], x), np.float32)
            assert a.size == b.size and a.size > 0, (n, args, a.size, b.size)
            assert _rel(a, b) <= 1e-5, (n, args)
    # 1 1 passes the bytes through like the reference's clone_ (which never returns at end of input, so only ours is run)
    x = np.random.default_rng(1).integers(0, 256, 10_000, dtype=np.uint8).tobytes()
    assert run_graph(ours, ["rational_resampler_ff 1 1"], x)[:len(x)] == x
    r = subprocess.run([ours, "rational_resampler_ff", "3"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
    assert r.returncode != 0 and b"interpolation, decimation" in r.stderr
