"""GPU tests (-m gpu) of the tone filters: the two banks (csdr_b200/csrc/tone.cu) at 1024 channels against the checker
tests/tone/tone_oracle.c bit for bit, apply_fir_cc against the compiled reference bit for bit and bfsk_demod_cf within the bound of
tests/tone/tone.py, L up to 4096; and the csdr commands bfsk_demod_cf, peaks_fir_cc and firdes_peak_c against the unmodified reference CLI
(its bytes, or within the bound for bfsk_demod_cf) at several buffer sizes through end of input, with their refusals.
tests/test_tone_cli_emulated.py runs the CLI bodies on the emulated library."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from test_gpu_cli import clis, run_graph  # noqa: F401  (the fixture: our CLI and the reference CLI)

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "tone"))
import tone  # noqa: E402

pytestmark = pytest.mark.gpu
TEXT = b"RYRYRY CQ CQ DE TEST 599 73\r\n"


def same_bits(a, b):
    """equal bit for bit, except that any NaN equals any NaN (the GPU writes the canonical NaN, a CPU keeps an input's payload)"""
    fa, fb = np.asarray(a).view(np.float32), np.asarray(b).view(np.float32)
    na, nb = np.isnan(fa), np.isnan(fb)
    return fa.shape == fb.shape and np.array_equal(na, nb) and np.array_equal(fa[~na].view(np.uint32), fb[~nb].view(np.uint32))


@pytest.fixture(scope="module")
def cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    return torch, csdr_b200


@pytest.mark.parametrize("L", [2, 44, 255, 1001, 4096])
def test_banks_equal_checker_at_1024_channels(cuda, L):
    torch, cb = cuda
    rng = np.random.default_rng(L)
    ch, n = 1024, L + 2000
    X = ((rng.standard_normal((ch, n)) + 1j * rng.standard_normal((ch, n))) * 10.0 ** rng.uniform(-3, 3, (ch, 1))).astype(np.complex64)
    X[5, 700] = np.nan; X[9, 100] = np.inf
    taps = cb.firdes_peak_c(0.1, L)
    xd = torch.from_numpy(X).cuda()
    y = cb.apply_fir_bank_cc(xd, taps).cpu().numpy()
    b = cb.bfsk_demod_bank_cf(xd, 0.085, L).cpu().numpy()
    mark, space = cb.firdes_peak_c(0.0425, L), cb.firdes_peak_c(-0.0425, L)
    assert y.shape == (ch, n - L + 1) and b.shape == (ch, n - L + 1)
    for c in list(range(0, ch, 37)) + [5, 9, ch - 1]:
        assert same_bits(y[c], tone.apply_fir_cc(X[c], taps)), c
        assert same_bits(b[c], tone.bfsk_demod_cf(X[c], mark, space)), c


@pytest.mark.skipif(not tone.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built")
def test_banks_against_reference(cuda):
    torch, cb = cuda
    rng = np.random.default_rng(11)
    for L, spacing in ((44, 0.085), (255, 0.02), (4096, 0.001)):
        n = L + 3000
        z = np.stack([tone.rtty_signal(TEXT, 44.0, rng, noise=0.05, tail_bits=(n / 44.0))[:n] for _ in range(4)])
        xd = torch.from_numpy(z).cuda()
        taps = tone.ref_peak(spacing, L)
        assert same_bits(taps, cb.firdes_peak_c(spacing, L))
        y = cb.apply_fir_bank_cc(xd, taps).cpu().numpy()
        b = cb.bfsk_demod_bank_cf(xd, spacing, L).cpu().numpy()
        mark, space = tone.bfsk_taps(spacing, L)
        for c in range(4):
            assert same_bits(y[c], tone.ref_apply_fir_cc(z[c], taps)), (L, c)
            err = np.abs(b[c].astype(np.float64) - tone.ref_bfsk_demod_cf(z[c], mark, space))
            assert np.all(err <= tone.bfsk_bound(z[c], mark, space)), (L, c)


def test_refusals(cuda):
    torch, cb = cuda
    x = torch.zeros((2, 100), dtype=torch.complex64, device="cuda")
    with pytest.raises(cb.CsdrB200Error, match="rc=-2"):
        cb.apply_fir_bank_cc(x, np.ones(1, np.complex64))
    with pytest.raises(cb.CsdrB200Error, match="rc=-1"):
        cb.apply_fir_bank_cc(x, np.ones(101, np.complex64))
    with pytest.raises(cb.CsdrB200Error, match="rc=-2"):
        cb.bfsk_demod_bank_cf(torch.zeros((1, 5000), dtype=torch.complex64, device="cuda"), 0.1, 4097)


# ---- the csdr commands --------------------------------------------------------------------------------------------------------------
def _run(cli, args, data, env=None):
    e = dict(os.environ); e.update(env or {})
    return subprocess.run(["bash", "-c", f"{cli} {args}"], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e, timeout=300)


def _signal(seed, n):
    rng = np.random.default_rng(seed)
    z = tone.rtty_signal(TEXT, 44.0, rng, freq=0.001, noise=0.05, tail_bits=40.0)
    return np.resize(z, n).astype(np.complex64)


def test_tone_commands_against_reference(clis):
    """bytes of the reference CLI for peaks_fir_cc and firdes_peak_c; for bfsk_demod_cf the same count, every value within the bound of the
    reference and equal to the checker bit for bit.  Stream lengths cut the memmove framing at different places; the output is the
    prefix of the valid convolution the reference's loop reaches before end of input"""
    ours, ref = clis
    for bufsize, n in ((None, 10_000), ("256", 7_777), ("4000", 20_001), ("64", 1_000)):
        env = {"CSDR_FIXED_BUFSIZE": bufsize} if bufsize else {}
        z = _signal(n, n)
        data = z.tobytes()
        for args in ("peaks_fir_cc 45 0.0425", "peaks_fir_cc 31 0.1 -0.2 0.33", "peaks_fir_cc 2 0.25"):
            a, b = _run(ours, args, data, env), _run(ref, args, data, env)
            assert a.returncode == b.returncode == 0 and a.stdout == b.stdout and len(a.stdout) > 0, (bufsize, args)
        for spacing, L in (("0.085", 44), ("0.2", 2), ("0.05", 63)):
            a, b = _run(ours, f"bfsk_demod_cf {spacing} {L}", data, env), _run(ref, f"bfsk_demod_cf {spacing} {L}", data, env)
            assert a.returncode == b.returncode == 0 and len(a.stdout) == len(b.stdout) > 0, (bufsize, spacing, L)
            got, want = np.frombuffer(a.stdout, np.float32), np.frombuffer(b.stdout, np.float32)
            mark, space = tone.bfsk_taps(float(spacing), L)
            full = tone.bfsk_demod_cf(z, mark, space)
            assert same_bits(got, full[:got.size]), (bufsize, spacing, L)
            bound = tone.bfsk_bound(z, mark, space)[:got.size]
            assert np.all(np.abs(got.astype(np.float64) - want) <= bound), (bufsize, spacing, L)
    for args in ("firdes_peak_c 0.1 45", "firdes_peak_c -0.0425 101 HAMMING", "firdes_peak_c 0.25 7 BOXCAR", "firdes_peak_c 0.3 1",
                 "firdes_peak_c 0.01 4095 HAMMING"):
        a, b = _run(ours, args, b""), _run(ref, args, b"")
        assert (a.returncode, a.stdout) == (b.returncode, b.stdout), args
        assert a.stderr.replace(ours.encode(), b"csdr") == b.stderr.replace(ref.encode(), b"csdr"), args


def test_tone_refusals(clis):
    """the reference's refusals with its code and message; a bfsk_demod_cf filter of fewer than 2 taps or not below the buffer refused"""
    ours, ref = clis
    for args, env in (("peaks_fir_cc", {}), ("peaks_fir_cc 45", {}), ("peaks_fir_cc 1024 0.1", {}), ("peaks_fir_cc 300 0.1", {"CSDR_FIXED_BUFSIZE": "256"}),
                      ("firdes_peak_c", {}), ("firdes_peak_c 0.1", {}), ("firdes_peak_c 0.1 44", {}), ("bfsk_demod_cf", {}), ("bfsk_demod_cf 0.1", {})):
        a, b = _run(ours, args, b"", env), _run(ref, args, b"", env)
        assert a.returncode != 0 and a.returncode == b.returncode, (args, a.returncode, b.returncode)
        assert a.stderr.replace(ours.encode(), b"csdr") == b.stderr.replace(ref.encode(), b"csdr"), args
    for args in ("bfsk_demod_cf 0.085 1", "bfsk_demod_cf 0.085 1024", "bfsk_demod_cf 0.085 5000", "peaks_fir_cc 1 0.1"):
        a = _run(ours, args, _signal(1, 3000).tobytes(), {"CSDR_FIXED_BUFSIZE": "8192"} if "5000" in args else {})
        assert a.returncode != 0 and a.stdout == b"" and b"must be between" in a.stderr, args
