"""GPU tests (-m gpu) of the transmit banks through the Python API at full size: fir_interpolate_bank at 1024 channels bit for bit against the
kernel's order restated in tests/tx/tx.py and within its bound of the compiled reference, a 2^24-sample row, calls cut with the carry; fmmod_bank
at 1024 channels with the build's phases bit for bit and the phase carried over calls; both through a tone loopback (fmmod -> interpolate ->
discriminator recovers the tone)."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "tx"))
import tx  # noqa: E402

pytestmark = pytest.mark.gpu
ULP1 = 2.0 ** -24


@pytest.fixture(scope="module")
def cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    return torch, csdr_b200


def same_bits(a, b):
    fa, fb = np.asarray(a).view(np.float32), np.asarray(b).view(np.float32)
    na, nb = np.isnan(fa), np.isnan(fb)
    return fa.shape == fb.shape and np.array_equal(na, nb) and np.array_equal(fa[~na].view(np.uint32), fb[~nb].view(np.uint32))


@pytest.mark.parametrize("I,T", [(1, 81), (3, 81), (50, 401), (256, 2049), (5, 9001)])
def test_interp_bank_at_1024_channels(cuda, I, T):
    torch, cb = cuda
    rng = np.random.default_rng(I)
    ch, n = 1024, 300
    X = ((rng.standard_normal((ch, n)) + 1j * rng.standard_normal((ch, n))) * 10.0 ** rng.uniform(-3, 3, (ch, 1))).astype(np.complex64)
    X[7, 100] = np.nan; X[9, 50] = np.inf
    taps = cb.firdes_lowpass_f(T, 0.5 / I)
    y = cb.fir_interpolate_bank(torch.from_numpy(X).cuda(), I, taps).cpu().numpy()
    assert y.shape == (ch, tx.groups(n, I, T) * I)
    for c in list(range(0, ch, 61)) + [7, 9, ch - 1]:
        assert same_bits(y[c], tx.fir_interpolate_cc(X[c], I, taps)), c
    if tx.have_ref():
        for c in (0, 500, ch - 1):
            want = tx.ref_fir_interpolate_cc(X[c], I, taps)
            bi, bq = tx.interp_bound(X[c], I, taps)
            assert np.all(np.abs(y[c].real.astype(np.float64) - want.real) <= bi) and np.all(np.abs(y[c].imag.astype(np.float64) - want.imag) <= bq)


def test_interp_long_row_and_carry(cuda):
    """2^24 outputs in one row, and the same row cut into calls that keep the unconsumed inputs"""
    torch, cb = cuda
    I, T = 50, 401
    keep = (T - 1 + I - 1) // I
    n = -(-(1 << 24) // I) + keep
    rng = np.random.default_rng(11)
    X = (rng.standard_normal((1, n)) + 1j * rng.standard_normal((1, n))).astype(np.complex64)
    taps = cb.firdes_lowpass_f(T, 0.5 / I)
    xd = torch.from_numpy(X).cuda()
    whole = cb.fir_interpolate_bank(xd, I, taps)
    assert whole.shape[1] >= 1 << 24
    parts, pos = [], 0
    while pos + keep < n:
        k = min(n - pos, keep + int(rng.integers(1, 60000)))
        p = cb.fir_interpolate_bank(xd[:, pos:pos + k].contiguous(), I, taps)
        parts.append(p); pos += p.shape[1] // I
    assert torch.equal(torch.cat(parts, dim=1).view(torch.float32), whole.view(torch.float32))
    for s in (0, 12345 * I, whole.shape[1] - 4000):
        seg = tx.fir_interpolate_cc(X[0, s // I:s // I + 80 + keep], I, taps)
        assert same_bits(whole[0, s:s + 80 * I].cpu().numpy(), seg[:80 * I]), s


def test_fmmod_bank_at_1024_channels(cuda):
    torch, cb = cuda
    ch, n = 1024, 2000
    rng = np.random.default_rng(12)
    X = rng.uniform(-1, 1, (ch, n)).astype(np.float32)
    X[::3] *= 9.0                                                    # several wraps per sample
    xd = torch.from_numpy(X).cuda()
    ph = torch.zeros(ch, dtype=torch.float32, device="cuda")
    y = torch.cat([cb.fmmod_bank(xd[:, a:b].contiguous(), ph) for a, b in ((0, 1), (1, 700), (700, 700), (700, n))], dim=1).cpu().numpy()
    phc = ph.cpu().numpy()
    for c in list(range(0, ch, 97)) + [ch - 1]:
        phases = tx.fmmod_phases(X[c])
        assert phc[c] == phases[-1], c
        assert np.abs(y[c] - np.exp(1j * phases.astype(np.float64))).max() < 1e-7, c
        if tx.have_ref():
            want, last = tx.ref_fmmod_fc(X[c])
            assert last == phc[c] and np.abs(y[c].view(np.float32) - want.view(np.float32)).max() <= ULP1, c


def test_tone_loopback(cuda):
    """audio tones -> fmmod_bank -> fir_interpolate_bank 50x -> a polar discriminator at the wide rate recovers each tone (correlation > 0.99)"""
    torch, cb = cuda
    ch, n, I = 8, 4800, 50
    t = np.arange(n) / 48000.0
    freqs = 400.0 + 150.0 * np.arange(ch)
    audio = (0.05 * np.sin(2 * np.pi * freqs[:, None] * t)).astype(np.float32)
    iq = cb.fmmod_bank(torch.from_numpy(audio).cuda())
    taps = cb.firdes_lowpass_f(8 * I + 1, 0.5 / I)
    wide = cb.fir_interpolate_bank(iq.contiguous(), I, taps).cpu().numpy().astype(np.complex128)
    d = np.angle(wide[:, 1:] * np.conj(wide[:, :-1]))                    # per wide sample: audio * PI / I
    rec = d[:, ::I][:, 200:-200] * I / np.pi
    for c in range(ch):
        best = max(np.corrcoef(rec[c], np.roll(audio[c], -k)[200:200 + rec.shape[1]])[0, 1] for k in range(0, 12))
        assert best > 0.99, (c, best)
