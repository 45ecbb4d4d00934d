"""GPU tests (-m gpu) of the synthesis bank through the Python API: against the project's own banks composed (fir_interpolate_bank, then
shift_addition_bank_cc with its chunks of 1024, then the pairwise channel tree restated with float32 adds) bit for bit at one channel, at 1024
channels x 48 000 inputs (I = 50, T = 401) and on one channel of 2^24 outputs; the streaming object against the one-shot call; and a loopback
through the receive side: three FM tones modulated (fmmod_bank), synthesised at three rates, received by DdcBank at -rate with the discriminator,
each channel peaking at its own tone with the others at least 40 dB below."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


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


def tree_(torch, Y):
    """the pairwise tree over dim 0 in place (float32 adds per component); returns the root row"""
    C, s = Y.shape[0], 1
    while s < C:
        for b in range(0, C - s, 2 * s):
            Y[b] += Y[b + s]
        s *= 2
    return Y[0]


def composed(torch, cb, x, rates, I, taps):
    """the existing banks: fir_interpolate_bank, shift_addition_bank_cc (chunk 1024), summed by the tree"""
    W = cb.fir_interpolate_bank(x, I, taps)
    Y, _ = cb.shift_addition_bank_cc(W.contiguous(), rates, chunk=1024)
    return tree_(torch, Y)


def rows(torch, rng, ch, n):
    return torch.from_numpy((rng.uniform(-1, 1, (ch, n)) + 1j * rng.uniform(-1, 1, (ch, n))).astype(np.complex64)).cuda()


@pytest.mark.parametrize("I,T", [(1, 81), (5, 41), (50, 401), (3, 100)])
def test_one_channel_is_the_composed_banks(cuda, I, T):
    torch, cb = cuda
    rng = np.random.default_rng(I)
    x = rows(torch, rng, 1, 5000)
    taps = cb.firdes_lowpass_f(T, 0.5 / I)
    y, _ = cb.synth_bank(x, [0.0831], I, taps)
    want = composed(torch, cb, x, [0.0831], I, taps)
    torch.cuda.synchronize()
    assert same_bits(y.cpu().numpy(), want.cpu().numpy())


def test_1024_channels_flagship(cuda):
    """1024 channels x 48 000 inputs, I = 50, T = 401: the composition per batch of 128 channels (an aligned block of the tree), then the tree
    over the eight batch nodes"""
    torch, cb = cuda
    rng = np.random.default_rng(7)
    ch, n, I, T = 1024, 48_000, 50, 401
    x = rows(torch, rng, ch, n)
    rates = rng.uniform(-0.49, 0.49, ch).astype(np.float32)
    taps = cb.firdes_lowpass_f(T, 0.5 / I)
    y, ph = cb.synth_bank(x, rates, I, taps)
    nodes = []
    for b in range(0, ch, 128):
        nodes.append(composed(torch, cb, x[b:b + 128], rates[b:b + 128], I, taps).clone())
        torch.cuda.empty_cache()
    want = tree_(torch, torch.stack(nodes))
    torch.cuda.synchronize()
    assert y.numel() == (n - 8) * I
    assert same_bits(y.cpu().numpy(), want.cpu().numpy())


def test_one_channel_of_2_24_outputs(cuda):
    torch, cb = cuda
    rng = np.random.default_rng(24)
    I, T = 256, 2049
    x = rows(torch, rng, 1, (1 << 16) + 8)
    taps = cb.firdes_lowpass_f(T, 0.5 / I)
    y, _ = cb.synth_bank(x, [-0.3], I, taps)
    assert y.numel() == 1 << 24
    want = composed(torch, cb, x, [-0.3], I, taps)
    torch.cuda.synchronize()
    assert same_bits(y.cpu().numpy(), want.cpu().numpy())


def test_streaming_equals_one_shot(cuda):
    torch, cb = cuda
    rng = np.random.default_rng(5)
    ch, I, T, total = 300, 50, 401, 20_000
    x = rows(torch, rng, ch, total)
    rates = rng.uniform(-0.49, 0.49, ch).astype(np.float32)
    taps = cb.firdes_lowpass_f(T, 0.5 / I)
    whole, _ = cb.synth_bank(x, rates, I, taps)
    bank = cb.SynthBank(rates, I, taps)
    got, pos, h = [], 0, (T - 1 + I - 1) // I
    try:
        while pos + h < total:
            n = min(total - pos, int(rng.integers(1, 3000)))
            out = bank.process(x[:, pos:pos + n].contiguous())
            got.append(out.clone())
            pos += out.numel() // I
    finally:
        bank.close()
    torch.cuda.synchronize()
    assert same_bits(torch.cat(got).cpu().numpy(), whole.cpu().numpy())


def test_loopback_through_the_receive_bank(cuda):
    torch, cb = cuda
    I, T, n = 50, 401, 40_000
    tones = np.array([0.011, 0.017, 0.029])                      # cycles per baseband sample
    rates = np.array([0.1, -0.15, 0.3], np.float32)              # cycles per wideband sample
    t = np.arange(n)
    audio = np.stack([0.2 * np.sin(2 * np.pi * f * t) for f in tones]).astype(np.float32)
    bb = cb.fmmod_bank(torch.from_numpy(audio).cuda())
    taps = cb.firdes_lowpass_f(T, 0.5 / I)
    wide, _ = cb.synth_bank(bb.contiguous(), rates, I, taps)
    rx = cb.DdcBank(-rates, I, taps, demod=True)
    try:
        dem = rx.process(wide).cpu().numpy()
    finally:
        rx.close()
    for c in range(3):
        s = dem[c, 2000:]
        spec = np.abs(np.fft.rfft(s * np.hanning(s.size)))
        bins = [int(round(f * s.size)) for f in tones]
        peak = [spec[max(b - 3, 0):b + 4].max() for b in bins]
        assert int(np.argmax(spec[5:])) + 5 in range(bins[c] - 3, bins[c] + 4), (c, int(np.argmax(spec[5:])) + 5, bins)
        for k in range(3):
            if k != c:
                assert 20 * np.log10(peak[k] / peak[c]) <= -40, (c, k, 20 * np.log10(peak[k] / peak[c]))
