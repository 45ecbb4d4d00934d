"""GPU parity tests (-m gpu) for the NFM audio tail of SURVEY 8(f) rank 1: deemphasis_nfm_ff (fixed FIRs, libcsdr.c:1099-1128) as the
libcsdr drop-in and as a bank with the preceding limit_ff fused in.  (CLI command and the README.md:87 graph: test_gpu_cli.py.)"""
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
GOLD = np.load(Path(__file__).parent / "golden" / "hotpath_golden.npz")
RATES = (48000, 44100, 11025, 8000)
TOL = 1e-5                                                               # north-star bar for float blocks (relative RMS)


@pytest.fixture(scope="module")
def gpu():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    csdr_b200.lib()
    return csdr_b200


def _rel(y, ref):
    from oracle.pyoracle import rel_rms
    return rel_rms(y, ref)


@pytest.mark.parametrize("rate", RATES)
def test_deemphasis_nfm_dropin_golden_and_oracle(gpu, oracle, rate):
    taps = GOLD[f"nfm_taps_{rate}"]
    y = gpu.libcsdr.deemphasis_nfm_ff(GOLD["nfm_in"], rate)
    assert y.size == GOLD["nfm_in"].size - taps.size == GOLD[f"nfm_out_{rate}"].size
    assert _rel(y, GOLD[f"nfm_out_{rate}"]) < TOL                        # the compiled reference (-ffast-math reduction order)
    assert _rel(y, oracle.deemphasis_nfm_ff(GOLD["nfm_in"], taps)) < 1e-6  # strict oracle: same order, only FMA contraction differs
    rng = np.random.default_rng(rate)
    for n in (taps.size + 1, taps.size + 1024, taps.size + 1025, 16384, 50_001):     # tile edges of the kernel (1024 outputs per CTA)
        x = rng.uniform(-1, 1, n).astype(np.float32)
        y = gpu.libcsdr.deemphasis_nfm_ff(x, rate)
        want = oracle.deemphasis_nfm_ff(x, taps)
        assert y.size == want.size == n - taps.size
        # each output is a ~200-term sum with cancellation: bound the error by the size of the terms, not of the (possibly tiny) result
        assert np.abs(y - want).max() <= 1e-6 * np.abs(taps).sum(), n
        if n >= 4096:
            assert _rel(y, want) < 1e-6, n


def test_deemphasis_nfm_dropin_degenerate_calls(gpu):
    x = np.ones(4096, np.float32)
    assert gpu.libcsdr.deemphasis_nfm_ff(x, 12345).size == 0            # no table for this rate -> 0 samples processed (libcsdr.c:1119)
    assert gpu.libcsdr.deemphasis_nfm_ff(x[:201], 48000).size == 0      # input_size == taps_length -> the reference loop does not run
    assert gpu.libcsdr.deemphasis_nfm_ff(x[:100], 48000).size == 0


def test_deemphasis_nfm_degenerate_calls(gpu):
    d = torch.ones((3, 4096), dtype=torch.float32, device="cuda")
    assert gpu.deemphasis_nfm_bank_ff(d, 22050).shape == (3, 0)


def test_deemphasis_nfm_bank_with_fused_limit(gpu, oracle):
    rng = np.random.default_rng(77)
    ch, n = 37, 48_000 + 201
    x = rng.uniform(-2.5, 2.5, (ch, n)).astype(np.float32)
    x[3, 17] = np.nan; x[5, 1000] = np.inf; x[6, 2000] = -np.inf       # limit_ff of the reference build: NaN -> +max
    dx = torch.from_numpy(x).cuda()
    taps = GOLD["nfm_taps_48000"]
    y = gpu.deemphasis_nfm_bank_ff(dx, 48000, limit_max=1.0).cpu().numpy()
    assert y.shape == (ch, n - taps.size)
    for c in range(ch):
        assert _rel(y[c], oracle.deemphasis_nfm_ff(oracle.limit_ff(x[c], 1.0), taps)) < 1e-6, c
    # strided rows, no limiter, another table
    wide = torch.zeros((ch, n + 64), dtype=torch.float32, device="cuda")
    xs = rng.uniform(-1, 1, (ch, n)).astype(np.float32)
    wide[:, :n] = torch.from_numpy(xs).cuda()
    y = gpu.deemphasis_nfm_bank_ff(wide[:, :n], 11025).cpu().numpy()
    for c in (0, 1, ch - 1):
        assert _rel(y[c], oracle.deemphasis_nfm_ff(xs[c], GOLD["nfm_taps_11025"])) < 1e-6

    # caller-supplied taps through the same kernel (odd length, maximum length, one tap)
    for T in (1, 77, 208):
        taps = rng.uniform(-1, 1, T).astype(np.float32)
        y = gpu.fir_valid_bank_ff(dx[:5], taps).cpu().numpy()
        assert y.shape == (5, n - T)
        xl = np.nan_to_num(x[4], nan=0.0, posinf=0.0, neginf=0.0)
        assert _rel(gpu.fir_valid_bank_ff(torch.from_numpy(xl[None]).cuda(), taps).cpu().numpy()[0], oracle.deemphasis_nfm_ff(xl, taps)) < 1e-6, T
    with pytest.raises(gpu.CsdrB200Error):
        gpu.fir_valid_bank_ff(dx[:1], np.ones(209, np.float32))


def test_readme_nfm_graph_as_a_bank(gpu, oracle):
    """README.md:87 for a whole bank, audio leaving the GPU as s16: fused shift|fir_decimate 50|fmdemod kernel -> limit fused into the
    de-emphasis FIR -> fastagc -> convert_f_s16, against the oracle running the seven blocks one channel at a time."""
    D, T = 50, 801
    taps = gpu.firdes_lowpass_f(T, 0.5 / D)
    N = 1_200_000
    rng = np.random.default_rng(123)
    t = np.arange(N)
    rates = np.array([-0.41, -0.2, 0.03, 0.27, 0.44], np.float32)
    audio = [np.sin(2 * np.pi * (700.0 + 300 * k) / 2.4e6 * t) for k in range(rates.size)]
    wide = sum(0.18 * np.exp(1j * (2 * np.pi * (-float(r)) * t + np.cumsum(2 * np.pi * 3000.0 / 2.4e6 * audio[k]))) for k, r in enumerate(rates))
    wide = (wide + 0.002 * (rng.normal(size=N) + 1j * rng.normal(size=N))).astype(np.complex64)
    demod, _, _ = gpu.ddc_bank(torch.from_numpy(wide).cuda(), rates, D, taps, demod=True, chunk=1024)
    deemph = gpu.deemphasis_nfm_bank_ff(demod, 48000, limit_max=1.0)
    agc, _, _ = gpu.fastagc_bank_ff(deemph, 1024, 1.0)
    pcm = gpu.convert_f_s16(agc.contiguous()).cpu().numpy()
    agc = agc.cpu().numpy()
    nfm_taps = GOLD["nfm_taps_48000"]
    for c, r in enumerate(rates):
        sh, _ = oracle.shift_addition_cc(wide, float(r), 0.0, 1024)
        d = oracle.fmdemod_quadri_cf(oracle.fir_decimate_cc(sh, D, taps))[0]
        want = oracle.fastagc_ff(oracle.deemphasis_nfm_ff(oracle.limit_ff(d, 1.0), nfm_taps), 1024, 1.0)
        assert agc[c].size == want.size and want.size >= 22 * 1024
        assert _rel(agc[c], want) < TOL, (c, _rel(agc[c], want))
        assert np.abs(pcm[c].astype(np.int32) - oracle.convert_f_s16(want).astype(np.int32)).max() <= 1
