"""GPU tests (-m gpu) of the BPSK31 transmit banks (csdr_b200/csrc/psk31_tx.cu): the checks of tests/psk31_tx/psk31_tx.py at full size --
1024 channels x 64 KiB of text through the encoder, 1024 channels x 2^20 bits through the codec, the whole modulator grid, every rate table up to
I = 8192, 1024 channels x 48 000 symbols at I = 256 through the interpolator -- and a loopback made only of the project's code: text -> the four banks -> synth_bank -> csdr-bankd --tail bpsk31 -> the same text.

The checks run once, together, under torch.profiler (the `profiled` fixture), and every kernel instantiation must be seen launching there.  A
profiler session around a handful of small launches alone is not enough: in a process that has run profiler sessions before, such a session
has been seen to return the runtime calls with only the last of its kernel records."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "psk31_tx"))
import psk31_tx as T  # noqa: E402

pytestmark = pytest.mark.gpu
KERNELS = ("varicode_encoder_bank_kernel", "differential_codec_bank_kernel<true>", "differential_codec_bank_kernel<false>",
           "psk_modulator_bank_kernel", "psk31_interpolate_sine_bank_kernel<true>", "psk31_interpolate_sine_bank_kernel<false>",
           "psk31_interpolate_sine_last_kernel")


@pytest.fixture(scope="module")
def drv():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    if not T.have_ref():
        pytest.fail("oracle/_ref/libcsdr_ref.so not built")
    import csdr_b200
    return T.GpuDriver(csdr_b200)


def check_encoder_full_size(drv):
    rng = np.random.default_rng(1)
    text = T.text_rows(rng, 1024, 65536)
    bits, ip, os_ = T.encoder_bank(drv, text)
    for c in range(1024):
        rb, rip, ros = T.ref_varicode_encode(text[c], 12 * 65536)
        assert (int(ip[c]), int(os_[c])) == (rip, ros) and np.array_equal(bits[c, :ros], rb), c
    T.check_encoder(drv, text[:8, :3000], lengths=[0, 1, 1024, 1025, 2999, 3000, 5, 77])
    T.check_encoder(drv, text[:4, :500], output_max_size=2000)


def check_codec_full_size(drv):
    import csdr_b200
    rng = np.random.default_rng(2)
    x = rng.integers(0, 2, (1024, 1 << 20)).astype(np.uint8)
    d_x = torch.from_numpy(x).cuda()
    for encode in (1, 0):
        st0 = torch.from_numpy(rng.integers(0, 3, 1024).astype(np.uint8)).cuda()
        s0 = st0.cpu().numpy().copy()
        out, st = csdr_b200.differential_codec_bank_u8_u8(d_x, encode, state=st0)
        out, st = out.cpu().numpy(), st.cpu().numpy()
        for c in range(0, 1024, 37):
            ro, rs = T.ref_differential_codec(x[c], encode, int(s0[c]))
            assert np.array_equal(out[c], ro) and int(st[c]) == rs, (encode, c)


def check_interpolator(drv, I):
    rng = np.random.default_rng(I)
    n = max(3, 20000 // I)
    x = T.with_specials((rng.standard_normal((5, n)) + 1j * rng.standard_normal((5, n))).astype(np.complex64), rng, 1)
    T.check_interp(drv, x, I, np.array([0, 1 - 1j, np.nan, 2, np.inf], np.complex64), lengths=[n, 0, n - 1, 1, n])


INTERP_I = (1, 2, 3, 7, 256, 1000, 9001)                                 # 9001: the rates copied per tile (I > 8192)
# run in this order: the rate tables' 16 384 launches come first, so that no kernel is seen only at the very start of the session
CHECKS = {"rates": (T.check_rates, range(1, 8193)), "encoder": (check_encoder_full_size,), "codec": (check_codec_full_size,),
          "modulator": (T.check_modulator_grid,), "refusals": (T.refusals,), **{f"interp {I}": (check_interpolator, I) for I in INTERP_I}}


@pytest.fixture(scope="module")
def profiled(drv):
    """every check of CHECKS once, the whole set under torch.profiler -> ({name: None or the failure}, kernel names launched)"""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, (fn, *args) in CHECKS.items():
            try:
                fn(drv, *args)
                res[name] = None
            except AssertionError as e:
                res[name] = e
        torch.cuda.synchronize()
    names = set()
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                names.add(k)
    return res, names


def _outcome(profiled, name):
    if profiled[0][name] is not None:
        raise profiled[0][name]


def test_encoder_full_size(profiled):
    _outcome(profiled, "encoder")


def test_codec_full_size(profiled):
    _outcome(profiled, "codec")


def test_modulator_grid(profiled):
    _outcome(profiled, "modulator")


def test_rate_tables_up_to_8192(profiled):
    _outcome(profiled, "rates")


@pytest.mark.parametrize("I", INTERP_I)
def test_interpolator_against_reference(profiled, I):
    _outcome(profiled, f"interp {I}")


def test_refusals(profiled):
    _outcome(profiled, "refusals")


def test_every_kernel_launches(profiled):
    """each kernel instantiation is seen launching in the profiled run of the checks"""
    missing = [k for k in KERNELS if k not in profiled[1]]
    assert not missing, (missing, sorted(profiled[1]))


def test_interpolator_full_size(drv):
    """1024 channels x 48 000 symbols at I = 256, in slices of 16 channels (100 GB of output in all), each slice against the same arithmetic
    in torch (separate float32 multiplies and adds) with the build's rate table"""
    import csdr_b200
    I, n = 256, 48000
    r = torch.from_numpy(T.ref_rates(I)).cuda()
    omr = 1 - r
    g = torch.Generator(device="cuda").manual_seed(3)
    for c0 in range(0, 1024, 16):
        x = torch.randn((16, n), dtype=torch.complex64, device="cuda", generator=g)
        last0 = torch.randn(16, dtype=torch.complex64, device="cuda", generator=g)
        y, last = csdr_b200.psk31_interpolate_sine_bank_cc(x, I, last=last0.clone())
        prev = torch.cat([last0[:, None], x[:, :-1]], 1)
        for k, comp in enumerate((torch.real, torch.imag)):
            want = comp(x)[:, :, None] * r + comp(prev)[:, :, None] * omr
            assert torch.equal(torch.view_as_real(y).reshape(16, n, I, 2)[..., k], want), c0
        assert torch.equal(last, x[:, -1])
        del y, x, prev


def modulate_texts(texts, sps, lead=64, tail=160):
    """text -> the four banks: varicode, lead/tail zero bits (idle reversals), differential encoder, BPSK, sine interpolation"""
    import csdr_b200
    ch, n = len(texts), max(len(t) for t in texts)
    rows = np.zeros((ch, n), np.uint8)
    for c, t in enumerate(texts):
        rows[c, :len(t)] = np.frombuffer(t, np.uint8)
    bits, _, size = csdr_b200.psk31_varicode_encoder_bank_u8_u8(torch.from_numpy(rows).cuda(),
                                                                lengths=torch.tensor([len(t) for t in texts], dtype=torch.int32, device="cuda"))
    size = size.cpu().numpy()
    m = lead + int(size.max()) + tail
    framed = torch.zeros((ch, m), dtype=torch.uint8, device="cuda")
    for c in range(ch):
        framed[c, lead:lead + int(size[c])] = bits[c, :int(size[c])]
    diff, _ = csdr_b200.differential_codec_bank_u8_u8(framed, True)
    sym = csdr_b200.psk_modulator_bank_u8_c(diff, 2)
    base, _ = csdr_b200.psk31_interpolate_sine_bank_cc(sym, sps)
    return (base * 0.25).contiguous()


TEXTS = (b"CQ de GPU one k", b"second channel 73", b"third: QRM?")
RATES = (-0.3, 0.05, 0.25)
PREFIX = b"vvv vvv "          # characters the receiver may spend on locking its symbol clock, as an operator sends before a call


def loopback(tmp_path, I, sps, bw, fmt):
    import csdr_b200
    base = modulate_texts([PREFIX + t for t in TEXTS], sps)
    taps = csdr_b200.firdes_lowpass_f(csdr_b200.firdes_filter_len(bw), 0.5 / I) * I        # unit gain through the interpolation by I
    wide, _ = csdr_b200.synth_bank(base, RATES, I, taps)
    # a little noise: on a noiseless signal the receiver's Gardner loop can settle between symbols
    rng = np.random.default_rng(I)
    z = wide.cpu().numpy() + 0.01 * (rng.standard_normal(wide.numel()) + 1j * rng.standard_normal(wide.numel()))
    if fmt == "f32":
        data = z.astype(np.complex64).tobytes()
    else:
        iq = np.empty(2 * z.size); iq[0::2] = z.real; iq[1::2] = z.imag
        data = np.clip(np.floor(iq * 127.5 + 128), 0, 255).astype(np.uint8).tobytes()
    sinks = [tmp_path / f"{fmt}{I}_{k}.txt" for k in range(3)]
    cmd = [str(ROOT / "csdr_b200" / "csdr-bankd"), f"--{fmt}", "--decimation", str(I), "--bw", str(bw), "--tail", "bpsk31", "--sps", str(sps),
           "--block", "16384"]                                               # several blocks even for the short f32 stream
    r = subprocess.run(cmd + [f"{-rt}:{p}" for rt, p in zip(RATES, sinks)], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = [p.read_bytes() for p in sinks]
    for k, g in enumerate(got):
        assert TEXTS[k] in g, (k, got)
        assert not any(TEXTS[j] in g for j in range(3) if j != k), (k, g)


def test_loopback_through_the_synthesis_bank_and_bankd(tmp_path):
    loopback(tmp_path, 10, 32, 0.05, "f32")


def test_loopback_at_the_skimmer_geometry(tmp_path):
    loopback(tmp_path, 300, 256, 0.001, "u8")
