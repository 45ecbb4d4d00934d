"""GPU tests (-m gpu) of the amplitude modulator banks (csdr_b200/csrc/modulate.cu) and of `csdr-synth --mod`:
- the four banks at 1024 channels x 480 000 samples through the Python API: gain_ff, dsb_fc and add_dcoffset_cc bit for bit against the
  restatements of tests/modulate/modulate.py (and, with the compiled reference, against the build), fixed_amplitude_cc bit for bit against its
  restatement and within the float64 bound; in-place calls; the refusals on device pointers;
- the real csdr-synth binary against SynthBank over the Python banks composed, byte for byte, for every mode;
- loopbacks made of the project's own programs: 4 tones between 1.5 and 3.3 kHz (48 kHz audio, I = 50, 2.4 Msps) through csdr-synth --mod X, then
  csdr-bankd --f32 --decimation 50 --bw 0.005 with the matching tail; each channel's audio peaks at its own tone with the others at least 40 dB
  down; and USB / LSB received as IQ keep the unwanted image at least 40 dB below the wanted tone (the Hamming filter gives about 56 dB at 1.5 kHz)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "modulate"))
import modulate as M  # noqa: E402

pytestmark = pytest.mark.gpu
SYNTH = ROOT / "csdr_b200" / "csdr-synth"
BANKD = ROOT / "csdr_b200" / "csdr-bankd"
CH, N = 1024, 480_000
ROWS = list(range(0, CH, 97)) + [CH - 1]
SSB_BAND = {"usb": (0.0, 0.1), "lsb": (-0.1, 0.0)}


@pytest.fixture(scope="module")
def cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    return torch, csdr_b200


def big_rows(torch, name, seed):
    """[CH, N] rows made on the device (uniform in (-1, 1), or 12 decades of magnitude at every angle for fixed_amplitude_cc), with the special
    values of tests/modulate/modulate.py in the first 1000 samples of the checked rows; returns the device rows and the checked rows on the host"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if M.BANKS[name][0] is np.float32:
        x = torch.rand((CH, N), generator=g, device="cuda") * 2 - 1
    elif name == "fixed_amplitude":
        mag = 10.0 ** (torch.rand((CH, N), generator=g, device="cuda") * 12 - 6)
        x = torch.polar(mag, (torch.rand((CH, N), generator=g, device="cuda") * 2 - 1) * np.pi)
    else:
        x = torch.complex(torch.rand((CH, N), generator=g, device="cuda") * 2 - 1, torch.rand((CH, N), generator=g, device="cuda") * 2 - 1)
    rng = np.random.default_rng(seed)
    for r in ROWS:
        x[r, :1000] = torch.from_numpy(M.rows_for(name, rng, 1, 1000)[0]).cuda()
    return x, x[ROWS].cpu().numpy()


def bits(t):
    import torch
    return (torch.view_as_real(t) if t.is_complex() else t).view(torch.int32)


def bank(cb, name, xd, arg, out=None):
    if name == "gain":
        return cb.gain_bank(xd, arg, out=out)
    if name == "dsb":
        return cb.dsb_bank(xd, arg)
    if name == "add_dcoffset":
        return cb.add_dcoffset_bank(xd, out=out)
    return cb.fixed_amplitude_bank(xd, arg, out=out)


@pytest.mark.parametrize("name,arg", [("gain", -1.7), ("dsb", 0.25), ("add_dcoffset", 0.0), ("fixed_amplitude", 2.0)])
def test_banks_at_1024_channels(cuda, name, arg):
    torch, cb = cuda
    xd, x = big_rows(torch, name, len(name))
    y = bank(cb, name, xd, arg)
    got = y[ROWS].cpu().numpy()
    for k, r in enumerate(ROWS):
        assert M.same_bits(got[k], M.restate(name, x[k], arg)), (name, r)
        if name == "fixed_amplitude":
            M.fixed_amplitude_ok(got[k], x[k], arg, M.ref_call(name, x[k], arg) if M.have_ref() else None)
        elif M.have_ref():
            assert M.same_bits(got[k], M.ref_call(name, x[k], arg)), (name, r)
    if name != "dsb":                                                    # in place over the whole bank gives the same bits
        bank(cb, name, xd, arg, out=xd)
        assert torch.equal(bits(xd), bits(y)), name


def test_refusals_on_the_device(cuda):
    torch, cb = cuda
    lib = M.bind(cb.lib())
    d_in = torch.zeros(64, dtype=torch.complex64, device="cuda"); d_out = torch.full((64,), 7.0, dtype=torch.complex64, device="cuda")
    torch.cuda.synchronize()
    before = lib.csdrb_kernel_launches()
    assert M.refusals(lib, d_in.data_ptr(), d_out.data_ptr()) == []
    torch.cuda.synchronize()
    assert lib.csdrb_kernel_launches() == before and torch.all(d_out == 7.0)


# ---- csdr-synth --mod -----------------------------------------------------------------------------------------------------------------------
def composed(torch, cb, mode, audio, gain):
    """the Python banks of the mode on [C, n] f32 audio -> [C, m] complex baseband"""
    a = cb.gain_bank(torch.from_numpy(audio).cuda(), gain)
    if mode == "fm":
        return cb.fmmod_bank(a)
    bb = cb.dsb_bank(a)
    if mode == "am":
        return cb.add_dcoffset_bank(bb, out=bb)
    if mode in SSB_BAND:
        _, _, unit, _ = cb.bandpass_geometry(0.05)
        m = bb.shape[1] // unit * unit
        y, _ = cb.bandpass_fir_fft_bank_cc(bb[:, :m].contiguous(), cb.bandpass_taps_fft(*SSB_BAND[mode], 0.05), unit)
        return y
    return bb


@pytest.mark.parametrize("mode", ["am", "dsb", "usb", "lsb", "fm"])
def test_csdr_synth_mod_equals_the_composed_banks(cuda, tmp_path, mode):
    torch, cb = cuda
    rng = np.random.default_rng(len(mode))
    lengths, rates, gain = [30_000, 21_111, 25_000], [-0.2, 0.0, 0.15], 0.8
    srcs = [rng.uniform(-1, 1, m).astype(np.float32) for m in lengths]
    for k, s in enumerate(srcs):
        s.tofile(tmp_path / f"a{k}.f32")
    for block in (1000, 16384):
        r = subprocess.run([str(SYNTH), "--interpolation", "50", "--block", str(block), "--mod", mode, "--gain", str(gain)] +
                           [f"{rates[k]}:{tmp_path / f'a{k}.f32'}" for k in range(3)], capture_output=True, timeout=600)
        assert r.returncode == 0, r.stderr.decode()
        L = min(lengths)
        bb = composed(torch, cb, mode, np.stack([s[:L] for s in srcs]), gain)
        sb = cb.SynthBank(rates, 50, cb.firdes_lowpass_f(cb.firdes_filter_len(0.05), 0.5 / 50))
        try:
            want = sb.process(bb.contiguous()).cpu().numpy()
        finally:
            sb.close()
        assert want.size > 0 and r.stdout == want.tobytes(), (mode, block, len(r.stdout), want.nbytes)


# ---- loopbacks through csdr-bankd ---------------------------------------------------------------------------------------------------------
TONES = np.array([1500.0, 2100.0, 2700.0, 3300.0])
RATES = [-0.3, -0.1, 0.1, 0.3]
FS = 48_000


def loopback(tmp_path, mode, tail, gain, seconds=1.0):
    n = int(FS * seconds)
    t = np.arange(n) / FS
    for k, f in enumerate(TONES):
        (0.5 * np.sin(2 * np.pi * f * t)).astype(np.float32).tofile(tmp_path / f"t{k}.f32")
    wide = subprocess.run([str(SYNTH), "--interpolation", "50", "--mod", mode, "--gain", str(gain)] +
                          [f"{r}:{tmp_path / f't{k}.f32'}" for k, r in enumerate(RATES)], capture_output=True, timeout=600)
    assert wide.returncode == 0, wide.stderr.decode()
    ext = "cf32" if tail == "iq" else "s16"
    sinks = [tmp_path / f"rx{k}.{ext}" for k in range(len(RATES))]
    rx = subprocess.run([str(BANKD), "--f32", "--decimation", "50", "--bw", "0.005", "--tail", tail] + [f"{-r}:{p}" for r, p in zip(RATES, sinks)],
                        input=wide.stdout, capture_output=True, timeout=600)
    assert rx.returncode == 0, rx.stderr.decode()[-2000:]
    return [np.fromfile(p, np.complex64 if tail == "iq" else np.int16) for p in sinks]


def spectrum_db(x, two_sided=False):
    x = np.asarray(x, np.complex128 if two_sided else np.float64)
    x = x[x.size // 4:]                                                 # past the AGC's and the filters' start
    s = np.abs(np.fft.fft(x * np.hanning(x.size)) if two_sided else np.fft.rfft(x * np.hanning(x.size)))
    return 20 * np.log10(s + 1e-30), x.size


def level(spec, size, f):
    k = int(round(f / FS * size))
    return spec[k - 3:k + 4].max()


@pytest.mark.parametrize("mode,tail,gain", [("am", "am", 1.0), ("usb", "usb", 1.0), ("dsb", "usb", 1.0), ("lsb", "lsb", 1.0), ("fm", "nfm", 0.1)])
def test_loopback_each_channel_hears_its_own_tone(cuda, tmp_path, mode, tail, gain):
    audio = loopback(tmp_path, mode, tail, gain)
    for c, a in enumerate(audio):
        assert a.size > FS // 2, (mode, c, a.size)
        spec, size = spectrum_db(a.astype(np.float64))
        band = slice(int(300 / FS * size), int(6000 / FS * size))
        peak = band.start + int(np.argmax(spec[band]))
        assert abs(peak * FS / size - TONES[c]) < 20, (mode, c, peak * FS / size)
        for j, f in enumerate(TONES):
            if j != c:
                assert level(spec, size, f) <= spec[peak] - 40, (mode, c, j, spec[peak] - level(spec, size, f))


@pytest.mark.parametrize("mode", ["usb", "lsb"])
def test_sideband_image_is_40_db_down(cuda, tmp_path, mode):
    bb = loopback(tmp_path, mode, "iq", 1.0)
    sign = 1 if mode == "usb" else -1
    for c, x in enumerate(bb):
        spec, size = spectrum_db(x, two_sided=True)
        wanted = level(spec, size, (sign * TONES[c]) % FS)
        image = level(spec, size, (-sign * TONES[c]) % FS)
        assert wanted - image >= 40, (mode, c, wanted - image)
