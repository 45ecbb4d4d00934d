"""CPU tier of `csdr-synth --mod` (csdr_b200/host/programs/synth.c) linked against the emulated library: for every mode its stdout equals, byte for
byte, the modulator banks composed through the emulated C ABI (gain_ff, then dsb_fc [| add_dcoffset_cc], dsb_fc | bandpass_fir_fft_cc or
fmmod_fc) and then the synthesis bank on the streams cut to the shortest source (for usb/lsb to whole filter units), for sources of unequal
lengths and two --block sizes, one of them not a multiple of the filter unit; and --gain without --mod or an unknown mode is refused."""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "synth"))
sys.path.insert(0, str(ROOT / "tests" / "modulate"))
sys.path.insert(0, str(ROOT))
import emul_build  # noqa: E402
import modulate as M  # noqa: E402
import synth  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402

SSB_BAND = {"usb": (0.0, 0.1), "lsb": (-0.1, 0.0)}


@pytest.fixture(scope="module")
def prog(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _ = emul_build.build_full_once(tmp_path_factory)
    exe = tmp_path_factory.mktemp("synth_mod_emul") / "csdr-synth_emul"
    subprocess.run(["gcc", "-std=gnu99", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "csdr_b200" / "host" / "programs" / "synth.c"), "-o",
                    str(exe), f"-L{lib.parent}", "-lcsdr_b200_emul", "-lm", f"-Wl,-rpath,{lib.parent}"], check=True, capture_output=True)
    L = M.bind(C.CDLL(str(lib)))
    vp, lg, it = C.c_void_p, C.c_long, C.c_int
    L.firdes_filter_len.argtypes = [C.c_float]; L.firdes_filter_len.restype = it
    L.firdes_lowpass_f.argtypes = [vp, it, C.c_float, it]
    L.firdes_bandpass_c.argtypes = [vp, it, C.c_float, C.c_float, it]
    L.next_pow2.argtypes = [it]; L.next_pow2.restype = it
    L.csdrb_fft_c2c_batch.argtypes = [vp, lg, vp, lg, it, it, it, vp]
    L.csdrb_bandpass_fir_fft_bank_cc.argtypes = [vp, lg, vp, lg, it, it, it, it, vp, lg, vp, vp]
    L.csdrb_fmmod_bank_fc.argtypes = [vp, lg, vp, lg, it, it, vp, vp]
    return str(exe), L


def modulate(L, mode, audio, gain):
    """[C, n] f32 audio -> [C, m] complex baseband by the mode's banks on the emulated C ABI (m = n, or whole filter units for usb/lsb)"""
    ch, n = audio.shape
    a = np.ascontiguousarray(audio, np.float32)
    g = np.empty_like(a)
    assert M.call(L, "gain", a.ctypes.data, n, g.ctypes.data, n, ch, n, gain) == n
    bb = np.empty((ch, n), np.complex64)
    if mode == "fm":
        ph = np.zeros(ch, np.float32)
        assert L.csdrb_fmmod_bank_fc(g.ctypes.data, n, bb.ctypes.data, n, ch, n, ph.ctypes.data, None) == n
        return bb
    assert M.call(L, "dsb", g.ctypes.data, n, bb.ctypes.data, n, ch, n, 0.0) == n
    if mode == "am":
        assert M.call(L, "add_dcoffset", bb.ctypes.data, n, bb.ctypes.data, n, ch, n) == n
    if mode in SSB_BAND:
        T = L.firdes_filter_len(0.05)
        N = L.next_pow2(T)
        N = N * 2 if N - T < 200 else N
        unit = N - T + 1
        taps = np.zeros(N, np.complex64)
        L.firdes_bandpass_c(taps.ctypes.data, T, *SSB_BAND[mode], 2)
        taps_fft = np.empty(N, np.complex64)
        assert L.csdrb_fft_c2c_batch(taps.ctypes.data, N, taps_fft.ctypes.data, N, N, 1, 0, None) >= 0
        nb = n // unit
        out = np.empty((ch, max(nb * unit, 1)), np.complex64)
        tail = np.zeros((ch, N), np.complex64)
        assert L.csdrb_bandpass_fir_fft_bank_cc(bb.ctypes.data, n, out.ctypes.data, out.shape[1], ch, N, unit, nb, taps_fft.ctypes.data, 0,
                                                tail.ctypes.data, None) >= 0
        return out[:, :nb * unit]
    return bb


@pytest.mark.parametrize("block", [500, 4096])
@pytest.mark.parametrize("mode", ["am", "dsb", "usb", "lsb", "fm"])
def test_stdout_is_the_composed_banks_then_the_synthesis_bank(prog, tmp_path, mode, block):
    exe, L = prog
    rng = np.random.default_rng(block + len(mode))
    lengths, rates, I, bw, gain = [2100, 1700, 1900], [-0.2, 0.05, 0.3], 5, 0.1, 0.7
    srcs = [rng.uniform(-1, 1, m).astype(np.float32) for m in lengths]
    for k, s in enumerate(srcs):
        s.tofile(tmp_path / f"a{k}.f32")
    r = subprocess.run([exe, "--interpolation", str(I), "--bw", str(bw), "--block", str(block), "--mod", mode, "--gain", str(gain)] +
                       [f"{rates[k]}:{tmp_path / f'a{k}.f32'}" for k in range(3)], capture_output=True, timeout=1200)
    assert r.returncode == 0, r.stderr.decode()
    n = min(lengths)
    bb = modulate(L, mode, np.stack([s[:n] for s in srcs]), gain)
    T = L.firdes_filter_len(bw)
    taps = np.zeros(T, np.float32)
    L.firdes_lowpass_f(taps.ctypes.data, T, 0.5 / I, 2)
    want, _ = synth.restate(Oracle(), bb, rates, I, taps, None, 1024, 0)
    assert want.size == (bb.shape[1] - (T - 1 + I - 1) // I) * I > 0
    assert r.stdout == want.tobytes()


def test_mod_refusals(prog, tmp_path):
    exe, _ = prog
    (tmp_path / "s.f32").write_bytes(np.zeros(64, np.float32).tobytes())
    s = f"0.1:{tmp_path / 's.f32'}"
    for args in (["--interpolation", "5", "--gain", "2", s], ["--interpolation", "5", "--mod", "ssb", s], ["--interpolation", "5", "--mod", "am",
                                                                                                            "--gain", "x", s]):
        r = subprocess.run([exe] + args, input=b"", capture_output=True, timeout=60)
        assert r.returncode != 0 and r.stderr and not r.stdout, args
