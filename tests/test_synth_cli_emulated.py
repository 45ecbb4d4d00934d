"""CPU tier of csdr-synth (csdr_b200/host/programs/synth.c) linked against the emulated library (built here, as the other programs are in
tests/host_shim/emul_build.build_full): stdout equals the synthesis bank's one-shot call on the
streams cut to the shortest source (csdrb_synth_bank_cc, which tests/test_synth_emulated.py holds to the restatement bit for bit), byte for byte,
for two --block sizes, with sources of unequal lengths, a `-` source and a FIFO; and every refusal exits non-zero with a message."""
import ctypes as C
import os
import subprocess
import sys
import threading
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "synth"))
sys.path.insert(0, str(ROOT))
import emul_build  # noqa: E402
import synth  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402


@pytest.fixture(scope="module")
def prog(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _ = emul_build.build_full_once(tmp_path_factory)
    exe = tmp_path_factory.mktemp("synth_emul") / "csdr-synth_emul"
    subprocess.run(["gcc", "-std=gnu99", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(ROOT / "csdr_b200" / "host" / "programs" / "synth.c"), "-o",
                    str(exe), f"-L{lib.parent}", "-lcsdr_b200_emul", "-lm", f"-Wl,-rpath,{lib.parent}"], check=True, capture_output=True)
    L = C.CDLL(str(lib))
    L.firdes_filter_len.argtypes = [C.c_float]; L.firdes_filter_len.restype = C.c_int
    L.firdes_lowpass_f.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int]
    return str(exe), L


def one_shot(L, srcs, rates, I, bw, window=2):
    """csdrb_synth_bank_cc on the streams cut to the shortest, with the fir_interpolate_cc command's taps"""
    T = L.firdes_filter_len(bw)
    taps = np.zeros(T, np.float32)
    L.firdes_lowpass_f(taps.ctypes.data, T, 0.5 / I, window)
    n = min(s.size for s in srcs)
    x = np.stack([s[:n] for s in srcs])
    y, _ = synth.restate(Oracle(), x, rates, I, taps, None, 1024, 0)
    return y


@pytest.mark.parametrize("block", [333, 4096])
def test_stdout_is_the_bank_on_the_shortest_stream(prog, tmp_path, block):
    exe, L = prog
    rng = np.random.default_rng(block)
    lengths = [1500, 1111, 1300]
    rates = [-0.2, 0.0, 0.15]
    srcs = [(rng.uniform(-1, 1, m) + 1j * rng.uniform(-1, 1, m)).astype(np.complex64) for m in lengths]
    srcs[0].tofile(tmp_path / "a.cf32")
    fifo = tmp_path / "c.fifo"
    os.mkfifo(fifo)

    def feed():
        with open(fifo, "wb") as f:
            f.write(srcs[2].tobytes())

    t = threading.Thread(target=feed)
    t.start()
    r = subprocess.run([exe, "--interpolation", "5", "--bw", "0.1", "--block", str(block), f"{rates[0]}:{tmp_path / 'a.cf32'}", f"{rates[1]}:-",
                        f"{rates[2]}:{fifo}"], input=srcs[1].tobytes(), capture_output=True, timeout=900)
    t.join()
    assert r.returncode == 0, r.stderr.decode()
    want = one_shot(L, srcs, rates, 5, 0.1)
    h = (L.firdes_filter_len(0.1) - 1 + 4) // 5
    assert want.size == (min(lengths) - h) * 5
    assert r.stdout == want.tobytes()


def test_window_and_a_single_source(prog, tmp_path):
    exe, L = prog
    rng = np.random.default_rng(1)
    s = (rng.uniform(-1, 1, 400) + 1j * rng.uniform(-1, 1, 400)).astype(np.complex64)
    s.tofile(tmp_path / "s.cf32")
    r = subprocess.run([exe, "--interpolation", "3", "--bw", "0.2", "--window", "BLACKMAN", "--block", "50", f"0.1:{tmp_path / 's.cf32'}"],
                       capture_output=True, timeout=600)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == one_shot(L, [s], [0.1], 3, 0.2, window=1).tobytes()


def test_refusals(prog, tmp_path):
    exe, _ = prog
    (tmp_path / "s.cf32").write_bytes(np.zeros(64, np.complex64).tobytes())
    s = f"0.1:{tmp_path / 's.cf32'}"
    cases = [
        ["--interpolation", "5"],                                   # no channel
        ["--interpolation", "0", s],
        ["--interpolation", "5", "--bw", "0", s],
        ["--interpolation", "5", "--bw", "1", s],
        ["--interpolation", "5", "--window", "KAISER", s],
        ["--interpolation", "5", "--chunk", "0", s],
        ["--interpolation", "5", "--block", "0", s],
        ["--interpolation", "5", "0.1:-", "0.2:-"],
        ["--interpolation", "5", f"0.1:{tmp_path / 'missing.cf32'}"],
        ["--interpolation", "5", "0.1"],
        ["--interpolation", "5", "x:-"],
        ["--interpolation", "5", ":-"],
        ["--interpolation", "five", s],
    ]
    for args in cases:
        r = subprocess.run([exe] + args, input=b"", capture_output=True, timeout=60)
        assert r.returncode != 0 and r.stderr and not r.stdout, args
