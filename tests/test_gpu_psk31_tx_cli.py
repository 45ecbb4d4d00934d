"""GPU tests (-m gpu) of the BPSK31 transmit commands of our csdr CLI against the unmodified reference CLI (oracle/_ref/csdr_ref), byte for
byte, in the default, CSDR_FIXED_BUFSIZE=4096 and dynamic framings: psk31_varicode_encoder_u8_u8 (whose reference loop re-encodes its first
block once per further read, DESIGN.md section 7), differential_encoder_u8_u8, differential_decoder_u8_u8, psk_modulator_u8_c and
psk31_interpolate_sine_cc, the four-stage pipe of the reference's BER harness, and the reference binary with libcsdr_b200.so preloaded.
tests/test_psk31_tx_cli_emulated.py runs these bodies on the emulated library."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import test_gpu_cli
from test_gpu_cli import clis  # noqa: F401  (the fixture: our CLI and the reference CLI)

# the shared every-command framing check (test_gpu_cli.test_every_command_frames_like_the_reference) needs a case for every command
test_gpu_cli.FRAMING_CASES.setdefault("psk31_varicode_encoder_u8_u8", (1, "u8", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("differential_encoder_u8_u8", (1, "u8", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("differential_decoder_u8_u8", (1, "u8", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("psk_modulator_u8_c", (1, "bits", ["2", "8"]))
test_gpu_cli.FRAMING_CASES.setdefault("psk31_interpolate_sine_cc", (8, "f", ["8"]))

pytestmark = pytest.mark.gpu
FRAMINGS = (("fixed", {}), ("small", {"CSDR_FIXED_BUFSIZE": "4096"}), ("dynamic", {"CSDR_DYNAMIC_BUFSIZE_ON": "1"}))


def run(cli, args, data, env, preload=None):
    e = dict(os.environ); e.update(env)
    if preload:
        e["LD_PRELOAD"] = preload; e["CSDRB_TRACE"] = "1"
    with tempfile.TemporaryFile() as fin, tempfile.TemporaryFile() as fout, tempfile.TemporaryFile() as ferr:
        fin.write(data); fin.seek(0)
        r = subprocess.run([cli] + args.split(), stdin=fin, stdout=fout, stderr=ferr, env=e, timeout=300)
        fout.seek(0); ferr.seek(0)
        return r.returncode, fout.read(), ferr.read()


def text(n, seed):
    rng = np.random.default_rng(seed)
    t = rng.integers(32, 127, n).astype(np.uint8)
    t[rng.random(n) < 0.05] = 0x90
    return t.tobytes()


def same_bytes(ours, ref, args, data, env):
    a, b = run(ours, args, data, env), run(ref, args, data, env)
    assert a[0] == b[0] and a[1] == b[1], (args, len(data), env, a[0], b[0], len(a[1]), len(b[1]))


def framed(data, name):
    return b"csdr" + np.array([4096], np.int32).tobytes() + data if name == "dynamic" else data


def test_varicode_encoder_against_reference_cli(clis):
    ours, ref = clis
    for name, env in FRAMINGS:
        for n in (0, 3, 1024, 1025, 3004, 5000):
            same_bytes(ours, ref, "psk31_varicode_encoder_u8_u8", framed(b"aaa" if n == 3 else text(n, n), name), env)
    a = run(ours, "psk31_varicode_encoder_u8_u8", b"aaa", {})[1]
    assert len(a) == 12270 and list(a[:18]) == [1, 0, 1, 1, 0, 0] * 3


def test_codec_modulator_interpolator_against_reference_cli(clis):
    ours, ref = clis
    rng = np.random.default_rng(5)
    for name, env in FRAMINGS:
        for n in (0, 1, 1024, 1025, 4097, 10000):
            u8 = framed(rng.integers(0, 3, n).astype(np.uint8).tobytes(), name)
            same_bytes(ours, ref, "differential_encoder_u8_u8", u8, env)
            same_bytes(ours, ref, "differential_decoder_u8_u8", u8, env)
            same_bytes(ours, ref, "psk_modulator_u8_c 2", framed(rng.integers(0, 2, n).astype(np.uint8).tobytes(), name), env)
            same_bytes(ours, ref, "psk_modulator_u8_c 4", framed(rng.integers(0, 4, n).astype(np.uint8).tobytes(), name), env)
            cf = framed(rng.uniform(-1, 1, 2 * n).astype(np.float32).tobytes(), name)
            same_bytes(ours, ref, "psk31_interpolate_sine_cc 8", cf, env)
            same_bytes(ours, ref, "psk31_interpolate_sine_cc 3", cf, env)
    for args in ("psk_modulator_u8_c", "psk_modulator_u8_c 0", "psk_modulator_u8_c 257", "psk31_interpolate_sine_cc", "psk31_interpolate_sine_cc 0"):
        assert run(ours, args, b"", {})[0] == run(ref, args, b"", {})[0] != 0, args


def pipe(cli, data, sps, preload=None):
    e = dict(os.environ)
    if preload:
        e["LD_PRELOAD"] = preload; e["CSDRB_TRACE"] = "1"
    stages = ["psk31_varicode_encoder_u8_u8", "differential_encoder_u8_u8", "psk_modulator_u8_c 2", f"psk31_interpolate_sine_cc {sps}"]
    cmd = " | ".join(f"{cli} {s}" for s in stages)
    r = subprocess.run(["bash", "-c", cmd], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout, r.stderr


def test_bpsk31_pipe_equals_the_reference_pipe(clis):
    ours, ref = clis
    for data in (b"CQ CQ de TEST k", text(1024, 9)):
        assert pipe(ours, data, 32)[0] == pipe(ref, data, 32)[0]


def test_reference_pipe_on_our_library(clis):
    """the reference's own csdr with libcsdr_b200.so preloaded gives the same bytes and its functions launch kernels"""
    ours, ref = clis
    data = b"CQ CQ de TEST k"
    plain, _ = pipe(ref, data, 32)
    pre, err = pipe(ref, data, 32, preload=str(test_gpu_cli.LIB))
    assert pre == plain
    counts = [int(ln.split()[1]) for ln in err.decode().splitlines() if ln.startswith("libcsdr_b200:") and "kernel launches" in ln]
    assert sum(c > 0 for c in counts) == 4, err[-2000:]              # the four csdr stages (the shell that runs the pipe launches none)
