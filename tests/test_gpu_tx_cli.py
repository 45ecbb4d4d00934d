"""GPU tests (-m gpu) of the transmit commands: `csdr fir_interpolate_cc` and `csdr fmmod_fc` of our CLI against the unmodified reference CLI,
across the buffer-size framings (the default big buffer, CSDR_FIXED_BUFSIZE, and dynamic sizes behind a preamble) at input lengths around the
block edges.  fir_interpolate_cc gives the reference's lengths and samples within 2e-6 (its taps and sums round differently in the last
bit); fmmod_fc its lengths and samples within one float ulp of the build's sincosf.
tests/test_tx_cli_emulated.py runs these bodies on the emulated library."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import test_gpu_cli
from test_gpu_cli import clis  # noqa: F401  (the fixture: our CLI and the reference CLI)

# test_gpu_cli.test_every_command_frames_like_the_reference runs every command `csdr --help` lists through its framing table and fails on a
# command without a case; the transmit commands add theirs to that table here, so that the shared framing check covers them like every other
# command (exit code, output length and the dynamic-mode preamble against the reference CLI at the same input lengths).
test_gpu_cli.FRAMING_CASES.setdefault("fir_interpolate_cc", (8, "f", ["4", "50 0.01 BLACKMAN"]))
test_gpu_cli.FRAMING_CASES.setdefault("fmmod_fc", (4, "f", [""]))

pytestmark = pytest.mark.gpu
ULP1 = 2.0 ** -24
LENGTHS = (0, 1, 1024, 1025, 16384, 16385, 40000)
FRAMINGS = (("fixed", {}), ("small", {"CSDR_FIXED_BUFSIZE": "4096"}), ("dynamic", {"CSDR_DYNAMIC_BUFSIZE_ON": "1"}))


def run(cli, args, data, env):
    e = dict(os.environ); e.update(env)
    with tempfile.TemporaryFile() as fin, tempfile.TemporaryFile() as fout, tempfile.TemporaryFile() as ferr:
        fin.write(data); fin.seek(0)
        r = subprocess.run([cli] + args.split(), stdin=fin, stdout=fout, stderr=ferr, env=e, timeout=300)
        fout.seek(0); ferr.seek(0)
        return r.returncode, fout.read(), ferr.read()


def cases(item, seed):
    for name, env in FRAMINGS:
        for n in LENGTHS:
            rng = np.random.default_rng(seed + n)
            data = rng.uniform(-1, 1, n * item // 4).astype(np.float32).tobytes()
            if name == "dynamic":
                data = b"csdr" + np.array([4096], np.int32).tobytes() + data
            yield (name, n), env, data


def test_fir_interpolate_cc_against_reference_cli(clis):
    ours, ref = clis
    for args in ("fir_interpolate_cc 4", "fir_interpolate_cc 50 0.01 BLACKMAN", "fir_interpolate_cc 3 0.2 BOXCAR"):
        for case, env, data in cases(8, 1):
            a, b = run(ours, args, data, env), run(ref, args, data, env)
            assert a[0] == b[0] and len(a[1]) == len(b[1]), (args, case, a[0], b[0], len(a[1]), len(b[1]))
            head = 8 if case[0] == "dynamic" and a[1] else 0
            assert a[1][:head] == b[1][:head], (args, case)
            fa, fb = np.frombuffer(a[1][head:], np.float32), np.frombuffer(b[1][head:], np.float32)
            assert np.all(np.abs(fa - fb) <= 2e-6), (args, case, float(np.abs(fa - fb).max()))      # taps and sums rounded in another order
            lines = lambda err: [ln.split(b": ", 1)[-1] for ln in err.splitlines() if b"window" in ln or b"taps_length" in ln]   # noqa: E731
            assert lines(a[2]) == lines(b[2]), (args, a[2], b[2])


def test_fmmod_fc_against_reference_cli(clis):
    ours, ref = clis
    for case, env, data in cases(4, 2):
        a, b = run(ours, "fmmod_fc", data, env), run(ref, "fmmod_fc", data, env)
        assert a[0] == b[0] and len(a[1]) == len(b[1]), (case, a[0], b[0], len(a[1]), len(b[1]))
        head = 8 if case[0] == "dynamic" and a[1] else 0
        assert a[1][:head] == b[1][:head], case
        fa, fb = np.frombuffer(a[1][head:], np.float32), np.frombuffer(b[1][head:], np.float32)
        assert np.all(np.abs(fa - fb) <= ULP1), (case, float(np.abs(fa - fb).max()))
    # values that wrap several times per sample
    x = np.random.default_rng(3).uniform(-12, 12, 5000).astype(np.float32).tobytes()
    a, b = run(ours, "fmmod_fc", x, {}), run(ref, "fmmod_fc", x, {})
    fa, fb = np.frombuffer(a[1], np.float32), np.frombuffer(b[1], np.float32)
    assert fa.size == fb.size > 0 and np.all(np.abs(fa - fb) <= ULP1)
