"""GPU tests (-m gpu) of the demodulator commands: `csdr dcblock_ff`, `fmdemod_atan_cf`, `fmdemod_quadri_novect_cf` and `amdemod_estimator_cf` of
our CLI against the unmodified reference CLI in the default, CSDR_FIXED_BUFSIZE=4096 and dynamic framings at input lengths around the block
edges, including inputs that end on a partial block: fmdemod_atan_cf writes whole blocks only, the other three write the stale final block.
dcblock_ff, amdemod_estimator_cf and fmdemod_quadri_novect_cf give the reference's bytes (novect also on an 8-bit receiver's repeating samples,
where the sign of a zero depends on the form of its numerator), fmdemod_atan_cf its bytes under the atan rounding rule of tests/demod/demod.py.
tests/test_demod_cli_emulated.py runs these bodies on the emulated library, where the atan rule leaves nothing to excuse."""
import sys
from pathlib import Path

import numpy as np
import pytest

import test_gpu_cli
from test_gpu_cli import clis  # noqa: F401  (the fixture: our CLI and the reference CLI)
from test_gpu_tx_cli import FRAMINGS, LENGTHS, cases, run

sys.path.insert(0, str(Path(__file__).resolve().parent / "demod"))
import demod as M  # noqa: E402

# the shared framing check (test_gpu_cli.test_every_command_frames_like_the_reference) needs a case for every command `csdr --help` lists
test_gpu_cli.FRAMING_CASES.setdefault("dcblock_ff", (4, "f", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("fmdemod_atan_cf", (8, "f", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("fmdemod_quadri_novect_cf", (8, "f", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("amdemod_estimator_cf", (8, "f", [""]))

pytestmark = pytest.mark.gpu


def both(ours, ref, args, data, env):
    a, b = run(ours, args, data, env), run(ref, args, data, env)
    assert a[0] == b[0] and len(a[1]) == len(b[1]), (args, a[0], b[0], len(a[1]), len(b[1]))
    return a[1], b[1]


@pytest.mark.parametrize("args,item", [("dcblock_ff", 4), ("amdemod_estimator_cf", 8)])
def test_bytes_equal_the_reference_cli(clis, args, item):
    ours, ref = clis
    for case, env, data in cases(item, 21):
        a, b = both(ours, ref, args, data, env)
        assert a == b, (args, case)


def quantised_cases(seed):
    """the framings and lengths of cases(), on an 8-bit receiver's samples"""
    for name, env in FRAMINGS:
        for n in LENGTHS:
            data = M.quantised_rows(np.random.default_rng(seed + n), 1, n)[0].tobytes()
            if name == "dynamic":
                data = b"csdr" + np.array([4096], np.int32).tobytes() + data
            yield (name, n), env, data


def test_novect_bytes_equal_the_reference_cli(clis):
    ours, ref = clis
    for case, env, data in list(cases(8, 22)) + list(quantised_cases(24)):
        a, b = both(ours, ref, "fmdemod_quadri_novect_cf", data, env)
        assert a == b, case


def test_atan_whole_blocks_under_the_rounding_rule(clis):
    ours, ref = clis
    near = 0
    for case, env, data in cases(8, 23):
        a, b = both(ours, ref, "fmdemod_atan_cf", data, env)
        head = 8 if case[0] == "dynamic" and a else 0
        assert a[:head] == b[:head], case
        ya, yb = np.frombuffer(a[head:], np.float32), np.frombuffer(b[head:], np.float32)
        x = np.frombuffer(data[head:], np.complex64)
        assert ya.size <= x.size, case                                  # whole blocks only: nothing past the input
        near += M.atan_matches(ya, yb, x[:ya.size])[0]
    assert near < 10, near
