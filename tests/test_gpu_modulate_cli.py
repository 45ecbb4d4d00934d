"""GPU tests (-m gpu) of the amplitude modulator commands: `csdr gain_ff`, `dsb_fc`, `add_dcoffset_cc` and `fixed_amplitude_cc` of our CLI against the
unmodified reference CLI in the default, CSDR_FIXED_BUFSIZE=4096 and dynamic framings at input lengths around the block edges.  gain_ff, dsb_fc and
add_dcoffset_cc give the reference's bytes; fixed_amplitude_cc its lengths and samples within the float64 bound of tests/modulate/modulate.py.
The reference CLI starts with FTZ/DAZ set (it is linked with -ffast-math), so the inputs stay normal here; subnormals are covered through the
library (tests/test_modulate_emulated.py).  tests/test_modulate_cli_emulated.py runs these bodies on the emulated library."""
import sys
from pathlib import Path

import numpy as np
import pytest

import test_gpu_cli
from test_gpu_cli import clis  # noqa: F401  (the fixture: our CLI and the reference CLI)
from test_gpu_tx_cli import cases, run

sys.path.insert(0, str(Path(__file__).resolve().parent / "modulate"))
import modulate as M  # noqa: E402

# the shared framing check (test_gpu_cli.test_every_command_frames_like_the_reference) needs a case for every command `csdr --help` lists
test_gpu_cli.FRAMING_CASES.setdefault("gain_ff", (4, "f", ["0.5"]))
test_gpu_cli.FRAMING_CASES.setdefault("dsb_fc", (4, "f", ["", "0.25"]))
test_gpu_cli.FRAMING_CASES.setdefault("add_dcoffset_cc", (8, "f", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("fixed_amplitude_cc", (8, "f", ["2"]))

pytestmark = pytest.mark.gpu


def both(ours, ref, args, data, env):
    a, b = run(ours, args, data, env), run(ref, args, data, env)
    assert a[0] == b[0] and len(a[1]) == len(b[1]), (args, a[0], b[0], len(a[1]), len(b[1]))
    return a[1], b[1]


@pytest.mark.parametrize("args,item", [("gain_ff 1.7", 4), ("gain_ff -0.25", 4), ("dsb_fc", 4), ("dsb_fc 0.3", 4), ("add_dcoffset_cc", 8)])
def test_bytes_equal_the_reference_cli(clis, args, item):
    ours, ref = clis
    for case, env, data in cases(item, 11):
        a, b = both(ours, ref, args, data, env)
        assert a == b, (args, case)


def test_fixed_amplitude_cc_within_bound_of_the_reference_cli(clis):
    ours, ref = clis
    for case, env, data in cases(8, 12):
        a, b = both(ours, ref, "fixed_amplitude_cc 2", data, env)
        head = 8 if case[0] == "dynamic" and a else 0
        assert a[:head] == b[:head], case
        x = np.frombuffer(data[head:], np.complex64)
        ya, yb = np.frombuffer(a[head:], np.complex64), np.frombuffer(b[head:], np.complex64)
        n = min(x.size, ya.size)                                    # the last block's tail repeats the block before: compare the read part
        M.fixed_amplitude_ok(ya[:n], x[:n], 2.0, yb[:n])


def test_missing_parameters_are_refused(clis):
    ours, _ = clis
    for cmd in ("gain_ff", "fixed_amplitude_cc"):
        code, out, err = run(ours, cmd, b"", {})
        assert code != 0 and not out and b"need required parameter" in err, cmd
