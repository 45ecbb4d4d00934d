"""GPU tests (-m gpu) of the sample-format commands `csdr convert_s8_f`, `convert_f_s8`, `convert_f_u8`, `convert_f_s24 [--bigendian]` and
`convert_s24_f [--bigendian]`: byte for byte against the unmodified reference CLI in the default, CSDR_FIXED_BUFSIZE=4096 and dynamic framings,
with out-of-range values, +-Inf and NaN in the float inputs; the round trips through both s24 byte orders; the reference's own binary with our
library preloaded.  The reference CLI's convert_s24_f cannot run: it allocates its byte buffer before the buffer size is known (csdr.c:623,
malloc(0)) and the fortified fread stops it with "buffer overflow detected".  Our command is checked against the reference library's
convert_s24_f called block by block the way the CLI's loop calls it.  tests/test_formats_cli_emulated.py runs these bodies on the emulated
library."""
import sys
from pathlib import Path

import numpy as np
import pytest

import test_gpu_cli
from test_gpu_cli import clis, run_graph  # noqa: F401  (the fixture: our CLI and the reference CLI)
from test_gpu_tx_cli import FRAMINGS, LENGTHS, run

sys.path.insert(0, str(Path(__file__).resolve().parent / "formats"))
import formats as M  # noqa: E402

# the shared framing check (test_gpu_cli.test_every_command_frames_like_the_reference) needs a case for every command `csdr --help` lists.
# convert_s24_f has no argument list there: the reference CLI aborts on it, so its framing is checked below against the reference library.
test_gpu_cli.FRAMING_CASES.setdefault("convert_s8_f", (1, "u8", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("convert_f_s8", (4, "f", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("convert_f_u8", (4, "f", [""]))
test_gpu_cli.FRAMING_CASES.setdefault("convert_f_s24", (4, "f", ["", "--bigendian"]))
test_gpu_cli.FRAMING_CASES.setdefault("convert_s24_f", (3, "u8", []))

pytestmark = pytest.mark.gpu


def cases(item, seed, floats):
    """(case, env, data) over the framings and lengths; float inputs mix uniform values, the wrap region, +-Inf and NaN"""
    for name, env in FRAMINGS:
        for n in LENGTHS:
            rng = np.random.default_rng(seed + n)
            if floats:
                x = rng.uniform(-1.2, 1.2, n).astype(np.float32)
                k = min(n, 64)
                x[rng.choice(n, k, replace=False) if n else []] = rng.choice(M.float_specials("f_s8"), k)
                data = x.tobytes()
            else:
                data = rng.integers(0, 256, n * item, dtype=np.uint8).tobytes()
            if name == "dynamic":
                data = b"csdr" + np.array([4096], np.int32).tobytes() + data
            yield (name, n), env, data


@pytest.mark.parametrize("args,item,floats", [("convert_s8_f", 1, False), ("convert_f_s8", 4, True), ("convert_f_u8", 4, True),
                                              ("convert_f_s24", 4, True), ("convert_f_s24 --bigendian", 4, True)])
def test_bytes_equal_the_reference_cli(clis, args, item, floats):
    ours, ref = clis
    for case, env, data in cases(item, 21, floats):
        a, b = run(ours, args, data, env), run(ref, args, data, env)
        assert a[0] == b[0] and len(a[1]) == len(b[1]), (args, case, a[0], b[0], len(a[1]), len(b[1]))
        # The reference's convert_f_s24 writes past its malloc(0) byte buffer (see above) into whatever the heap holds behind it: the head of
        # its float buffer, so a block written again past the end of the input converts floats the previous block overwrote, and in dynamic
        # mode also stdin's buffer, allocated while the preamble is read, so every block after the first converts overwritten input.  Only
        # the bytes of values the reference read intact are compared there.
        cut = len(a[1]) if "s24" not in args else 3 * case[1] if case[0] != "dynamic" else 8 + 3 * min(case[1], 4096)
        assert a[1][:cut] == b[1][:cut], (args, case)


def cli_loop_with_the_reference_library(data, block, bigendian):
    """what the CLI's convert_s24_f loop (csdr.c:620-633) computes with a buffer of `block` values: the end-of-file test before each read, a
    short last read converted over the previous block's tail, every block written whole"""
    buf = np.zeros(3 * block, np.uint8)
    out, pos = [], 0
    while True:
        chunk = np.frombuffer(data[pos:pos + 3 * block], np.uint8)
        buf[:chunk.size] = chunk; pos += chunk.size
        out.append(np.asarray(M.ref_call("s24_f", buf, bigendian)).tobytes())
        if chunk.size < 3 * block:
            return b"".join(out)


@pytest.mark.parametrize("bigendian", [0, 1])
def test_convert_s24_f_is_the_reference_library_in_the_cli_loop(clis, bigendian):
    ours, _ = clis
    for case, env, data in cases(3, 22, False):
        code, out, err = run(ours, "convert_s24_f" + (" --bigendian" if bigendian else ""), data, env)
        assert code == 0, (case, err[-300:])
        head = data[:8] if case[0] == "dynamic" else b""
        block = 4096 if case[0] != "fixed" else 1024
        assert out == head + cli_loop_with_the_reference_library(data[len(head):], block, bigendian), case


def test_s24_round_trips(clis):
    """convert_f_s24 | convert_s24_f in both byte orders, and a mismatched pair reading the other order"""
    ours, _ = clis
    x = np.random.default_rng(23).uniform(-1, 1, 50_000).astype(np.float32)
    for be in ("", " --bigendian"):
        y = np.frombuffer(run_graph(ours, ["convert_f_s24" + be, "convert_s24_f" + be], x.tobytes()), np.float32)
        want = M.s24_f(M.f_s24(x, bool(be)), bool(be))
        assert M.same(y[:x.size], want) and np.abs(y[:x.size] - x).max() < 2.0 ** -22, be
    crossed = np.frombuffer(run_graph(ours, ["convert_f_s24", "convert_s24_f --bigendian"], x.tobytes()), np.float32)
    assert M.same(crossed[:x.size], M.s24_f(M.f_s24(x, 0), 1))


def test_reference_binary_runs_on_our_library(clis):
    """the reference's own csdr with our library preloaded gives its own bytes, and our library did the work.  Not convert_f_s24: its
    writes past its malloc(0) buffer corrupt a heap that the preloaded library shares, and glibc may abort it"""
    _, ref = clis
    rng = np.random.default_rng(24)
    x = rng.uniform(-1.2, 1.2, 30_000).astype(np.float32).tobytes()
    b = rng.integers(0, 256, 30_000, dtype=np.uint8).tobytes()
    pre = {"LD_PRELOAD": str(test_gpu_cli.LIB), "CSDRB_TRACE": "1"}
    for args, data in (("convert_s8_f", b), ("convert_f_s8", x), ("convert_f_u8", x)):
        plain = run(ref, args, data, {})
        loaded = run(ref, args, data, pre)
        assert loaded[0] == plain[0] == 0 and loaded[1] == plain[1], args
        assert b"libcsdr_b200: " in loaded[2] and b" 0 kernel launches" not in loaded[2], (args, loaded[2][-300:])
