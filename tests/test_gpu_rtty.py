"""GPU tests (-m gpu) of the RTTY receive chain: the two banks against the checker tests/rtty/rtty_oracle.c bit for bit at 1024 channels,
the libcsdr drop-in, and the csdr commands against the unmodified reference CLI stage for stage (at the CLI's buffer size and a small one,
through end of input) and as the three-stage pipe.  tests/test_rtty_cli_emulated.py runs the CLI bodies on the emulated library."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from test_gpu_cli import clis, run_graph  # noqa: F401  (the fixture: our CLI and the reference CLI)

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "rtty"))
import rtty  # noqa: E402

pytestmark = pytest.mark.gpu
TEXT = b"RYRYRY CQ CQ DE TEST TEST 599 73, 14.080 MHZ (K1ABC/P) 'OK?' = 100 + -5 $1 #2 @3 *4 :5\r\n"


def signal(spb, seed, text=TEXT, tail=None, noise=0.01):
    rng = np.random.default_rng(seed)
    return rtty.modulate(text, spb, rng, freq=0.001, noise=noise, lead_bits=float(rng.uniform(2, 12)),
                         tail_bits=(16384 / spb + 4) if tail is None else tail)


# ---- banks --------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    return torch, csdr_b200


@pytest.mark.parametrize("spb,databits,stopbits,ratio", [(44.0, 5, 1.5, 0.4), (5.0, 8, 1.0, 0.4), (176.02, 7, 2.0, 0.9)])
def test_banks_equal_checker_at_1024_channels(cuda, spb, databits, stopbits, ratio):
    """1024 channels: RTTY discriminator rows, heavy-tailed noise, +-0 / denormal / NaN / Inf rows; ragged starts, calls of 4096 samples"""
    torch, cb = cuda
    rng = np.random.default_rng(int(spb))
    ch, bufsize = 1024, 4096
    base = [rtty.discriminator(signal(spb, 50 + k, tail=bufsize / spb + 4)) for k in range(4)]
    n = max(min(b.size for b in base), 3 * bufsize)
    X = np.empty((ch, n), np.float32)
    for c in range(ch):
        kind = c % 8
        if kind < 4:
            X[c] = np.resize(base[kind], n)
        elif kind == 4:
            X[c] = rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)
        elif kind == 5:
            X[c] = rng.choice(np.array([0.0, -0.0, 1e-45, -1e-45, 1.0, -1.0, np.nan, np.inf, -np.inf], np.float32), n)
        else:
            X[c] = np.resize(base[kind - 6], n) + rng.standard_normal(n).astype(np.float32)
    starts = rng.integers(0, 200, ch).astype(np.int32)
    codes, cnt, st, stuck = cb.serial_line_decoder_bank_f_u8(torch.from_numpy(X).cuda(), spb, databits, stopbits, ratio, bufsize=bufsize,
                                                             start=torch.from_numpy(starts.copy()).cuda())
    codes, cnt, st, stuck = codes.cpu().numpy(), cnt.cpu().numpy(), st.cpu().numpy(), stuck.cpu().numpy()
    want = []
    for c in range(ch):
        w, pos, stk = rtty.serial_stream(X[c], spb, databits, stopbits, ratio, bufsize, int(starts[c]), n)
        assert codes[c, :cnt[c]].tobytes() == w and st[c] == pos and stuck[c] == int(stk), c
        want.append(w)
    modes = rng.integers(0, 2, ch).astype(np.uint8)
    chars, ccnt, m = cb.rtty_baudot2ascii_bank_u8_u8(torch.from_numpy(codes).cuda(), torch.from_numpy(cnt).cuda(), torch.from_numpy(modes.copy()).cuda())
    chars, ccnt, m = chars.cpu().numpy(), ccnt.cpu().numpy(), m.cpu().numpy()
    for c in range(ch):
        t, wm = rtty.baudot_decode(want[c], int(modes[c]))
        assert chars[c, :ccnt[c]].tobytes() == t and m[c] == wm, c
    if databits == 5 and stopbits == 1.5:
        assert all(TEXT in chars[c, :ccnt[c]].tobytes() for c in range(0, ch, 8))


def test_chain_in_blocks_equals_one_pass(cuda):
    """the daemon's use: rows fed in blocks, the start carried per channel and the FIGS/LTRS mode carried: the text of one pass"""
    torch, cb = cuda
    ch, spb, bufsize = 512, 44.0, 16384
    base = [rtty.discriminator(signal(spb, 7 + k)) for k in range(4)]
    n = min(b.size for b in base)
    X = torch.from_numpy(np.stack([base[c % 4][:n] for c in range(ch)])).cuda()
    start = torch.zeros(ch, dtype=torch.int32, device="cuda"); mode = None; out = [b""] * ch
    for end in list(range(3000, n, 3000)) + [n]:
        codes, cnt, start, stuck = cb.serial_line_decoder_bank_f_u8(X, spb, 5, 1.5, 0.4, bufsize=bufsize, start=start, end=end)
        assert not stuck.any()
        chars, ccnt, mode = cb.rtty_baudot2ascii_bank_u8_u8(codes, cnt, mode)
        chars, ccnt = chars.cpu().numpy(), ccnt.cpu().numpy()
        out = [t + chars[c, :ccnt[c]].tobytes() for c, t in enumerate(out)]
    for k in range(4):
        want = rtty.baudot_decode(rtty.serial_stream(base[k][:n], spb, 5, 1.5, 0.4, bufsize)[0])[0]
        assert TEXT in want
        assert all(out[c] == want for c in range(k, ch, 4))


def test_dropin(cuda):
    torch, cb = cuda
    d = rtty.discriminator(signal(44.0, 3))
    for n in (0, 1, 100, 16384, d.size):
        for ratio in (0.4, 1.0):
            want = rtty.serial_line_decoder(d[:n], 44.0, 5, 1.5, ratio)
            assert cb.libcsdr.serial_line_decoder_f_u8(d[:n], 44.0, 5, 1.5, ratio) == want
            if rtty.have_ref():
                assert want == rtty.ref_serial_line_decoder(d[:n], 44.0, 5, 1.5, ratio)


# ---- the csdr commands --------------------------------------------------------------------------------------------------------------
def _run(cli, args, data, env=None):
    import os
    e = dict(os.environ); e.update(env or {})
    return subprocess.run(["bash", "-c", f"{cli} {args}"], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e, timeout=300)


def test_rtty_commands_stage_for_stage(clis):
    """serial_line_decoder_f_u8 on the reference's discriminator output and rtty_baudot2ascii_u8_u8 on the reference's codes give the reference
    CLI's bytes, end of input included (the last call runs on a buffer whose tail still holds the call before's samples)"""
    ours, ref = clis
    disc = run_graph(ref, ["fmdemod_quadri_cf"], signal(44.0, 5).tobytes())
    for bufsize in ("16384", "512"):
        env = {"CSDR_FIXED_BUFSIZE": bufsize}
        for args in ("44 5 1.5", "44", "44 5", "40.5 7 2", "44.004 5 1.5", "4 5 1"):
            a, b = _run(ours, "serial_line_decoder_f_u8 " + args, disc, env), _run(ref, "serial_line_decoder_f_u8 " + args, disc, env)
            assert (a.returncode, a.stdout, a.stderr) == (b.returncode, b.stdout, b.stderr.replace(str(ref).encode(), str(ours).encode())), (bufsize, args)
    codes = run_graph(ref, ["serial_line_decoder_f_u8 44 5 1.5"], disc)
    rng = np.random.default_rng(1)
    for data in (codes, rng.integers(0, 256, 5000).astype(np.uint8).tobytes(), rng.choice([27, 31, 3, 16, 0, 255], 3000).astype(np.uint8).tobytes(), b""):
        assert run_graph(ours, ["rtty_baudot2ascii_u8_u8"], data) == run_graph(ref, ["rtty_baudot2ascii_u8_u8"], data)


def test_rtty_pipe_decodes_seeded_text(clis):
    ours, ref = clis
    x = signal(44.0, 9).tobytes()
    stages = ["fmdemod_quadri_cf", "serial_line_decoder_f_u8 44 5 1.5", "rtty_baudot2ascii_u8_u8"]
    want = run_graph(ref, stages, x)
    assert TEXT in want
    assert run_graph(ours, stages[1:], run_graph(ref, stages[:1], x)) == want


def test_rtty_refusals_and_stuck_exit(clis):
    """bad syntax and "got stuck" exit like the reference CLI: same code, same message"""
    ours, ref = clis
    stuck_input = np.r_[np.ones(1), -np.ones(200000)].astype(np.float32).tobytes()
    cases = [("serial_line_decoder_f_u8", b"", {}), ("serial_line_decoder_f_u8 0.5", b"", {}), ("serial_line_decoder_f_u8 44 9", b"", {}),
             ("serial_line_decoder_f_u8 44 0", b"", {}), ("serial_line_decoder_f_u8 44 5 0.5", b"", {}),
             ("serial_line_decoder_f_u8 44 5 1.5", stuck_input, {"CSDR_FIXED_BUFSIZE": "64"})]
    for args, data, env in cases:
        a, b = _run(ours, args, data, env), _run(ref, args, data, env)
        assert a.returncode != 0 and a.returncode == b.returncode, (args, a.returncode, b.returncode)
        assert a.stderr.replace(str(ours).encode(), b"csdr") == b.stderr.replace(str(ref).encode(), b"csdr"), args
