"""GPU tests (-m gpu) of the AM / SSB receiver blocks (csdr_b200/csrc/agc.cu): the bank calls and the host drop-ins against the CPU
restatement tests/am_ssb/am_ssb_oracle.c, bit for bit (amdemod_cf included: both sides take the correctly rounded square root), and the
reference's own csdr binary running amdemod_cf, fastdcblock_ff and agc_ff on top of our library."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "am_ssb"))
import am_ssb  # noqa: E402

LIB = ROOT / "csdr_b200" / "libcsdr_b200.so"
REF = ROOT / "oracle" / "_ref" / "csdr_ref"
AMDEMOD_ULP = 3                                   # measured bound between the reference build and the correctly rounded form (test_oracle_am_ssb.py)


@pytest.fixture(scope="module")
def cb():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    csdr_b200.lib()
    return csdr_b200


def signal(rng, n, c):
    t = np.arange(n)
    x = (0.2 * (1 + (c % 7)) * np.sin(2 * np.pi * t / (13.0 + c % 29)) * (1 + 0.8 * np.sin(2 * np.pi * t / 4000.0))).astype(np.float32)
    x += (0.003 * rng.standard_normal(n)).astype(np.float32)
    x[n // 4: n // 4 + 3000] = 0.0
    x[n // 2: n // 2 + 300] *= 30.0
    x[rng.integers(0, n, n // 40)] = 0.0
    return x


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def test_amdemod_bank_bit_exact(cb):
    rng = np.random.default_rng(1)
    x = (rng.standard_normal(300_001) + 1j * rng.standard_normal(300_001)).astype(np.complex64) * np.float32(7)
    y = cb.amdemod_cf(torch.from_numpy(x).cuda()).cpu().numpy()
    assert np.array_equal(bits(y), bits(am_ssb.amdemod_cf(x)))


@pytest.mark.parametrize("block", [1024, 1000, 777])
def test_am_front_bank_split_calls(cb, block):
    """amdemod_cf | fastdcblock_ff over 130 channels, in two calls (9 + 14 blocks), equals the CLI loop per channel"""
    rng = np.random.default_rng(block)
    ch, nb = 130, 23
    x = ((rng.standard_normal((ch, nb * block)) + 1j * rng.standard_normal((ch, nb * block))) + (0.5 + 0.2j)).astype(np.complex64)
    xd = torch.from_numpy(x).cuda()
    y1, last = cb.fastdcblock_bank_ff(xd[:, :9 * block], block)
    y2, last = cb.fastdcblock_bank_ff(xd[:, 9 * block:], block, last)
    y = torch.cat([y1, y2], 1).cpu().numpy(); last = last.cpu().numpy()
    for c in range(0, ch, 7):
        want, lw = am_ssb.am_front(x[c], block)
        assert np.array_equal(bits(y[c]), bits(want)), c
        assert np.float32(lw) == last[c]


@pytest.mark.parametrize("chunk", [1024, 333])
def test_agc_bank_split_stream(cb, chunk):
    """agc_ff over 100 channels (not a multiple of 32), a stream cut into calls of uneven sizes, equals agc_ff's CLI loop"""
    rng = np.random.default_rng(chunk)
    ch, n = 100, 40_000
    x = np.stack([signal(rng, n, c) for c in range(ch)])
    kw = dict(hang_time=50, attack_rate=0.05, decay_rate=0.001, attack_wait=3, max_gain=1000.0, alpha=0.99, reference=0.3)
    p = cb.AgcParams(reference=0.3, attack_rate=0.05, decay_rate=0.001, max_gain=1000.0, hang_time=50, attack_wait_time=3, gain_filter_alpha=0.99, chunk=chunk)
    xd = torch.from_numpy(x).cuda()
    state = None; outs = []
    for s0, s1 in ((0, 1), (1, 5000), (5000, 5031), (5031, 40_000)):
        y, state = cb.agc_bank_ff(xd[:, s0:s1].contiguous(), p, state)
        outs.append(y)
    y = torch.cat(outs, 1).cpu().numpy()
    for c in range(0, ch, 3):
        want, _ = am_ssb.agc_stream(x[c], chunk, **kw)
        assert np.array_equal(bits(y[c]), bits(want)), c


@pytest.mark.parametrize("limit", [0.0, 0.6])
def test_ssb_tail_bank_s16(cb, oracle, limit):
    """realpart_cf | agc_ff | limit_ff | convert_f_s16 from cf32 rows with the CLI defaults"""
    rng = np.random.default_rng(5)
    ch, n = 45, 30_000
    x = np.stack([signal(rng, n, c) + 1j * rng.standard_normal(n).astype(np.float32) for c in range(ch)]).astype(np.complex64)
    y, _ = cb.agc_bank_ff(torch.from_numpy(x).cuda(), None, None, limit, True)
    y = y.cpu().numpy()
    for c in range(ch):
        assert np.array_equal(bits(y[c]), bits(am_ssb.agc_tail(x[c], oracle, 1024, limit, True))), c


def test_host_dropins(cb):
    """amdemod_cf, fastdcblock_ff and agc_ff with the reference's signatures, host pointers"""
    rng = np.random.default_rng(9)
    iq = (rng.standard_normal(5000) + 1j * rng.standard_normal(5000)).astype(np.complex64)
    assert np.array_equal(bits(cb.libcsdr.amdemod_cf(iq)), bits(am_ssb.amdemod_cf(iq)))
    for n in (1, 3, 7, 1024, 1027):
        x = rng.standard_normal(n).astype(np.float32) + np.float32(0.4)
        y, avg = cb.libcsdr.fastdcblock_ff(x, 0.25)
        w, aw = am_ssb.fastdcblock_ff(x, 0.25)
        assert np.array_equal(bits(y), bits(w)) and np.float32(avg) == np.float32(aw), n
    x = signal(rng, 3000, 2)
    y, g = cb.libcsdr.agc_ff(x, 0.3, 0.05, 0.001, 500.0, 20, 2, 0.9, 1.7)
    w, gw = am_ssb.agc_ff(x, 1.7, reference=0.3, attack_rate=0.05, decay_rate=0.001, max_gain=500.0, hang_time=20, attack_wait=2, alpha=0.9)
    assert np.array_equal(bits(y), bits(w)) and np.float32(g) == np.float32(gw)


def run(cmd, data, env=None):
    e = dict(os.environ); e.update(env or {})
    r = subprocess.run(["bash", "-c", cmd], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e, timeout=120)
    assert r.returncode == 0, (cmd, r.stderr[-2000:])
    return r.stdout, r.stderr


@pytest.mark.parametrize("stage", ["amdemod_cf", "fastdcblock_ff", "fastdcblock_ff 1000", "agc_ff", "agc_ff 20 0.3 0.05 0.001 300 4 0.9"])
def test_reference_binary_on_our_library(cb, stage):
    """the reference csdr with libcsdr_b200.so preloaded runs the stage on the GPU (CSDRB_TRACE reports the kernel launches) and gives
    the oracle's bytes; the plain reference binary agrees bit for bit (agc_ff, fastdcblock_ff) or within the ulp bound (amdemod_cf)"""
    if not REF.exists():
        pytest.skip("oracle/_ref/csdr_ref not built")
    rng = np.random.default_rng(len(stage))
    n = 1024 * 40
    if stage == "amdemod_cf":
        x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 3).astype(np.complex64)
    else:
        x = signal(rng, n, 4) + np.float32(0.05)
    pre, err = run(f"{REF} {stage}", x.tobytes(), {"LD_PRELOAD": str(LIB), "CSDRB_TRACE": "1"})
    plain, _ = run(f"{REF} {stage}", x.tobytes())
    import re
    m = re.search(rb"libcsdr_b200: (\d+) kernel launches", err)
    assert m and int(m.group(1)) > 0, err[-500:]                        # the preloaded library ran kernels, not the reference's own code
    pre = np.frombuffer(pre, np.float32); plain = np.frombuffer(plain, np.float32)
    assert pre.size == plain.size >= n                                   # the reference writes one more, stale block at EOF (FEOF_CHECK before fread)
    a = stage.split()
    if a[0] == "amdemod_cf":
        want = am_ssb.amdemod_cf(x)
        d = np.abs(plain[:n].view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert d.max() <= AMDEMOD_ULP
    elif a[0] == "fastdcblock_ff":
        block = int(a[1]) if len(a) > 1 else 1024
        want, _ = am_ssb.fastdcblock_stream(x, block)
        n = want.size
        assert np.array_equal(bits(plain), bits(pre))
    else:
        v = [float(t) for t in a[1:]]
        names = ["hang_time", "reference", "attack_rate", "decay_rate", "max_gain", "attack_wait", "alpha"]
        kw = {k: (int(t) if k in ("hang_time", "attack_wait") else t) for k, t in zip(names, v)}
        want, _ = am_ssb.agc_stream(x, 1024, **kw)
        assert np.array_equal(bits(plain), bits(pre))
    assert np.array_equal(bits(pre[:n]), bits(want))
