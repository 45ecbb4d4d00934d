"""GPU tests (-m gpu) of the BPSK31 receive chain: the four banks against the checker tests/psk31/psk31_oracle.c (bit for bit, at sizes a
band skimmer runs), the libcsdr drop-ins, and the csdr commands against the unmodified reference CLI stage for stage and as the four-stage
pipe.  tests/test_psk31_cli_emulated.py runs the CLI bodies on the emulated library."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from test_gpu_cli import clis, run_graph  # noqa: F401  (the fixture: our CLI and the reference CLI)

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "psk31"))
import psk31  # noqa: E402

pytestmark = pytest.mark.gpu
TEXT = b"CQ CQ CQ de TEST TEST The quick brown fox jumps over the lazy dog 0123456789 pse k"


def bits_of(a):
    return np.ascontiguousarray(a).view(np.uint8)


def same(a, b):
    """bit for bit, except that a NaN equals any NaN (the GPU writes the canonical NaN where the CPU propagates the input's payload)"""
    a = np.ascontiguousarray(a).view(np.float32); b = np.ascontiguousarray(b).view(np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def signal(sps, seed, text=TEXT):
    rng = np.random.default_rng(seed)
    enc = psk31.ref_varicode_encode(text) if psk31.have_ref() else rng.integers(0, 2, 8 * len(text)).astype(np.uint8)
    return psk31.modulate(enc, sps, rng, freq=0.2 / (2 * np.pi * sps), noise=0.03)


def dbpsk_mismatches_near_half_pi(x, got, want):
    """indexes where the decisions differ must be phase steps within a few ulps of +-pi/2"""
    prev = np.concatenate([[np.complex64(0)], x[:-1]])
    for i in np.nonzero(np.asarray(got) != np.asarray(want))[0]:
        d = np.float32(np.arctan2(x[i].imag, x[i].real)) - np.float32(np.arctan2(prev[i].imag, prev[i].real))
        d = (d + np.pi) % (2 * np.pi) - np.pi
        assert abs(abs(d) - np.pi / 2) < 1e-6, (i, d)


# ---- banks --------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    return torch, csdr_b200


def test_banks_equal_checker(cuda):
    torch, cb = cuda
    rng = np.random.default_rng(1)
    ch, sps = 131, 64
    rows = [signal(sps, 100 + c)[:40000] for c in range(ch)]
    n = min(r.size for r in rows)
    X = np.stack([r[:n] for r in rows])
    X[5, 100:110] = np.nan; X[6, 200] = np.inf; X[7, 300:400] = 0
    g0 = rng.uniform(0.5, 2, ch).astype(np.float32)
    y, g = cb.simple_agc_bank_cc(torch.from_numpy(X).cuda(), 0.001, 0.5, 65535.0, torch.from_numpy(g0).cuda())
    y = y.cpu().numpy(); g = g.cpu().numpy()
    for c in range(ch):
        yc, gc = psk31.simple_agc_cc(X[c], 0.001, 0.5, 65535.0, float(g0[c]))
        assert same(y[c], yc) and np.float32(gc) == g[c], c
    for alg in (psk31.GARDNER, psk31.EARLYLATE):
        for use_q in (False, True):
            starts = rng.integers(0, 50, ch).astype(np.int32); sizes = (n - starts - rng.integers(0, 50, ch)).astype(np.int32)
            st0 = np.zeros((ch, 3), np.int32); st0[:, 0] = rng.integers(-sps // 4 + 1, sps // 4, ch)
            o, e, ix, st = cb.timing_recovery_bank_cc(torch.from_numpy(y).cuda(), alg, sps, use_q, start=torch.from_numpy(starts).cuda(),
                                                      size=torch.from_numpy(sizes).cuda(), state=torch.from_numpy(st0.copy()).cuda())
            o, e, ix, st = o.cpu().numpy(), e.cpu().numpy(), ix.cpu().numpy(), st.cpu().numpy()
            for c in range(ch):
                yo, eo, io, so = psk31.timing_recovery_cc(y[c, starts[c]:starts[c] + sizes[c]], alg, sps, use_q, 0.5, 2.0, int(st0[c, 0]))
                m = so[2]
                assert tuple(st[c]) == so
                assert same(o[c, :m], yo) and same(e[c, :m], eo) and np.array_equal(ix[c, :m], io)
    counts = torch.from_numpy(st[:, 2].copy()).cuda()
    b, last = cb.dbpsk_decoder_bank_c_u8(torch.from_numpy(o).cuda(), counts)
    b = b.cpu().numpy(); last = last.cpu().numpy()
    for c in range(ch):
        m = st[c, 2]
        want, wl = psk31.dbpsk_decoder_c_u8(o[c, :m])
        dbpsk_mismatches_near_half_pi(o[c, :m], b[c, :m], want)
        assert same(np.complex64(wl), last[c])
    chars, cnt, hist = cb.psk31_varicode_decoder_bank_u8_u8(torch.from_numpy(b).cuda(), counts)
    chars, cnt, hist = chars.cpu().numpy(), cnt.cpu().numpy(), hist.cpu().numpy()
    for c in range(ch):
        want, wh = psk31.varicode_decode(b[c, :st[c, 2]])
        assert chars[c, :cnt[c]].tobytes() == want and int(hist[c]) & (2 ** 64 - 1) == wh


def test_chain_at_256_sps_over_1024_channels_in_blocks(cuda):
    """the chain of a band skimmer: 1024 channels at 8 kHz baseband and 31.25 Bd, fed in blocks of 4096 samples.  The timing recovery bank
    starts every channel where it stopped (per-channel offsets into the stream) and the AGC gain, timing state, last dbpsk input and
    varicode history are carried; every channel decodes what the checker's chain decodes from the same stream"""
    torch, cb = cuda
    ch, sps, blk, text = 1024, 256, 4096, b"CQ de TEST pse k"
    base = [signal(sps, 7 + k, text) for k in range(4)]
    n = min(b.size for b in base)
    X = np.stack([base[c % 4][:n] for c in range(ch)])
    dev = torch.from_numpy(X).cuda()
    A = torch.empty_like(dev)
    gain = None; tr_state = None; last = None; hist = None; out = [b""] * ch
    consumed = torch.zeros(ch, dtype=torch.int32, device="cuda")
    for pos in range(0, n, blk):
        A[:, pos:pos + blk], gain = cb.simple_agc_bank_cc(dev[:, pos:pos + blk].contiguous(), 0.001, 0.5, 65535.0, gain)
        filled = min(pos + blk, n)
        size = (filled - consumed).to(torch.int32)
        o, _, _, tr_state = cb.timing_recovery_bank_cc(A[:, :filled], psk31.GARDNER, sps, True, start=consumed, size=size, state=tr_state)
        consumed = (consumed + tr_state[:, 1]).to(torch.int32)
        counts = tr_state[:, 2].contiguous()
        b, last = cb.dbpsk_decoder_bank_c_u8(o, counts, last)
        chars, cnt, hist = cb.psk31_varicode_decoder_bank_u8_u8(b, counts, hist)
        chars, cnt = chars.cpu().numpy(), cnt.cpu().numpy()
        out = [t + chars[c, :cnt[c]].tobytes() for c, t in enumerate(out)]
    for c in range(4):
        want = psk31.chain(X[c], sps)
        assert text in want
        assert all(out[k] == want for k in range(c, ch, 4)), (c, want, out[c])


def test_dropins(cuda):
    torch, cb = cuda
    x = signal(32, 3)[:50000]
    y, g = cb.libcsdr.simple_agc_cc(x, 0.001, 0.5)
    yc, gc = psk31.simple_agc_cc(x, 0.001, 0.5)
    assert np.array_equal(bits_of(y), bits_of(yc)) and np.float32(g) == np.float32(gc)
    for alg in (psk31.GARDNER, psk31.EARLYLATE):
        got = cb.libcsdr.timing_recovery_cc(y, alg, 32, True, 0.5, 2.0, 3)
        want = psk31.timing_recovery_cc(y, alg, 32, True, 0.5, 2.0, 3)
        assert got[3] == want[3] and all(np.array_equal(bits_of(a), bits_of(b)) for a, b in zip(got[:3], want[:3]))
    s = want[0]
    b1 = cb.libcsdr.dbpsk_decoder_c_u8(s[:100]); b2 = cb.libcsdr.dbpsk_decoder_c_u8(s[100:])      # the previous sample carries over
    w, _ = psk31.dbpsk_decoder_c_u8(s)
    dbpsk_mismatches_near_half_pi(s, np.concatenate([b1, b2]), w)


# ---- the csdr commands --------------------------------------------------------------------------------------------------------------
def test_psk31_commands_stage_for_stage(clis):
    """every stage gets the reference CLI's output of the previous stage and must give the reference CLI's bytes (simple_agc_cc: within the
    relative bound of tests/test_oracle_psk31.py, the reference build's rsqrtss seed being vendor-dependent)"""
    ours, ref = clis
    x = signal(32, 5).tobytes()
    want, got = run_graph(ref, ["simple_agc_cc 0.001 0.5"], x), run_graph(ours, ["simple_agc_cc 0.001 0.5"], x)
    a, b = np.frombuffer(want, np.complex64), np.frombuffer(got, np.complex64)
    assert a.size == b.size and np.max(np.abs(a - b) / np.maximum(np.abs(a), 1e-30)) < 2e-5
    for args in ("GARDNER 32 0.5 2 --add_q", "EARLYLATE 32", "GARDNER 32 0.25 2 --add_q --output_error", "EARLYLATE 32 0.5 2 --add_q --output_indexes",
                 "GARDNER 32 0.5 2 xx --output_indexes", "GARDNER 32 1 2 --add_q", "EARLYLATE 32 0.5 2 --add_q --octave"):
        assert run_graph(ours, ["timing_recovery_cc " + args], want) == run_graph(ref, ["timing_recovery_cc " + args], want), args
    sym = run_graph(ref, ["timing_recovery_cc GARDNER 32 0.5 2 --add_q"], want)
    d_ref, d_ours = run_graph(ref, ["dbpsk_decoder_c_u8"], sym), run_graph(ours, ["dbpsk_decoder_c_u8"], sym)
    assert len(d_ref) == len(d_ours)
    s = np.frombuffer(sym, np.complex64)
    dbpsk_mismatches_near_half_pi(s, np.frombuffer(d_ours, np.uint8)[:s.size], np.frombuffer(d_ref, np.uint8)[:s.size])
    assert run_graph(ours, ["psk31_varicode_decoder_u8_u8"], d_ref) == run_graph(ref, ["psk31_varicode_decoder_u8_u8"], d_ref)


def test_psk31_pipe_decodes_seeded_text(clis):
    ours, ref = clis
    x = signal(256, 9).tobytes()
    stages = ["simple_agc_cc 0.001 0.5", "timing_recovery_cc GARDNER 256 0.5 2 --add_q", "dbpsk_decoder_c_u8", "psk31_varicode_decoder_u8_u8"]
    want = run_graph(ref, stages, x)
    assert TEXT in want
    assert run_graph(ours, stages, x) == want


def test_psk31_refusals(clis):
    ours, _ = clis
    for args in ("timing_recovery_cc GARDNER 30", "timing_recovery_cc GARDNER 4", "timing_recovery_cc GARDNER 32 0.5 2 --add_q --octave 10",
                 "timing_recovery_cc GARDNER 32 1.5 2", "simple_agc_cc 0", "simple_agc_cc 0.1 -1", "simple_agc_cc 0.1 1 0"):
        r = subprocess.run(["bash", "-c", f"{ours} {args}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and r.stderr, args


def test_reference_binary_runs_psk31_on_our_library(clis):
    """the reference's own csdr binary with libcsdr_b200.so preloaded runs timing_recovery_cc and simple_agc_cc on the GPU"""
    ours, ref = clis
    lib = ROOT / "csdr_b200" / "libcsdr_b200.so"
    x = signal(32, 6).tobytes()
    e = dict(os.environ); e.update({"LD_PRELOAD": str(lib), "CSDRB_TRACE": "1"})
    for stage in ("simple_agc_cc 0.001 0.5", "timing_recovery_cc GARDNER 32 0.5 2 --add_q"):
        r = subprocess.run(["bash", "-c", f"{ref} {stage}"], input=x, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e, timeout=120)
        assert r.returncode == 0, r.stderr[-500:]
        tail = r.stderr.decode(errors="replace").split("libcsdr_b200: ")[-1]
        assert "kernel launches" in tail and int(tail.split()[0]) > 0, r.stderr[-500:]
        plain = run_graph(ref, [stage], x)
        if stage.startswith("timing"):
            assert r.stdout == plain
