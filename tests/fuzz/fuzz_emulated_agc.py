"""Fuzz the SHIPPED AM / SSB kernels (csdr_b200/csrc/agc.cu) on the CPU (tests/host_shim/cuda_emul.h) against the CPU restatement
tests/am_ssb/am_ssb_oracle.c, bit for bit: random agc_ff parameters, chunks, channel counts, row strides, input / output kinds and stream cuts;
random fastdcblock block sizes and call splits, f32 or cf32 input.  usage: python tests/fuzz/fuzz_emulated_agc.py [seed] [seconds]"""
import sys, time, tempfile, numpy as np
from pathlib import Path
_ROOT = str(Path(__file__).resolve().parents[2])
sys.path.insert(0, _ROOT); sys.path.insert(0, _ROOT + '/tests/host_shim'); sys.path.insert(0, _ROOT + '/tests/am_ssb')
import emul_build as eb
import am_ssb
from oracle.pyoracle import Oracle
o = Oracle()
agc, _ = eb.build_file(Path(tempfile.mkdtemp(prefix='fuzz_agc_')), 'agc.cu')
P = lambda a: a.ctypes.data
rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
t_end = time.time() + (float(sys.argv[2]) if len(sys.argv) > 2 else 120)
DT = [("r", "<f4"), ("a", "<f4"), ("d", "<f4"), ("m", "<f4"), ("h", "<i4"), ("w", "<i4"), ("al", "<f4"), ("c", "<i4")]


def signal(n):
    x = (rng.uniform(-1, 1, n) * np.exp(rng.uniform(-6, 2, n // 64 + 1)).repeat(64)[:n]).astype(np.float32)
    for _ in range(int(rng.integers(0, 4))):
        s = int(rng.integers(0, n)); x[s:s + int(rng.integers(1, 500))] = 0.0
    return x


it = 0; cases = {'agc': 0, 'dc': 0}
while time.time() < t_end:
    it += 1
    if rng.integers(0, 2) == 0:
        ch = int(rng.integers(1, 70)); n = int(rng.integers(1, 3000)); chunk = int(rng.choice([1, 2, 7, 100, 1000, 1024, 4096]))
        kw = dict(hang_time=int(rng.integers(-5, 300)), reference=float(np.float32(rng.uniform(0.01, 2))), attack_rate=float(np.float32(rng.uniform(0, 0.5))),
                  decay_rate=float(np.float32(rng.uniform(0, 0.05))), max_gain=float(np.float32(rng.choice([5, 100, 65536]))), attack_wait=int(rng.integers(-2, 20)),
                  alpha=float(np.float32(rng.uniform(0, 1))))
        p = np.array([(kw["reference"], kw["attack_rate"], kw["decay_rate"], kw["max_gain"], kw["hang_time"], kw["attack_wait"], kw["alpha"], chunk)], dtype=DT)
        cf32 = bool(rng.integers(0, 2)); s16 = bool(rng.integers(0, 2)); limit = float(rng.choice([0.0, 0.5, 1.0]))
        stride = n + int(rng.integers(0, 9))
        x = np.zeros((ch, stride), np.complex64 if cf32 else np.float32)
        for c in range(ch):
            x[c, :n] = signal(n) + (1j * rng.standard_normal(n) if cf32 else 0)
        y = np.zeros((ch, stride), np.int16 if s16 else np.float32)
        st = np.zeros((ch, 5), np.int32); st[:, 0] = np.array([1.0], np.float32).view(np.int32)[0]
        cuts = np.unique(np.r_[0, np.sort(rng.integers(0, n + 1, int(rng.integers(0, 5)))), n])
        for s0, s1 in zip(cuts[:-1], cuts[1:]):
            rc = agc.emul_launch_agc_bank(P(x) + int(s0) * x.itemsize, stride, int(cf32), P(y) + int(s0) * y.itemsize, stride, int(s16), ch, int(s1 - s0), P(p), P(st), limit)
            assert rc >= 0, agc.emul_last_error()
        for c in range(ch):
            want = am_ssb.agc_tail(x[c, :n], o, chunk, limit, s16, **kw)
            assert np.array_equal(y[c, :n].view(np.uint8), want.view(np.uint8)), ('agc', ch, n, chunk, kw, cf32, s16, limit, c)
        cases['agc'] += 1
    else:
        block = int(rng.integers(1, 1500)); nb = int(rng.integers(1, 20)); ch = int(rng.integers(1, 6)); cf32 = bool(rng.integers(0, 2))
        n = block * nb; stride = n + int(rng.integers(0, 5))
        x = (rng.standard_normal((ch, stride)) + (1j * rng.standard_normal((ch, stride)) if cf32 else 0) + rng.uniform(-3, 3)).astype(np.complex64 if cf32 else np.float32)
        y = np.zeros((ch, stride), np.float32); last = rng.uniform(-1, 1, ch).astype(np.float32); last0 = last.copy()
        split = int(rng.integers(0, nb + 1))
        for b0, k in ((0, split), (split, nb - split)):
            if k:
                assert agc.emul_launch_fastdcblock_bank(P(x) + b0 * block * x.itemsize, stride, int(cf32), P(y) + b0 * block * 4, stride, ch, block, k, P(last)) >= 0, agc.emul_last_error()
        for c in range(ch):
            src = am_ssb.amdemod_cf(x[c, :n]) if cf32 else x[c, :n]
            want, lw = am_ssb.fastdcblock_stream(src, block, float(last0[c]))
            assert np.array_equal(y[c, :n].view(np.int32), want.view(np.int32)) and np.float32(lw) == last[c], ('dc', block, nb, split, cf32, c)
        cases['dc'] += 1
print("iterations", it, "cases", cases)
