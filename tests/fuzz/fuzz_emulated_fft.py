"""Fuzz the SHIPPED FFT-family kernels on the CPU (tests/host_shim/cuda_emul.h): random overlap-add geometries against numpy, random fastddc
geometries against the oracle, each also within the per-output bounds of tests/test_fft_bound_emulated.py.  usage: python tests/fuzz/fuzz_emulated_fft.py [seed] [seconds]   -- test infrastructure."""
import sys, time, tempfile, ctypes as C, numpy as np
from pathlib import Path
_ROOT = str(Path(__file__).resolve().parents[2])
sys.path.insert(0, _ROOT); sys.path.insert(0, _ROOT + '/tests/host_shim'); sys.path.insert(0, _ROOT + '/tests')
import emul_build as eb
import test_fft_bound_emulated as B
from oracle.pyoracle import Oracle, rel_rms, _CF, _p, WINDOWS
o = Oracle()
fft, _ = eb.build_file(Path(tempfile.mkdtemp(prefix='fuzz_fft_')), 'fft.cu')
P = lambda a: a.ctypes.data
rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
t_end = time.time() + (float(sys.argv[2]) if len(sys.argv) > 2 else 120)
def cplx(*s): return (rng.uniform(-1, 1, s) + 1j * rng.uniform(-1, 1, s)).astype(np.complex64)
it = 0; worst = {}
while time.time() < t_end:
    it += 1
    if rng.integers(0, 2) == 0:
        N = int(2 ** rng.integers(2, 13)); isz = int(rng.integers(1, N + 1)); nb = int(rng.integers(1, 12)); bpc = int(rng.integers(0, 9)); ch = int(rng.integers(1, 3))
        x = cplx(ch, nb * isz); H = cplx(ch, N); y = np.zeros_like(x); tail0 = cplx(ch, N); tail = tail0.copy()
        assert fft.emul_launch_olafir_bank(P(x), x.shape[1], P(y), y.shape[1], ch, N, isz, nb, P(H), N, P(tail), bpc) >= 0, fft.emul_last_error()
        for c in range(ch):
            out = np.zeros(nb * isz + N - isz, np.complex128); out[:N - isz] = tail0[c, :N - isz]      # a stream that continues: the carried tail comes first
            for b in range(nb):
                blk = np.zeros(N, np.complex128); blk[:isz] = x[c, b * isz:(b + 1) * isz]
                out[b * isz:b * isz + N] += np.fft.ifft(np.fft.fft(blk) * H[c].astype(np.complex128))
            e = rel_rms(y[c], out[:nb * isz]); worst['ola'] = max(worst.get('ola', 0), e); assert e < 3e-6, ('ola', N, isz, nb, bpc, e)
            want, bound = B.ola_model(x[c], H[c], N, isz, B.ola_form(N), tail=tail0[c])
            r = float(np.max(np.abs(y[c] - want) / bound)); worst['ola bound'] = max(worst.get('ola bound', 0), r); assert r <= 1, ('ola bound', N, isz, nb, bpc, r)
            if N > isz:
                scale = np.sqrt(np.mean(np.abs(out) ** 2))                         # a one-sample tail is all cancellation: normalise by the stream's level
                e = float(np.abs(tail[c, :N - isz] - out[nb * isz:]).max() / scale); assert e < 1e-5, ('ola tail', N, isz, nb, bpc, e)
    else:
        bw = float(np.float32(rng.uniform(0.02, 0.2))); dec = int(rng.integers(1, 40)); shift = float(np.float32(rng.uniform(-0.5, 0.5)))
        g, err = o.fastddc_init(bw, dec, shift)
        if err or g.fft_size > 4096 or g.fft_inv_size < 2: continue
        nb = int(rng.integers(1, 5)); chn = int(rng.integers(1, 6))
        x = (cplx(nb * g.input_size) * 0.3).astype(np.complex64)
        sp = np.zeros((nb, g.fft_size), np.complex64); carry = np.zeros(max(g.overlap_length, 1), np.complex64)
        assert fft.emul_launch_fastddc_fwd(P(x), P(sp), P(carry), g.fft_size, g.input_size, nb) >= 0
        want_sp = np.stack(o.fastddc_fwd(x, g)); e = rel_rms(sp, want_sp); worst['fwd'] = max(worst.get('fwd', 0), e); assert e < 2e-6, ('fwd', bw, dec, e)
        shifts = [shift] + [float(np.float32(rng.uniform(-0.5, 0.5))) for _ in range(chn - 1)]
        gs = [o.fastddc_init(bw, dec, s)[0] for s in shifts]
        tf = np.empty((chn, g.fft_size), np.complex64)
        for k, (gk, s) in enumerate(zip(gs, shifts)): o.L.oracle_fastddc_make_taps_fft(C.byref(gk), s, dec, WINDOWS["HAMMING"], _p(tf[k], _CF))
        chan = np.zeros(chn, np.dtype([("offsetbin", np.int32), ("sindelta", np.float32), ("cosdelta", np.float32), ("rate", np.float32)]))
        for k, gk in enumerate(gs): chan[k] = (gk.offsetbin, gk.dsadata.sindelta, gk.dsadata.cosdelta, gk.dsadata.rate)
        remain = np.zeros(chn, np.int32); phase = np.zeros(chn, np.float32); total = np.zeros(chn, np.int32)
        out = np.zeros((chn, nb * (g.post_input_size // g.post_decimation + 1) + 2), np.complex64)
        sb = fft.emul_fastddc_inv_scratch_bytes(chn, nb); scr = np.zeros(sb + 16, np.uint8)
        rc = fft.emul_launch_fastddc_inv_bank(P(want_sp), nb, P(tf), P(chan), chn, g.fft_size, g.fft_inv_size, g.pre_decimation, g.scrap, g.post_input_size, g.post_decimation,
                                              P(remain), P(phase), P(out), out.shape[1], P(total), P(scr), sb)
        assert rc >= 0, fft.emul_last_error()
        for k, s in enumerate(shifts):
            w = o.fastddc_inv(list(want_sp), bw, dec, s)
            assert total[k] == w.size, ('inv count', bw, dec, s, total[k], w.size)
            if w.size:
                e = rel_rms(out[k, :w.size], w); worst['inv'] = max(worst.get('inv', 0), e); assert e < 1e-5, ('inv', bw, dec, s, e)
                m, bound, _, _, _ = B.fastddc_inv_model(o, want_sp, tf[k], chan[k], gs[k], B.inv_path(g, nb, chn))
                r = float(np.max(np.abs(out[k, :w.size] - m) / bound)); worst['inv bound'] = max(worst.get('inv bound', 0), r); assert r <= 1, ('inv bound', bw, dec, s, r)
print("iterations", it, "worst", worst)
