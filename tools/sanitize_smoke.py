"""Every kernel once on small, awkward sizes -- meant to run under `compute-sanitizer --tool memcheck` (and racecheck)."""
import sys, numpy as np, torch
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import csdr_b200 as cb
dev = "cuda"; rng = np.random.default_rng(0)
def cplx(*shape): return torch.view_as_complex(torch.rand(shape + (2,), device=dev) * 2 - 1)
cb.convert_u8_f(torch.randint(0, 256, (4099,), dtype=torch.uint8, device=dev)); cb.convert_s16_f(torch.randint(-30000, 30000, (4099,), dtype=torch.int16, device=dev))
f = torch.rand(4099, device=dev); cb.convert_f_s16(f); cb.limit_ff(f, 0.5)
taps = cb.firdes_lowpass_f(199, 0.05)
for n in (199, 208, 9999, 30011):
    for v in (-1, 0, 1, 2, 3): cb.fir_decimate_bank_cc(cplx(3, n + (n & 1))[:, :n] if False else cplx(3, n + (n & 1)), 10, taps, variant=v)
cb.fir_decimate_bank_cc(cplx(2, 5001), 7, cb.firdes_lowpass_f(79, 0.07))            # generic kernel, odd stride
cb.fir_decimate_bank_cc(cplx(2, 70000), 50, cb.firdes_lowpass_f(801, 0.01))
y = cb.fmdemod_quadri_bank_cf(cplx(3, 10001))
cb.shift_addition_bank_cc(cplx(16384 + 777), [0.1, -0.3, 0.45], chunk=1024); cb.shift_addition_bank_cc(cplx(3, 1000), [0.1, -0.3, 0.45], chunk=37)
a = torch.rand((3, 20000), device=dev); cb.fractional_decimator_bank_ff(a, 5.0, 12); cb.fractional_decimator_bank_ff(a, 2.5, 4, taps=cb.firdes_lowpass_f(31, 0.15))
cb.fastagc_bank_ff(a[:, :19 * 1024], 1024, 1.0); cb.fastagc_bank_ff(a[:, :1000], 1000, 1.0); cb.deemphasis_wfm_bank_ff(a[:37 if False else 3, :10001].contiguous(), 50e-6, 48000)
for n in (2, 4, 8, 16, 64, 512, 4096, 16384): cb.fft_c2c(cplx(2, n)); cb.fft_c2c(cplx(2, n), inverse=True)
for bw in (0.002, 0.05, 0.005):
    T, N, isz, ov = cb.bandpass_geometry(bw); cb.bandpass_fir_fft_bank_cc(cplx(3, 9 * isz), cb.bandpass_taps_fft(-0.1, 0.1, bw), isz)
for bw, dec, sh in ((0.002, 64, [0.1, -0.3, 0.0, 0.2, 0.44]), (0.01, 6, [0.25]), (0.05, 8, [0.123, -0.2])):
    d = cb.fastddc_init(bw, dec, 0.0); sp, ov = cb.fastddc_fwd_cc(cplx(3 * d.input_size), d); cb.fastddc_inv_bank_cc(sp, sh, dec, bw)
for D, bw in ((50, 0.005), (10, 0.0201), (10, 0.05)):
    T = cb.firdes_filter_len(bw)
    for demod in (True, False): cb.ddc_bank(cplx(40000 + 14), np.linspace(-0.4, 0.4, 37), D, cb.firdes_lowpass_f(T, 0.5 / D), demod=demod, chunk=1024, offset=100)
x = rng.integers(0, 256, 5000).astype(np.uint8); cb.libcsdr.convert_u8_f(x); cb.libcsdr.fir_decimate_cc(rng.normal(size=4000).astype(np.complex64), 10, taps)
for sr in (48000, 44100, 11025, 8000):
    for n in (202, 1024 + 201, 1024 + 202, 5000): cb.deemphasis_nfm_bank_ff(a[:, :n], sr, limit_max=0.5 if n & 1 else 0.0)
cb.shift_addfast_bank_cc(cplx(16384 + 777), [0.1, -0.3, 0.45], chunk=1024); cb.shift_addfast_bank_cc(cplx(3, 1001), [0.1, -0.3, 0.45], chunk=37)
cb.libcsdr.shift_addfast_cc(rng.normal(size=1022).astype(np.complex64), 0.2); cb.libcsdr.deemphasis_nfm_ff(rng.normal(size=3000).astype(np.float32), 48000)
# round 2: u8 front end (fused and two-launch), long phase chains on the wrap table, fold-path fastddc on ragged banks, fused AGC + s16, streaming bank + retune
u8 = torch.randint(0, 256, (3, 20008, 2), dtype=torch.uint8, device=dev)
cb.fir_decimate_bank_u8_cc(u8[:, :20001], 10, taps); cb.fir_decimate_bank_u8_cc(u8[:, :20001], 50, cb.firdes_lowpass_f(801, 0.01)); cb.fir_decimate_bank_u8_cc(u8[:, :9999].contiguous(), 7, cb.firdes_lowpass_f(33, 0.1))
cb.shift_addition_bank_cc(cplx(130 * 1024 + 5), [0.1, -0.3, 0.45, 1e-4], chunk=1024); cb.shift_addfast_bank_cc(cplx(9000), [0.2, -0.4], chunk=64)
d = cb.fastddc_init(0.002, 64, 0.0); sp, ov = cb.fastddc_fwd_cc(cplx(130 * d.input_size), d); cb.fastddc_inv_bank_cc(sp, list(np.linspace(-0.4, 0.4, 17)), 64, 0.002)
cb.fastagc_bank_f_s16(a[:, :19 * 1024], 1024, 1.0); cb.fastagc_bank_f_s16(a[:, :19 * 1000], 1000, 1.0); cb.fastagc_bank_f_s16(a[:, :8 * 2048], 2048, 1.0)
bank = cb.DdcBank(np.linspace(-0.4, 0.4, 37), 50, cb.firdes_lowpass_f(801, 0.5 / 50), demod=True, chunk=1024)
w = cplx(60000); o1 = bank.process(w[:20000]); bank.set_rate(3, 0.11); bank.process(w[o1.shape[1] * 50:o1.shape[1] * 50 + 30000]); bank.close()
# round 2, late: fastddc plan object (look-ahead, retune), sliced K2 chain (>= 512 chunks), ragged sizes
plan = cb.FastddcInvPlan(list(np.linspace(-0.4, 0.4, 5)), 64, 0.002, 7)
sp7, _ = cb.fastddc_fwd_cc(cplx(7 * d.input_size), d)
plan.run(sp7); plan.set_shift(2, 0.123); plan.run(sp7); plan.state(); plan.run(sp7); plan.close()
cb.shift_addition_bank_cc(cplx(2, 600 * 64 + 13), [0.31, -0.07], chunk=64); cb.shift_addition_bank_cc(cplx(1100 * 1024 + 1), [0.2], chunk=1024)
torch.cuda.synchronize(); print("sanitize_smoke: all kernels ran")
# transmit banks: fir_interpolate (staged taps and taps past the shared-memory tile, ragged rows, odd strides), fmmod with several wraps per sample
for I, T, n in ((1, 7, 999), (3, 81, 1001), (50, 401, 333), (256, 2049, 37), (5, 9001, 2000)):
    cb.fir_interpolate_bank(cplx(3, n + 1)[:, :n], I, cb.firdes_lowpass_f(T, 0.5 / I))
ph = torch.zeros(5, device=dev); cb.fmmod_bank((torch.rand((5, 1037), device=dev) * 2 - 1) * 9, ph); cb.fmmod_bank(torch.rand((5, 31), device=dev), ph)
# BPSK31 transmit banks at awkward sizes: rows across scan chunks, a cut encoder, odd lengths, both interpolator rate paths
txt = torch.randint(0, 256, (3, 1031), dtype=torch.uint8, device=dev)
cb.psk31_varicode_encoder_bank_u8_u8(txt); cb.psk31_varicode_encoder_bank_u8_u8(txt, output_max_size=777)
cb.differential_codec_bank_u8_u8(txt, True); cb.differential_codec_bank_u8_u8(txt, False)
cb.psk_modulator_bank_u8_c(txt, 256)
cb.psk31_interpolate_sine_bank_cc(cplx(3, 37), 257); cb.psk31_interpolate_sine_bank_cc(cplx(2, 3), 9001)
torch.cuda.synchronize()
# synthesis bank: the register window at h = 1 and 8, the general path with taps in shared memory and past it, ragged warps, two CTAs of
# channels (the second tree pass), chunks of 1 and 7 with offsets, n below one group, the streaming object
for ch, I, T, n, chunk, off in ((1, 1, 1, 300, 7, 3), (33, 50, 401, 40, 1024, 17), (257, 2, 2, 100, 7, 2), (5, 3, 40, 200, 1, 0), (3, 50, 9001, 190, 1024, 0),
                               (100, 256, 2049, 11, 1024, 1023), (2, 50, 401, 8, 1024, 0)):
    cb.synth_bank(cplx(ch, n + 1)[:, :n], np.linspace(-0.45, 0.45, ch), I, rng.uniform(-1, 1, T).astype(np.float32), chunk=chunk, offset=off)
sb = cb.SynthBank(np.linspace(-0.4, 0.4, 40), 50, cb.firdes_lowpass_f(401, 0.01)); w = cplx(40, 3000); sb.process(w[:, :1000].contiguous()); sb.process(w[:, 992:2500].contiguous()); sb.close()
torch.cuda.synchronize()
# amplitude modulator banks: 128-bit rows, rows off 16-byte alignment (odd strides, offset starts), ragged tails, in place
r = (torch.rand((3, 1037), device=dev) * 2 - 1)
cb.gain_bank(r[:, :1035], 0.7); cb.gain_bank(r[:, 1:1030], 2.0); cb.gain_bank(r, 0.5, out=r)
cb.dsb_bank(r[:, :1033], 0.1); cb.dsb_bank(r[:, 3:], 0.0)
z = cplx(3, 1037)
cb.add_dcoffset_bank(z[:, :1035]); cb.add_dcoffset_bank(z[:, 1:]); cb.add_dcoffset_bank(z, out=z)
cb.fixed_amplitude_bank(z[:, :1031], 2.0); cb.fixed_amplitude_bank(z[:, 1:], 1.0); cb.fixed_amplitude_bank(z, 0.5, out=z)
torch.cuda.synchronize()
# demodulator banks: atan tiles with ragged ends and rows off 16-byte alignment, novect, the estimator's pair and single paths, dcblock in place
z = cplx(3, 2051)
for n in (1, 5, 1023, 1025, 2051): cb.fmdemod_atan_bank_cf(z[:, :n]); cb.fmdemod_atan_bank_cf(z[:, 1:n + 1] if n < 2051 else z[:, :n], last=torch.zeros(3, device=dev))
cb.fmdemod_atan_bank_cf(z, return_last=True); cb.fmdemod_quadri_novect_bank_cf(z[:, :2049]); cb.fmdemod_quadri_novect_bank_cf(z[:, 1:], return_last=True)
cb.amdemod_estimator_bank_cf(z[:, :1]); cb.amdemod_estimator_bank_cf(z[:, 1:1030], 0.5, 0.25); cb.amdemod_estimator_bank_cf(z)
r = (torch.rand((37, 1037), device=dev) * 2 - 1)
cb.dcblock_bank_ff(r[:, :1035]); cb.dcblock_bank_ff(r[:, 1:1030].contiguous(), 0.9, return_state=True); cb.dcblock_bank_ff(r, out=r)
torch.cuda.synchronize()
