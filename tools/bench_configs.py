"""Throughput of the non-headline BASELINE configs and of the standalone streaming kernels on one H100 (device-resident data).
Prints one line per measurement and writes gpurun_out/configs.json.  Parity for all of these is in tests/ (-m gpu)."""
import json, os, sys, time
from pathlib import Path
import numpy as np, torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import csdr_b200 as cb

PEAK = json.loads(Path("MEASURED_PEAKS.json").read_text())["hbm_gbs"] if Path("MEASURED_PEAKS.json").exists() else 3350.0
res = {}


def timed(fn, reps=5, warm=2):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def report(name, ms, samples, algo_bytes, extra=""):
    gbs = algo_bytes / ms / 1e6
    res[name] = dict(ms=ms, msps=samples / ms / 1e3, gbs=gbs, frac_hbm=gbs / PEAK)
    print(f"{name:58s} {ms:9.3f} ms  {samples / ms / 1e3:12,.0f} Msps  {gbs:8,.0f} GB/s algorithmic ({gbs / PEAK:6.1%} of HBM) {extra}", flush=True)


which = set(sys.argv[1:]) or {"k", "c3", "c4", "c5"}
dev = "cuda"
if "k" in which:
    n = 1 << 28
    u8 = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev); f = torch.empty(n, dtype=torch.float32, device=dev)
    report("K1 convert_u8_f", timed(lambda: cb.convert_u8_f(u8, out=f)), n / 2, n * 5)
    s16 = torch.empty(n, dtype=torch.int16, device=dev)
    report("K1 convert_f_s16", timed(lambda: cb.convert_f_s16(f, out=s16)), n, n * 6)
    report("K1 convert_s16_f", timed(lambda: cb.convert_s16_f(s16, out=f)), n, n * 6)
    del u8, s16
    taps3 = cb.firdes_lowpass_f(199, 0.05)
    u8b = torch.randint(0, 256, (256, 2_400_000, 2), dtype=torch.uint8, device=dev)
    n3 = cb.fir_out_len(2_400_000, 10, 199); y3 = torch.empty((256, n3 + (n3 & 1)), dtype=torch.complex64, device=dev)
    report("K1+K3 u8 front end fused into the FIR bank 256x2.4M (2 + 8/D B/sample)", timed(lambda: cb.fir_decimate_bank_u8_cc(u8b, 10, taps3, out=y3)), 256 * 2_400_000, 256 * 2_400_000 * 2.8,
           f"{256 * n3 * 199 * 4 / 1e9:.0f} Gflop per launch")
    del u8b, y3
    C, N = 64, 2_400_000
    x = torch.rand((C, N, 2), device=dev) * 2 - 1
    y = torch.empty((C, N), dtype=torch.float32, device=dev)
    report("K4 fmdemod_quadri bank 64x2.4M", timed(lambda: cb.fmdemod_quadri_bank_cf(x, out=y)), C * N, C * N * 12)
    rates = np.linspace(-0.4, 0.4, C).astype(np.float32)
    xc = torch.view_as_complex(x)
    out = torch.empty((C, N), dtype=torch.complex64, device=dev)
    report("K2 shift_addition bank 64x2.4M chunk 1024", timed(lambda: cb.shift_addition_bank_cc(xc, rates, chunk=1024, out=out)), C * N, C * N * 16)
    steps = np.stack([cb.shift_addfast_init(float(r)) for r in rates]); table = torch.from_numpy(cb.libcsdr.shift_table_init(65536)).to(dev)
    report("K2 shift_addfast bank 64x2.4M chunk 1024", timed(lambda: cb.shift_addfast_bank_cc(xc, steps=steps, chunk=1024, out=out)), C * N, C * N * 16)
    report("K2 shift_math bank 64x2.4M", timed(lambda: cb.shift_math_bank_cc(xc, rates, out=out)), C * N, C * N * 16)
    report("K2 shift_table bank 64x2.4M (65536-entry table)", timed(lambda: cb.shift_table_bank_cc(xc, rates, table, out=out)), C * N, C * N * 16)
    a = y[:, :N // 10 * 10].contiguous()
    report("K5 fractional_decimator bank 64x2.4M rate 5", timed(lambda: cb.fractional_decimator_bank_ff(a, 5.0, 12)), C * a.shape[1], C * a.shape[1] * 4.8)
    a2 = a[:, :2343 * 1024].contiguous()
    report("K6 fastagc bank 64x2.4M block 1024", timed(lambda: cb.fastagc_bank_ff(a2, 1024, 1.0)), C * a2.shape[1], C * a2.shape[1] * 8)
    del x, y, out, a, a2, xc
    for nfft in (512, 4096, 16384):
        b = (1 << 26) // nfft
        z = torch.view_as_complex(torch.rand((b, nfft, 2), device=dev))
        report(f"K7 fft_c2c {nfft} x {b}", timed(lambda: cb.fft_c2c(z)), b * nfft, b * nfft * 16)
        del z
    torch.cuda.empty_cache()

if "c3" in which:
    bw, dec, C = 0.002, 64, 64
    ddc = cb.fastddc_init(bw, dec, 0.0)
    nblocks = int(os.environ.get("C3_BLOCKS", "256"))
    x = torch.view_as_complex(torch.rand((nblocks * ddc.input_size, 2), device=dev) * 2 - 1)
    shifts = list(np.linspace(-0.45, 0.45, C))
    sp, ov = cb.fastddc_fwd_cc(x, ddc)
    out, counts, st = cb.fastddc_inv_bank_cc(sp, shifts, dec, bw)
    t_f = timed(lambda: cb.fastddc_fwd_cc(x, ddc, overlap=ov))
    t_i = timed(lambda: cb.fastddc_inv_bank_cc(sp, shifts, dec, bw, state=st))
    nsamp = nblocks * ddc.input_size
    algo = nsamp * 16
    report("cfg3 fastddc fwd 16384-pt", t_f, nsamp, nsamp * 8 + nblocks * ddc.fft_size * 8)
    report("cfg3 fastddc inv bank 64 ch", t_i, nsamp, nblocks * ddc.fft_size * 8 + C * nblocks * 224 * 8)
    report("cfg3 fastddc fwd+inv (16 B/wideband sample)", t_f + t_i, nsamp, algo, f"= {nsamp / (t_f + t_i) / 1e3 / 61.44:.0f}x real time at 61.44 Msps")
    plan = cb.FastddcInvPlan(shifts, dec, bw, nblocks)
    t_p = timed(lambda: plan.run(sp))
    report("cfg3 fastddc inv bank 64 ch, plan object (look-ahead)", t_p, nsamp, nblocks * ddc.fft_size * 8 + C * nblocks * 224 * 8)

    def both():
        cb.fastddc_fwd_cc(x, ddc, overlap=ov)
        plan.run(sp)
    t_b = timed(both)
    report("cfg3 fastddc fwd + plan.run, one loop", t_b, nsamp, algo, f"= {nsamp / t_b / 1e3 / 61.44:.0f}x real time at 61.44 Msps")
    plan.close()
    del x, sp, out
    torch.cuda.empty_cache()

if "c4" in which:
    C, N, D, bw = 128, 1 << 21, 50, 0.005
    T = cb.firdes_filter_len(bw)
    taps = cb.firdes_lowpass_f(T, 0.5 / D)
    x = torch.view_as_complex(torch.rand((N, 2), device=dev) * 2 - 1)
    rates = np.linspace(-0.45, 0.45, C).astype(np.float32)
    shifted = torch.empty((C, N), dtype=torch.complex64, device=dev)
    n_out = cb.fir_out_len(N, D, T)
    base = torch.empty((C, n_out + (n_out & 1)), dtype=torch.complex64, device=dev)
    audio = torch.empty((C, n_out + (n_out & 1)), dtype=torch.float32, device=dev)

    def chain():
        cb.shift_addition_bank_cc(x, rates, chunk=1024, out=shifted)
        cb.fir_decimate_bank_cc(shifted, D, taps, out=base)
        cb.fmdemod_quadri_bank_cf(base[:, :n_out], out=audio)
    t1 = timed(lambda: cb.shift_addition_bank_cc(x, rates, chunk=1024, out=shifted), reps=3)
    t2 = timed(lambda: cb.fir_decimate_bank_cc(shifted, D, taps, out=base), reps=3)
    t3 = timed(lambda: cb.fmdemod_quadri_bank_cf(base[:, :n_out], out=audio), reps=3)
    report(f"cfg4 shift (shared in) 128 ch x {N}", t1, N, N * 8 + C * N * 8)
    report(f"cfg4 fir_decimate d=50 T={T} 128 ch (independent-input bank kernel)", t2, N, C * N * 8.16, f"{C * n_out * T * 4 / t2 / 1e9:.1f} TFLOP/s")
    report("cfg4 fmdemod 128 ch", t3, N, C * n_out * 12)
    report("cfg4 unfused chain, wideband Msps per GPU (18.24 B/sample algorithmic)", timed(chain, reps=3), N, N * 18.24)
    fo = torch.empty((C, n_out + (n_out & 1)), dtype=torch.float32, device=dev)
    tfu = timed(lambda: cb.ddc_bank(x, rates, D, taps, demod=True, chunk=1024, out=fo), reps=5)
    report("cfg4 FUSED ddc_bank (shift|fir d=50 T=801|fmdemod) 128 ch", tfu, N, N * 18.24, f"{C * N * (10 + 4 * 17 * 1.0) / tfu / 1e9:.1f} TFLOP/s fp32 (10+4M flop per sample-channel)")
    bank = cb.DdcBank(rates, D, taps, demod=True, chunk=1024)
    tbk = timed(lambda: bank.process(x, out=fo), reps=8, warm=3)
    report("cfg4 FUSED via bank object (pre-pass of block k+1 overlaps block k)", tbk, N, N * 18.24, f"{C * N * (10 + 4 * 17 * 1.0) / tbk / 1e9:.1f} TFLOP/s fp32")
    bank.close()
    del shifted, base, audio
    torch.cuda.empty_cache()

if "c5" in which:
    T, NF, isz, ov = cb.bandpass_geometry(0.002)
    tf = cb.bandpass_taps_fft(-0.05, 0.05, 0.002)
    C = 512
    for L in (65536, 262144, 1048576):
        nb = L // isz
        x = torch.view_as_complex(torch.rand((C, nb * isz, 2), device=dev) * 2 - 1)
        tail = torch.zeros((C, NF), dtype=torch.complex64, device=dev)
        t = timed(lambda: cb.bandpass_fir_fft_bank_cc(x, tf, isz, tail=tail), reps=3)
        report(f"cfg5 bandpass_fir_fft bank 512 ch x {L} (4096-pt)", t, C * nb * isz, C * nb * isz * 16)
        del x
        torch.cuda.empty_cache()

Path("gpurun_out").mkdir(exist_ok=True)
prev = json.loads(Path("gpurun_out/configs.json").read_text()) if Path("gpurun_out/configs.json").exists() else {}
prev.update(res)
Path("gpurun_out/configs.json").write_text(json.dumps(prev, indent=1))
