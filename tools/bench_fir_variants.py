"""Time every compiled tiling of the fir_decimate_cc bank kernel on BASELINE config 2 (256 ch, T=199, D=10)."""
import json, sys
from pathlib import Path
import numpy as np, torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import csdr_b200

C, N, T, D = 256, 2_400_000, 199, 10
if len(sys.argv) > 1: N = int(sys.argv[1])
taps = csdr_b200.firdes_lowpass_f(T, 0.5 / D)
x = torch.rand((C, N, 2), device="cuda") * 2 - 1
n_out = csdr_b200.fir_out_len(N, D, T)
out = torch.empty((C, n_out + (n_out & 1)), dtype=torch.complex64, device="cuda")
peaks = json.loads(Path("MEASURED_PEAKS.json").read_text()) if Path("MEASURED_PEAKS.json").exists() else {"hbm_gbs": 3350.0}
res = {}
nv = csdr_b200.lib().csdrb_fir_bank_variants()
for v in range(nv):
    for _ in range(3): csdr_b200.fir_decimate_bank_cc(x, D, taps, out=out, variant=v)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps): csdr_b200.fir_decimate_bank_cc(x, D, taps, out=out, variant=v)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    msps = C * N / ms / 1e3
    gbs = (C * N * 8 + C * n_out * 8) / ms / 1e6
    tf = C * n_out * T * 4 / ms / 1e9
    res[v] = dict(ms=ms, msps=msps, gbs=gbs, frac_hbm=gbs / peaks["hbm_gbs"], fp32_tflops=tf)
    print(f"variant {v}: {ms:.3f} ms  {msps:,.0f} Msps  {gbs:,.0f} GB/s ({gbs / peaks['hbm_gbs']:.1%} of measured HBM)  {tf:.1f} TFLOP/s fp32", flush=True)
Path("gpurun_out").mkdir(exist_ok=True)
Path("gpurun_out/fir_variants.json").write_text(json.dumps(res, indent=1))
