"""Times the amplitude modulator banks and the transmit chains they feed on the GPU: each bank (gain_ff, dsb_fc, add_dcoffset_cc,
fixed_amplitude_cc) on 1024 channels of 60 s of 48 kHz audio (2 880 000 samples per channel), with its bytes moved per second as a share of the
H100's 3.35 TB/s HBM3 bandwidth (each is a stream: read once, write once); and the whole `csdr-synth --mod usb` and `--mod am` chains into the
synthesis bank at I = 50 (401 taps) on 1024 channels of 1 s of audio, with the modulators' share of the chain's GPU time.  CUDA events after a
warm-up.  Prints one JSON line with the card's name and power limit."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import csdr_b200 as cb  # noqa: E402

RATE, SECONDS, CH, HBM = 48_000, 60, 1024, 3.35e12


def timed(fn, reps=10):
    for _ in range(2):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps / 1e3


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": q.splitlines()[0] if q else torch.cuda.get_device_name(), "channels": CH, "sample_rate": RATE}
    n = RATE * SECONDS
    audio = torch.rand((CH, n), device="cuda") * 2 - 1                 # 11.8 GB; the complex rows twice that, so one set of rows at a time
    res["banks"] = {"signal_seconds": SECONDS}

    def record(name, fn, bytes_per_sample):
        t = timed(fn)
        res["banks"][name] = {"ms": round(t * 1e3, 3), "GBps": round(CH * n * bytes_per_sample / t / 1e9, 1),
                              "share_of_hbm": round(CH * n * bytes_per_sample / t / HBM, 3)}

    out_f = torch.empty_like(audio)
    record("gain_ff", lambda: cb.gain_bank(audio, 0.5, out=out_f), 8)
    del out_f
    record("dsb_fc", lambda: cb.dsb_bank(audio, 0.0), 12)
    bb = cb.dsb_bank(audio)
    del audio
    record("add_dcoffset_cc", lambda: cb.add_dcoffset_bank(bb, out=bb), 16)
    record("fixed_amplitude_cc", lambda: cb.fixed_amplitude_bank(bb, 1.0, out=bb), 16)
    del bb
    torch.cuda.empty_cache()
    # the chains of csdr-synth --mod usb / am at I = 50, one second of audio per channel (48 000 baseband samples, 2.4 M wideband outputs)
    I, m = 50, RATE
    taps = cb.firdes_lowpass_f(cb.firdes_filter_len(0.05), 0.5 / I)
    rates = np.linspace(-0.45, 0.45, CH).astype(np.float32)
    T, N, unit, _ = cb.bandpass_geometry(0.05)
    usable = m // unit * unit
    a = torch.rand((CH, m), device="cuda") * 2 - 1
    g = torch.empty_like(a)
    tfft = cb.bandpass_taps_fft(0.0, 0.1, 0.05)
    tail = torch.zeros((CH, N), dtype=torch.complex64, device="cuda")
    res["chains"] = {"interpolation": I, "signal_seconds": m / RATE}
    for mode in ("usb", "am"):
        def mods():
            cb.gain_bank(a, 1.0, out=g)
            d = cb.dsb_bank(g)
            if mode == "am":
                return cb.add_dcoffset_bank(d, out=d)
            return cb.bandpass_fir_fft_bank_cc(d[:, :usable], tfft, unit, tail)[0]
        base = mods()
        t_mod = timed(mods)
        t_syn = timed(lambda: cb.synth_bank(base, rates, I, taps), reps=3)
        res["chains"][mode] = {"modulators_ms": round(t_mod * 1e3, 3), "synth_bank_ms": round(t_syn * 1e3, 3),
                               "modulators_share": round(t_mod / (t_mod + t_syn), 4), "realtime_factor": round(CH * m / RATE / (t_mod + t_syn), 0)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
