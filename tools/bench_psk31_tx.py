"""Times the BPSK31 transmit banks on the GPU for 128 and 1024 channels of 60 s of 8 kHz baseband at sps 256 (1875 symbols, 480 000
outputs per channel): each bank's GPU time from CUDA events after a warm-up, the interpolator's stored bytes per second as a share of the
H100's 3.35 TB/s HBM3 bandwidth (it is bound by its stores: 8 bytes out per output), and real-time factors (signal seconds per GPU second).
Prints one JSON line with the card's name and power limit."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import csdr_b200  # noqa: E402

RATE, SECONDS, SPS, HBM = 8000, 60, 256, 3.35e12


def timed(fn, reps=20):
    for _ in range(3):
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
    symbols = RATE * SECONDS // SPS
    chars = symbols // 12                                            # about one character per 12 bits
    res = {"gpu": q.splitlines()[0] if q else torch.cuda.get_device_name(), "signal_seconds": SECONDS, "sample_rate": RATE, "sps": SPS}
    for ch in (128, 1024):
        text = torch.randint(32, 127, (ch, chars), dtype=torch.uint8, device="cuda")
        bits = torch.randint(0, 2, (ch, symbols), dtype=torch.uint8, device="cuda")
        sym = csdr_b200.psk_modulator_bank_u8_c(bits, 2)
        last = torch.zeros(ch, dtype=torch.complex64, device="cuda")
        t_enc = timed(lambda: csdr_b200.psk31_varicode_encoder_bank_u8_u8(text))
        t_dc = timed(lambda: csdr_b200.differential_codec_bank_u8_u8(bits, True))
        t_mod = timed(lambda: csdr_b200.psk_modulator_bank_u8_c(bits, 2))
        out = torch.empty((ch, symbols * SPS), dtype=torch.complex64, device="cuda")
        t_int = timed(lambda: csdr_b200.lib().csdrb_psk31_interpolate_sine_bank_cc(sym.data_ptr(), sym.stride(0), out.data_ptr(), out.stride(0), ch,
                                                                                   symbols, None, SPS, last.data_ptr(), csdr_b200._stream()))
        stored = ch * symbols * SPS * 8
        total = t_enc + t_dc + t_mod + t_int
        res[f"ch{ch}"] = {"encoder_ms": round(t_enc * 1e3, 4), "codec_ms": round(t_dc * 1e3, 4), "modulator_ms": round(t_mod * 1e3, 4),
                          "interpolator_ms": round(t_int * 1e3, 4), "interpolator_store_GBps": round(stored / t_int / 1e9, 1),
                          "interpolator_share_of_hbm": round(stored / t_int / HBM, 3), "bound": "stores",
                          "realtime_factor_chain": round(ch * SECONDS / total, 0), "realtime_factor_interpolator": round(ch * SECONDS / t_int, 0)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
