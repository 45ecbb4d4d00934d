"""GPU time of the BPSK31 receive chain per second of signal: simple_agc_cc | timing_recovery_cc GARDNER 256 | dbpsk_decoder_c_u8 | varicode
decoder for 128 and 1024 channels of 8 kHz baseband (31.25 Bd at 256 samples per symbol), one bank call of each per second of signal.
CUDA events around the four launches after warm-up; prints one line per channel count with the card name and power limit."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import csdr_b200 as cb  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    rate, sps, reps = 8000, 256, 20
    rng = np.random.default_rng(0)
    for ch in (128, 1024):
        bits = rng.integers(0, 2, (ch, rate // sps + 2))
        sym = np.cumprod(np.where(bits, 1.0, -1.0), axis=1)
        x = torch.from_numpy((0.3 * np.repeat(sym, sps, axis=1)[:, :rate] + 0.01 * rng.standard_normal((ch, rate))).astype(np.complex64)).cuda()
        gain = torch.ones(ch, dtype=torch.float32, device="cuda")

        def step():
            a, _ = cb.simple_agc_bank_cc(x, 0.001, 0.5, 65535.0, gain)
            o, _, _, st = cb.timing_recovery_bank_cc(a, 0, sps, True)
            counts = st[:, 2].contiguous()
            b, _ = cb.dbpsk_decoder_bank_c_u8(o, counts)
            cb.psk31_varicode_decoder_bank_u8_u8(b, counts)

        for _ in range(3):
            step()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            step()
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / reps
        print(f"bpsk31 chain: {ch} channels x 1 s at {rate} Hz, sps {sps}: {ms:.3f} ms GPU per second of signal  [{card()}]", flush=True)


if __name__ == "__main__":
    main()
