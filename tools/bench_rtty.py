"""GPU time of the RTTY decoder banks per second of signal: serial_line_decoder_f_u8 44 5 1.5 (2 kHz baseband, 45.45 Bd) and
rtty_baudot2ascii_u8_u8 for 128 and 1024 channels.  The decoder runs calls of 16384 samples, as csdr-bankd --tail rtty does: one call decodes
about 8 s of signal, so each timed step is one call of each bank over rows of 16384 + 400 samples, and the time is divided by the seconds of
signal the call consumed.  CUDA events around the two launches after warm-up; prints one line per channel count with the card name and
power limit."""
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


def discriminator_rows(rng, ch, n, spb):
    """noisy +-1 discriminator output of random ITA2 characters: start bit, 5 data bits, 1.5 stop bits, 2 samples of mark between them"""
    rows = np.empty((ch, n), np.float32)
    for c in range(ch):
        lev = [np.ones(int(rng.integers(10, 200)))]
        while sum(v.size for v in lev) < n:
            bits = np.r_[0, rng.integers(0, 2, 5)]
            lev.append(np.repeat(np.where(bits, 1.0, -1.0), spb))
            lev.append(np.ones(int(1.5 * spb) + 2))
        rows[c] = np.concatenate(lev)[:n] + 0.3 * rng.standard_normal(n)
    return rows


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    rate, spb, bufsize, reps = 2000, 44, 16384, 20
    n = bufsize + 400
    rng = np.random.default_rng(0)
    for ch in (128, 1024):
        x = torch.from_numpy(discriminator_rows(rng, ch, n, spb)).cuda()
        start0 = torch.zeros(ch, dtype=torch.int32, device="cuda")

        def step():
            codes, cnt, start, _ = cb.serial_line_decoder_bank_f_u8(x, float(spb), 5, 1.5, 0.4, bufsize=bufsize, start=start0.clone())
            cb.rtty_baudot2ascii_bank_u8_u8(codes, cnt)
            return start

        for _ in range(3):
            start = step()
        torch.cuda.synchronize()
        seconds = float(start.double().mean()) / rate                  # signal one call consumes per channel
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            step()
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / reps
        print(f"rtty decoder: {ch} channels at {rate} Hz, spb {spb}: {ms:.3f} ms per call of {bufsize} samples ({seconds:.2f} s of signal), "
              f"{ms / seconds:.3f} ms GPU per second of signal  [{card()}]", flush=True)


if __name__ == "__main__":
    main()
