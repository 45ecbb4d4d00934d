"""Time the AM / SSB audio-rate blocks on cuda:0 and print one JSON line: milliseconds of GPU time per second of 48 kHz audio for the AM
front (amdemod_cf | fastdcblock_ff 1024 from cf32 rows) and the AGC tail (realpart_cf | agc_ff | limit_ff | convert_f_s16 with the CLI
defaults), at 128 and 1024 channels, plus the card's name and power limit read in the same run.  CUDA events, after warm-up."""
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def power_limit_w():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def time_ms(fn, reps=20, warm=3):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record(); b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    import torch
    import csdr_b200
    torch.cuda.set_device(0)
    rate = 48_000
    res = {"metric": "gpu_ms_per_second_of_audio", "audio_rate": rate, "device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}
    g = torch.Generator(device="cuda").manual_seed(0)
    n = (rate // 1024 + 1) * 1024                                         # whole 1024-sample blocks covering one second
    for ch in (128, 1024):
        x = torch.randn((ch, n), dtype=torch.complex64, device="cuda", generator=g)
        last = torch.zeros(ch, dtype=torch.float32, device="cuda")
        front = time_ms(lambda: csdr_b200.fastdcblock_bank_ff(x, 1024, last))
        state = csdr_b200.agc_state(ch)
        p = csdr_b200.AgcParams()
        tail = time_ms(lambda: csdr_b200.agc_bank_ff(x, p, state, 1.0, True))
        res[f"am_front_{ch}ch_ms"] = round(front * rate / n, 4)
        res[f"agc_tail_{ch}ch_ms"] = round(tail * rate / n, 4)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
