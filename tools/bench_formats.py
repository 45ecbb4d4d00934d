"""Times the sample-format conversion kernels on the GPU: convert_s8_f, convert_f_s8, convert_f_u8, convert_s24_f and convert_f_s24 on 2^28
values each, CUDA events after a warm-up, each timed over at least 0.5 s.  Reports the algorithmic bytes moved per second (read + write) and
their share of the H100's 3.35 TB/s HBM3 bandwidth.  Prints one JSON line with the card's name and power limit, read in the same run."""
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import csdr_b200 as cb  # noqa: E402

N, HBM, MIN_SECONDS = 1 << 28, 3.35e12, 0.5


def timed(fn):
    """seconds per call: two warm-up calls, then enough calls for at least MIN_SECONDS"""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 4
    while True:
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        t = a.elapsed_time(b) / 1e3
        if t >= MIN_SECONDS:
            return t / reps
        reps *= 2


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": q.splitlines()[0] if q else torch.cuda.get_device_name(), "values": N, "kernels": {}}
    f = torch.rand(N, device="cuda") * 2.2 - 1.1
    s8 = torch.randint(-128, 128, (N,), dtype=torch.int8, device="cuda")
    b8 = torch.empty(N, dtype=torch.uint8, device="cuda")
    b24 = torch.randint(0, 256, (3 * N,), dtype=torch.uint8, device="cuda")
    out = torch.empty(N, device="cuda")

    def record(name, fn, bytes_per_value):
        t = timed(fn)
        res["kernels"][name] = {"ms": round(t * 1e3, 3), "GBps": round(N * bytes_per_value / t / 1e9, 1),
                                "share_of_hbm": round(N * bytes_per_value / t / HBM, 3)}

    record("convert_s8_f", lambda: cb.convert_s8_f(s8, out=out), 5)
    record("convert_f_s8", lambda: cb.convert_f_s8(f, out=s8), 5)
    record("convert_f_u8", lambda: cb.convert_f_u8(f, out=b8), 5)
    record("convert_s24_f", lambda: cb.convert_s24_f(b24, out=out), 7)
    record("convert_f_s24", lambda: cb.convert_f_s24(f, out=b24), 7)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
