"""Writes tests/golden/resampler_golden.npz: rational_resampler_ff as the compiled, unmodified reference computes it (oracle/_ref/libcsdr_ref.so),
so that the GPU tier can check the resampler without the reference sources.  Run from the repository root where oracle/_ref has been built:

    python tests/golden/make_resampler_golden.py

Per case <name>: <name>_x (input), <name>_taps (rational_resampler_get_lowpass_f of the reference), <name>_y (output), <name>_state
(input_processed, output_size, last_taps_delay) and <name>_geom (I, D, T, block; block 0 = one call on all of x, else the CLI loop's block).
"""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent / "resampler"))
import resampler as R  # noqa: E402

CASES = {                 # name: (I, D, taps, n, block)
    "r3_4": (3, 4, 79, 2048, 0),
    "r3_2": (3, 2, 79, 2048, 0),
    "r5_2": (5, 2, 201, 2048, 0),                 # transition bandwidth 0.02
    "r1_3": (1, 3, 79, 2048, 0),
    "r4_1": (4, 1, 79, 2048, 0),
    "r24_25": (24, 25, 201, 2048, 0),             # 0.02: T >= I
    "r147_160": (147, 160, 79, 2048, 0),          # default 79 taps < I: every output is 0 (reference behaviour)
    "cap1_100": (1, 100, 79, 4096, 0),            # the output cap ends the call: state (3900, 40, 0)
    "stream3_4": (3, 4, 79, 8192, 1024),          # the CLI loop with 1024-sample blocks
}


def main():
    ref = R.Ref()
    rng = np.random.default_rng(2026)
    out = {}
    for name, (I, D, T, n, block) in CASES.items():
        t = np.arange(n)
        x = (0.6 * np.sin(2 * np.pi * 0.013 * t) + 0.3 * np.sin(2 * np.pi * 0.21 * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)
        taps = ref.lowpass(T, I, D)
        if block:
            y = ref.stream(x, I, D, taps, block); st = (0, y.size, 0)
        else:
            y, st = ref.rational_resampler_ff(x, I, D, taps)
        out.update({f"{name}_x": x, f"{name}_taps": taps, f"{name}_y": y, f"{name}_state": np.array(st, np.int32),
                    f"{name}_geom": np.array([I, D, T, block], np.int32)})
        print(name, I, D, T, st, y.size)
    np.savez_compressed(HERE / "resampler_golden.npz", **out)


if __name__ == "__main__":
    main()
