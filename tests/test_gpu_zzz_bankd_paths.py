"""GPU tests (-m gpu) of csdr-bankd's two loops: the single-GPU loop, where the bank writes into the tail's rows, and the --devices loop, where the
bank's rows come back to the host and go to the same tail on the first device.  Every tail must give its sinks the same bytes on both paths.
The bodies also run on the emulated library with two pretend devices (tests/test_bankd_paths_emulated.py)."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))
import test_gpu_zzz_bankd as base  # noqa: E402  (stream generator, runner, device lists)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
bankd = base.bankd
BLOCK, N, CHANNELS = 16384, 4 * 16384 + 1000, 2
D10 = ["--decimation", "10", "--bw", "0.05"]                                 # about 1600 outputs per block: every tail fills its first call
RESAMPLE = ["--decimation", "32", "--bw", "0.01", "--resample", "3:4"]          # the geometry of tests/test_gpu_zzz_bankd_resample.py
TAILS = {"nfm": D10, "none": D10, "iq": D10, "am": D10, "usb": D10, "lsb": D10, "bpsk31": D10 + ["--sps", "16"],
         "rtty": D10 + ["--sps", "12", "--rtty-bufsize", "1024"], "wfm": D10, "nfm-resample": RESAMPLE, "none-resample": RESAMPLE}


def both_paths(bankd, tmp_path, args, data):
    """the sinks of one run on one device and of one run with --devices, as bytes"""
    out = []
    for tag, extra in (("single", []), ("devices", ["--devices", base.MULTI_DEVICES()[-1]])):
        sinks = [tmp_path / f"{tag}{k}.out" for k in range(CHANNELS)]
        base.run(bankd, ["--block", str(BLOCK)] + args + extra, data, sinks)
        out.append([p.read_bytes() for p in sinks])
    return out


@pytest.mark.parametrize("tail", sorted(TAILS))
def test_every_tail_gets_the_same_bytes_on_both_paths(bankd, tmp_path, tail):
    noise = np.random.default_rng(31).integers(0, 256, 2 * N, dtype=np.uint8)      # u8 IQ noise: the text tails decode characters from it too
    single, devices = both_paths(bankd, tmp_path, ["--tail", tail.split("-")[0]] + TAILS[tail], noise.tobytes())
    for k in range(CHANNELS):
        assert len(single[k]) > 0 and single[k] == devices[k], (tail, k, len(single[k]), len(devices[k]))


@pytest.mark.parametrize("tail", ["none", "iq", "usb"])
def test_real_f32_gets_the_same_bytes_on_both_paths(bankd, tmp_path, tail):
    u8 = base.wideband_u8(N, seed=32)
    x = ((u8[0::2].astype(np.float32) - 127.5) / 127.5).astype(np.float32)          # the I samples as a real stream
    single, devices = both_paths(bankd, tmp_path, D10 + ["--real-f32", "--tail", tail], x.tobytes())
    for k in range(CHANNELS):
        assert len(single[k]) > 0 and single[k] == devices[k], (tail, k, len(single[k]), len(devices[k]))
