"""GPU tests (-m gpu) of csdr-bankd --waterfall SINK (csdr_b200/host/bankd.c): the waterfall sink must hold, byte for byte, the first L lines of
the product CLI pipe `csdr [convert_u8_f |] fft_cc N E W | logaveragepower_cf X N A | fft_exchange_sides_ff N [| compress_fft_adpcm_f_u8 N]` on the
samples the daemon processed (L = the whole lines they complete; the CLI's stale lines at end of input are not compared), for u8 and f32 input,
two block sizes, E < N and E > N and both compressions; the channel sinks do not change; --devices gives the same bytes; a FIFO nobody reads for
a while holds only whole lines; the option combinations the daemon refuses exit with a message; --fft-compression none is within 5e-3 dB of the
compiled reference CLI chain.  tests/test_bankd_waterfall_emulated.py runs the same bodies on the emulated library."""
import os
import subprocess
import threading
import time
from pathlib import Path

import numpy as np
import pytest

from test_gpu_zzz_bankd import bankd  # noqa: F401  (the fixture)
import test_gpu_zzz_bankd as base

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
REF_CLI = ROOT / "oracle" / "_ref" / "csdr_ref"
CLI = [ROOT / "csdr_b200" / "csdr"]                                    # the product CLI next to the daemon (the emulated tier points it elsewhere)
RATES = base.RATES


def product_cli():
    return str(CLI[0])


def cli_pipe(cli, stages, data):
    cmd = " | ".join(f"{cli} {s}" for s in stages)
    r = subprocess.run(["bash", "-c", cmd], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, (cmd, r.stderr[-2000:])
    return r.stdout


def frames_at(N, E, total):
    return total // E if E <= N else ((total - N) // E + 1 if total >= N else 0)


def wf_stages(fmt, N, E, A, W, add_db, compress):
    st = ["convert_u8_f"] if fmt == "u8" else []
    st += [f"fft_cc {N} {E} {W}", f"logaveragepower_cf {add_db} {N} {A}", f"fft_exchange_sides_ff {N}"]
    return st + ([f"compress_fft_adpcm_f_u8 {N}"] if compress else [])


def run(bankd, args, data, sinks, timeout=900):
    cmd = [bankd] + args + [f"{r}:{p}" for r, p in zip(RATES, sinks)]
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stderr.decode()


def stream(fmt, n, seed):
    u8 = base.wideband_u8(n, seed)
    if fmt == "u8":
        return u8.tobytes()
    return ((u8.astype(np.float32) - 127.5) / 127.5).astype(np.float32).tobytes()


@pytest.mark.parametrize("fmt", ["u8", "f32"])
@pytest.mark.parametrize("block", [16384, 40000])
@pytest.mark.parametrize("N,E,A,compress", [(1024, 300, 3, True), (256, 700, 2, False), (2048, 2048, 2, False), (512, 100, 5, True)])
def test_waterfall_equals_the_cli_pipe(bankd, oracle, tmp_path, fmt, block, N, E, A, compress):
    n = 5 * block + 777
    data = stream(fmt, n, 5)
    used = base.stream_used(oracle, n, block)
    wf = tmp_path / "wf.bin"
    chan_wf = [tmp_path / f"w{k}.f32" for k in range(len(RATES))]
    chan_plain = [tmp_path / f"p{k}.f32" for k in range(len(RATES))]
    fmt_args = [f"--{fmt}", "--tail", "none", "--block", str(block)]
    wf_args = ["--waterfall", str(wf), "--fft-size", str(N), "--fft-every", str(E), "--fft-averages", str(A), "--fft-add-db", "-60",
               "--fft-window", "HAMMING", "--fft-compression", "adpcm" if compress else "none"]
    run(bankd, fmt_args + wf_args, data, chan_wf)
    run(bankd, fmt_args, data, chan_plain)
    for a, b in zip(chan_wf, chan_plain):                               # the channels do not notice the waterfall
        assert a.read_bytes() == b.read_bytes() and a.stat().st_size > 0
    lb = (N + 10) // 2 if compress else 4 * N
    L = frames_at(N, E, used) // A
    sample_bytes = 2 if fmt == "u8" else 8
    want = cli_pipe(product_cli(), wf_stages(fmt, N, E, A, "HAMMING", -60, compress), data[:used * sample_bytes])
    got = wf.read_bytes()
    assert L >= 3 and len(got) == L * lb and len(want) >= L * lb, (L, len(got), len(want))
    assert got == want[:L * lb]


def test_waterfall_over_several_devices(bankd, tmp_path):
    data = stream("u8", 6 * 16384 + 5, 8)
    args = ["--u8", "--block", "16384", "--tail", "none", "--fft-size", "512", "--fft-every", "200", "--fft-averages", "3"]
    one = tmp_path / "one.bin"
    run(bankd, args + ["--waterfall", str(one)], data, [tmp_path / f"o{k}.f32" for k in range(len(RATES))])
    assert one.stat().st_size > 0
    for devices in base.MULTI_DEVICES():
        many = tmp_path / f"m{devices.replace(',', '_')}.bin"
        run(bankd, args + ["--waterfall", str(many), "--devices", devices], data, [tmp_path / f"m{k}.f32" for k in range(len(RATES))])
        assert many.read_bytes() == one.read_bytes(), devices


def test_slow_fifo_gets_whole_lines_only(bankd, tmp_path):
    """nobody reads the FIFO for a while, then everything is drained: only whole lines arrive, in order, each equal to a line of the
    unhindered run, and the first ones (written before the pipe filled) are the first lines of that run"""
    N = 256
    lb = 4 * N
    data = stream("u8", 24 * 16384, 9)
    args = ["--u8", "--block", "16384", "--tail", "none", "--fft-size", str(N), "--fft-compression", "none"]
    ref = tmp_path / "ref.bin"
    run(bankd, args + ["--waterfall", str(ref)], data, [tmp_path / f"r{k}.f32" for k in range(len(RATES))])
    ref_lines = np.frombuffer(ref.read_bytes(), np.uint8).reshape(-1, lb)
    assert ref_lines.shape[0] * lb > 4 * 65536                          # far more than a pipe holds
    fifo = tmp_path / "wf.fifo"
    os.mkfifo(fifo)
    got = bytearray()

    def reader():
        fd = os.open(fifo, os.O_RDONLY)
        time.sleep(3.0)                                                 # the pipe fills, lines are dropped
        while True:
            b = os.read(fd, 1 << 16)
            if not b:
                break
            got.extend(b)
        os.close(fd)

    t = threading.Thread(target=reader, daemon=True)
    t.start()
    err = run(bankd, args + ["--waterfall", str(fifo)], data, [tmp_path / f"f{k}.f32" for k in range(len(RATES))])
    t.join(60)
    assert len(got) % lb == 0 and len(got) > 0
    lines = np.frombuffer(bytes(got), np.uint8).reshape(-1, lb)
    index = {ref_lines[i].tobytes(): i for i in range(ref_lines.shape[0])}
    pos = [index.get(l.tobytes(), -1) for l in lines]
    assert min(pos) >= 0 and all(b > a for a, b in zip(pos, pos[1:]))
    assert pos[:8] == list(range(8))
    if len(pos) < ref_lines.shape[0]:
        assert "lost" in err


def test_waterfall_refusals(bankd, tmp_path):
    for args in (["--fft-size", "1024"], ["--fft-every", "10"], ["--fft-averages", "2"], ["--fft-compression", "none"], ["--fft-add-db", "3"],
                 ["--fft-window", "BLACKMAN"], ["--waterfall", str(tmp_path / "w"), "--fft-size", "1000"],
                 ["--waterfall", str(tmp_path / "w"), "--fft-size", "32768"], ["--waterfall", str(tmp_path / "w"), "--fft-every", "0"],
                 ["--waterfall", str(tmp_path / "w"), "--fft-averages", "0"], ["--waterfall", str(tmp_path / "w"), "--fft-compression", "zip"]):
        r = subprocess.run([bankd] + args + [f"0.1:{tmp_path / 'x.f32'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and b"csdr-bankd:" in r.stderr, args


def test_waterfall_against_the_reference_cli(bankd, oracle, tmp_path):
    """the daemon's float dB lines against the compiled reference chain (FFTW replaced by the float64 shim): E >= N, so no frame of the
    reference is built from its uninitialised buffer"""
    if not REF_CLI.exists():
        pytest.skip("oracle/_ref/csdr_ref not built")
    N, E, A, block = 2048, 2500, 4, 65536
    n = 6 * block
    data = stream("u8", n, 13)
    used = base.stream_used(oracle, n, block)
    wf = tmp_path / "wf.f32"
    run(bankd, ["--u8", "--tail", "none", "--block", str(block), "--waterfall", str(wf), "--fft-size", str(N), "--fft-every", str(E),
                "--fft-averages", str(A), "--fft-compression", "none"], data, [tmp_path / f"c{k}.f32" for k in range(len(RATES))])
    got = np.fromfile(wf, np.float32)
    want = np.frombuffer(cli_pipe(str(REF_CLI), wf_stages("u8", N, E, A, "HAMMING", -70, False), data[:2 * used]), np.float32)
    L = frames_at(N, E, used) // A
    assert got.size == L * N and L >= 10 and want.size >= got.size
    assert np.abs(got - want[:got.size]).max() < 5e-3                   # dB; FFT rounding differences on weak bins, as for the CLI commands
