"""GPU tests (-m gpu) of the real-stream waterfall: `csdr fft_fc` against the compiled reference CLI, and csdr-bankd --real-s16 | --real-f32
--waterfall SINK --fft-real (csdr_b200/host/bankd.c), whose sink must hold, byte for byte, the whole lines of the product CLI pipe
`csdr [convert_s16_f |] fft_fc N E W | logaveragepower_cf X N A [| compress_fft_adpcm_f_u8 N]` on the samples the daemon processed, for E < 2N and
E > 2N, both compressions and two block sizes; the channel sinks do not change; --devices gives the same bytes; every refusal exits with a
message.  On the H100 also: the daemon's dB lines within 5e-3 dB of the reference chain, and the FT8-at-64.8-Msps command of the README end to end.
tests/test_bankd_spectrum_real_emulated.py runs the same bodies (except the ones that need the real library) on the emulated library."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent / "spectrum"))
import spectrum_real as SR  # noqa: E402
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_real as real  # noqa: E402
from test_gpu_zzz_bankd import bankd  # noqa: E402,F401  (the fixture)

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
REF_CLI = ROOT / "oracle" / "_ref" / "csdr_ref"
CLI = [ROOT / "csdr_b200" / "csdr"]                                    # the product CLI next to the daemon (the emulated tier points it elsewhere)
RATES = real.RATES
U = 2.0 ** -24


def cli_pipe(cli, stages, data):
    cmd = " | ".join(f"{cli} {s}" for s in stages)
    r = subprocess.run(["bash", "-c", cmd], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, (cmd, r.stderr[-2000:])
    return r.stdout


def noise_stream(n, seed):
    """a real float32 stream with tones and noise (no near-empty bins)"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = 0.3 * np.cos(2 * np.pi * 0.1234 * t) + 0.05 * np.cos(2 * np.pi * 0.377 * t) + 0.02 * rng.standard_normal(n)
    return x.astype(np.float32)


# ---- csdr fft_fc against the reference CLI --------------------------------------------------------------------------------------------------
FFT_FC_CASES = [(256, 100, "HAMMING"), (256, 512, "BLACKMAN"), (64, 300, "BOXCAR"), (1024, 2048, "HAMMING"), (16, 70, "BLACKMAN")]


def check_fft_fc_against_the_reference(cli, ref, N, E, W):
    """same frame count; every frame that lies wholly inside the stream within the r2c bound of the float64 reference transform"""
    T = SR.stream_for(N, E, 9 + 2 * N // E) + 17
    x = noise_stream(T, N + E)
    ours = np.frombuffer(cli_pipe(cli, [f"fft_fc {N} {E} {W}"], x.tobytes()), np.complex64).reshape(-1, N)
    theirs = np.frombuffer(cli_pipe(ref, [f"fft_fc {N} {E} {W}"], x.tobytes()), np.complex64).reshape(-1, N)
    assert ours.shape == theirs.shape and ours.shape[0] >= SR.frames_at(N, E, T)
    inside = [k for k in range(SR.frames_at(N, E, T)) if SR.frame_start(N, E, k) >= 0]
    assert len(inside) >= 5
    for k in inside:
        s = SR.frame_start(N, E, k)
        bound = (10 * np.log2(2 * N) + 14) * U * np.abs(x[s:s + 2 * N].astype(np.float64)).sum()      # window <= 1; + the reference's rounding
        assert np.abs(ours[k].astype(np.complex128) - theirs[k]).max() <= bound, (k, np.abs(ours[k] - theirs[k]).max(), bound)


def check_fft_fc_pipe_against_the_reference(cli, ref):
    """fft_fc | logaveragepower_cf, E = 2N and E > 2N (no frame reaches before the stream): within 5e-3 dB"""
    for N, E, A in ((512, 1024, 3), (256, 900, 2)):
        x = noise_stream(SR.stream_for(N, E, 10 * A), 7 * N)
        st = [f"fft_fc {N} {E} HAMMING", f"logaveragepower_cf -70 {N} {A}"]
        ours = np.frombuffer(cli_pipe(cli, st, x.tobytes()), np.float32)
        theirs = np.frombuffer(cli_pipe(ref, st, x.tobytes()), np.float32)
        whole = SR.frames_at(N, E, x.size) // A * N
        assert ours.size == theirs.size and whole >= 10 * N
        assert np.abs(ours[:whole] - theirs[:whole]).max() < 5e-3


def check_fft_fc_refusals(cli):
    for args in ("fft_fc 1 2", "fft_fc 2097152 4194304", "fft_fc 100 200", "fft_fc 64"):
        r = subprocess.run(["bash", "-c", f"{cli} {args}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and r.stderr, args


@pytest.fixture(scope="module")
def ref_cli():
    if not REF_CLI.exists():
        pytest.skip("oracle/_ref/csdr_ref not built")
    return str(REF_CLI)


@pytest.mark.parametrize("N,E,W", FFT_FC_CASES)
def test_fft_fc_against_the_reference(bankd, ref_cli, N, E, W):
    check_fft_fc_against_the_reference(str(CLI[0]), ref_cli, N, E, W)


def test_fft_fc_pipe_against_the_reference(bankd, ref_cli):
    check_fft_fc_pipe_against_the_reference(str(CLI[0]), ref_cli)


def test_fft_fc_refusals(bankd):
    check_fft_fc_refusals(str(CLI[0]))


# ---- csdr-bankd --fft-real ----------------------------------------------------------------------------------------------------------------------
def wf_stages(fmt, N, E, A, W, add_db, compress):
    st = ["convert_s16_f"] if fmt == "real-s16" else []
    st += [f"fft_fc {N} {E} {W}", f"logaveragepower_cf {add_db} {N} {A}"]
    return st + ([f"compress_fft_adpcm_f_u8 {N}"] if compress else [])


def stream(fmt, n, seed):
    s16 = real.real_stream(n, seed)
    return s16.tobytes() if fmt == "real-s16" else (s16.astype(np.float32) / 32768.0).astype(np.float32).tobytes()


def run(bankd, args, data, sinks, timeout=900):
    r = real.run(bankd, args, data, sinks, timeout=timeout)
    return r.stderr.decode()


@pytest.mark.parametrize("fmt", ["real-s16", "real-f32"])
@pytest.mark.parametrize("block", [16384, 40000])
@pytest.mark.parametrize("N,E,A,compress", [(1024, 700, 3, True), (256, 700, 2, False)])
def test_real_waterfall_equals_the_cli_pipe(bankd, oracle, tmp_path, fmt, block, N, E, A, compress):
    n = 5 * block + 777
    data = stream(fmt, n, 5)
    used = real.used(oracle, n, block)
    wf = tmp_path / "wf.bin"
    chan_wf = [tmp_path / f"w{k}.f32" for k in range(len(RATES))]
    chan_plain = [tmp_path / f"p{k}.f32" for k in range(len(RATES))]
    fmt_args = [f"--{fmt}", "--tail", "none", "--block", str(block)]
    wf_args = ["--waterfall", str(wf), "--fft-real", "--fft-size", str(N), "--fft-every", str(E), "--fft-averages", str(A), "--fft-add-db", "-60",
               "--fft-window", "HAMMING", "--fft-compression", "adpcm" if compress else "none"]
    run(bankd, fmt_args + wf_args, data, chan_wf)
    run(bankd, fmt_args, data, chan_plain)
    for a, b in zip(chan_wf, chan_plain):                               # the channels do not notice the waterfall
        assert a.read_bytes() == b.read_bytes() and a.stat().st_size > 0
    lb = (N + 10) // 2 if compress else 4 * N
    L = SR.frames_at(N, E, used) // A
    sample_bytes = 2 if fmt == "real-s16" else 4
    want = cli_pipe(str(CLI[0]), wf_stages(fmt, N, E, A, "HAMMING", -60, compress), data[:used * sample_bytes])
    got = wf.read_bytes()
    assert L >= 3 and len(got) == L * lb and len(want) >= L * lb, (L, len(got), len(want))
    assert got == want[:L * lb]


@pytest.mark.parametrize("fmt", ["real-s16", "real-f32"])
def test_real_waterfall_over_several_devices(bankd, tmp_path, fmt):
    data = stream(fmt, 6 * 16384 + 5, 8)
    args = [f"--{fmt}", "--block", "16384", "--tail", "none", "--fft-real", "--fft-size", "256", "--fft-every", "900", "--fft-averages", "3"]
    one = tmp_path / "one.bin"
    run(bankd, args + ["--waterfall", str(one)], data, [tmp_path / f"o{k}.f32" for k in range(len(RATES))])
    assert one.stat().st_size > 0
    for devices in base.MULTI_DEVICES():
        many = tmp_path / f"m{devices.replace(',', '_')}.bin"
        run(bankd, args + ["--waterfall", str(many), "--devices", devices], data, [tmp_path / f"m{k}.f32" for k in range(len(RATES))])
        assert many.read_bytes() == one.read_bytes(), devices


def test_real_waterfall_refusals(bankd, tmp_path):
    w = str(tmp_path / "w")
    for args in (["--real-s16", "--fft-real"], ["--fft-real", "--waterfall", w], ["--f32", "--fft-real", "--waterfall", w],
                 ["--real-s16", "--waterfall", w, "--fft-real", "--fft-size", "32768"], ["--real-f32", "--waterfall", w, "--fft-real", "--fft-size", "1"],
                 ["--real-f32", "--waterfall", w, "--fft-real", "--fft-size", "1000"], ["--real-s16", "--waterfall", w, "--fft-real", "--fft-every", "0"]):
        r = subprocess.run([str(bankd)] + args + [f"0.1:{tmp_path / 'x.f32'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and b"csdr-bankd:" in r.stderr, args
    r = subprocess.run([str(bankd), "--real-s16", "--waterfall", w, f"0.1:{tmp_path / 'x.f32'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       timeout=60)
    assert r.returncode != 0 and b"--waterfall needs a complex input" in r.stderr and b"--fft-real" in r.stderr


def test_real_waterfall_against_the_reference_cli(bankd, oracle, ref_cli, tmp_path):
    """the daemon's float dB lines against the compiled reference chain (FFTW replaced by the float64 shim), E >= 2N: within 5e-3 dB"""
    N, E, A, block = 2048, 5000, 4, 65536
    n = 6 * block
    data = stream("real-s16", n, 13)
    used = real.used(oracle, n, block)
    wf = tmp_path / "wf.f32"
    run(bankd, ["--real-s16", "--tail", "none", "--block", str(block), "--waterfall", str(wf), "--fft-real", "--fft-size", str(N), "--fft-every", str(E),
                "--fft-averages", str(A), "--fft-compression", "none"], data, [tmp_path / f"c{k}.f32" for k in range(len(RATES))])
    got = np.fromfile(wf, np.float32)
    want = np.frombuffer(cli_pipe(ref_cli, wf_stages("real-s16", N, E, A, "HAMMING", -70, False), data[:2 * used]), np.float32)
    L = SR.frames_at(N, E, used) // A
    assert got.size == L * N and L >= 10 and want.size >= got.size
    assert np.abs(got - want[:got.size]).max() < 5e-3


def test_ft8_at_64_8_msps_end_to_end(bankd, oracle, tmp_path):
    """the README's RX888 command with the waterfall beside the channel: the sink equals convert_s16_f | fft_fc 16384 32768 |
    logaveragepower_cf -70 16384 1 | compress_fft_adpcm_f_u8 16384 on the samples the daemon processed"""
    block, D = 1 << 18, 1350
    n = 5 * block
    rng = np.random.default_rng(21)
    t = np.arange(n)
    x = 0.2 * np.cos(2 * np.pi * 0.10916667 * t + 0.3) + 0.01 * rng.standard_normal(n)
    data = np.clip(np.round(x * 32767), -32768, 32767).astype(np.int16).tobytes()
    wf, ch = tmp_path / "wf.bin", tmp_path / "ft8.s16"
    cmd = [str(bankd), "--real-s16", "--decimation", str(D), "--bw", "0.0008", "--tail", "usb", "--waterfall", str(wf), "--fft-real", "--fft-size", "16384",
           f"-0.10916667:{ch}"]
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    T = oracle.firdes_filter_len(0.0008)
    consumed = ((block - T) // D + 1) * D
    used = block + ((n - block) // consumed) * consumed
    L = SR.frames_at(16384, 32768, used)
    lb = (16384 + 10) // 2
    want = cli_pipe(str(CLI[0]), ["convert_s16_f", "fft_fc 16384 32768", "logaveragepower_cf -70 16384 1", "compress_fft_adpcm_f_u8 16384"], data[:2 * used])
    got = wf.read_bytes()
    assert ch.stat().st_size > 0 and L >= 30 and len(got) == L * lb and got == want[:L * lb]
