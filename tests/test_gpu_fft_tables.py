"""GPU tests (-m gpu): every FFT path that reads a cached twiddle table gives the same bytes on a second device of the same process.  The tables
are cached per device, so sizes first run on cuda:0 and then on cuda:1 read cuda:1's own copies.  Needs two devices; skipped on one."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def csdr():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    from csdr_b200.build import build
    build()
    import csdr_b200
    return csdr_b200


def run_on(csdr, device, body):
    """body(torch device) on `device`, as host tensors; the library's current device goes back to 0 afterwards"""
    with torch.cuda.device(device):
        assert csdr.lib().csdrb_set_device(device) == 0
        try:
            outs = body(torch.device("cuda", device))
            torch.cuda.synchronize(device)
            return [o.cpu().contiguous() for o in outs]
        finally:
            csdr.lib().csdrb_set_device(0)


def test_fft_paths_give_the_same_bytes_on_a_second_device(csdr):
    rng = np.random.default_rng(11)
    cplx = lambda *s: (rng.standard_normal(s) + 1j * rng.standard_normal(s)).astype(np.complex64) * np.float32(0.3)
    xc = [cplx(4, n) for n in (16, 64, 4096, 16384)]                   # radix-8 and radix-16 row transforms
    xr = [rng.standard_normal((3, n)).astype(np.float32) for n in (32, 128, 8192)]
    ddc = csdr.fastddc_init(0.005, 20, 0.1)
    wide = cplx(3 * ddc.input_size)
    sc, sr = cplx(2, 9000), rng.standard_normal((2, 20000)).astype(np.float32)

    def body(dev):
        outs = []
        for x in xc:
            t = torch.from_numpy(x).to(dev)
            outs += [csdr.fft_c2c(t), csdr.fft_c2c(t, inverse=True)]
        outs += [csdr.fft_r2c(torch.from_numpy(x).to(dev)) for x in xr]
        outs += list(csdr.fastddc_fwd_cc(torch.from_numpy(wide).to(dev), ddc))
        for real, x in ((False, sc), (True, sr)):
            for N in (16, 1024):
                outs.append(csdr.SpectrumBank(2, N, N // 2, 2, -70.0, device=dev, real=real).process(torch.from_numpy(x).to(dev)))
        return outs

    a, b = run_on(csdr, 0, body), run_on(csdr, 1, body)
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert u.numel() > 0 and u.numpy().tobytes() == v.numpy().tobytes(), f"output {i} differs between cuda:0 and cuda:1"
