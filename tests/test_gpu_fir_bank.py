"""GPU tier of the FIR bank contract (-m gpu): the case matrix and checks of tests/fir_ref.py through the C ABI on the device.

Every output is within the per-output error bound of the float64 reference, the bit-exact invariants hold (tiling, tile boundaries, channel sets,
row padding, output stride, I/Q symmetry, u8 front end), a non-finite sample reaches exactly the outputs whose window holds it, and the host
pipeline and the libcsdr drop-in give the device call's bits.  The matrix runs once under torch.profiler, whose kernel names carry the template
arguments <D, M, R, NPAIR, MINB, U8>: it must launch every compiled FIR kernel and nothing else of this file.
"""
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import fir_ref as F  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

CASES = F.cases(max_work=3_000_000, tiles=3)
TILING_T = [1, 9, 79, 80, 81, 150, 199, 200]
U8_CASES = [(10, 79, 16_384 + 5), (10, 80, 30_001), (10, 199, 40_007), (10, 200, 8_321), (10, 81, 205), (50, 801, 30_011), (50, 900, 61_003), (50, 1, 7)]
KERNEL_NAME = re.compile(r"(fir_bank_fast_kernel<[^>]*>|fir_bank_generic_kernel|u8_rows_to_cf32_kernel)")


class GpuDriver:
    def __init__(self, pkg):
        self.pkg, self.L = pkg, pkg.lib()

    @property
    def stream(self):
        return self.pkg._stream()

    def dev(self, a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def ptr(self, t):
        return t.data_ptr()

    def host(self, t):
        torch.cuda.synchronize()
        return t.cpu().numpy()


@pytest.fixture(scope="module")
def gpu():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    import csdr_b200
    csdr_b200.lib()
    return csdr_b200


def _run(results, key, fn, *a, **kw):
    try:
        results[key] = ("ok", fn(*a, **kw))
    except AssertionError as e:
        results[key] = ("fail", str(e))


@pytest.fixture(scope="module")
def matrix(gpu):
    """every check of the matrix, run once under torch.profiler -> ({key: (status, value or message)}, kernel names launched)"""
    from torch.profiler import ProfilerActivity, profile
    drv = GpuDriver(gpu)
    res = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case in CASES:
            _run(res, "case " + F.case_id(case), F.check_case, drv, case)
        for D, T in ((10, 79), (10, 199), (50, 801)):
            c = dict(D=D, T=T, variant=-1, layout="pad", kind="firdes", n=T + 3 * 832 * D + 7, channels=64, seed=D + T)
            _run(res, f"firdes D{D} T{T}", F.check_case, drv, c, taps=gpu.firdes_lowpass_f(T, 0.5 / D))
        for T in TILING_T:
            _run(res, f"tilings T{T}", F.check_tilings, drv, 10, T, T + 2000 * 10 + 3, seed=T)
        for D, T, v in F.NONFINITE:
            _run(res, f"nonfinite D{D} T{T} v{v}", F.check_nonfinite, drv, D, T, v, F.nonfinite_n(D, T, v), seed=T + v)
        for D, T, n in U8_CASES:
            _run(res, f"u8 D{D} T{T} n{n}", F.check_u8, drv, D, T, n, seed=n)
        torch.cuda.synchronize()
    names = set()
    for e in prof.key_averages():
        m = KERNEL_NAME.search(e.key)
        if m:
            names.add(m.group(1))
    return res, names


def _outcome(matrix, key):
    status, val = matrix[0][key]
    if status != "ok":
        pytest.fail(val)
    return val


@pytest.mark.parametrize("case", CASES, ids=F.case_id)
def test_gpu_fir_bank_contract(matrix, case):
    """bound at every output; tight rows / output stride, channel subset, shifted start, I/Q swap, sign and scale give the same bits"""
    worst = _outcome(matrix, "case " + F.case_id(case))
    print(f"{F.case_id(case)} [{F.kernel_name(F.kernel_for(case['D'], case['T'], case['variant'], case['layout'] == 'pad'))}]: worst err/bound {worst:.3f}")


@pytest.mark.parametrize("D,T", [(10, 79), (10, 199), (50, 801)])
def test_gpu_fir_bank_firdes_taps(matrix, D, T):
    """the product's lowpass taps (symmetric) at the headline shapes"""
    print(f"firdes D={D} T={T}: worst err/bound {_outcome(matrix, f'firdes D{D} T{T}'):.3f}")


@pytest.mark.parametrize("T", TILING_T)
def test_gpu_fir_bank_tilings_agree(matrix, T):
    _outcome(matrix, f"tilings T{T}")


@pytest.mark.parametrize("D,T,variant", F.NONFINITE)
def test_gpu_fir_bank_nonfinite_stays_in_its_windows(matrix, D, T, variant):
    _outcome(matrix, f"nonfinite D{D} T{T} v{variant}")


@pytest.mark.parametrize("D,T,n", U8_CASES)
def test_gpu_fir_bank_u8_equals_convert_then_filter(matrix, D, T, n):
    _outcome(matrix, f"u8 D{D} T{T} n{n}")


def test_gpu_fir_bank_coverage(matrix):
    """the matrix launched the 13 fast instantiations, the generic kernel and the u8 conversion of the two-launch path, and each case's kernel
    is the one fir_ref.kernel_for names"""
    want = {F.kernel_name(k) for k in F.KERNELS} | {F.GENERIC, F.U8_ROWS}
    assert matrix[1] == want, (sorted(matrix[1] - want), sorted(want - matrix[1]))
    assert {F.kernel_for(c["D"], c["T"], c["variant"], c["layout"] == "pad") for c in CASES} == set(F.CF32_KERNELS) | {F.GENERIC}


@pytest.mark.parametrize("u8", [False, True])
def test_gpu_fir_bank_host_calls(gpu, u8):
    """fir_decimate_bank_cc_host / _u8_host over padded host rows, chunk_channels 0, 1, 2 and C: the device call's bits, host padding untouched"""
    drv = GpuDriver(gpu)
    D, T, ch, n = 10, 199, 5, 30_011
    h = np.random.default_rng(3).uniform(-1, 1, T).astype(np.float32)
    if u8:
        u = F.u8_inputs(ch, n, 4)
        want = F.bank(drv, F.convert_u8(u), D, h)
        src = np.full((ch, n + 24, 2), 0x5A, np.uint8); src[:, :n] = u
        xin = src[:, :n]
    else:
        x, _ = F.make_inputs(dict(seed=4, channels=ch, n=n, T=T))
        want = F.bank(drv, x, D, h)
        src = np.full((ch, n + 5), np.nan, np.complex64); src[:, :n] = x
        xin = src[:, :n]
    n_out = want.shape[1]
    for cc in (0, 1, 2, ch):
        ob = np.full((ch, 2 * (n_out + 3)), F.SENTINEL, np.uint32).view(np.complex64)
        (gpu.fir_decimate_bank_u8_host if u8 else gpu.fir_decimate_bank_cc_host)(xin, D, h, out=ob[:, :n_out], chunk_channels=cc)
        F.assert_bits_equal(ob[:, :n_out], want, f"host call, chunk_channels={cc}")
        assert np.all(ob.view(np.uint32)[:, 2 * n_out:] == F.SENTINEL), "the host call wrote into the output padding"


@pytest.mark.parametrize("D,T,n", [(10, 199, 9_999), (10, 79, 20_001), (50, 801, 70_000), (7, 79, 5_001), (10, 81, 81)])
def test_gpu_fir_decimate_cc_dropin_equals_one_channel_bank(gpu, D, T, n):
    drv = GpuDriver(gpu)
    x, h = F.make_inputs(dict(seed=n, channels=1, n=n, T=T))
    F.assert_bits_equal(gpu.libcsdr.fir_decimate_cc(x[0], D, h), F.bank(drv, x, D, h)[0], "libcsdr.fir_decimate_cc against the bank")


def _fir64_and_bound_on_device(x, taps, D):
    """fir64 and fir_ref.bound of rows x [r, n] (complex64, numpy) with torch in float64 on the device, one row at a time -> two complex arrays"""
    T = taps.size
    h = torch.from_numpy(taps.astype(np.float64)).cuda()
    k = (T + 2) * F.U * (1 + 1e-3)
    want, bnd = [], []
    for row in x:
        t = torch.from_numpy(np.ascontiguousarray(row)).cuda()
        w = [p.to(torch.float64).unfold(0, T, D) @ h for p in (t.real, t.imag)]
        b = [k * (p.to(torch.float64).abs().unfold(0, T, D) @ h.abs()) for p in (t.real, t.imag)]
        want.append(torch.complex(w[0], w[1]).cpu().numpy())
        bnd.append(torch.complex(b[0], b[1]).cpu().numpy())
    return np.stack(want), np.stack(bnd)


def test_gpu_fir_bank_headline_size(gpu):
    """256 channels x 2^20 + 7 samples, the default tiling: the bound at every output of 8 seeded rows, reference and bound in float64 on the device"""
    D, T, ch, n = 10, 199, 256, (1 << 20) + 7
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.complex(torch.rand(ch, n, device="cuda", generator=g) * 2 - 1, torch.rand(ch, n, device="cuda", generator=g) * 2 - 1)
    h = np.random.default_rng(2).uniform(-1, 1, T).astype(np.float32)
    y = gpu.fir_decimate_bank_cc(x, D, h)
    rows = np.random.default_rng(3).choice(ch, 8, replace=False)
    xs, ys = x[rows].cpu().numpy(), y[rows].cpu().numpy()
    want, bnd = _fir64_and_bound_on_device(xs, h, D)
    assert want.shape == ys.shape
    for part in (np.real, np.imag):
        err = np.abs(part(ys.astype(np.complex128)) - part(want))
        i = np.unravel_index(np.argmax(err / part(bnd)), err.shape)
        print(f"headline size: worst err/bound {float(err[i] / part(bnd)[i]):.3f}")
        assert np.all(err <= part(bnd)), (rows[i[0]], i[1], float(err[i]), float(part(bnd)[i]))


def test_gpu_fir_bank_65535_channels(gpu):
    """the grid's channel limit with a short row: the last channel within the bound and equal to its one-channel call"""
    drv = GpuDriver(gpu)
    D, T, ch = 10, 79, 65535
    n = T + 12 * D + 1
    rng = np.random.default_rng(9)
    x = (rng.uniform(-1, 1, (ch, n)) + 1j * rng.uniform(-1, 1, (ch, n))).astype(np.complex64)
    h = rng.uniform(-1, 1, T).astype(np.float32)
    y = F.bank(drv, x, D, h)
    F.assert_within_bound(y[-1:], x[-1:], h, D, "last of 65535 channels")
    F.assert_bits_equal(F.bank(drv, x[-1:], D, h), y[-1:], "last channel against its own call")
