"""GPU tier of the NCO shift banks (-m gpu): the checks of tests/shift_ref.py through the C ABI on the device, at full size.

On top of the CPU tier's matrix: 1024-channel banks of 2^17 samples (shift_addition at chunk 1024 is 128 chunks x 1024 channels: the
side-stream chain at the product's slice threshold, in one slice of 128 chunks; chunk 512 reaches two slices, chunk 8 three), every bank at 65535 channels (the grid.y limit), and shift_math
over 2^27 samples, where the host's and CUDA's double cos/sin are expected to round a few seeds differently: every big case prints the
ambiguous seeds it met.  The matrix runs once under torch.profiler: it must launch all ten kernel instantiations of the shift banks.
"""
import re
import sys
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import shift_ref as S  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KERNEL_NAME = re.compile(r"(shift_phase_chain_kernel|shift_bank_kernel<float2?>|addfast_phase_chain_kernel|shift_addfast_bank_kernel|"
                         r"shift_math_chain_kernel|shift_math_bank_kernel|shift_table_bank_kernel|dshift_kernel|shift_unroll_bank_kernel)")
WANT_KERNELS = {"shift_phase_chain_kernel", "shift_bank_kernel<float2>", "shift_bank_kernel<float>", "addfast_phase_chain_kernel",
                "shift_addfast_bank_kernel", "shift_math_chain_kernel", "shift_math_bank_kernel", "shift_table_bank_kernel", "dshift_kernel",
                "shift_unroll_bank_kernel"}
BIG, N17 = 1024, 1 << 17
# (kind, channels, n, chunk, table size, input layout, output layout)
BIG_CASES = [("cc", BIG, N17, 1024, None, "tight", "tight"), ("cc", BIG, N17, 512, None, "pad", "pad"), ("cc", BIG, N17, 8, None, "tight", "odd"), ("fc", BIG, N17, 1024, None, "pad", "tight"),
             ("fc", BIG, N17, 8, None, "tight", "tight"), ("addfast", BIG, N17, 1022, None, "tight", "pad"), ("math", BIG, N17, 0, None, "tight", "tight"),
             ("table", BIG, 1 << 14, 0, 65536, "tight", "tight"), ("unroll", BIG, N17, 0, 1024, "shared", "tight"),
             ("cc", 65535, 64, 16, None, "tight", "tight"), ("fc", 65535, 33, 0, None, "tight", "odd"), ("addfast", 65535, 40, 8, None, "tight", "tight"),
             ("math", 65535, 300, 0, None, "tight", "tight"), ("table", 65535, 64, 0, 1024, "tight", "tight"), ("unroll", 65535, 50, 0, 16, "tight", "tight")]
BIG_DEC = (256, 16, [4001, 1001, 3])


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


def _run(res, key, fn, *a, **kw):
    try:
        res[key] = ("ok", fn(*a, **kw))
    except AssertionError as e:
        res[key] = ("fail", f"{type(e).__name__}: {e}")


def _big_rates(ch, seed):
    """rates and phases of a big bank: the edge values of the small matrix first, then random ones"""
    rng = np.random.default_rng(seed)
    r, p = S.rates_phases(min(ch, 13))
    rates = np.concatenate([r, rng.uniform(-0.5, 0.5, ch - r.size)]).astype(np.float32)
    phases = np.concatenate([p, rng.uniform(-np.pi, np.pi, ch - p.size)]).astype(np.float32)
    return rates, phases


@pytest.fixture(scope="module")
def matrix(gpu, oracle):
    """every check once under torch.profiler -> ({key: (status, value or message)}, kernel names launched, seconds)"""
    from torch.profiler import ProfilerActivity, profile
    drv = GpuDriver(gpu)
    res = {}
    t0 = time.perf_counter()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case in S.BANK_CASES:
            kind, ch, n, chunk, tsize, lin, lout = case
            rates, ph0 = S.rates_phases(ch, shift=n % 7)
            _run(res, "bank " + S.case_id(case), S.check_bank, drv, oracle, kind, rates, ph0, n, chunk, tsize, lin, lout, seed=n + ch)
        for case in BIG_CASES:
            kind, ch, n, chunk, tsize, lin, lout = case
            rates, ph0 = _big_rates(ch, n)
            _run(res, "big " + S.case_id(case), S.check_bank, drv, oracle, kind, rates, ph0, n, chunk, tsize, lin, lout, seed=n + ch)
        for case in S.INV_CASES:
            kind, ch, n, chunk, tsize = case
            rates, ph0 = S.rates_phases(ch, shift=3)
            _run(res, "inv " + S.case_id(case), S.check_invariants, drv, oracle, kind, rates, ph0, n, chunk, tsize, seed=n)
        for case in S.NONFINITE_CASES:
            kind, n, chunk, tsize = case
            _run(res, "nonfinite " + S.case_id(case), S.check_nonfinite, drv, oracle, kind, n, chunk, tsize, seed=n)
        for dec, sizes in S.DEC_CASES:
            rates, ph0 = S.rates_phases(5, shift=dec)
            _run(res, f"dec {dec}", S.check_decimating, drv, oracle, rates, ph0, [0, 1, dec - 1, sizes[0] + 2, sizes[0] + dec], dec, sizes, seed=dec)
        ch, dec, sizes = BIG_DEC
        rates, ph0 = _big_rates(ch, 5)
        _run(res, "dec big", S.check_decimating, drv, oracle, rates, ph0, np.arange(ch) % (dec + 2), dec, sizes, seed=5)
        _run(res, "refusals", S.check_refusals, drv, oracle)
        for n, call, rate, phase in S.DROPIN_CASES:
            _run(res, f"dropins {n} {call}", S.check_dropins, drv, oracle, n, call, rate, phase, seed=n)
        torch.cuda.synchronize()
    names = set()
    for e in prof.key_averages():
        m = KERNEL_NAME.search(e.key)
        if m:
            names.add(m.group(1))
    return res, names, time.perf_counter() - t0


def _outcome(matrix, key):
    status, val = matrix[0][key]
    if status != "ok":
        pytest.fail(val)
    return val


@pytest.mark.parametrize("case", S.BANK_CASES, ids=[S.case_id(c) for c in S.BANK_CASES])
def test_gpu_shift_bank(matrix, case):
    amb, worst = _outcome(matrix, "bank " + S.case_id(case))
    print(f"{S.case_id(case)}: ambiguous seeds {amb}, worst err/bound {worst:.3f}")


@pytest.mark.parametrize("case", BIG_CASES, ids=[S.case_id(c) for c in BIG_CASES])
def test_gpu_shift_big_bank(matrix, case):
    kind, ch, n, chunk, tsize, _, _ = case
    amb, worst = _outcome(matrix, "big " + S.case_id(case))
    print(f"{S.case_id(case)} ({S.shift_path(ch, n, tsize if kind == 'unroll' else chunk, kind)}): ambiguous seeds {amb}, worst err/bound {worst:.3f}")


@pytest.mark.parametrize("case", S.INV_CASES, ids=[S.case_id(c) for c in S.INV_CASES])
def test_gpu_shift_invariants(matrix, case):
    _outcome(matrix, "inv " + S.case_id(case))


@pytest.mark.parametrize("case", S.NONFINITE_CASES, ids=[S.case_id(c) for c in S.NONFINITE_CASES])
def test_gpu_shift_nonfinite(matrix, case):
    _outcome(matrix, "nonfinite " + S.case_id(case))


@pytest.mark.parametrize("dec", [d for d, _ in S.DEC_CASES] + ["big"])
def test_gpu_decimating_shift_bank(matrix, dec):
    amb, worst = _outcome(matrix, f"dec {dec}")
    print(f"decimating {dec}: ambiguous seeds {amb}, worst err/bound {worst:.3f}")


def test_gpu_shift_refusals(matrix):
    _outcome(matrix, "refusals")


@pytest.mark.parametrize("n,call", [(n, c) for n, c, _, _ in S.DROPIN_CASES])
def test_gpu_shift_dropins(matrix, n, call):
    _outcome(matrix, f"dropins {n} {call}")


def test_gpu_shift_coverage(matrix):
    """the matrix launched every kernel instantiation of the shift banks, the big banks reached the 2- and 3-slice chains, and nothing of the
    shift banks is left out of WANT_KERNELS"""
    print(f"shift matrix: {matrix[2]:.1f} s")
    assert matrix[1] == WANT_KERNELS, (sorted(matrix[1] - WANT_KERNELS), sorted(WANT_KERNELS - matrix[1]))
    paths = {(p["side"], p["slices"]) for p in (S.shift_path(ch, n, chunk, kind) for kind, ch, n, chunk, _, _, _ in BIG_CASES + S.BANK_CASES
                                                  if kind in ("cc", "fc"))}
    assert {(False, 1), (True, 1), (True, 2), (True, 3)} <= paths, paths
