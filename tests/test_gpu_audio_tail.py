"""GPU tier of the FM chain's audio-rate kernels (-m gpu): the checks of tests/audio_ref.py through the C ABI on the device, at full size.

On top of the CPU tier's matrix: 1024-channel banks of every kernel, fmdemod's 64-CTA grid looping over long rows, and fracdec's sequential
fallback (fracdec_positions_kernel + fracdec_interp_kernel, rows of 2^22 samples and more) against the oracle.  The matrix runs once under
torch.profiler: it must launch every kernel instantiation of the five banks that audio_ref's restatements of the launchers name.
"""
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import audio_ref as A  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KERNEL_NAME = re.compile(r"(fmdemod_quadri_bank_kernel|fracdec_\w+_kernel(?:<\d+>)?|fastagc_\w+_kernel(?:<(?:true|false)>)?|"
                         r"nfm_deemph_bank_kernel<(?:true|false)>|deemphasis_wfm_bank_kernel)")
WANT_KERNELS = {"fmdemod_quadri_bank_kernel", "fracdec_segments_kernel", "fracdec_interp_seg_kernel<12>", "fracdec_interp_seg_kernel<0>",
                "fracdec_positions_kernel", "fracdec_interp_kernel", "fastagc_fused_kernel<false>", "fastagc_fused_kernel<true>",
                "fastagc_peaks_kernel", "fastagc_apply_kernel<false>", "fastagc_apply_kernel<true>", "fastagc_carry_kernel",
                "nfm_deemph_bank_kernel<true>", "nfm_deemph_bank_kernel<false>", "deemphasis_wfm_bank_kernel"}
BIG = 1024
FD_BIG = dict(rate=5.0, points=12, where=[None, 5.75], n=(1 << 22) + 1001, T=0, B=None, note="the sequential fallback, 2 rows")
FD_BIG_TAPS = dict(rate=2.5, points=4, where=[None], n=(1 << 22) + 17, T=5, B=None, note="the fallback with a prefilter")


class GpuDriver:
    def __init__(self, pkg):
        self.pkg, self.L = pkg, pkg.lib()

    @property
    def stream(self):
        return self.pkg._stream()

    def dev(self, a):
        """a device copy; structured arrays (the fracdec state) travel as bytes and come back with their dtype"""
        a = np.ascontiguousarray(a)
        t = torch.from_numpy(a.view(np.uint8).reshape(-1).copy() if a.dtype.fields else a).cuda()
        t.np_view = (a.dtype, a.shape) if a.dtype.fields else None
        return t

    def ptr(self, t):
        return t.data_ptr()

    def host(self, t):
        torch.cuda.synchronize()
        h = t.cpu().numpy()
        return h.view(t.np_view[0]).reshape(t.np_view[1]) if getattr(t, "np_view", None) else h


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


FM_CASES = [(ch, n, lay) for n in A.FM_N + [A.FM_BIG, 3 * 32768 + 3] for ch, lay in ((5, "pad"), (4, "view"), (5, "oddstride"))] + \
           [(BIG, 4001, "pad"), (BIG, 4001, "oddstride")]
AGC_CASES = [(b, c) for b in A.AGC_BLOCKS for c in ("1", "2", "3", "16", "17", "33", "1-block calls")]
FV_CASES = [(T, n_out, lim) for T in A.FV_T for n_out in A.FV_OUT + [5000] for lim in (0.0, 1.0)]
WFM_CASES = [(ch, n) for ch in A.WFM_ROWS + [BIG] for n in A.WFM_N + [3001]]


@pytest.fixture(scope="module")
def matrix(gpu, oracle):
    """every check once under torch.profiler -> ({key: (status, value or message)}, kernel names launched)"""
    from torch.profiler import ProfilerActivity, profile
    drv = GpuDriver(gpu)
    res = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for ch, n, lay in FM_CASES:
            _run(res, f"fm {ch} {n} {lay}", A.check_fmdemod, drv, ch, n, lay, seed=n + ch)
        for lay in A.FM_LAYOUTS:
            _run(res, f"fm nonfinite {lay}", A.check_fmdemod_nonfinite, drv, A.FM_BIG, lay, seed=3)
        _run(res, "fm refusals", A.check_fmdemod_refusals, drv)
        for c in A.FD_CASES:
            _run(res, "fd " + A.fd_id(c), A.check_fracdec, drv, oracle, c, seed=int(c["rate"] * 10) + c["points"], ch_rep=3)
        for c in (FD_BIG, FD_BIG_TAPS):
            _run(res, "fd " + A.fd_id(c), A.check_fracdec_big, drv, oracle, c)
        _run(res, "fd bank", A.check_fracdec, drv, oracle, dict(rate=5.0, points=12, where=[None, 5.5] * (BIG // 2), n=48_000, T=0, B=None), seed=9,
             detail_rows=range(0, BIG, 128))
        _run(res, "fd refusals", A.check_fracdec_refusals, drv)
        for b, cut in AGC_CASES:
            _run(res, f"agc {b} {cut}", A.check_fastagc, drv, oracle, 3, b, A.AGC_CUTS[cut], seed=b)
        for b in (1024, 2048):
            _run(res, f"agc bank {b}", A.check_fastagc, drv, oracle, BIG, b, [9, 1, 6], seed=b, bound_rows=range(0, BIG, 97))
        for b, cuts in ((256, [3, 1, 1]), (1025, [2, 1]), (1024, [17, 2])):
            _run(res, f"agc nonfinite {b}", A.check_fastagc_nonfinite, drv, oracle, b, cuts, seed=b + 1)
        _run(res, "agc refusals", A.check_fastagc_refusals, drv)
        for T, n_out, lim in FV_CASES:
            _run(res, f"fv {T} {n_out} {lim}", A.check_fir_valid, drv, oracle, 4, T, n_out, lim, seed=T + n_out)
        _run(res, "fv bank", A.check_fir_valid, drv, oracle, BIG, 201, 4799, 1.0, seed=5)
        for T, n_out, lim in ((201, 3000, 0.0), (2, 300, 0.0), (208, 1030, 1.0), (1, 1025, 0.0)):
            _run(res, f"fv nonfinite {T} {n_out} {lim}", A.check_fir_valid_nonfinite, drv, T, n_out, lim, seed=T)
        _run(res, "fv refusals", A.check_fir_valid_refusals, drv)
        for ch, n in WFM_CASES:
            _run(res, f"wfm {ch} {n}", A.check_wfm, drv, oracle, ch, n, seed=ch * 100 + n, cuts=32 if n > 32 else None)
        _run(res, "wfm refusals", A.check_wfm_refusals, drv)
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


@pytest.mark.parametrize("ch,n,layout", FM_CASES, ids=[f"ch{c}-n{n}-{lay}" for c, n, lay in FM_CASES])
def test_gpu_fmdemod_bank(matrix, ch, n, layout):
    print(f"fmdemod ch={ch} n={n} {layout}: worst err/bound {_outcome(matrix, f'fm {ch} {n} {layout}'):.3f}")


@pytest.mark.parametrize("layout", A.FM_LAYOUTS)
def test_gpu_fmdemod_nonfinite(matrix, layout):
    _outcome(matrix, f"fm nonfinite {layout}")


@pytest.mark.parametrize("case", A.FD_CASES + [FD_BIG, FD_BIG_TAPS], ids=A.fd_id)
def test_gpu_fracdec_bank(matrix, case):
    print(f"{A.fd_id(case)}: worst err/bound {_outcome(matrix, 'fd ' + A.fd_id(case)):.3f}")


@pytest.mark.parametrize("block,cut", AGC_CASES)
def test_gpu_fastagc_bank(matrix, block, cut):
    _outcome(matrix, f"agc {block} {cut}")


@pytest.mark.parametrize("block", [1024, 256, 1025])
def test_gpu_fastagc_nonfinite(matrix, block):
    _outcome(matrix, f"agc nonfinite {block}")


@pytest.mark.parametrize("T,n_out,limit", FV_CASES)
def test_gpu_fir_valid_bank(matrix, T, n_out, limit):
    _outcome(matrix, f"fv {T} {n_out} {limit}")


@pytest.mark.parametrize("T,n_out,limit", [(201, 3000, 0.0), (2, 300, 0.0), (208, 1030, 1.0), (1, 1025, 0.0)])
def test_gpu_fir_valid_nonfinite(matrix, T, n_out, limit):
    _outcome(matrix, f"fv nonfinite {T} {n_out} {limit}")


@pytest.mark.parametrize("ch,n", WFM_CASES)
def test_gpu_deemphasis_wfm_bank(matrix, ch, n):
    _outcome(matrix, f"wfm {ch} {n}")


def test_gpu_1024_channel_banks(matrix):
    """every kernel at 1024 channels"""
    for key in ("fm 1024 4001 pad", "fm 1024 4001 oddstride", "fd bank", "agc bank 1024", "agc bank 2048", "fv bank", "wfm 1024 3001"):
        _outcome(matrix, key)


@pytest.mark.parametrize("what", ["fm", "fd", "agc", "fv", "wfm"])
def test_gpu_refusals(matrix, what):
    _outcome(matrix, f"{what} refusals")


def test_gpu_audio_coverage(matrix):
    """the matrix launched every kernel instantiation of the five banks, and nothing of them is left out of WANT_KERNELS"""
    assert matrix[1] == WANT_KERNELS, (sorted(matrix[1] - WANT_KERNELS), sorted(WANT_KERNELS - matrix[1]))
    assert {A.fracdec_path(c["n"], c["points"], c["T"] or None)[1] for c in (FD_BIG, FD_BIG_TAPS)} == {"fracdec_interp_kernel"}
