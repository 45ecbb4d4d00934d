"""CPU tier of the FM chain's audio-rate kernels: the checks of tests/audio_ref.py on the emulated library (tests/host_shim/emul_build.build_full_once,
every product translation unit executed on the host, the C ABI included) under the three fiber orders, at small sizes.

There is no profiler here, so coverage is stated through the host restatements of each launcher's choice (audio_ref.fm_path, fracdec_path,
agc_path, fv_path, wfm_path) and of fracdec's segment walk (audio_ref.fracdec_walk): test_matrix_reaches_every_path lists what each part of the
matrix reaches.  The big paths (fracdec from 2^22 samples on, 1024-channel banks, fmdemod's grid loop at full width) run in the GPU tier.
"""
import os
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import audio_ref as A  # noqa: E402
import emul_build  # noqa: E402

ORDERS = ["alternate", "reverse", "random"]

FM_CASES = [(ch, n, lay) for n in A.FM_N for ch, lay in ((3, "pad"), (2, "view"), (3, "oddstride"))] + [(1, 33_001, "pad")]
AGC_CASES = [(1, ["1-block calls", "33"]), (2, ["2", "16+1+2"]), (255, ["3"]), (256, ["17"]), (257, ["1-block calls"]), (1000, ["3"]), (1023, ["2"]),
             (1024, ["17+16"]), (1025, ["1", "3"]), (4096, ["2"])]
FV_CASES = [(1, 1, 0.0), (1, 1025, 1.0), (2, 255, 0.0), (2, 769, 0.7), (201, 256, 0.0), (201, 1023, 1.0), (201, 257, 0.0), (208, 767, 0.0),
            (208, 1024, 1.0), (208, 2049, 0.0)]
WFM_CASES = [(1, 33), (31, 32), (32, 1), (33, 31), (127, 33), (128, 32), (129, 100)]


class EmulDriver:
    """'device' buffers are 256-byte aligned host copies (cudaMalloc's alignment)"""
    stream = None

    def __init__(self, pkg):
        self.pkg, self.L = pkg, pkg.lib()

    def dev(self, a):
        a = np.ascontiguousarray(a)
        raw = np.empty(a.nbytes + 256, np.uint8)
        off = (-raw.ctypes.data) % 256
        d = raw[off:off + a.nbytes].view(a.dtype).reshape(a.shape)
        d[...] = a
        return d

    def ptr(self, d):
        return d.ctypes.data

    def host(self, d):
        return d.copy()


@pytest.fixture(scope="module", params=ORDERS)
def drv(request, tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    import csdr_b200
    lib, _ = emul_build.build_full_once(tmp_path_factory)
    copy = Path(lib).with_name(f"libcsdr_b200_emul_audio_{request.param}.so")
    if not copy.exists():
        shutil.copy(lib, copy)
    saved_env = os.environ.get("CUDA_EMUL_ORDER")
    saved = csdr_b200.LIB_PATH, csdr_b200._lib
    os.environ["CUDA_EMUL_ORDER"] = request.param
    csdr_b200.LIB_PATH, csdr_b200._lib = copy, None
    try:
        yield EmulDriver(csdr_b200)
    finally:
        csdr_b200.LIB_PATH, csdr_b200._lib = saved
        if saved_env is None:
            os.environ.pop("CUDA_EMUL_ORDER", None)
        else:
            os.environ["CUDA_EMUL_ORDER"] = saved_env


# ---- coverage and the segment table's margin (host only) ----------------------------------------------------------------------------------
def test_matrix_reaches_every_path():
    """every kernel instantiation and launcher branch of the five banks, and every segment branch and segment end of fracdec's walk, is reached
    by a case of this file (fracdec's sequential fallback and the 1024-channel banks by the GPU file)"""
    fm = set()
    for ch, n, lay in FM_CASES:
        stride, col0 = A.fm_layout(n, lay)
        fm |= {A.fm_path(256 + 8 * col0 + 8 * stride * c, n) for c in range(ch)}
    assert {p[0] for p in fm} == {"vector", "scalar"} and ("vector", True, False) in fm and ("vector", True, True) in fm, fm
    br, ends, kern = A.fd_coverage(A.FD_CASES)
    assert br == A.FD_BRANCHES, br
    assert ends == A.FD_ENDS, ends
    assert {k[1] for k in kern} == {"fracdec_interp_seg_kernel<12>", "fracdec_interp_seg_kernel<0>"}
    assert {k[2] for k in kern if len(k) > 2} == {"unrolled16", "loop"}
    assert {p for c in A.FD_CASES for p in [c["points"]]} >= {2, 4, 12, 16, 18, 64} and any(c["T"] for c in A.FD_CASES)
    agc = set()
    for block, cuts in AGC_CASES:
        for name in cuts:
            for nb in A.AGC_CUTS[name]:
                agc |= set(A.agc_path(block, nb)) | set(A.agc_path(block, nb, s16=True))
    assert {"fastagc_fused_kernel<false>", "fastagc_fused_kernel<true>", "fastagc_peaks_kernel", "fastagc_apply_kernel<false>",
            "fastagc_apply_kernel<true>", "fastagc_carry_kernel", "carry: shift history", "carry: copy two blocks", "runs: 2", "runs: 3"} <= agc, agc
    fv = set()
    for T, n_out, lim in FV_CASES:
        fv |= set(A.fv_path(T, n_out + T, lim))
    assert {"nfm_deemph_bank_kernel<true>", "nfm_deemph_bank_kernel<false>"} <= fv
    assert {f"last tile accumulators: {s}" for s in ("0", "01", "012", "0123")} <= fv, fv
    wfm = set()
    for ch, _ in WFM_CASES:
        wfm |= set(A.wfm_path(ch))
    assert {"CTAs: 2", "warps: 5", "rows of the last warp: 1", "rows of the last warp: 31", "rows of the last warp: 32"} <= wfm, wfm


def test_fracdec_segment_table_margin():
    """the segment walk never comes near FD_MAX_SEGS - 2 (from there on it falls back to single steps, and entries past the table would be lost)"""
    worst, at = A.fd_segment_sweep()
    assert worst < A.FD_MAX_SEGS - 2, (worst, at)
    print(f"most segments: {worst} at {at}")


# ---- fmdemod ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ch,n,layout", FM_CASES, ids=[f"ch{c}-n{n}-{lay}" for c, n, lay in FM_CASES])
def test_fmdemod_bank(drv, ch, n, layout):
    A.check_fmdemod(drv, ch, n, layout, seed=n + ch)


@pytest.mark.parametrize("layout", A.FM_LAYOUTS)
def test_fmdemod_nonfinite(drv, layout):
    A.check_fmdemod_nonfinite(drv, 515, layout, seed=3)


def test_fmdemod_refusals(drv):
    A.check_fmdemod_refusals(drv)


# ---- fractional decimator -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", A.FD_CASES, ids=A.fd_id)
def test_fracdec_bank(drv, oracle, case):
    A.check_fracdec(drv, oracle, case, seed=int(case["rate"] * 10) + case["points"])


def test_fracdec_refusals(drv):
    A.check_fracdec_refusals(drv)


# ---- fastagc ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("block,cuts", [(b, c) for b, cs in AGC_CASES for c in cs], ids=[f"b{b}-{c}" for b, cs in AGC_CASES for c in cs])
def test_fastagc_bank(drv, oracle, block, cuts):
    A.check_fastagc(drv, oracle, 2, block, A.AGC_CUTS[cuts], seed=block)


@pytest.mark.parametrize("block,cuts", [(256, [3, 1, 1]), (1025, [2, 1])])
def test_fastagc_nonfinite(drv, oracle, block, cuts):
    A.check_fastagc_nonfinite(drv, oracle, block, cuts, seed=block + 1)


def test_fastagc_refusals(drv):
    A.check_fastagc_refusals(drv)


# ---- fir_valid (NFM de-emphasis) ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,n_out,limit", FV_CASES)
def test_fir_valid_bank(drv, oracle, T, n_out, limit):
    A.check_fir_valid(drv, oracle, 3, T, n_out, limit, seed=T + n_out)


@pytest.mark.parametrize("T,n_out,limit", [(201, 1100, 0.0), (2, 300, 0.0), (208, 1030, 1.0)])
def test_fir_valid_nonfinite(drv, T, n_out, limit):
    A.check_fir_valid_nonfinite(drv, T, n_out, limit, seed=T)


def test_fir_valid_refusals(drv):
    A.check_fir_valid_refusals(drv)


# ---- deemphasis_wfm -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ch,n", WFM_CASES)
def test_deemphasis_wfm_bank(drv, oracle, ch, n):
    A.check_wfm(drv, oracle, ch, n, seed=ch * 100 + n, cuts=31 if n > 31 else None)


def test_deemphasis_wfm_refusals(drv):
    A.check_wfm_refusals(drv)
