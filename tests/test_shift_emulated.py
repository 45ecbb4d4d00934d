"""CPU tier of the NCO shift banks: the checks of tests/shift_ref.py on the emulated library (tests/host_shim/emul_build.build_full_once, every
product translation unit executed on the host, the C ABI and the drop-ins included) under the three fiber orders, at small sizes.

CSDRB_SHIFT_SLICE_MIN is 3000 here (as in tests/test_kernels_emulated.py), so that banks of a few thousand chunk-channels reach the 2- and
3-slice side-stream chains.  There is no profiler, so coverage is stated through shift_ref.shift_path, the restatement of each launcher's
choice that every check also asserts the returned launch count against: test_matrix_reaches_every_path lists what each case reaches.
"""
import os
import shutil
import sys
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
os.environ.setdefault("CSDRB_SHIFT_SLICE_MIN", "3000")
import emul_build  # noqa: E402
import shift_ref as S  # noqa: E402

ORDERS = ["alternate", "reverse", "random"]
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
    copy = Path(lib).with_name(f"libcsdr_b200_emul_shift_{request.param}.so")
    if not copy.exists():
        shutil.copy(lib, copy)
    saved_env = os.environ.get("CUDA_EMUL_ORDER")
    saved = csdr_b200.LIB_PATH, csdr_b200._lib
    os.environ["CUDA_EMUL_ORDER"] = request.param
    csdr_b200.LIB_PATH, csdr_b200._lib = copy, None
    t0 = time.perf_counter()
    try:
        yield EmulDriver(csdr_b200)
    finally:
        print(f"\nshift checks under fiber order {request.param}: {time.perf_counter() - t0:.1f} s")
        csdr_b200.LIB_PATH, csdr_b200._lib = saved
        if saved_env is None:
            os.environ.pop("CUDA_EMUL_ORDER", None)
        else:
            os.environ["CUDA_EMUL_ORDER"] = saved_env


# ---- coverage (host only) -----------------------------------------------------------------------------------------------------------------
def test_matrix_reaches_every_path():
    """every launcher path of the shift banks is reached by a case of this file: the direct and the wrap-table chain of each chained bank,
    unsliced and 2- and 3-slice side-stream chains of both shift_addition forms, chunk > n, n % chunk != 0, a chunk not a multiple of 4"""
    assert S.slice_min() == int(os.environ["CSDRB_SHIFT_SLICE_MIN"])
    reached = {}
    for kind, ch, n, chunk, tsize, _, _ in S.BANK_CASES:
        p = S.shift_path(ch, n, tsize if kind == "unroll" else chunk, kind)
        key = (kind, "table" if p["table"] else "direct", "side stream" if p["side"] else "one stream", p["slices"])
        reached.setdefault(key, []).append((ch, n, chunk, tsize))
    for key in sorted(reached):
        print(key, "<-", reached[key][:3])
    for kind in ("cc", "fc", "addfast", "unroll"):
        assert {(kind, "direct", "one stream", 1), (kind, "table", "one stream", 1)} <= set(reached), kind
    for kind in ("cc", "fc"):
        assert {(kind, "table", "side stream", 2), (kind, "table", "side stream", 3)} <= set(reached), kind
    assert ("cc", "table", "side stream", 1) in reached                  # cut into slices of whole 128-chunk CTAs: a short chain is one slice
    assert any(k == "cc" and c > n for k, _, n, c, _, _, _ in S.BANK_CASES)
    assert any(k == "addfast" and c % 4 for k, _, _, c, _, _, _ in S.BANK_CASES)
    assert any(k == "unroll" and t > n for k, _, n, _, t, _, _ in S.BANK_CASES)
    chunks = {c for k, _, _, c, _, _, _ in S.BANK_CASES if k == "cc"}
    assert {0, 1, 2, 3, 4, 5, 31, 32, 33, 1023, 1024, 1025} <= chunks
    nch = {S.shift_path(ch, n, c)["nchunks"] for k, ch, n, c, _, _, _ in S.BANK_CASES if k == "cc"}
    assert {96, 97, 127, 128, 129} <= nch
    assert {lay for *_, lay, _ in S.BANK_CASES} == {"tight", "pad", "shared"} and {lay for *_, lay in S.BANK_CASES} == {"tight", "pad", "odd"}
    # the invariant cases compare the table chain with the direct chain, and a sliced bank with its unsliced channels
    inv = set()
    for kind, ch, n, chunk, tsize in S.INV_CASES:
        ck = tsize if kind == "unroll" else chunk
        bank, one = S.shift_path(ch, n, ck, kind), S.shift_path(1, n, ck, kind)
        if bank["table"]:
            inv.add((kind, "table vs direct"))
        if bank["slices"] > 1 and one["slices"] == 1:
            inv.add((kind, "sliced vs unsliced"))
    assert {("cc", "table vs direct"), ("fc", "table vs direct"), ("addfast", "table vs direct"), ("unroll", "table vs direct"),
            ("cc", "sliced vs unsliced"), ("fc", "sliced vs unsliced")} <= inv, inv


# ---- the banks ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", S.BANK_CASES, ids=[S.case_id(c) for c in S.BANK_CASES])
def test_shift_bank(drv, oracle, case):
    kind, ch, n, chunk, tsize, lin, lout = case
    rates, ph0 = S.rates_phases(ch, shift=n % 7)
    amb, worst = S.check_bank(drv, oracle, kind, rates, ph0, n, chunk, tsize, lin, lout, seed=n + ch)
    print(f"{S.case_id(case)}: ambiguous seeds {amb}, worst err/bound {worst:.3f}")


@pytest.mark.parametrize("case", S.INV_CASES, ids=[S.case_id(c) for c in S.INV_CASES])
def test_shift_invariants(drv, oracle, case):
    kind, ch, n, chunk, tsize = case
    rates, ph0 = S.rates_phases(ch, shift=3)
    S.check_invariants(drv, oracle, kind, rates, ph0, n, chunk, tsize, seed=n)


@pytest.mark.parametrize("case", S.NONFINITE_CASES, ids=[S.case_id(c) for c in S.NONFINITE_CASES])
def test_shift_nonfinite(drv, oracle, case):
    kind, n, chunk, tsize = case
    S.check_nonfinite(drv, oracle, kind, n, chunk, tsize, seed=n)


@pytest.mark.parametrize("dec,sizes", S.DEC_CASES, ids=[f"d{d}-{'+'.join(map(str, s))}" for d, s in S.DEC_CASES])
def test_decimating_shift_bank(drv, oracle, dec, sizes):
    rates, ph0 = S.rates_phases(5, shift=dec)
    remain = [0, 1, dec - 1, sizes[0] + 2, sizes[0] + dec]                # the last two skip the whole first call
    S.check_decimating(drv, oracle, rates, ph0, remain, dec, sizes, seed=dec)


def test_shift_refusals(drv, oracle):
    S.check_refusals(drv, oracle)


@pytest.mark.parametrize("n,call,rate,phase", S.DROPIN_CASES)
def test_shift_dropins(drv, oracle, n, call, rate, phase):
    S.check_dropins(drv, oracle, n, call, rate, phase, seed=n)
