"""CPU tier of the FIR bank contract: the checks of tests/fir_ref.py on the emulated library (tests/host_shim/emul_build.build_full_once: every
product translation unit executed on the host, the C ABI and the host pipeline included), under the three fiber orders.

There is no profiler here, so coverage is stated through fir_ref.kernel_for: the subset below reaches every compiled fir_bank_fast_kernel
instantiation, the generic kernel and the u8 two-launch path (u8_rows_to_cf32_kernel) at least once.
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
import emul_build  # noqa: E402
import fir_ref as F  # noqa: E402

ORDERS = ["alternate", "reverse", "random"]
MAX_WORK = 12_000                                                    # channels x samples of a matrix case


def _subset():
    """the first case of the matrix for every kernel, the edges of the tap range and the generic layouts"""
    out, seen = [], set()
    for c in F.cases(max_work=MAX_WORK, tiles=1):
        k = F.kernel_for(c["D"], c["T"], c["variant"], c["layout"] == "pad")
        edge = c["T"] in (1, 200, 900) or c["layout"] != "pad" or c["kind"] == "odd"
        if k not in seen or (edge and c["seed"] % 10 == 0):
            seen.add(k)
            out.append(c)
    return out


CASES = _subset()
NONFINITE = [(10, 79, -1), (10, 81, 0), (10, 199, -1), (10, 81, 1), (10, 81, 2), (10, 81, 3), (10, 150, 4), (10, 81, 5), (10, 81, 6), (10, 81, 7),
             (50, 801, -1), (50, 51, -1), (7, 79, -1)]
U8_CASES = [(10, 79, 2_405), (10, 199, 8_321), (50, 801, 3_011), (10, 81, 205)]


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
    copy = Path(lib).with_name(f"libcsdr_b200_emul_fir_{request.param}.so")
    if not copy.exists():
        shutil.copy(lib, copy)
    saved_env = os.environ.get("CUDA_EMUL_ORDER")
    saved = csdr_b200.LIB_PATH, csdr_b200._lib
    os.environ["CUDA_EMUL_ORDER"] = request.param
    csdr_b200.LIB_PATH, csdr_b200._lib = copy, None
    try:
        d = EmulDriver(csdr_b200)
        yield d
    finally:
        csdr_b200.LIB_PATH, csdr_b200._lib = saved
        if saved_env is None:
            os.environ.pop("CUDA_EMUL_ORDER", None)
        else:
            os.environ["CUDA_EMUL_ORDER"] = saved_env


def test_subset_reaches_every_kernel():
    ran = {F.kernel_for(c["D"], c["T"], c["variant"], c["layout"] == "pad") for c in CASES}
    ran |= {F.kernel_for(D, T, v) for D, T, v in NONFINITE}
    ran |= {F.kernel_for(D, T, u8=True) for D, T, _ in U8_CASES}
    assert ran == set(F.KERNELS) | {F.GENERIC}, sorted(map(str, set(F.KERNELS) | {F.GENERIC} - ran))


@pytest.mark.parametrize("case", CASES, ids=F.case_id)
def test_fir_bank_contract(drv, case):
    """bound at every output, and the bit-exact invariants of fir_ref.check_case"""
    F.check_case(drv, case)


@pytest.mark.parametrize("D,T", [(10, 79), (10, 199), (50, 801)])
def test_fir_bank_firdes_taps(drv, oracle, D, T):
    c = dict(D=D, T=T, variant=-1, layout="pad", kind="firdes", n=T + 700 * D + 7, channels=3, seed=D + T)
    F.check_case(drv, c, taps=oracle.firdes_lowpass_f(T, 0.5 / D), invariants=False)


@pytest.mark.parametrize("T", [79, 199])
def test_fir_bank_tilings_agree(drv, T):
    F.check_tilings(drv, 10, T, T + 1000 * 10 + 3, ch=2, seed=T)


@pytest.mark.parametrize("D,T,variant", NONFINITE)
def test_fir_bank_nonfinite_stays_in_its_windows(drv, D, T, variant):
    F.check_nonfinite(drv, D, T, variant, F.nonfinite_n(D, T, variant), ch=3, seed=T + variant)


@pytest.mark.parametrize("D,T,n", U8_CASES)
def test_fir_bank_u8_equals_convert_then_filter(drv, D, T, n):
    F.check_u8(drv, D, T, n, ch=3, seed=n)


def test_fir_bank_host_calls_and_dropin(drv):
    """fir_decimate_bank_cc_host / _u8_host with chunk_channels 0, 1, 2, C over padded host rows give the device call's bits and leave the output
    padding alone; libcsdr's fir_decimate_cc equals the one-channel bank call"""
    pkg = drv.pkg
    D, T, ch, n = 10, 199, 4, 4_001
    h = np.random.default_rng(3).uniform(-1, 1, T).astype(np.float32)
    x, _ = F.make_inputs(dict(seed=4, channels=ch, n=n, T=T))
    u = F.u8_inputs(ch, n, 5)
    for u8 in (False, True):
        want = F.bank(drv, F.convert_u8(u) if u8 else x, D, h)
        if u8:
            src = np.full((ch, n + 24, 2), 0x5A, np.uint8); src[:, :n] = u
        else:
            src = np.full((ch, n + 5), np.nan, np.complex64); src[:, :n] = x
        n_out = want.shape[1]
        for cc in (0, 1, 2, ch):
            ob = np.full((ch, 2 * (n_out + 3)), F.SENTINEL, np.uint32).view(np.complex64)
            (pkg.fir_decimate_bank_u8_host if u8 else pkg.fir_decimate_bank_cc_host)(src[:, :n], D, h, out=ob[:, :n_out], chunk_channels=cc)
            F.assert_bits_equal(ob[:, :n_out], want, f"host call u8={u8}, chunk_channels={cc}")
            assert np.all(ob.view(np.uint32)[:, 2 * n_out:] == F.SENTINEL), "the host call wrote into the output padding"
    for D, T, n in ((10, 199, 2_001), (10, 79, 1_001), (50, 801, 5_000), (7, 79, 501)):
        x, h = F.make_inputs(dict(seed=n, channels=1, n=n, T=T))
        F.assert_bits_equal(pkg.libcsdr.fir_decimate_cc(x[0], D, h), F.bank(drv, x, D, h)[0], f"libcsdr.fir_decimate_cc D={D} T={T}")
