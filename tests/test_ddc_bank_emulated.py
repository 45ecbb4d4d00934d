"""CPU tier: the fused DDC bank (csrc/ddc_bank.cu, ddc_bank_fused2_kernel) executed on the host under tests/host_shim, all 12 instantiations.

Contract (DESIGN.md 8b): output o of channel c depends only on its own samples, its phasors and the taps, so the bank gives the same bits for one or
two channels per lane (CSDRB_DDC_CPL), any segmentation, any channel count or subset, and any split of the stream into blocks.  Against the float64
reference every output is inside the error bound of the kernel's arithmetic (tests/ddc_ref.py), the NCO is the reference's bit for bit, and the
discriminator is fmdemod_quadri_cf on the bank's own baseband bit for bit.

CSDRB_DDC_CPL is read once per launch_fused<D, M> instantiation, at its first call, so one channel per lane needs its own loaded copy of the library
with the variable set while that copy is first called (the fixture below); the barrier count of the emulator (one __syncthreads per CTA) shows which
geometry each copy launched.
"""
import ctypes as C
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
from ddc_ref import (NONFINITE, assert_bits_equal, case_id, cases, check_against_reference, check_nonfinite, kernel_for, make_inputs, n_out_of,  # noqa: E402
                     nco)

ORDERS = ["alternate", "reverse", "random"]
SM_COUNT, WARPS_PER_SM = 132, 12                                     # kSmCount (common.cuh), kDdcWarpsPerSm (ddc_bank.cu)
SENTINEL = np.uint32(0x7FC0DEAD)                                     # a NaN the kernel never produces: padding must keep it
_built = {}
_ORACLE = None                                                       # the session's oracle (shift_addition_init for the NCO parameters)


def _load(so, tag, order, cpl):
    copy = so.with_name(f"{so.stem}_{order}_{tag}.so")
    if not copy.exists():
        shutil.copy(so, copy)
    saved = {k: os.environ.get(k) for k in ("CUDA_EMUL_ORDER", "CSDRB_DDC_CPL")}
    os.environ["CUDA_EMUL_ORDER"] = order
    if cpl == 1:
        os.environ["CSDRB_DDC_CPL"] = "1"
    else:
        os.environ.pop("CSDRB_DDC_CPL", None)
    try:
        lib = C.CDLL(str(copy))
        for n in _built["names"]:
            f = getattr(lib, "emul_" + n); g = getattr(_built["proto"], "emul_" + n)
            f.argtypes, f.restype = g.argtypes, g.restype
        lib.emul_last_error.restype = C.c_char_p; lib.emul_barriers.restype = C.c_long
        lib.cpl = cpl
        for D, T in ((50, 801), (10, 79), (10, 199)):               # first call of every launch_fused<D, M>: fixes its channels per lane
            x = np.ones(T, np.complex64); rates = np.zeros(1, np.float32)
            _run(lib, x, rates, np.zeros(1, np.float32), 1024, 0, D, np.ones(T, np.float32), 0, None)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return lib


@pytest.fixture(scope="module", params=ORDERS)
def banks(request, tmp_path_factory, oracle):
    """(two channels per lane, one channel per lane): two private copies of the emulated ddc_bank.cu per fiber order"""
    global _ORACLE
    _ORACLE = oracle
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if "so" not in _built:
        lib, names = emul_build.build_file(tmp_path_factory.mktemp("emul_ddc_cpl"), "ddc_bank.cu")
        _built.update(so=Path(lib._name), names=names, proto=lib)
    return _load(_built["so"], "cpl2", request.param, 2), _load(_built["so"], "cpl1", request.param, 1)


# ---- write guards, as in test_kernels_emulated.py: an out-of-bounds write of a kernel trips the canaries -------------------------------------
_GUARD = 512
_guarded = []


def Z(shape, dtype):
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = np.full(n + 2 * _GUARD + 32, 0xA5, np.uint8)
    off = _GUARD + ((-(raw.ctypes.data + _GUARD)) % 16)
    raw[off:off + n] = 0
    _guarded.append((raw, off, n))
    return raw[off:off + n].view(dtype).reshape(shape)


@pytest.fixture(autouse=True)
def _check_guards():
    _guarded.clear()
    yield
    for raw, off, n in _guarded:
        assert np.all(raw[:off] == 0xA5) and np.all(raw[off + n:] == 0xA5), "a kernel wrote outside one of its buffers"
    _guarded.clear()


def P(a):
    return a.ctypes.data


def expected_ctas(channels, n_out, M, cpl):
    """launch_fused's grid: segments sized to fill SM_COUNT * WARPS_PER_SM warps, at least 2M outputs each, one warp per (segment, channel set)"""
    wps = -(-channels // (32 * cpl))
    want = -(-SM_COUNT * WARPS_PER_SM // wps)
    seg = max(-(-n_out // want), 2 * M)
    return (-(-n_out // seg) * wps + 3) // 4


def _prepass(lib, x, rates, ph0, chunk, offset, D, T):
    """the phase-chain pre-pass of one block: (wideband copy, NCO parameters, scratch with the chunk seeds, carried phases).  It does not depend on
    the channels per lane, so the main kernels of both library copies may share it."""
    ch, n = rates.size, x.size
    xa = Z(n, np.complex64); xa[:] = x
    params = Z((ch, 3), np.float32); params[:] = [_ORACLE.shift_addition_init(float(r)) for r in rates]
    ph = Z(ch, np.float32); ph[:] = ph0
    sb = lib.emul_ddc_bank_scratch_bytes(ch, n, chunk, offset); scratch = Z(sb + 64, np.uint8)
    assert lib.emul_launch_ddc_prepass(n, ch, P(params), P(ph), chunk, offset, D, T, P(scratch), sb, None) > 0, lib.emul_last_error()
    return xa, params, scratch, ph.copy()


def _main(lib, pre, chunk, offset, D, taps, demod, last_in):
    """the main kernel on a pre-pass -> (out [C, n_out], last_out or None).  The output has a spare row and three spare columns, last_out a spare
    entry, all holding SENTINEL: they must come back untouched.  The emulator's barrier count (one per CTA) must match the grid launch_fused
    computes for this copy's channels per lane."""
    xa, params, scratch, _ = pre
    ch, n, T = params.shape[0], xa.size, taps.size
    n_out = n_out_of(n, D, T)
    stride = n_out + 3
    out = Z((ch + 1, stride), np.float32 if demod else np.complex64); out.view(np.uint32)[:] = SENTINEL
    last_out = Z(ch + 1, np.complex64); last_out.view(np.uint32)[:] = SENTINEL
    li = None
    if last_in is not None:
        li = Z(ch, np.complex64); li[:] = last_in
    b0 = lib.emul_barriers()
    rc = lib.emul_launch_ddc_main(P(xa), n, ch, P(params), chunk, offset, D, taps.ctypes.data_as(C.c_void_p), T, demod, P(out), stride,
                                  P(li) if li is not None else None, P(last_out) if demod else None, P(scratch))
    assert rc == n_out, lib.emul_last_error()
    assert lib.emul_barriers() - b0 == expected_ctas(ch, n_out, kernel_for(D, T)[1], lib.cpl), "the copy did not run the channels per lane it was loaded for"
    words = out.view(np.uint32)
    assert np.all(words[:, n_out if demod else 2 * n_out:] == SENTINEL) and np.all(words[ch] == SENTINEL), "a store beyond n_out or channels"
    assert np.all(last_out.view(np.uint32)[2 * ch if demod else 0:] == SENTINEL), "a last_out store beyond channels, or without demod"
    return out[:ch, :n_out].copy(), (last_out[:ch].copy() if demod else None)


def _run(lib, x, rates, ph0, chunk, offset, D, taps, demod, last_in):
    """one whole bank call, pre-pass and main kernel -> (out, carried phases, last_out or None)"""
    pre = _prepass(lib, x, rates, ph0, chunk, offset, D, taps.size)
    out, lo = _main(lib, pre, chunk, offset, D, taps, demod, last_in)
    return out, pre[3], lo


def _firdes_case(oracle, case):
    return oracle.firdes_lowpass_f(case["T"], 0.5 / case["D"]) if case.get("firdes") else None


FIRDES = [dict(D=50, T=801, channels=65, chunk=1024, offset=0, n=801 + 60 * 50, seed=7, firdes=True),
          dict(D=10, T=199, channels=33, chunk=1024, offset=517, n=199 + 300 * 10 + 7, seed=8, firdes=True),
          dict(D=10, T=79, channels=97, chunk=1000, offset=999, n=79 + 200 * 10 + 3, seed=9, firdes=True)]
CASES = cases(large=90, extra=FIRDES, chain_budget=6000)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_fused_ddc_bank_contract(banks, oracle, case):
    """one case of the matrix, both kernels (DEMOD false / true) and both channels-per-lane copies:
    reference bound and bit-exact invariants (tests/ddc_ref.py), CPL=1 == CPL=2, a channel subset == the full bank, two blocks == one"""
    cpl2, cpl1 = banks
    D, T, chunk, offset = case["D"], case["T"], case["chunk"], case["offset"]
    x, rates, ph0, last, taps = make_inputs(case, _firdes_case(oracle, case))
    ch = rates.size
    pre = _prepass(cpl2, x, rates, ph0, chunk, offset, D, T)
    ph_b = pre[3]
    base, _ = _main(cpl2, pre, chunk, offset, D, taps, 0, None)
    dem, lo = _main(cpl2, pre, chunk, offset, D, taps, 1, last)
    check_against_reference(oracle, case, x, rates, ph0, last, taps, base, ph_b, dem, ph_b, lo)

    for demod, want in ((0, (base, None)), (1, (dem, lo))):
        got = _main(cpl1, pre, chunk, offset, D, taps, demod, last if demod else None)
        for g, w, what in zip(got, want, ("output", "last_out")):
            if w is not None:
                assert_bits_equal(g, w, f"CPL=1 against CPL=2, demod={demod}: {what}")

    sub = np.unique([0, ch // 2, ch - 1])
    got, ph_s, _ = _run(cpl2, x, rates[sub], ph0[sub], chunk, offset, D, taps, 0, None)
    assert_bits_equal(got, base[sub], "channel subset against the full bank")
    assert_bits_equal(ph_s, ph_b[sub], "channel subset: carried phase")

    n_out = base.shape[1]
    if chunk > 0 and n_out >= 2:                                     # chunk = 0 means "one chunk per call": a split changes the NCO by definition
        k = n_out // 2
        n1 = T + k * D - 1                                           # k outputs, the last D - 1 samples already belong to output k
        o1, p1, l1 = _run(cpl1, x[:n1], rates, ph0, chunk, offset, D, taps, 1, last)
        consumed = o1.shape[1] * D
        o2, p2, l2 = _run(cpl2, x[consumed:], rates, p1, chunk, (offset + consumed) % chunk, D, taps, 1, l1)
        assert_bits_equal(np.concatenate([o1, o2], 1), dem, "two blocks with the tail re-presented against one")
        assert_bits_equal(p2, ph_b, "two blocks: carried phase")
        assert_bits_equal(l2, lo, "two blocks: last_out")


@pytest.mark.parametrize("chunk,offset", [(1024, 0), (7, 3), (13, 12)])
def test_fused_ddc_bank_unit_tap_is_the_reference_nco(banks, oracle, chunk, offset):
    """x = 1 and a single unit tap at k: output o is the reference phasor at sample oD + k, bit for bit, in every instantiation and copy"""
    rng = np.random.default_rng(chunk)
    ch = 33
    rates = np.linspace(-0.4999, 0.4999, ch).astype(np.float32)
    ph0 = rng.uniform(-3, 3, ch).astype(np.float32)
    for D, T in ((50, 801), (10, 80), (10, 199)):
        n = T + 47 * D + 3
        x = np.ones(n, np.complex64)
        refs = [nco(oracle, r, ph0[c], chunk, offset, n) for c, r in enumerate(rates)]
        pre = _prepass(banks[0], x, rates, ph0, chunk, offset, D, T)
        for k in (0, 3, 9, 79):
            taps = np.zeros(T, np.float32); taps[k] = 1.0
            for lib in banks:
                out, _ = _main(lib, pre, chunk, offset, D, taps, 0, None)
                for c in range(ch):
                    assert_bits_equal(out[c], refs[c][k::D][:out.shape[1]], f"D={D} T={T} k={k} CPL={lib.cpl} channel {c}")


@pytest.mark.parametrize("D,T", NONFINITE)
@pytest.mark.parametrize("chunk,offset", [(1024, 0), (13, 12)])
def test_fused_ddc_bank_nonfinite_stays_in_its_windows(banks, D, T, chunk, offset):
    """NaN / +-Inf wideband samples reach exactly the outputs whose window holds them (ddc_ref.check_nonfinite), both DEMOD kernels and both
    channels-per-lane copies; the two copies give the same bits"""
    case = dict(D=D, T=T, channels=33, chunk=chunk, offset=offset, n=T + 60 * D + 7, seed=D + T + chunk)
    outs = []
    for lib in banks:
        got = {}

        def run(x, rates, ph0, last, taps, demod):
            out, _, lo = _run(lib, x, rates, ph0, chunk, offset, D, taps, demod, last if demod else None)
            got[(x.tobytes(), demod)] = (out, lo)
            return out, lo
        check_nonfinite(run, case)
        outs.append(got)
    for k in outs[0]:
        for a, b in zip(outs[0][k], outs[1][k]):
            if a is not None:
                assert_bits_equal(b, a, "CPL=1 against CPL=2")
