"""GPU tier (-m gpu) of the fused DDC bank at every served decimation: the geometry matrix of tests/ddc_generic_ref.py at larger sizes, through
csdr_b200.ddc_bank and DdcBank, against the contract of tests/ddc_ref.py (float64 bound, NCO / discriminator / last_out bit for bit, the bits
independent of channels per lane, channel subset, block split and DdcBank block sizes).

Every generic geometry must run ddc_bank_generic_kernel<M, CPL, DEMOD> with its bucket M and never ddc_bank_fused2_kernel; torch.profiler lists
the kernels.  One channel per lane (CSDRB_DDC_CPL=1) is fixed when the library first launches a bank kernel, so a child process runs the matrix
with it and hands back a digest of every output array.

Run directly (python tests/test_gpu_ddc_generic.py --child DIR), this file is that child.
"""
import hashlib
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import ddc_ref  # noqa: E402
from ddc_generic_ref import BUCKETS, NONFINITE, case_id, cases, kernel_for, nonfinite_positions  # noqa: E402
from ddc_ref import assert_bits_equal, check_against_reference, check_nonfinite, make_inputs, n_out_of, nco  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SENTINEL = np.uint32(0x7FC0DEAD)
EXTRA = [dict(D=40, T=641, channels=700, chunk=1024, offset=100, n=641 + 1999 * 40 + 10, seed=21, firdes=True),     # hundreds of channels,
         dict(D=200, T=3201, channels=300, chunk=1024, offset=0, n=3201 + 999 * 200 + 17, seed=22, firdes=True),    # the product's taps,
         dict(D=48, T=769, channels=257, chunk=7, offset=3, n=769 + 1999 * 48 + 5, seed=23, firdes=True),          # thousands of outputs
         dict(D=12, T=193, channels=1000, chunk=1000, offset=999, n=193 + 99 * 12 + 9, seed=24),                   # segments at the 2M floor
         dict(D=2, T=48, channels=513, chunk=13, offset=12, n=48 + 4999 * 2 + 1, seed=25, firdes=True),
         dict(D=400, T=8000, channels=129, chunk=1024, offset=517, n=8000 + 299 * 400 + 3, seed=26, firdes=True)]
CASES = cases(outputs=300, max_wide=150_000, chain_budget=300_000, extra=EXTRA)
KERNEL_NAME = re.compile(r"ddc_bank_(fused2|generic)_kernel<([\d, ]+), (true|false)>")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bank(gpu, x, rates, ph0, chunk, offset, D, taps, demod, last):
    """one csdrb_ddc_bank call into an output with a spare row and spare columns that hold SENTINEL -> (out, carried phases, last_out or None)"""
    ch, n_out = rates.size, n_out_of(x.size, D, taps.size)
    stride = n_out + (n_out & 1) + 2
    init = np.full((ch + 1, stride * (1 if demod else 2)), SENTINEL, np.uint32).view(np.float32 if demod else np.complex64)
    out = _dev(init)
    _, ph, lo = gpu.ddc_bank(_dev(x), rates, D, taps, demod=bool(demod), chunk=chunk, offset=offset, phases=_dev(ph0),
                             last=_dev(last) if last is not None else None, out=out)
    full = out.cpu().numpy()
    words = full.view(np.uint32)
    assert np.all(words[:, n_out * (1 if demod else 2):] == SENTINEL) and np.all(words[ch] == SENTINEL), "a store beyond n_out or channels"
    return full[:ch, :n_out].copy(), ph.cpu().numpy(), (lo.cpu().numpy() if demod else None)


def run_matrix(gpu):
    """every case (both DEMOD kernels, a 3-channel subset, a two-block split), the unit-tap probes and the non-finite runs -> {name: array}"""
    res = {}
    for case in CASES:
        key = case_id(case)
        D, T, chunk, offset = case["D"], case["T"], case["chunk"], case["offset"]
        x, rates, ph0, last, taps = make_inputs(case)
        if case.get("firdes"):
            taps = gpu.firdes_lowpass_f(T, 0.5 / D)
        res[key + "__taps"] = taps
        res[key + "__base"], res[key + "__phase"], _ = _bank(gpu, x, rates, ph0, chunk, offset, D, taps, 0, None)
        res[key + "__demod"], res[key + "__demod_phase"], res[key + "__last_out"] = _bank(gpu, x, rates, ph0, chunk, offset, D, taps, 1, last)
        sub = np.unique([0, rates.size // 2, rates.size - 1])
        res[key + "__subset"], res[key + "__subset_phase"], _ = _bank(gpu, x, rates[sub], ph0[sub], chunk, offset, D, taps, 0, None)
        n_out = n_out_of(x.size, D, T)
        if chunk > 0 and n_out >= 2:
            n1 = T + (n_out // 2) * D - 1
            o1, p1, l1 = _bank(gpu, x[:n1], rates, ph0, chunk, offset, D, taps, 1, last)
            consumed = o1.shape[1] * D
            o2, p2, l2 = _bank(gpu, x[consumed:], rates, p1, chunk, (offset + consumed) % chunk, D, taps, 1, l1)
            res[key + "__split"], res[key + "__split_phase"], res[key + "__split_last"] = np.concatenate([o1, o2], 1), p2, l2
    rates = np.linspace(-0.4999, 0.4999, 67).astype(np.float32)
    ph0 = np.random.default_rng(5).uniform(-3, 3, rates.size).astype(np.float32)
    res["probe_phase0"] = ph0
    for D, T in NONFINITE:
        x = np.ones(T + 300 * D + 3, np.complex64)
        for k in sorted({0, D - 1, T - 1}):
            taps = np.zeros(T, np.float32); taps[k] = 1.0
            res[f"probe_D{D}T{T}_k{k}"], _, _ = _bank(gpu, x, rates, ph0, 13, 12, D, taps, 0, None)
    saved = ddc_ref.nonfinite_positions
    ddc_ref.nonfinite_positions = nonfinite_positions                # this bucket's last zero-padded tap among the poisoned samples
    try:
        for D, T in NONFINITE:
            for chunk, offset in ((1024, 0), (13, 12)):
                key = f"nonfinite_D{D}T{T}_{chunk}+{offset}"
                case = dict(D=D, T=T, channels=97, chunk=chunk, offset=offset, n=T + 300 * D + 7, seed=D + T + chunk)
                runs = []

                def run(x, rates, ph0, last, taps, demod):
                    out, _, lo = _bank(gpu, x, rates, ph0, chunk, offset, D, taps, demod, last if demod else None)
                    res[f"{key}__run{len(runs)}"] = out
                    runs.append(out)
                    return out, lo
                try:
                    check_nonfinite(run, case)
                    res[key] = np.array("ok")
                except AssertionError as e:
                    res[key] = np.array(str(e))
    finally:
        ddc_ref.nonfinite_positions = saved
    return res


def run_profiled(gpu):
    """run_matrix under torch.profiler -> (results, the set of bank kernels that ran: ("generic", M, CPL, DEMOD) or ("fused2", D, M, CPL, DEMOD))"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = run_matrix(gpu)
        torch.cuda.synchronize()
    ran = set()
    for e in prof.key_averages():
        m = KERNEL_NAME.search(e.key)
        if m:
            ran.add((m.group(1),) + tuple(int(v) for v in m.group(2).split(", ")) + (m.group(3) == "true",))
    return res, ran


def digest(res):
    return {k: hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest() for k, v in res.items()}


@pytest.fixture(scope="module")
def gpu():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    if os.environ.get("CSDRB_DDC_CPL"):
        pytest.fail("run the suite without CSDRB_DDC_CPL: this module compares the default against one channel per lane itself")
    import csdr_b200
    csdr_b200.lib()
    return csdr_b200


@pytest.fixture(scope="module")
def cpl2(gpu):
    return run_profiled(gpu)


@pytest.fixture(scope="module")
def cpl1(gpu, tmp_path_factory):
    out = tmp_path_factory.mktemp("ddc_generic_cpl1")
    env = dict(os.environ, CSDRB_DDC_CPL="1")
    r = subprocess.run([sys.executable, str(Path(__file__).resolve()), "--child", str(out)], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, f"CSDRB_DDC_CPL=1 child failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    got = json.loads((out / "results.json").read_text())
    return got["digest"], {tuple(t) for t in got["kernels"]}


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_gpu_generic_ddc_bank_contract(cpl2, oracle, case):
    """reference bound, carried phase, discriminator and last_out (ddc_ref.check_against_reference); a channel subset and a two-block split give the
    full bank's bits"""
    res, _ = cpl2
    key = case_id(case)
    x, rates, ph0, last, _ = make_inputs(case)
    taps = res[key + "__taps"]
    base, phase = res[key + "__base"], res[key + "__phase"]
    check_against_reference(oracle, case, x, rates, ph0, last, taps, base, phase, res[key + "__demod"], res[key + "__demod_phase"], res[key + "__last_out"])
    sub = np.unique([0, rates.size // 2, rates.size - 1])
    assert_bits_equal(res[key + "__subset"], base[sub], "channel subset against the full bank")
    assert_bits_equal(res[key + "__subset_phase"], phase[sub], "channel subset: carried phase")
    if key + "__split" in res:
        assert_bits_equal(res[key + "__split"], res[key + "__demod"], "two blocks with the tail re-presented against one")
        assert_bits_equal(res[key + "__split_phase"], phase, "two blocks: carried phase")
        assert_bits_equal(res[key + "__split_last"], res[key + "__last_out"], "two blocks: last_out")


def test_gpu_generic_unit_tap_is_the_reference_nco(cpl2, oracle):
    """x = 1 and a single unit tap at k: output o is the host reference phasor at sample oD + k, bit for bit"""
    res, _ = cpl2
    rates = np.linspace(-0.4999, 0.4999, 67).astype(np.float32)
    ph0 = res["probe_phase0"]
    for D, T in NONFINITE:
        n = T + 300 * D + 3
        refs = [nco(oracle, r, ph0[c], 13, 12, n) for c, r in enumerate(rates)]
        for k in sorted({0, D - 1, T - 1}):
            out = res[f"probe_D{D}T{T}_k{k}"]
            for c in range(rates.size):
                assert_bits_equal(out[c], refs[c][k::D][:out.shape[1]], f"D={D} T={T} k={k} channel {c}")


@pytest.mark.parametrize("D,T", NONFINITE)
@pytest.mark.parametrize("chunk,offset", [(1024, 0), (13, 12)])
def test_gpu_generic_nonfinite_stays_in_its_windows(cpl2, D, T, chunk, offset):
    verdict = str(cpl2[0][f"nonfinite_D{D}T{T}_{chunk}+{offset}"])
    assert verdict == "ok", verdict


def test_gpu_generic_kernels_and_one_channel_per_lane(cpl2, cpl1):
    """every generic geometry ran ddc_bank_generic_kernel<M, CPL, DEMOD> of its bucket and never ddc_bank_fused2_kernel, in both runs; the
    CSDRB_DDC_CPL=1 child produced every array of the matrix with the same bits"""
    res2, ran2 = cpl2
    dig1, ran1 = cpl1
    assert all(kernel_for(c["D"], c["T"])[0] == "generic" for c in CASES)
    want = {kernel_for(c["D"], c["T"])[1] for c in CASES}
    assert want == set(BUCKETS)
    assert ran2 == {("generic", b, 2, dm) for b in BUCKETS for dm in (False, True)}, sorted(ran2)
    assert ran1 == {("generic", b, 1, dm) for b in BUCKETS for dm in (False, True)}, sorted(ran1)
    dig2 = digest(res2)
    assert sorted(dig1) == sorted(dig2)
    differ = [k for k in dig2 if dig1[k] != dig2[k]]
    assert not differ, f"CPL=1 against CPL=2 differ in {differ[:10]}"


@pytest.mark.parametrize("D,T,demod", [(200, 3201, True), (40, 641, False), (52, 1248, True), (1000, 7001, False)])
def test_gpu_generic_ddc_bank_object_equals_one_shot(gpu, D, T, demod):
    """DdcBank over blocks of several sizes (look-ahead pre-pass kept, dropped, and the scratch grown), tail re-presented, gives the bits of one
    ddc_bank call over the whole stream; (200, 3201) is DdcBank(rates, 200, firdes_lowpass_f(3201, 0.0025))"""
    rng = np.random.default_rng(D + T)
    ch, chunk = 97, 1024
    rates = np.linspace(-0.4999, 0.4999, ch).astype(np.float32)
    taps = gpu.firdes_lowpass_f(T, 0.5 / D)
    x = (rng.uniform(-1, 1, 1_200_000) + 1j * rng.uniform(-1, 1, 1_200_000)).astype(np.complex64)
    dx = _dev(x)
    bank = gpu.DdcBank(rates, D, taps, demod=demod, chunk=chunk)
    try:
        pos, outs = 0, []
        for sz in (90_000, 90_000, 51_002, 51_002, 180_008, T, T + D - 1, 90_000, 90_000):
            assert bank.offset == pos % chunk
            o = bank.process(dx[pos:pos + sz])                       # pos is a multiple of D: 16-byte aligned
            outs.append(o.cpu().numpy().copy())
            pos += o.shape[1] * D
    finally:
        bank.close()
    got = np.concatenate(outs, 1)
    whole, _, _ = gpu.ddc_bank(dx[:pos - D + T], rates, D, taps, demod=demod, chunk=chunk)
    assert_bits_equal(got, whole.cpu().numpy(), "DdcBank blocks against one call")


def test_gpu_generic_refusals(gpu):
    """odd D, M above 24 and D * MP above 8000 raise, for the one-shot call and the bank object"""
    x = torch.zeros(20_000, dtype=torch.complex64, device="cuda")
    for D, T in ((7, 79), (10, 241), (446, 7137)):
        with pytest.raises(gpu.CsdrB200Error, match="no fused kernel"):
            gpu.ddc_bank(x, np.zeros(3, np.float32), D, np.ones(T, np.float32))
        with pytest.raises(gpu.CsdrB200Error, match="no fused kernel"):
            gpu.DdcBank(np.zeros(3, np.float32), D, np.ones(T, np.float32))


if __name__ == "__main__" and sys.argv[1:2] == ["--child"]:
    sys.path.insert(0, str(ROOT))
    import csdr_b200
    csdr_b200.lib()
    results, kernels = run_profiled(csdr_b200)
    (Path(sys.argv[2]) / "results.json").write_text(json.dumps({"digest": digest(results), "kernels": sorted(kernels)}))
