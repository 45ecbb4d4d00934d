"""GPU tier of the fused DDC bank contract (-m gpu): the case matrix of tests/ddc_ref.py at larger sizes, through csdr_b200.ddc_bank / DdcBank.

Every output is within the per-output error bound of the float64 reference, the NCO is the host reference's bit for bit, the discriminator is
fmdemod_quadri_cf on the bank's own baseband bit for bit, and the bits do not depend on the channels per lane, the channel subset, the block split
or the DdcBank block sizes (DESIGN.md 8b).  One channel per lane (CSDRB_DDC_CPL=1) is fixed when the library first launches a bank kernel, so a
child process runs the whole matrix with it and hands its outputs back through files; the kernels the child launched are listed with
torch.profiler, whose kernel names carry the template arguments <D, M, CPL, DEMOD>.

Run directly (python tests/test_gpu_ddc_bank.py --child DIR), this file is that child.
"""
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
from ddc_ref import (KERNELS, NONFINITE, assert_bits_equal, case_id, cases, check_against_reference, check_nonfinite, make_inputs, n_out_of,  # noqa: E402
                     nco)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SENTINEL = np.uint32(0x7FC0DEAD)                                     # a NaN the kernel never produces: padding must keep it
EXTRA = [dict(D=50, T=801, channels=700, chunk=1024, offset=100, n=801 + 59 * 50 + 10, seed=11),          # several hundred channels, short segments:
         dict(D=10, T=199, channels=1000, chunk=7, offset=3, n=199 + 99 * 10 + 5, seed=12),                 # every segment at the 2M-output floor
         dict(D=10, T=79, channels=513, chunk=1000, offset=999, n=79 + 150 * 10 + 9, seed=13),
         dict(D=50, T=801, channels=129, chunk=1024, offset=0, n=801 + 3999 * 50 + 17, seed=14, firdes=True),  # the product's taps, a long block
         dict(D=10, T=199, channels=97, chunk=1024, offset=517, n=199 + 5000 * 10 + 3, seed=15, firdes=True),
         dict(D=10, T=79, channels=65, chunk=1000, offset=999, n=79 + 3000 * 10 + 1, seed=16, firdes=True)]
CASES = cases(large=2000, extra=EXTRA)
PROBE_CHUNKS = [(1024, 0), (7, 3), (13, 12)]
PROBE_T = {(50, 17): 801, (10, 8): 80, (10, 20): 199}
PROBE_K = (0, 3, 9, 79)
PROBE_RATES = np.linspace(-0.4999, 0.4999, 67).astype(np.float32)
KERNEL_NAME = re.compile(r"ddc_bank_fused2_kernel<(\d+), (\d+), (\d+), (true|false)>")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _taps(gpu, case, rng_taps):
    return gpu.firdes_lowpass_f(case["T"], 0.5 / case["D"]) if case.get("firdes") else rng_taps


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
    """every case (both DEMOD kernels, a 3-channel subset, a two-block split) and the unit-tap NCO probes -> {name: array}"""
    res = {}
    for case in CASES:
        key = case_id(case)
        D, T, chunk, offset = case["D"], case["T"], case["chunk"], case["offset"]
        x, rates, ph0, last, taps = make_inputs(case)
        taps = res[key + "__taps"] = _taps(gpu, case, taps)
        res[key + "__base"], res[key + "__phase"], _ = _bank(gpu, x, rates, ph0, chunk, offset, D, taps, 0, None)
        res[key + "__demod"], res[key + "__demod_phase"], res[key + "__last_out"] = _bank(gpu, x, rates, ph0, chunk, offset, D, taps, 1, last)
        sub = np.unique([0, rates.size // 2, rates.size - 1])
        res[key + "__subset"], res[key + "__subset_phase"], _ = _bank(gpu, x, rates[sub], ph0[sub], chunk, offset, D, taps, 0, None)
        n_out = n_out_of(x.size, D, T)
        if chunk > 0 and n_out >= 2:                                 # chunk = 0 means "one chunk per call": a split changes the NCO by definition
            n1 = T + (n_out // 2) * D - 1
            o1, p1, l1 = _bank(gpu, x[:n1], rates, ph0, chunk, offset, D, taps, 1, last)
            consumed = o1.shape[1] * D
            o2, p2, l2 = _bank(gpu, x[consumed:], rates, p1, chunk, (offset + consumed) % chunk, D, taps, 1, l1)
            res[key + "__split"], res[key + "__split_phase"], res[key + "__split_last"] = np.concatenate([o1, o2], 1), p2, l2
    ph0 = np.random.default_rng(5).uniform(-3, 3, PROBE_RATES.size).astype(np.float32)
    for chunk, offset in PROBE_CHUNKS:
        for (D, M), T in PROBE_T.items():
            x = np.ones(T + 300 * D + 3, np.complex64)
            for k in PROBE_K:
                taps = np.zeros(T, np.float32); taps[k] = 1.0
                res[f"probe_{chunk}+{offset}_D{D}T{T}_k{k}"], _, _ = _bank(gpu, x, PROBE_RATES, ph0, chunk, offset, D, taps, 0, None)
    res["probe_phase0"] = ph0
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
    return res


def run_profiled(gpu):
    """run_matrix under torch.profiler -> (results, the set of (D, M, CPL, DEMOD) bank kernels that ran)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = run_matrix(gpu)
        torch.cuda.synchronize()
    ran = set()
    for e in prof.key_averages():
        m = KERNEL_NAME.search(e.key)
        if m:
            ran.add((int(m.group(1)), int(m.group(2)), int(m.group(3)), m.group(4) == "true"))
    return res, ran


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
    out = tmp_path_factory.mktemp("ddc_cpl1")
    env = dict(os.environ, CSDRB_DDC_CPL="1")
    r = subprocess.run([sys.executable, str(Path(__file__).resolve()), "--child", str(out)], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"CSDRB_DDC_CPL=1 child failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    with np.load(out / "results.npz") as z:
        res = {k: z[k] for k in z.files}
    return res, {tuple(t) for t in json.loads((out / "kernels.json").read_text())}


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_gpu_fused_ddc_bank_contract(cpl2, oracle, case):
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


def test_gpu_unit_tap_is_the_reference_nco(cpl2, oracle):
    """x = 1 and a single unit tap at k: output o is the host reference phasor at sample oD + k, bit for bit.  The chunk seeds come from device
    double cos / sin rounded to float, the host's from the C library's; both are the correctly rounded float in all but ~2^-29 of the cases, and
    this test pins that they agree here."""
    res, _ = cpl2
    ph0 = res["probe_phase0"]
    for chunk, offset in PROBE_CHUNKS:
        for (D, M), T in PROBE_T.items():
            n = T + 300 * D + 3
            refs = [nco(oracle, r, ph0[c], chunk, offset, n) for c, r in enumerate(PROBE_RATES)]
            for k in PROBE_K:
                out = res[f"probe_{chunk}+{offset}_D{D}T{T}_k{k}"]
                for c in range(PROBE_RATES.size):
                    assert_bits_equal(out[c], refs[c][k::D][:out.shape[1]], f"chunk {chunk}+{offset} D={D} T={T} k={k} channel {c}")


def test_gpu_one_channel_per_lane_gives_the_same_bits(cpl2, cpl1):
    """CSDRB_DDC_CPL=1 (child process) against the default two channels per lane: every array of the matrix bit for bit, and each run launched
    all six <D, M, CPL, DEMOD> kernels of its CPL and none of the other"""
    res2, ran2 = cpl2
    res1, ran1 = cpl1
    assert ran1 == {(D, M, 1, dm) for D, M in KERNELS for dm in (False, True)}, sorted(ran1)
    assert ran2 == {(D, M, 2, dm) for D, M in KERNELS for dm in (False, True)}, sorted(ran2)
    assert sorted(res1) == sorted(res2)
    for k in res2:
        assert_bits_equal(res1[k], res2[k], f"CPL=1 against CPL=2: {k}")


@pytest.mark.parametrize("D,T", NONFINITE)
@pytest.mark.parametrize("chunk,offset", [(1024, 0), (13, 12)])
def test_gpu_ddc_bank_nonfinite_stays_in_its_windows(cpl2, D, T, chunk, offset):
    """NaN / +-Inf wideband samples reach exactly the outputs whose window holds them, both DEMOD kernels (ddc_ref.check_nonfinite); the
    one-channel-per-lane child ran the same calls, and test_gpu_one_channel_per_lane_gives_the_same_bits compares its outputs"""
    verdict = str(cpl2[0][f"nonfinite_D{D}T{T}_{chunk}+{offset}"])
    assert verdict == "ok", verdict


@pytest.mark.parametrize("D,T,demod", [(50, 801, True), (10, 199, False), (10, 79, True)])
def test_gpu_ddc_bank_object_equals_one_shot(gpu, D, T, demod):
    """DdcBank over blocks of several sizes (look-ahead pre-pass kept, dropped, and the scratch grown), tail re-presented, gives the bits of one
    ddc_bank call over the whole stream"""
    rng = np.random.default_rng(D + T)
    ch, chunk = 97, 1024
    rates = np.linspace(-0.4999, 0.4999, ch).astype(np.float32)
    taps = gpu.firdes_lowpass_f(T, 0.5 / D)
    x = (rng.uniform(-1, 1, 400_000) + 1j * rng.uniform(-1, 1, 400_000)).astype(np.complex64)
    dx = _dev(x)
    bank = gpu.DdcBank(rates, D, taps, demod=demod, chunk=chunk)
    try:
        pos, outs = 0, []
        for sz in (30_000, 30_000, 17_001, 17_001, 60_007, T, T + D - 1, 30_000, 30_000):
            assert bank.offset == pos % chunk
            o = bank.process(dx[pos:pos + sz])                       # pos is a multiple of D: 16-byte aligned
            outs.append(o.cpu().numpy().copy())
            pos += o.shape[1] * D
    finally:
        bank.close()
    got = np.concatenate(outs, 1)
    whole, _, _ = gpu.ddc_bank(dx[:pos - D + T], rates, D, taps, demod=demod, chunk=chunk)
    assert_bits_equal(got, whole.cpu().numpy(), "DdcBank blocks against one call")


if __name__ == "__main__" and sys.argv[1:2] == ["--child"]:
    sys.path.insert(0, str(ROOT))
    import csdr_b200
    csdr_b200.lib()
    results, kernels = run_profiled(csdr_b200)
    out_dir = Path(sys.argv[2])
    np.savez(out_dir / "results.npz", **results)
    (out_dir / "kernels.json").write_text(json.dumps(sorted(kernels)))
