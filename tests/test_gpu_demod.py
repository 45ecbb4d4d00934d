"""GPU tests (-m gpu) of the demodulator banks at full size, 1024 channels x 480 000 samples, against the compiled reference (oracle/_ref/
libcsdr_ref.so, one call per channel): dcblock_ff, amdemod_estimator_cf and fmdemod_quadri_novect_cf bit for bit (novect also on an 8-bit
receiver's repeating samples, where the sign of a zero depends on the form of its numerator), fmdemod_atan_cf bit for bit except at samples whose float64 phase lies within 4 ulp (double) of a float rounding
midpoint, where outputs k and k+1 are held to the bound of tests/demod/demod.py.  The test reports how many such samples occurred and asserts
their fraction is at most 1e-6.  Plus the Python banks' carries over calls in pieces, and the refusals on device pointers."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "demod"))
import demod as M  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
CH, N, CHUNK = 1024, 480_000, 64


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    if not M.have_ref():
        pytest.skip("oracle/_ref/libcsdr_ref.so not built")
    import csdr_b200
    return csdr_b200


def rows(seed, c0, complex_=True):
    """channels c0 .. c0 + CHUNK - 1 of the full-size input, generated per chunk so the host never holds the whole bank"""
    rng = np.random.default_rng(seed * 100003 + c0)
    x = M.complex_rows(rng, CHUNK, N) if complex_ else M.real_rows(rng, CHUNK, N)
    if complex_ and c0 == 0:
        x[0, :M.edge_row().size] = M.edge_row()
    return x


def full_bank(seed, complex_=True):
    dt = torch.complex64 if complex_ else torch.float32
    d = torch.empty((CH, N), dtype=dt, device="cuda")
    for c0 in range(0, CH, CHUNK):
        d[c0:c0 + CHUNK] = torch.from_numpy(rows(seed, c0, complex_)).cuda()
    return d


def test_atan_bank_under_the_rounding_rule(pkg):
    x = full_bank(1)
    y, last = pkg.fmdemod_atan_bank_cf(x, return_last=True)
    torch.cuda.synchronize()
    near = diff = 0
    for c0 in range(0, CH, CHUNK):
        h = rows(1, c0)
        got = y[c0:c0 + CHUNK].cpu().numpy()
        lo = last[c0:c0 + CHUNK].cpu().numpy()
        for c in range(CHUNK):
            want, wlast = M.ref_atan(h[c])
            a, b = M.atan_matches(got[c], want, h[c])
            near += a; diff += b
            assert lo[c] == wlast or (np.isnan(lo[c]) and np.isnan(wlast)) or M.atan_near_midpoint(h[c, -1:])[0], (c0 + c, lo[c], wlast)
    frac = near / (CH * N)
    print(f"fmdemod_atan bank: {near} of {CH * N} samples within 4 ulp (double) of a float rounding midpoint ({frac:.2e}), {diff} outputs differ")
    assert frac <= 1e-6, frac


def test_estimator_and_novect_banks_equal_the_reference(pkg):
    x = full_bank(2)
    est = pkg.amdemod_estimator_bank_cf(x)
    est2 = pkg.amdemod_estimator_bank_cf(x, 0.75, 0.25)
    nov = pkg.fmdemod_quadri_novect_bank_cf(x)
    torch.cuda.synchronize()
    for c0 in range(0, CH, 4 * CHUNK):                                # every fourth chunk: the reference's scalar loops are slow on 5e8 samples
        h = rows(2, c0)
        e, e2, nv = est[c0:c0 + CHUNK].cpu().numpy(), est2[c0:c0 + CHUNK].cpu().numpy(), nov[c0:c0 + CHUNK].cpu().numpy()
        for c in range(CHUNK):
            assert M.same_bits(e[c], M.ref_estimator(h[c])), c0 + c
            assert M.same_bits(e2[c], M.ref_estimator(h[c], 0.75, 0.25)), c0 + c
            assert M.same_bits(nv[c], M.ref_novect(h[c])[0]), c0 + c
    q = M.quantised_rows(np.random.default_rng(5), CHUNK, 100_001)
    nq = pkg.fmdemod_quadri_novect_bank_cf(torch.from_numpy(q).cuda()).cpu().numpy()
    for c in range(CHUNK):
        assert M.same_bits(nq[c], M.ref_novect(q[c])[0]), c


def test_dcblock_bank_equals_the_reference(pkg):
    x = full_bank(3, complex_=False)
    y, st = pkg.dcblock_bank_ff(x, return_state=True)
    ya = pkg.dcblock_bank_ff(x, a=0.95)
    torch.cuda.synchronize()
    for c0 in range(0, CH, 4 * CHUNK):
        h = rows(3, c0, complex_=False)
        g, ga, s = y[c0:c0 + CHUNK].cpu().numpy(), ya[c0:c0 + CHUNK].cpu().numpy(), st[c0:c0 + CHUNK].cpu().numpy()
        for c in range(CHUNK):
            want, wst = M.ref_dcblock(h[c])
            assert M.same_bits(g[c], want) and M.same_bits(s[c], np.array(wst, np.float32)), c0 + c
            assert M.same_bits(ga[c], M.ref_dcblock(h[c], 0.95)[0]), c0 + c


def test_carries_over_calls_in_pieces(pkg):
    """the Python banks' carries: pieces of a stream give the bits of one call; dcblock in place gives what separate buffers give"""
    rng = np.random.default_rng(4)
    x = torch.from_numpy(M.complex_rows(rng, 300, 20011)).cuda()
    r = torch.from_numpy(M.real_rows(rng, 300, 20011)).cuda()
    whole_a, whole_n, whole_d = pkg.fmdemod_atan_bank_cf(x), pkg.fmdemod_quadri_novect_bank_cf(x), pkg.dcblock_bank_ff(r, 0.9)
    la = ln = sd = None
    pa, pn, pd = [], [], []
    for a, b in ((0, 1), (1, 1024), (1024, 7777), (7777, 20011)):
        ya, la = pkg.fmdemod_atan_bank_cf(x[:, a:b], last=la, return_last=True)
        yn, ln = pkg.fmdemod_quadri_novect_bank_cf(x[:, a:b], last=ln, return_last=True)
        yd, sd = pkg.dcblock_bank_ff(r[:, a:b].contiguous(), 0.9, state=sd, return_state=True)
        pa.append(ya); pn.append(yn); pd.append(yd)
    for whole, parts in ((whole_a, pa), (whole_n, pn), (whole_d, pd)):
        assert M.same_bits(torch.cat(parts, 1).cpu().numpy(), whole.cpu().numpy())
    buf = r.clone()
    pkg.dcblock_bank_ff(buf, 0.9, out=buf)
    assert M.same_bits(buf.cpu().numpy(), whole_d.cpu().numpy())


def test_python_banks_refuse_carries_they_cannot_pass_as_device_rows(pkg):
    """a carry or output that is not a contiguous CUDA tensor of the right dtype and shape is refused before any pointer reaches the device"""
    x = torch.zeros((3, 100), dtype=torch.complex64, device="cuda")
    r = torch.zeros((3, 100), device="cuda")
    for last in (torch.zeros(3), torch.zeros(3, dtype=torch.float64, device="cuda"), torch.zeros(4, device="cuda"),
                 torch.zeros(6, device="cuda")[::2], [0.0, 0.0, 0.0]):
        with pytest.raises(ValueError):
            pkg.fmdemod_atan_bank_cf(x, last=last)
    for last in (torch.zeros(3, dtype=torch.complex64), torch.zeros(3, device="cuda"), torch.zeros(2, dtype=torch.complex64, device="cuda")):
        with pytest.raises(ValueError):
            pkg.fmdemod_quadri_novect_bank_cf(x, last=last)
    for state in (torch.zeros((3, 2)), torch.zeros((3, 2), dtype=torch.float64, device="cuda"), torch.zeros((2, 3), device="cuda"),
                  torch.zeros((2, 3), device="cuda").t(), torch.zeros(6, device="cuda")):
        with pytest.raises(ValueError):
            pkg.dcblock_bank_ff(r, state=state)
    for out in (torch.zeros((3, 100)), torch.zeros((3, 100), dtype=torch.float64, device="cuda"), torch.zeros((3, 99), device="cuda"),
                torch.zeros((100, 3), device="cuda").t()):
        with pytest.raises(ValueError):
            pkg.dcblock_bank_ff(r, out=out)
        with pytest.raises(ValueError):
            pkg.amdemod_estimator_bank_cf(x, out=out)
        with pytest.raises(ValueError):
            pkg.fmdemod_atan_bank_cf(x, out=out)
    with pytest.raises(ValueError):
        pkg.dcblock_bank_ff(r.double())


def test_refusals_on_device_pointers(pkg):
    L = M.bind(pkg.lib())
    d_cf = torch.zeros(64, dtype=torch.complex64, device="cuda")
    d_f = torch.zeros(512, dtype=torch.float32, device="cuda")
    d_state = torch.zeros(16, dtype=torch.float32, device="cuda")
    assert M.refusals(L, d_cf.data_ptr(), d_f.data_ptr(), d_state.data_ptr()) == []
