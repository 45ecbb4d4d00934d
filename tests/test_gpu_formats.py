"""GPU tests (-m gpu) of the sample-format kernels (csdr_b200/csrc/elementwise.cu) on the H100, bit for bit against the restatements of
tests/formats/formats.py and the compiled reference: all 256 s8 codes, all 2^24 s24 codes in both byte orders, every truncation boundary of
every s8, u8 and s24 code with the wrap region, +-0, subnormals, |s| at 2^31, +-Inf and NaN; lengths 1..40 at odd offsets; the refusals; the
torch functions and the drop-ins."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "formats"))
import formats as M  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
CASES = [(k, be) for k in M.KINDS for be in ((0, 1) if M.KINDS[k][2] else (0,))]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    return M.CudaDev()


@pytest.mark.parametrize("kind,bigendian", CASES)
def test_every_code_and_boundary(dev, kind, bigendian):
    M.check_against(dev, kind, M.inputs(kind, np.random.default_rng(11), full=True), bigendian, with_ref=M.have_ref())


@pytest.mark.parametrize("kind,bigendian", CASES)
def test_lengths_and_offsets(dev, kind, bigendian):
    rng = np.random.default_rng(12)
    x = M.inputs(kind, rng)
    item = M.KINDS[kind][0]
    x = np.concatenate([x[:20], rng.permutation(x)[:20]]) if item == 4 else rng.permutation(x.reshape(-1, item))[:40].reshape(-1)
    M.check_lengths_and_offsets(dev, kind, x, bigendian, with_ref=M.have_ref())


def test_refusals_launch_nothing(dev):
    assert M.refusals(dev) == []


def test_torch_functions_and_dropins():
    import csdr_b200
    rng = np.random.default_rng(13)
    x = M.float_inputs("f_s24", rng)
    b8 = M.byte_inputs("s8_f", rng)
    b24 = M.byte_inputs("s24_f", rng)
    xt = torch.from_numpy(x).cuda()
    assert M.same(csdr_b200.convert_s8_f(torch.from_numpy(b8.view(np.int8)).cuda()).cpu().numpy(), M.s8_f(b8.view(np.int8)))
    assert M.same(csdr_b200.convert_f_s8(xt).cpu().numpy(), M.f_s8(x))
    assert M.same(csdr_b200.convert_f_u8(xt).cpu().numpy(), M.f_u8(x))
    for be in (False, True):
        assert M.same(csdr_b200.convert_f_s24(xt, bigendian=be).cpu().numpy(), M.f_s24(x, be))
        assert M.same(csdr_b200.convert_s24_f(torch.from_numpy(b24).cuda(), bigendian=be).cpu().numpy(), M.s24_f(b24, be))
        assert M.same(csdr_b200.libcsdr.convert_f_s24(x, be), M.f_s24(x, be))
        assert M.same(csdr_b200.libcsdr.convert_s24_f(b24, be), M.s24_f(b24, be))
    assert M.same(csdr_b200.libcsdr.convert_s8_f(b8.view(np.int8)), M.s8_f(b8.view(np.int8)))
    assert M.same(csdr_b200.libcsdr.convert_f_s8(x), M.f_s8(x))
    assert M.same(csdr_b200.libcsdr.convert_f_u8(x), M.f_u8(x))
    torch.cuda.synchronize()
