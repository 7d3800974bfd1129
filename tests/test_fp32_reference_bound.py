"""The bounds and rules of tests/fp32_reference.py are honest and not vacuous (no GPU needed): fp32 emulations of the upsampling,
stem, depthwise and depth-head kernels, operation for operation, pass; each planted defect fails.  Also measures the upsampling
constants (C_UP_POS, C_UP_BLEND >= 8x the worst measured)."""
import numpy as np
import pytest
import torch

from tests import fp32_reference as R
from tests.tc_reference import ACT_RELU, ACT_SIGMOID, U, check


def _rand(shape, seed, scale=1.0):
    return (np.random.RandomState(seed).randn(*shape) * scale).astype(np.float32)


def _nchw(a):
    return torch.from_numpy(np.ascontiguousarray(a)).permute(0, 3, 1, 2)


UP_SHAPES = [(2, 5, 7, 3), (1, 8, 8, 16), (1, 64, 64, 1), (1, 17, 9, 4)]


@pytest.mark.parametrize("shape", UP_SHAPES)
def test_upsample_emulation_within_bound(shape):
    x = _rand(shape, sum(shape))
    y, b = R.upsample_reference(_nchw(x))
    print("upsample %s err/bound %.3f" % (shape, check("upsample", _nchw(R.emulate_upsample(x)), y, b)[0]))


def test_upsample_constants():
    """the worst err / (u (max |tap| + (H + W - 2) range)) of the emulation: both constants are >= 8x it"""
    worst = 0.0
    saved = R.C_UP_POS, R.C_UP_BLEND
    for shape in UP_SHAPES:
        x = _rand(shape, sum(shape))
        try:
            R.C_UP_POS, R.C_UP_BLEND = 1.0, 1.0
            y, unit = R.upsample_reference(_nchw(x))
        finally:
            R.C_UP_POS, R.C_UP_BLEND = saved
        err = (_nchw(R.emulate_upsample(x)).double() - y).abs()
        worst = max(worst, float((err / unit.clamp_min(1e-300)).max()))
    print("upsample: worst err / (u (max|tap| + (H+W-2) range)) = %.3f (C_UP_POS = %g, C_UP_BLEND = %g)" % (worst, R.C_UP_POS, R.C_UP_BLEND))
    assert worst * 8 <= min(R.C_UP_POS, R.C_UP_BLEND)


def test_upsample_defect_rejected():
    x = _rand((1, 6, 9, 4), 3)
    y, b = R.upsample_reference(_nchw(x))
    with pytest.raises(AssertionError):
        check("upsample last_row_clamp", _nchw(R.emulate_upsample(x, "last_row_clamp")), y, b)


@pytest.mark.parametrize("variant", [None, "pad0"])
def test_stem(variant):
    img = _rand((2, 3, 15, 13), 1)
    w, b = _rand((3, 3, 3, 32), 2, 0.3), _rand((32,), 3, 0.1)
    ref = R.stem_reference(torch.from_numpy(img), torch.from_numpy(w), torch.from_numpy(b))
    got = _nchw(R.emulate_stem(img, w, b, variant))
    if variant is None:
        print("stem err/bound %.3f" % check("stem", got, ref.y, ref.bound)[0])
    else:
        with pytest.raises(AssertionError):
            check("stem " + variant, got, ref.y, ref.bound)


@pytest.mark.parametrize("variant", [None, "stride_y_only"])
def test_dwconv(variant):
    x = _rand((1, 9, 11, 8), 4)
    w, b = _rand((5, 5, 8), 5, 0.3), _rand((8,), 6, 0.1)
    ref = R.dwconv_reference(_nchw(x), torch.from_numpy(w), torch.from_numpy(b), 2, ACT_RELU)
    got = R.emulate_dwconv(x, w, b, 2, ACT_RELU, variant)
    if variant is None:
        print("dwconv err/bound %.3f" % check("dwconv", _nchw(got), ref.y, ref.bound)[0])
    else:
        with pytest.raises(AssertionError):
            check("dwconv " + variant, _nchw(got), ref.y, ref.bound)


@pytest.mark.parametrize("variant", [None, "no_bias", "aux_pre_activation"])
@pytest.mark.parametrize("lanes", [8, 32])
def test_head(lanes, variant):
    x = _rand((1, 6, 7, 128), 7)
    w, b = _rand((3, 3, 128, 1), 8, (2.0 / (9 * 128)) ** 0.5), _rand((1,), 9, 0.5)
    aux = (3.9, 0.05)
    ref = R.conv_reference([(_nchw(x), False)], torch.from_numpy(w), 1, torch.from_numpy(b), act=ACT_SIGMOID, aux=aux,
                           chain=3 * 128 // lanes + 2 + int(np.log2(lanes)))
    y, a = R.emulate_head(x, w, b, ACT_SIGMOID, aux, lanes, variant)

    def run():
        w1 = check("head", _nchw(y), ref.y, ref.bound)[0]
        w2 = check("head aux", _nchw(a), ref.aux, ref.aux_bound)[0]
        return max(w1, w2)
    if variant is None:
        print("head<%d> err/bound %.3f" % (lanes, run()))
    else:
        with pytest.raises(AssertionError):
            run()


def _staged(x, c_offset, c_cover, Cs, variant=None):
    """an emulated split_planes call into a sentinel-filled (…, Cs) plane pair"""
    sentinel = torch.tensor(7.0).half().view(torch.int16)
    hi = torch.full(x.shape[:-1] + (Cs,), 7.0).half()
    lo = hi.clone()
    eh, el = R.emulate_split(x, "lo_without_fp32_subtraction" if variant == "lo" else None)
    C = x.shape[-1]
    cover = c_cover + (1 if variant == "past_cover" else 0)
    hi[..., c_offset:c_offset + cover] = 0
    lo[..., c_offset:c_offset + cover] = 0
    hi[..., c_offset:c_offset + C], lo[..., c_offset:c_offset + C] = eh, el
    return hi, lo, sentinel


@pytest.mark.parametrize("variant", [None, "lo", "past_cover"])
def test_staging_rules(variant):
    x = _rand((2, 3, 5, 12), 10)
    hi, lo, sentinel = _staged(x, 8, 16, 32, variant)
    if variant is None:
        R.check_staged("staging", hi, lo, torch.from_numpy(x), 8, 16, sentinel)
    else:
        with pytest.raises(AssertionError):
            R.check_staged("staging " + variant, hi, lo, torch.from_numpy(x), 8, 16, sentinel)
