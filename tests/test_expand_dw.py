"""The fused MnasNet expansion + depthwise launch (ops.expand_dwconv, csrc/expand_dw.cu) against its two-launch composition:
conv2d_tc of the 1x1 expansion (fp32 output) followed by dwconv2d (fp16 pair planes).  Equal bit for bit, for every trunk
block shape of FeatureExtractor, on ragged maps, at batch 1 / 3 / 12, with 1-term and 3-term operands; and the whole
FeatureExtractor equals its two-launch form."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _bn(c, gen):
    bn = torch.nn.BatchNorm2d(c)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=gen) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=gen) * 0.2)
        bn.running_mean.copy_(torch.randn(c, generator=gen) * 0.1)
        bn.running_var.copy_(torch.rand(c, generator=gen) + 0.5)
    return bn.eval()


def _block(cin, mid, k, stride, seed):
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    gen = torch.Generator().manual_seed(seed)
    we = torch.randn(mid, cin, 1, 1, generator=gen) * (2.0 / cin) ** 0.5
    wd = torch.randn(mid, 1, k, k, generator=gen) * (2.0 / (k * k)) ** 0.5
    expand = ops.ConvLayer(ops.PackedConv(we.to(DEV), None, _bn(mid, gen).to(DEV), act=N.ACT_RELU))
    dw = ops.PackedDepthwise(wd.to(DEV), _bn(mid, gen).to(DEV), stride=stride)
    return expand, dw


def _trunk_shapes():
    """(cin, mid, k, stride, input map side) of the 16 inverted-residual blocks at the engines' 256 x 256 input, deduplicated"""
    from dvmvs._blocks import FeatureExtractor
    fe = FeatureExtractor()
    shapes, side = [], 128
    for layer in (fe.layer2, fe.layer3, fe.layer4, fe.layer5):
        for stack in layer:
            for blk in stack:
                L = blk.layers
                s = (L[0].in_channels, L[0].out_channels, L[3].kernel_size[0], blk.stride, side)
                if s not in shapes:
                    shapes.append(s)
                side //= blk.stride
    return shapes


SHAPES = _trunk_shapes()


def _check(expand, dw, B, H, W, cin, terms, seed):
    from dvmvs import _ops as ops
    gen = torch.Generator().manual_seed(seed)
    x = ops.Act(ops.to_nhwc((torch.randn(B, cin, H, W, generator=gen)).to(DEV)))
    with torch.no_grad():
        fused = ops.expand_dwconv(x, expand, dw, terms)
        ptc = ops.PackedConvTC(expand.pc, [cin], DEV)
        mid_f32, _ = ops.conv2d_tc([x.get_planes()], ptc, terms=terms, want_f32=True, want_planes=False)
        _, ref = ops.dwconv2d(mid_f32, dw, want_f32=False, want_planes=True)
    assert fused.shape == ref.shape
    assert torch.equal(fused[0], ref[0])
    if terms == 3:
        assert torch.equal(fused[1], ref[1])


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("B", [1, 3, 12])
@pytest.mark.parametrize("shape", SHAPES, ids=["%d-%d-k%d-s%d-%d" % s for s in SHAPES])
def test_expand_dw_trunk_shapes(shape, B, terms):
    cin, mid, k, stride, side = shape
    expand, dw = _block(cin, mid, k, stride, seed=cin * 7 + k)
    _check(expand, dw, B, side, side, cin, terms, seed=B * 31 + terms)


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("hw", [(17, 15), (9, 8)])
@pytest.mark.parametrize("shape", SHAPES, ids=["%d-%d-k%d-s%d" % s[:4] for s in SHAPES])
def test_expand_dw_ragged_maps(shape, hw, terms):
    cin, mid, k, stride, _ = shape
    expand, dw = _block(cin, mid, k, stride, seed=cin * 5 + k)
    _check(expand, dw, 3, hw[0], hw[1], cin, terms, seed=hw[0] + terms)


def test_expand_dw_rejects_unsupported_shapes():
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    expand, dw = _block(24, 72, 3, 1, seed=1)
    ptc = ops.PackedConvTC(expand.pc, [24], DEV)
    x = torch.zeros((2, 1, 16, 16, 24), dtype=torch.float16, device=DEV)
    y = torch.empty((2, 1, 16, 16, 72), dtype=torch.float16, device=DEV)

    def call(ksize=3, stride=1, mid=72, terms=1, cs=24, ktot=ptc.ktot):
        return N.lib().dvmvs_expand_dwconv(x.data_ptr(), 1, 16, 16, cs, ptc.w_hi.data_ptr(), ptc.w_lo.data_ptr(), ptc.rows, ktot,
                                           ptc.bias.data_ptr(), N.ACT_RELU, dw.weight.data_ptr(), dw.bias.data_ptr(), ksize, stride,
                                           N.ACT_RELU, mid, terms, 0, y.data_ptr(), ops._stream())
    assert call() == 0
    torch.cuda.synchronize()
    for bad in ({"ksize": 7}, {"stride": 3}, {"mid": 76}, {"terms": 2}, {"cs": 20}, {"ktot": 64}):
        assert call(**bad) != 0, bad


def _two_launch_run(fe, x):
    """FeatureExtractor.run(part="all") on the CUDA-core stem, with every block's front half as conv2d_tc + dwconv2d"""
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    stem, levels = fe.packed()

    def depthwise(t, dw):
        return ops.Act(None, ops.dwconv2d(t.f32, dw, want_f32=False, want_planes=True)[1])

    x = stem[2].run([(depthwise(stem[0].run([(x, N.SRC_DIRECT)]), stem[1]), N.SRC_DIRECT)])
    outs = [x]
    for blocks in levels:
        for expand, dw, project, residual in blocks:
            y = depthwise(expand.run([(x, N.SRC_DIRECT)], want_planes=False), dw)
            x = project.run([(y, N.SRC_DIRECT)], residual=x if residual else None,
                            residual_mode=N.RES_SAME if residual else N.RES_NONE)
        outs.append(x)
    return outs


@pytest.mark.parametrize("terms", [1, 3])
def test_feature_extractor_equals_two_launch_form(terms):
    from dvmvs import _ops as ops
    from dvmvs._blocks import FeatureExtractor
    old = (ops._BACKEND, ops._TC_TERMS)
    ops.set_conv_backend("tc", terms=terms)
    try:
        torch.manual_seed(3)
        fe = FeatureExtractor()
        gen = torch.Generator().manual_seed(4)
        for m in fe.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.load_state_dict(_bn(m.num_features, gen).state_dict())
        fe = fe.to(DEV).eval()
        image = torch.randn(3, 3, 256, 256, generator=gen).to(DEV)
        with torch.no_grad():
            x = ops.Act(ops.to_nhwc(image))
            fused = fe.run(x)
            ref = _two_launch_run(fe, x)
        assert len(fused) == len(ref) == 5
        for a, b in zip(fused, ref):
            assert torch.equal(a.f32, b.f32)
    finally:
        ops.set_conv_backend(old[0], terms=old[1])
