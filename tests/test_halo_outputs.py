"""Output pruning on the halo path of ConvLayer.run: each want_* flag yields exactly the requested outputs, bit for bit
what the unpruned launch writes, and a layer reads a blocked-planes-only activation as its source."""
import pytest
import torch

from tests.helpers import T

pytestmark = pytest.mark.gpu

DEV = "cuda"
FLAGS = [  # want_f32, want_planes, want_blk
    (True, False, False),
    (False, False, True),
    (False, True, False),
    (True, True, False),
    (False, True, True),
]


def _layer(synth, name, cin, cout, k):
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    w = T(synth.tensor("halo_out/%s/w" % name, (cout, cin, k, k), seed=2, scale=(2.0 / (cin * k * k)) ** 0.5)).to(DEV)
    b = T(synth.tensor("halo_out/%s/b" % name, (cout,), seed=3, scale=0.1)).to(DEV)
    return ops.ConvLayer(ops.PackedConv(w, b, None, stride=1, act=N.ACT_RELU))


@pytest.mark.parametrize("terms", [1, 3])
def test_halo_output_flags(synth, terms):
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    old = (ops._BACKEND, ops._TC_TERMS)
    ops.set_conv_backend("tc", terms=terms)
    try:
        B, H, W, C = 1, 72, 80, 32                                  # ragged in both tile directions
        x = ops.Act(ops.to_nhwc(T(synth.tensor("halo_out/x", (B, C, H, W), seed=1)).to(DEV)))
        c1, c2 = _layer(synth, "c1", C, 32, 5), _layer(synth, "c2", 32, 32, 5)
        assert c1.path(H, W) == "halo" and c2.path(H, W) == "halo"
        with torch.no_grad():
            full = c1.run([(x, N.SRC_DIRECT)])
            assert full.f32 is not None and full.planes is not None and full.blk is not None
            for want_f32, want_planes, want_blk in FLAGS:
                y = c1.run([(x, N.SRC_DIRECT)], want_f32=want_f32, want_planes=want_planes, want_blk=want_blk)
                assert (y.f32 is not None, y.planes is not None, y.blk is not None) == (want_f32, want_planes, want_blk)
                planes = 2 if terms == 3 else 1                     # 1-term operands: only the hi plane is written
                if want_f32:
                    assert torch.equal(y.f32, full.f32)
                if want_planes:
                    assert torch.equal(y.planes[:planes], full.planes[:planes])
                if want_blk:
                    assert torch.equal(y.blk[:planes], full.blk[:planes])
            # the next halo layer reads the blocked planes of an activation that carries nothing else
            ref = c2.run([(full, N.SRC_DIRECT)])
            blk_only = c1.run([(x, N.SRC_DIRECT)], want_f32=False, want_planes=False)
            out = c2.run([(blk_only, N.SRC_DIRECT)], want_planes=False, want_blk=False)
            assert out.planes is None and out.blk is None
            assert torch.equal(out.f32, ref.f32)
    finally:
        ops.set_conv_backend(old[0], terms=old[1])


@pytest.mark.parametrize("upsample", [False, True])
def test_split_blocked_hi_only_flag(synth, upsample):
    """SPLIT_HI_ONLY writes the same hi plane as the full split and leaves the lo plane untouched."""
    from dvmvs import _native as N
    from dvmvs import _ops as ops
    B, H, W, C = 2, 24, 40, 20
    x = ops.to_nhwc(T(synth.tensor("halo_out/split_x", (B, C, H, W), seed=5)).to(DEV))
    f = 2 if upsample else 1
    C8 = (C + 7) // 8
    full = ops.split_blocked([(x, upsample)])
    sentinel = torch.full((2, B, C8, H * f, W * f, 8), 7.0, dtype=torch.float16, device=DEV)
    flags = (N.SPLIT_UPSAMPLE2X if upsample else 0) | N.SPLIT_HI_ONLY
    N.check(N.lib().dvmvs_split_blocked(x.data_ptr(), sentinel.data_ptr(), B, H, W, C, C8, flags, 0, C8 * 8, ops._stream()), "split_blocked")
    torch.cuda.synchronize()
    assert torch.equal(sentinel[0], full[0])
    assert bool((sentinel[1] == 7.0).all())
    assert N.lib().dvmvs_split_blocked(x.data_ptr(), sentinel.data_ptr(), B, H, W, C, C8, 4, 0, C8 * 8, ops._stream()) != 0
