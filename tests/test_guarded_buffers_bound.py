"""The guarded-buffer mechanism (tests/guarded.py) catches what it claims, without a GPU: an honest torch-on-CPU stand-in of a small
staged convolution passes under guard_allocations(), and each planted defect -- a store one element past either end, a store into
a channel outside the call's window, a skipped store, a masked read one element past the end, a modified input, a split-K counter
left set -- is rejected with a message that names it."""
import sys

import pytest
import torch

from tests import guarded as G
from tests import tc_reference as R

THIS = sys.modules[__name__]
DEFECTS = ["write_past_end", "write_before_start", "write_outside_window", "skip_one_store", "masked_read_past_end", "modify_input",
           "counter_left_set"]


def stage_conv1x1(x, w, into, c_offset, ws, defect=None):
    """Stand-in of a staging convolution: relu(x @ w) for x (B,H,W,C) and w (C,Cout) stored into channels [c_offset, c_offset+Cout)
    of `into` (B,H,W,Cs), or of a fresh tensor when `into` is None.  The K sum runs in two halves through the partial-sum region
    of the split-K workspace, with an arrival counter at its head that the second half returns to zero."""
    B, H, W, C = x.shape
    cout = w.shape[1]
    y = torch.empty((B, H, W, cout), dtype=x.dtype, device=x.device) if into is None else into
    half = C // 2
    counter = ws[:1]
    part = ws[G.COUNTER_BYTES // 4:G.COUNTER_BYTES // 4 + B * H * W * cout].view(B, H, W, cout)
    part.copy_(x[..., :half] @ w[:half])
    counter += 1
    acc = part + x[..., half:] @ w[half:]
    if defect != "counter_left_set":
        counter -= 1
    if defect == "masked_read_past_end":        # a tap with weight 0 one element past the operand
        acc = acc + 0.0 * torch.as_strided(x, (1,), (1,), x.storage_offset() + x.numel())
    if defect == "modify_input":
        x.view(-1)[5] = 0.0
    r = torch.relu(acc)
    dst = y[..., c_offset:c_offset + cout] if into is not None else y
    if defect == "skip_one_store":
        keep = torch.zeros(r.shape, dtype=torch.bool)
        keep.view(-1)[7] = True
        r = torch.where(keep, dst, r)                    # element 7 keeps whatever the memory held
    dst.copy_(r)
    if defect == "write_outside_window":
        y[..., c_offset - 1] = 0.0                       # the last channel of the previous call's window
    if defect == "write_past_end":
        torch.as_strided(y, (1,), (1,), y.storage_offset() + y.numel()).fill_(0.0)
    if defect == "write_before_start":
        torch.as_strided(y, (1,), (1,), y.storage_offset() - 1).fill_(0.0)
    return y


def _operands():
    g = torch.Generator().manual_seed(3)
    x1 = torch.randn((2, 5, 7, 16), generator=g)
    x2 = torch.randn((2, 5, 7, 8), generator=g)
    w1 = torch.randn((16, 12), generator=g)
    w2 = torch.randn((8, 4), generator=g)
    return x1, x2, w1, w2


def _run(defect):
    """two staging calls into one 16-channel operand (windows [0,12) and [12,16)) and one call into a fresh output, all guarded,
    each checked against the float64 reference; then verify()"""
    x1, x2, w1, w2 = _operands()
    with G.guard_allocations(modules=[THIS], device_type="cpu") as g:
        gx1, gx2, gw1, gw2 = G.guard_inputs(x1, x2, w1, w2)
        into = torch.empty((2, 5, 7, 16), dtype=torch.float32, device="cpu")
        stage_conv1x1(gx1, gw1, into, 0, g.workspace)
        stage_conv1x1(gx2, gw2, into, 12, g.workspace, defect=defect)
        fresh = stage_conv1x1(gx1, gw1, None, 0, g.workspace, defect=defect if defect != "write_outside_window" else None)
        ref = torch.cat([torch.relu(x1.double() @ w1.double()), torch.relu(x2.double() @ w2.double())], -1)
        bound = 1e-5 * ref.abs() + 1e-5
        R.check("staged operand", into, ref, bound)
        R.check("fresh output", fresh, ref[..., :12], bound[..., :12])
        G.verify()


def test_honest_stand_in_passes_under_the_guard():
    _run(None)


@pytest.mark.parametrize("defect", DEFECTS)
def test_planted_defect_is_rejected(defect):
    expect = {
        "write_past_end": r"output .* fringe after the tensor modified at byte offset \+0 ",
        "write_before_start": r"output .* fringe before the tensor modified at byte offset -4 ",
        "write_outside_window": r"staged operand: .*exceeds the bound",
        "skip_one_store": r"staged operand: .*non-finite output",
        "masked_read_past_end": r"non-finite output",
        "modify_input": r"input \S+ _run \(\(2, 5, 7, 8\) float32\): modified at byte offset 20 ",
        "counter_left_set": r"workspace .* split-K counter region not zero at byte offset 0",
    }[defect]
    with pytest.raises(AssertionError, match=expect):
        _run(defect)


def test_fringes_sizes_and_alignment():
    for shape, dtype in (((3,), torch.float32), ((2, 3, 5, 7), torch.float16), ((300, 1000), torch.float32), ((5,), torch.int32)):
        with G.guard_allocations(modules=[THIS], device_type="cpu"):
            t = G.guarded(shape, dtype, "cpu")
            g = G.REGISTRY.lookup(t)
            assert g.fringe % G.ALIGN == 0 and g.fringe >= max(G.MIN_FRINGE, t.numel() * t.element_size())
            assert (t.data_ptr() - g.base.data_ptr()) % G.ALIGN == 0
            if dtype.is_floating_point:
                assert bool(torch.isnan(t).all())          # output interior: NaN until written
            before = g.base[:g.fringe].view(dtype)
            assert bool(torch.isnan(before).all()) if dtype.is_floating_point else bool((before.view(torch.uint8) == 0xa5).all())
            G.verify()
    x = G.guard_inputs(torch.ones(4, 6))
    g = G.REGISTRY.lookup(x)
    assert g.base[:g.fringe].view(torch.int32).eq(0x7fc0dead).all()
    h = G.guard_inputs(torch.ones(4, 6, dtype=torch.float16))
    assert G.REGISTRY.lookup(h).base[:16].view(torch.int16).eq(0x7e5a).all()
    s = G.guard_inputs(torch.ones(4, 6), shift=4)
    assert s.data_ptr() % 16 == 4 and bool((s == 1).all())
    G.verify()


def test_views_keep_fills_alignment_and_registry():
    with G.guard_allocations(modules=[THIS], device_type="cpu"):
        t = torch.empty((2, 3, 4, 8), dtype=torch.float32, device="cpu")         # through the proxy: a guarded output
        nchw = t.permute(0, 3, 1, 2)
        for v in (t.view(-1), nchw, nchw.permute(0, 2, 3, 1).contiguous(), t.view(6, 32)[1:], t.contiguous()):
            assert G.REGISTRY.lookup(v) is G.REGISTRY.lookup(t) and v.data_ptr() % 16 == 0
        nchw.copy_(torch.arange(t.numel(), dtype=torch.float32).view(2, 8, 3, 4))
        G.verify(clear=False)
        x = G.guard_inputs(torch.randn(2, 8, 3, 4).contiguous(memory_format=torch.channels_last))
        assert x.stride() == (96, 1, 32, 8) and x.permute(0, 2, 3, 1).is_contiguous()
        assert G.REGISTRY.lookup(x.permute(0, 2, 3, 1).contiguous()) is G.REGISTRY.lookup(x)
        with pytest.raises(AssertionError, match=r"fringe after the tensor modified at byte offset \+0 "):
            torch.as_strided(x, (1,), (1,), x.storage_offset() + x.numel()).fill_(1.0)
            G.verify()


def test_row_slice_of_poisoned():
    t = torch.randn(2, 3, 4)
    v = G.row_slice_of_poisoned(t, 1, 3)
    assert torch.equal(v, t)
    full = torch.as_strided(v, (5, 3, 4), v.stride(), v.storage_offset() - v.stride(0))
    assert bool(torch.isnan(full[0]).all()) and bool(torch.isnan(full[3:]).all())
    G.verify()


def test_proxy_forwards_everything_else_and_restores():
    before = THIS.torch
    with G.guard_allocations(modules=[THIS], device_type="cpu") as g:
        assert THIS.torch is g.proxy and torch.float16 is THIS.torch.float16 and torch.randn is THIS.torch.randn
        z = torch.zeros(3, 4)
        e = torch.empty_like(z)
        f = torch.full((2, 2), 3.0)
        assert G.REGISTRY.lookup(z).role == G.ZEROS and G.REGISTRY.lookup(e).role == G.OUTPUT and bool((f == 3).all())
        assert bool((z == 0).all()) and bool(torch.isnan(e).all()) and g.proxy.allocations == 3
        G.verify()
    assert THIS.torch is before
