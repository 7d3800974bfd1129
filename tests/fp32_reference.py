"""fp64 reference of the fp32 CUDA-core kernels the benchmark engine runs between its tensor-core convolutions -- the depth heads
and the direct convolution (dvmvs_conv2d), the MnasNet stem, the depthwise convolution, the x2 bilinear upsampling -- and the
bit-exact rules of the operand staging (dvmvs_split_planes, dvmvs_split_blocked).  Shared by the GPU tests
(tests/test_fp32_reference.py) and the CPU test that checks the bounds against fp32 emulations and planted defects
(tests/test_fp32_reference_bound.py); nothing here needs a GPU.  Tensors are NCHW torch (any device).

Convolutions: every output is a sum of fmaf products in some order.  Summed sequentially in fp32 over a chain of n roundings,
|y - y64| <= gamma_n * S, gamma_n = n u / (1 - n u), S = the convolution of |x| and |w| (+ |bias| where the chain starts from it).
n is the longest chain the kernel runs:
    conv_head_kernel<LPP>   three accumulators over Cin / LPP products each (taps t with t % 3 equal), their sum and log2(LPP)
                            shuffle additions: 3 Cin / LPP + 2 + log2 LPP
    conv2d_direct_kernel    k*k*8 products per 8-channel chunk over the chunks of one split part, plus one addition per part
    stem_conv_kernel        27 products onto the bias;  dwconv_kernel  k*k products onto the bias
Bias / residual additions are charged EPS_EP of their magnitude, and the bound is carried through the activation and aux as in
tests/tc_reference.py.  A source read through the fused x2 upsampling carries the upsampling bound below, times |w|.

x2 bilinear upsampling (align_corners=True): the kernel's fp32 coordinate sh * oy errs by |d lambda| <= 2u(H - 1) (same along x),
charged C_UP_POS u ((H - 1) + (W - 1)) times the range of the 4x4 input pixels around the cell, plus C_UP_BLEND u max |tap| for
the blend's roundings."""
import numpy as np
import torch
import torch.nn.functional as F

from tests.tc_reference import EPS_EP, U, activation, aux_reference, conv64

C_UP_POS = 8.0          # units of u (H - 1 + W - 1) * range and of u * max |tap|: >= 8x the worst measured by the fp32 emulation
C_UP_BLEND = 8.0        # (0.577 of the two together; tests/test_fp32_reference_bound.py prints it)
CK = 8                  # conv2d_direct_kernel's input-channel chunk
TH, TW, TN = 8, 16, 32  # its output tile


def gamma(n):
    return n * U / (1 - n * U)


def upsample_reference(x):
    """x (B,C,H,W) -> (y, bound) of the x2 align_corners upsampling, float64"""
    x = x.double()
    B, C, H, W = x.shape
    y = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
    xp = F.pad(x, (1, 2, 1, 2), mode="replicate")
    rng = F.max_pool2d(xp, 4, 1) + F.max_pool2d(-xp, 4, 1)          # (B,C,H,W): range of rows i-1..i+2, cols j-1..j+2
    mx = F.max_pool2d(xp.abs(), 4, 1)
    oy = torch.arange(2 * H, dtype=torch.float64, device=x.device)
    ox = torch.arange(2 * W, dtype=torch.float64, device=x.device)
    y0 = torch.floor(oy * (H - 1) / max(2 * H - 1, 1)).long().clamp(0, H - 1)
    x0 = torch.floor(ox * (W - 1) / max(2 * W - 1, 1)).long().clamp(0, W - 1)
    r = rng[:, :, y0][:, :, :, x0]
    m = mx[:, :, y0][:, :, :, x0]
    bound = C_UP_POS * U * ((H - 1) + (W - 1)) * r + C_UP_BLEND * U * m
    return y, bound


class Ref:
    def __init__(self, y, bound, aux=None, aux_bound=None):
        self.y, self.bound, self.aux, self.aux_bound = y, bound, aux, aux_bound


def direct_ksplit(B, Hout, Wout, Cout, src_channels, workspace_bytes):
    """dvmvs_conv2d's split of conv2d_direct_kernel over input-channel chunks (1 = none)"""
    chunks = sum((c + CK - 1) // CK for c in src_channels)
    ctas = -(-Wout // TW) * -(-Hout // TH) * -(-Cout // TN) * B
    if ctas < 96 and chunks >= 8 and workspace_bytes:
        want = -(-296 // ctas)
        fit = workspace_bytes // (B * Hout * Wout * Cout * 4)
        return max(1, min(min(want, chunks // 4), fit))
    return 1


def head_lanes(B, Hout, Wout, Cin):
    """conv_head_kernel's lanes per pixel: 32 on small maps with many channels, else 8"""
    return 32 if (B * Hout * Wout <= 4096 and Cin >= 128) else 8


def conv_reference(sources, w32, stride=1, bias=None, residual=None, residual_mode=0, act=0, aux=None, chain=None):
    """sources: [(x (B,C,Hs,Ws), upsample)]; w32 [k][k][Cin][Cout] fp32; residual NCHW (same size or coarse for nearest-up);
    chain: the longest fmaf chain of the kernel (see the module docstring)"""
    xs, bs = [], []
    for x, up in sources:
        if up:
            y, b = upsample_reference(x)
        else:
            y, b = x.double(), torch.zeros_like(x, dtype=torch.float64)
        xs.append(y)
        bs.append(b)
    x, bx = torch.cat(xs, 1), torch.cat(bs, 1)
    w = w32.double().to(x.device)
    y = conv64(x, w, stride)
    S = conv64(x.abs(), w.abs(), stride)
    bz = gamma(chain) * S + conv64(bx, w.abs(), stride)
    z, mag = y, y.abs()
    if bias is not None:
        b = bias.double().to(x.device).view(1, -1, 1, 1)
        z, mag = z + b, mag + b.abs()
    if residual_mode:
        r = residual.double().to(x.device)
        if residual_mode == 2:
            r = F.interpolate(r, size=z.shape[2:], mode="nearest")
        z, mag = z + r, mag + r.abs()
    bz = bz + EPS_EP * mag
    out, bound = activation(z, bz, act)
    ref = Ref(out, bound)
    if aux is not None:
        ref.aux, ref.aux_bound = aux_reference(out, bound, *aux)
    return ref


def stem_reference(img, w32, bias):
    """img (B,3,H,W); w32 [3][3][3][32]; 3x3 stride 2 pad 1 + bias + ReLU"""
    x = img.double()
    w = w32.double().to(x.device)
    y = conv64(x, w, 2)
    S = conv64(x.abs(), w.abs(), 2)
    if bias is not None:
        b = bias.double().to(x.device).view(1, -1, 1, 1)
        y, S = y + b, S + b.abs()
    return Ref(y.clamp_min(0.0), gamma(28) * S)


def dwconv_reference(x, w_kkc, bias, stride, act):
    """x (B,C,H,W); w_kkc [k][k][C]"""
    x = x.double()
    k = w_kkc.shape[0]
    wd = w_kkc.double().to(x.device).permute(2, 0, 1).unsqueeze(1)
    y = F.conv2d(x, wd, None, stride, k // 2, groups=x.shape[1])
    S = F.conv2d(x.abs(), wd.abs(), None, stride, k // 2, groups=x.shape[1])
    if bias is not None:
        b = bias.double().to(x.device).view(1, -1, 1, 1)
        y, S = y + b, S + b.abs()
    out, bound = activation(y, gamma(k * k + 1) * S, act)
    return Ref(out, bound)


def split_expected(v):
    """fp32 values -> the (hi, lo) fp16 planes every staging kernel must write, bit for bit"""
    v = v.float()
    hi = v.half()
    return hi, (v - hi.float()).half()


# ------------------------------------------------------------------------------------------------ fp32 emulation of the kernels
def _f32(x):
    return np.asarray(x, dtype=np.float32)


def fmaf(a, b, c):
    return _f32(np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64))


def emulate_upsample(x, variant=None):
    """upsample2x_kernel in fp32 numpy, x (B,H,W,C) -> (B,2H,2W,C); variant "last_row_clamp": y1 clamps one row early"""
    x = _f32(x)
    B, H, W, C = x.shape
    Ho, Wo = 2 * H, 2 * W
    sh = np.float32(H - 1) / np.float32(Ho - 1) if Ho > 1 else np.float32(0)
    sw = np.float32(W - 1) / np.float32(Wo - 1) if Wo > 1 else np.float32(0)
    fy = _f32(np.float32(sh) * np.arange(Ho, dtype=np.float32))
    fx = _f32(np.float32(sw) * np.arange(Wo, dtype=np.float32))
    y0, x0 = fy.astype(np.int64), fx.astype(np.int64)
    y1 = y0 + (y0 < (H - 2 if variant == "last_row_clamp" else H - 1))
    x1 = x0 + (x0 < W - 1)
    ly1, lx1 = _f32(fy - y0), _f32(fx - x0)
    ly0, lx0 = _f32(1 - ly1), _f32(1 - lx1)
    g = lambda yy, xx: x[:, yy][:, :, xx]
    lx0_, lx1_ = lx0[None, None, :, None], lx1[None, None, :, None]
    ly0_, ly1_ = ly0[None, :, None, None], ly1[None, :, None, None]
    # bilerp (common.cuh): the roundings of every copy of the blend, spelled out
    top = fmaf(lx1_, g(y0, x1), _f32(lx0_ * g(y0, x0)))
    bot = fmaf(lx0_, g(y1, x0), _f32(lx1_ * g(y1, x1)))
    return fmaf(ly0_, top, _f32(ly1_ * bot))


def emulate_stem(img, w, bias, variant=None):
    """stem_conv_kernel: img (B,3,H,W) NCHW, w [3][3][3][32] -> (B,Ho,Wo,32); variant "pad0": taps read without the 1-pixel pad"""
    img, w = _f32(img), _f32(w)
    B, _, H, W = img.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    pad = 0 if variant == "pad0" else 1
    acc = np.broadcast_to(_f32(bias) if bias is not None else np.zeros(32, np.float32), (B, Ho, Wo, 32)).copy()
    oy, ox = np.arange(Ho)[:, None], np.arange(Wo)[None, :]
    for ky in range(3):
        for kx in range(3):
            iy, ix = oy * 2 - pad + ky, ox * 2 - pad + kx
            ok = (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
            for c in range(3):
                v = img[:, c][:, np.clip(iy, 0, H - 1), np.clip(ix, 0, W - 1)] * ok
                acc = np.where(ok[None, :, :, None], fmaf(v[..., None], w[ky, kx, c][None, None, None, :], acc), acc)
    return np.maximum(acc, np.float32(0))


def emulate_dwconv(x, w, bias, stride, act, variant=None):
    """dwconv_kernel: x (B,H,W,C), w [k][k][C]; variant "stride_y_only": the stride applied to rows only"""
    x, w = _f32(x), _f32(w)
    B, H, W, C = x.shape
    k = w.shape[0]
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    sx = 1 if variant == "stride_y_only" else stride
    acc = np.broadcast_to(_f32(bias) if bias is not None else np.zeros(C, np.float32), (B, Ho, Wo, C)).copy()
    oy, ox = np.arange(Ho)[:, None], np.arange(Wo)[None, :]
    for ky in range(k):
        for kx in range(k):
            iy, ix = oy * stride - pad + ky, ox * sx - pad + kx
            ok = (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
            v = x[:, np.clip(iy, 0, H - 1), np.clip(ix, 0, W - 1)]
            acc = np.where(ok[None, :, :, None], fmaf(v, w[ky, kx][None, None, None, :], acc), acc)
    return np.maximum(acc, np.float32(0)) if act == 1 else acc


def emulate_head(x, w, bias, act, aux, lanes, variant=None):
    """conv_head_kernel<lanes>: x (B,H,W,Cin), w [3][3][Cin][1]; returns (out (B,H,W,1), aux_out or None).
    variant "no_bias": the bias is dropped; "aux_pre_activation": aux from the value before the activation"""
    x, w = _f32(x), _f32(w)[..., 0]
    B, H, W, C = x.shape
    xp = np.zeros((B, H + 2, W + 2, C), np.float32)
    xp[:, 1:-1, 1:-1] = x
    subs = []
    for sub in range(lanes):
        acc = [np.zeros((B, H, W), np.float32) for _ in range(3)]
        for c in range(sub * 4, C, lanes * 4):
            for t in range(9):
                ky, kx = t // 3, t % 3
                xv = xp[:, ky:ky + H, kx:kx + W, c:c + 4]
                wv = w[ky, kx, c:c + 4]
                a = acc[t % 3]
                a = fmaf(xv[..., 0], wv[0], fmaf(xv[..., 1], wv[1], fmaf(xv[..., 2], wv[2], fmaf(xv[..., 3], wv[3], a))))
                acc[t % 3] = a
        subs.append(_f32(_f32(acc[0] + acc[1]) + acc[2]))
    o = 1
    while o < lanes:                       # __shfl_xor_sync butterfly: lane s adds lane s ^ o
        subs = [_f32(subs[s] + subs[s ^ o]) for s in range(lanes)]
        o <<= 1
    z = subs[0]
    if bias is not None and variant != "no_bias":
        z = _f32(z + np.float32(bias[0]))
    v = np.maximum(z, np.float32(0)) if act == 1 else (_f32(1 / _f32(1 + np.exp(-z.astype(np.float64)).astype(np.float32))) if act == 2 else z)
    a = None
    if aux is not None:
        src = z if variant == "aux_pre_activation" else v
        a = _f32(np.float32(1) / fmaf(np.float32(aux[0]), src, np.float32(aux[1])))
    return v[..., None], (a[..., None] if a is not None else None)


def emulate_split(v, variant=None):
    """the staging kernels' (hi, lo) of fp32 values; variant "lo_without_fp32_subtraction": lo = rn16(x) - hi in fp16"""
    v = torch.as_tensor(_f32(v))
    hi = v.half()
    if variant == "lo_without_fp32_subtraction":
        return hi, (v.half().float() - hi.float()).half()
    return hi, (v - hi.float()).half()


def check_staged(what, hi, lo, values, c_offset, c_cover, sentinel_bits, hi_only=False, others=True):
    """hi / lo: the staged fp16 planes (..., Cs) of one call, filled with the fp16 bit pattern `sentinel_bits` beforehand; values
    (..., C): the fp32 values staged (x, or upsample2x's output for the same tensor: every copy of the interpolation computes the
    same fp32 value).  Channels [c_offset, c_offset + C) must be split_expected(values) bit for bit, [c_offset + C,
    c_offset + c_cover) +0 in both planes, every other channel -- and the lo plane under hi_only -- untouched.  others=False: the
    other channels belong to other calls (a staged concatenation) and are not checked."""
    C = values.shape[-1]
    eh, el = split_expected(values)
    hb, lb = hi.view(torch.int16), lo.view(torch.int16)
    win = slice(c_offset, c_offset + C)
    pad = slice(c_offset + C, c_offset + c_cover)
    assert torch.equal(hb[..., win], eh.view(torch.int16)), "%s: hi plane != fp16_rn(x)" % what
    if hi_only:
        assert bool((lb == sentinel_bits).all()), "%s: hi-only staging wrote the lo plane" % what
    else:
        assert torch.equal(lb[..., win], el.view(torch.int16)), "%s: lo plane != fp16_rn(x - hi)" % what
        assert bool((lb[..., pad] == 0).all()), "%s: padding channels of the lo plane are not +0" % what
    assert bool((hb[..., pad] == 0).all()), "%s: padding channels of the hi plane are not +0" % what
    if not others:
        return
    outside = torch.ones(hb.shape[-1], dtype=torch.bool, device=hb.device)
    outside[c_offset:c_offset + c_cover] = False
    assert bool((hb[..., outside] == sentinel_bits).all()) and bool((lb[..., outside] == sentinel_bits).all()), \
        "%s: a channel outside [%d, %d) was written" % (what, c_offset, c_offset + c_cover)
