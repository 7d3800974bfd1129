"""Steady-state timing (CUDA events, warm caches, back-to-back launches) of individual convolution layers on both
backends, for the layer shapes that dominate the keyframe.  Usage: python tools/tc_bench.py [terms]

    python tools/tc_bench.py halo [terms]

times every halo convolution (dvmvs_conv2d_halo) of bench.py's default engine at the shape and with the outputs the engine
runs it: the engine is built and primed, each conv2d_halo call it makes is recorded with its operands, and each distinct
call is then replayed alone.  Prints us and achieved TFLOP/s (2 x MACs / time) per layer, then a JSON record.

    python tools/tc_bench.py tc

does the same for every dvmvs_conv2d_tc call of the engine.  Both modes mark the calls the engine issues on its recurrent
(loop-carried) stage with "rec".

    python tools/tc_bench.py expand [terms]

times the front half (1x1 expansion + depthwise) of every MnasNet trunk block at batch 12 and 3: the two-launch composition
beside the fused dvmvs_expand_dwconv, with algorithmic HBM bytes, TB/s and TFLOP/s."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "deep-video-mvs_b200"))
import torch

import synth_data as synth
from dvmvs import _native as N
from dvmvs import _ops as ops
from tools.engine_record import engine_calls, layer_names

DEV = "cuda"
LAYERS = [
    # name, B, H, W, [src channels], Cout, k, stride
    ("refine.1 5x5 32->32 @256^2", 1, 256, 256, [32], 32, 5, 1),
    ("refine.0 5x5 36->32 @256^2 (packed)", 1, 256, 256, [36], 32, 5, 1),
    ("db4.conv1 5x5 65->32 @128^2", 1, 128, 128, [32, 32, 1], 32, 5, 1),
    ("aggregator0 5x5 96->32 @128^2", 1, 128, 128, [32, 64], 32, 5, 1),
    ("fpn.layer0 3x3 32->32 @128^2 B=3", 3, 128, 128, [32], 32, 3, 1),
    ("eb0.conv 5x5 64->64 @64^2", 1, 64, 64, [64], 64, 5, 1),
    ("eb1.conv 3x3 128->128 @32^2", 1, 32, 32, [128], 128, 3, 1),
    ("eb2.conv 3x3 256->256 @16^2", 1, 16, 16, [256], 256, 3, 1),
    ("eb3.conv 3x3 512->512 @8^2", 1, 8, 8, [512], 512, 3, 1),
    ("lstm 3x3 1024->2048 @8^2", 1, 8, 8, [512, 512], 2048, 3, 1),
    ("mnas pw 1x1 96->576 @16^2 B=3", 3, 16, 16, [96], 576, 1, 1),
    ("mnas pw 1x1 1152->192 @8^2 B=3", 3, 8, 8, [1152], 192, 1, 1),
    ("mnas pw 1x1 16->48 @128^2 B=3", 3, 128, 128, [16], 48, 1, 1),
]


def timeit(fn, iters=30):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def graph_timeit(fn, calls=20, replays=20):
    """us per call of `fn` with `calls` back-to-back calls captured in one CUDA graph: the device time the engine's graphs see.
    Timing eager calls instead measures the host (Python, descriptor, allocation: ~20-30 us per call), not these kernels."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(calls):
            fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (calls * replays) * 1e3


def halo_layers(terms):
    import json
    mods, calls = engine_calls(("conv2d_halo",))
    names = layer_names(mods)
    rows = []
    with torch.no_grad():
        for key, (args, kw, lay, on_rec) in calls.items():
            blks, ph = args[0], args[1]
            kw = dict(kw, terms=terms)
            B, Hh, Ww = blks[0].shape[1], blks[0].shape[3], blks[0].shape[4]
            t = graph_timeit(lambda: ops.conv2d_halo(*args, **kw))
            t_eager = timeit(lambda: ops.conv2d_halo(*args, **kw), iters=100)
            macs = B * Hh * Ww * ph.cout * ph.cin * ph.ksize * ph.ksize
            rows.append({"layer": names.get(id(lay), "?"), "recurrent": on_rec, "B": B, "H": Hh, "W": Ww, "cin": ph.cin, "cout": ph.cout,
                         "k": ph.ksize, "kc": ph.kc, "block_n": ph.block_n,
                         "outputs": [o for o in ("f32", "blk", "nhwc") if kw.get("want_" + o, o != "blk")],
                         "us": t, "us_eager": t_eager, "tflops": 2.0 * macs / (t * 1e-6) / 1e12})
    rows.sort(key=lambda r: -r["us"])
    for r in rows:
        print("%-28s %s B=%-2d %3dx%-3d %3d->%-3d k%d kc%d N%d %-14s %8.1f us %6.1f TFLOP/s (eager %5.1f us)" % (
            r["layer"], "rec" if r["recurrent"] else "   ", r["B"], r["H"], r["W"], r["cin"], r["cout"], r["k"], r["kc"], r["block_n"],
            "+".join(r["outputs"]), r["us"], r["tflops"], r["us_eager"]))
    print(json.dumps({"device": torch.cuda.get_device_name(0), "timing": "graph_timeit", "terms": terms, "total_us": sum(r["us"] for r in rows),
                      "recurrent_us": sum(r["us"] for r in rows if r["recurrent"]), "layers": rows}))


def tc_layers():
    """every conv2d_tc call of the engine (stride 1 and 2, split-K or not, deferred finishing pass or not) replayed alone"""
    import json
    mods, calls = engine_calls(("conv2d_tc",))
    names = layer_names(mods)
    rows = []
    with torch.no_grad():
        for key, (args, kw, lay, on_rec) in calls.items():
            planes, ptc = args[0], args[1]
            B, Hin, Win = planes[0].shape[1], planes[0].shape[2], planes[0].shape[3]
            pad = (ptc.ksize - 1) // 2
            Ho, Wo = (Hin + 2 * pad - ptc.ksize) // ptc.stride + 1, (Win + 2 * pad - ptc.ksize) // ptc.stride + 1
            t = graph_timeit(lambda: ops.conv2d_tc(*args, **kw))
            t_eager = timeit(lambda: ops.conv2d_tc(*args, **kw), iters=100)
            macs = B * Ho * Wo * ptc.cout * ptc.cin * ptc.ksize * ptc.ksize
            rows.append({"layer": names.get(id(lay), "?"), "recurrent": on_rec, "B": B, "Hin": Hin, "Win": Win, "Hout": Ho, "Wout": Wo,
                         "cin": ptc.cin, "sources": [int(p.shape[4]) for p in planes], "cout": ptc.cout, "k": ptc.ksize,
                         "stride": ptc.stride, "deferred_finish": bool(kw.get("defer_finish")), "us": t, "us_eager": t_eager,
                         "tflops": 2.0 * macs / (t * 1e-6) / 1e12})
    rows.sort(key=lambda r: -r["us"])
    for r in rows:
        print("%-28s %s B=%-2d %3dx%-3d s%d %4d->%-4d k%d%s %8.1f us %6.1f TFLOP/s (eager %5.1f us)" % (
            r["layer"], "rec" if r["recurrent"] else "   ", r["B"], r["Hout"], r["Wout"], r["stride"], r["cin"], r["cout"], r["k"],
            " deferred" if r["deferred_finish"] else "", r["us"], r["tflops"], r["us_eager"]))
    print(json.dumps({"device": torch.cuda.get_device_name(0), "timing": "graph_timeit", "total_us": sum(r["us"] for r in rows),
                      "recurrent_us": sum(r["us"] for r in rows if r["recurrent"]), "layers": rows}))


def expand_layers(terms):
    """every MnasNet trunk block's front half (1x1 expansion + depthwise) at the engine's shapes -- batch 12 (the lookahead
    engine's trunk graphs: 4 keyframes x 3 images) and batch 3 -- as the two launches conv2d_tc (fp32 out) + dwconv2d (planes
    out) and as the fused expand_dwconv; algorithmic HBM bytes (operands in, outputs out, weights ignored) and FLOP/s
    (expansion at the input resolution + depthwise taps) over graph-timed us"""
    import json
    from dvmvs._blocks import FeatureExtractor
    fe = FeatureExtractor()
    shapes, side = [], 128
    for layer in (fe.layer2, fe.layer3, fe.layer4, fe.layer5):
        for stack in layer:
            for blk in stack:
                L = blk.layers
                shapes.append((L[0].in_channels, L[0].out_channels, L[3].kernel_size[0], blk.stride, side))
                side //= blk.stride
    rows = []
    planes_in = 2 if terms == 3 else 1
    with torch.no_grad():
        for B in (12, 3):
            for shape in sorted(set(shapes), key=shapes.index):
                cin, mid, k, s, H = shape
                w = torch.from_numpy(synth.tensor("tb/we", (mid, cin, 1, 1), seed=2, scale=(2.0 / cin) ** 0.5)).to(DEV)
                bias = torch.from_numpy(synth.tensor("tb/be", (mid,), seed=3, scale=0.1)).to(DEV)
                expand = ops.ConvLayer(ops.PackedConv(w, bias, None, act=N.ACT_RELU))
                bn = torch.nn.BatchNorm2d(mid).to(DEV).eval()
                dw = ops.PackedDepthwise(torch.from_numpy(synth.tensor("tb/wd", (mid, 1, k, k), seed=4, scale=0.3)).to(DEV), bn, stride=s)
                x = ops.Act(torch.from_numpy(synth.tensor("tb/x", (B, H, H, cin), seed=1)).to(DEV))
                planes = x.get_planes()
                ptc = ops.PackedConvTC(expand.pc, [cin], DEV)
                Ho = (H + 2 * (k // 2) - k) // s + 1

                def two_launch():
                    f32, _ = ops.conv2d_tc([planes], ptc, terms=terms, want_f32=True, want_planes=False)
                    ops.dwconv2d(f32, dw, want_f32=False, want_planes=True)

                t_old = graph_timeit(two_launch)
                t_new = graph_timeit(lambda: ops.expand_dwconv(x, expand, dw, terms))
                x_bytes, e_bytes, y_bytes = planes_in * B * H * H * cin * 2, B * H * H * mid * 4, B * Ho * Ho * mid * 2
                old_bytes = x_bytes + 2 * e_bytes + 2 * y_bytes                  # dwconv_kernel writes both planes
                new_bytes = x_bytes + planes_in * y_bytes
                flops = 2.0 * B * H * H * cin * mid * terms + 2.0 * B * Ho * Ho * mid * k * k
                rows.append({"B": B, "cin": cin, "mid": mid, "k": k, "stride": s, "Hin": H, "Hout": Ho, "blocks": shapes.count(shape),
                             "us_two_launch": t_old, "us_fused": t_new, "mb_two_launch": old_bytes / 1e6, "mb_fused": new_bytes / 1e6,
                             "tbs_two_launch": old_bytes / (t_old * 1e-6) / 1e12, "tbs_fused": new_bytes / (t_new * 1e-6) / 1e12,
                             "tflops_two_launch": flops / (t_old * 1e-6) / 1e12, "tflops_fused": flops / (t_new * 1e-6) / 1e12})
    for r in rows:
        print("B=%-2d %3d->%-4d k%d s%d %3d^2->%3d^2 x%d | two launches %7.1f us %6.1f MB %5.2f TB/s %5.1f TFLOP/s | fused %7.1f us %6.1f MB "
              "%5.2f TB/s %5.1f TFLOP/s | x%.2f" % (
                  r["B"], r["cin"], r["mid"], r["k"], r["stride"], r["Hin"], r["Hout"], r["blocks"], r["us_two_launch"], r["mb_two_launch"],
                  r["tbs_two_launch"], r["tflops_two_launch"], r["us_fused"], r["mb_fused"], r["tbs_fused"], r["tflops_fused"],
                  r["us_two_launch"] / r["us_fused"]))
    for B in (12, 3):
        sel = [r for r in rows if r["B"] == B]
        print("B=%d, all 16 blocks: two launches %.1f us, fused %.1f us" % (
            B, sum(r["us_two_launch"] * r["blocks"] for r in sel), sum(r["us_fused"] * r["blocks"] for r in sel)))
    print(json.dumps({"device": torch.cuda.get_device_name(0), "timing": "graph_timeit", "terms": terms, "blocks": rows}))


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "halo":
        return halo_layers(int(sys.argv[2]) if len(sys.argv) > 2 else 1)
    if len(sys.argv) > 1 and sys.argv[1] == "tc":
        return tc_layers()
    if len(sys.argv) > 1 and sys.argv[1] == "expand":
        return expand_layers(int(sys.argv[2]) if len(sys.argv) > 2 else 1)
    terms = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    for name, B, H, W, chans, Cout, k, stride in LAYERS:
        cin = sum(chans)
        xs = [torch.from_numpy(synth.tensor("tb/x%d" % i, (B, H, W, c), seed=1)).to(DEV) for i, c in enumerate(chans)]
        w = torch.from_numpy(synth.tensor("tb/w", (Cout, cin, k, k), seed=2, scale=(2.0 / (cin * k * k)) ** 0.5))
        pc = ops.PackedConv(w, None, None, stride=stride, act=N.ACT_RELU)
        ptc = ops.PackedConvTC(pc, chans, DEV)
        pc.weight = pc.weight.to(DEV)
        planes = [ops.split_planes(x) for x in xs]
        t_fp32 = timeit(lambda: ops.conv2d([(x, N.SRC_DIRECT) for x in xs], pc))
        res = []
        for bn in (32, 64, 128):
            if bn > 32 and Cout <= 32:
                continue
            for split in (False, True):
                t = timeit(lambda: ops.conv2d_tc(planes, ptc, terms=terms, block_n=bn, allow_split=split))
                res.append("N%d%s %.1f" % (bn, "+splitK" if split else "", t))
        t1 = timeit(lambda: ops.conv2d_tc(planes, ptc, terms=1, allow_split=True))
        if stride == 1 and k >= 3 and Cout <= 64 * 8:
            for kc in (16, 32):
                try:
                    ph = ops.PackedConvHalo(pc, chans, DEV, kc=kc, concat_padded=True)
                    blk = ops.split_blocked([(x, False) for x in xs])
                    th = timeit(lambda: ops.conv2d_halo([blk], ph, terms=terms, want_f32=True, want_blk=True, want_nhwc=False))
                    res.append("HALO kc%d %.1f" % (kc, th))
                except Exception as e:  # noqa: BLE001
                    res.append("HALO kc%d FAILED %s" % (kc, str(e)[:60]))
        macs = B * (H // stride) * (W // stride) * Cout * cin * k * k
        print("%-38s %7.1f MMAC | fp32 %7.1f us | tc x%d: %s | tc x1 auto %.1f us" % (name, macs / 1e6, t_fp32, terms, "  ".join(res), t1), flush=True)


if __name__ == "__main__":
    main()
