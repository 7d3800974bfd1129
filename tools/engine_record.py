"""Records the calls bench.py's default engine makes while it primes: used by tools/tc_bench.py to time each layer alone and by the
fp64 reference tests (tests/test_tc_reference.py, tests/test_engine_coverage.py) to check each call on the engine's own buffers, and
to list every dvmvs_* entry point of the native library the engine launches."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (REPO, os.path.join(REPO, "deep-video-mvs_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import torch

import synth_data as synth
from dvmvs import _ops as ops


def layer_names(mods):
    """id(ConvLayer) -> 'tag.module[index]' for every packed layer of the modules"""
    names = {}

    def walk(obj, path):
        if isinstance(obj, ops.ConvLayer):
            names[id(obj)] = path
        elif isinstance(obj, (list, tuple)):
            for i, o in enumerate(obj):
                walk(o, "%s[%d]" % (path, i))

    for tag, m in mods.items():
        for name, sub in m.named_modules():
            walk(getattr(sub, "_packed", None), tag + ("." + name if name else ""))
    return names


def _key(name, a, kw):
    """one entry per distinct call site: (op, packed weights, operand shape[, deferred finish])"""
    if name == "lstm_gates":
        return name, tuple(a[1].shape), kw.get("parts") is not None
    if name == "expand_dwconv":
        return name, id(a[1]), tuple(a[0].get_planes().shape)
    if name == "plane_sweep_tc":          # (reference planes, measurement planes, poses, K, depth range, D); no packed weights
        return name, tuple(a[0][0].shape), len(a[1]), kw.get("terms")
    if name in ("conv2d_tc", "conv2d_halo"):
        return name, id(a[1]), tuple(a[0][0].shape), bool(kw.get("defer_finish"))
    return (name,) + tuple(_signature(v) for v in a) + tuple(sorted((k, _signature(v)) for k, v in kw.items()))


def _signature(v):
    """a call argument reduced to what tells call sites apart: tensor shapes, packed weights by identity, plain values as they are"""
    if isinstance(v, torch.Tensor):
        return ("tensor",) + tuple(v.shape)
    if isinstance(v, (list, tuple)):
        return tuple(_signature(x) for x in v)
    if v is None or isinstance(v, (int, float, bool, str)):
        return v
    return ("object", id(v))


def conv2d_branch(d, launches):
    """the kernel dvmvs_conv2d dispatches a descriptor to (csrc/conv.cu) -- "head8" / "head32" (conv_head_kernel), "direct K/S" or
    "direct K/S split" (conv2d_direct_kernel, + conv_epilogue_kernel: two launches) -- given the kernels the call launched"""
    cin = sum(d.src_channels[i] for i in range(d.n_src))
    if (d.Cout == 1 and d.n_src == 1 and d.src_mode[0] == 0 and d.ksize == 3 and d.stride == 1 and cin % 32 == 0 and d.residual_mode == 0
            and d.src[0] % 16 == 0 and d.weight % 16 == 0):
        return "head32" if (d.B * d.Hin * d.Win <= 4096 and cin >= 128) else "head8"
    return "direct %d/%d%s" % (d.ksize, d.stride, " split" if launches > 1 else "")


def engine_calls(ops_recorded=("conv2d_tc",), height=None, width=None, device="cuda", native=None):
    """Builds and primes bench.py's default engine (seed-7 weights, tensor-core backend with 1-term operands; bench.py's input
    size unless height / width are given) with every call of the named functions of dvmvs._ops ("conv2d_tc", "conv2d_halo",
    "expand_dwconv", "lstm_gates", "plane_sweep_tc") recorded: returns (mods, {key: (args, kwargs, ConvLayer or None, on the recurrent stage?)}).
    The recorded tensors are the engine's own buffers: their contents are whatever the engine left in them.
    native: a dict filled with {dvmvs_* entry point: number of calls} of every native call made while priming, and for dvmvs_conv2d
    {"dvmvs_conv2d " + conv2d_branch: number of calls}."""
    import bench
    from dvmvs import pipeline
    from dvmvs.fusionnet.model import CostVolumeDecoder, CostVolumeEncoder, FeatureExtractor, FeatureShrinker, LSTMFusion
    ops.set_conv_backend("tc", terms=1, stride2=True)
    dev = torch.device(device, 0)
    H, W, D, M = height or bench.H, width or bench.W, bench.D, bench.M
    mods = {"fe": FeatureExtractor(), "fpn": FeatureShrinker(), "cve": CostVolumeEncoder(), "lstm": LSTMFusion(), "cvd": CostVolumeDecoder()}
    for m in mods.values():
        shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes, seed=7).items()}, strict=True)
        m.to(dev).eval()
    clip = [synth.make_clip(0, 1, H, W, M)]
    ref, rpose, meas, mpose, K = bench.stack_frame(clip, 0)
    frame = (torch.from_numpy(ref).to(dev), torch.from_numpy(rpose).to(dev), [torch.from_numpy(x).to(dev) for x in meas],
             [torch.from_numpy(p).to(dev) for p in mpose], torch.from_numpy(K).to(dev))
    real = {name: getattr(ops, name) for name in ops_recorded}
    real_run, real_deferred = ops.ConvLayer.run, ops.ConvLayer.run_deferred
    calls, current, rec_stream = {}, [], []

    def within(fn):
        def wrapped(self, *a, **k):
            current.append(self)
            try:
                return fn(self, *a, **k)
            finally:
                current.pop()
        return wrapped

    def recorder(name):
        def record(*a, **kw):
            key = _key(name, a, kw)
            if key not in calls:
                on_rec = bool(rec_stream) and torch.cuda.current_stream(dev) == rec_stream[0]
                args = (list(a[0]),) + a[1:] if isinstance(a[0], list) else a
                calls[key] = (args, kw, current[-1] if current else None, on_rec)
            return real[name](*a, **kw)
        return record

    for name in ops_recorded:
        setattr(ops, name, recorder(name))
    from dvmvs import _native as N
    L = N.lib()
    real_native = {}
    if native is not None:
        count = L.dvmvs_kernel_launch_count

        def native_recorder(sym):
            fn = real_native[sym] = getattr(L, sym)

            def record(*a):
                native[sym] = native.get(sym, 0) + 1
                if sym != "dvmvs_conv2d":
                    return fn(*a)
                before = count()
                rc = fn(*a)
                key = sym + " " + conv2d_branch(a[0]._obj, count() - before)
                native[key] = native.get(key, 0) + 1
                return rc
            return record

        for sym in N.EXPORTED_SYMBOLS:
            if hasattr(L, sym):
                setattr(L, sym, native_recorder(sym))
    ops.ConvLayer.run, ops.ConvLayer.run_deferred = within(real_run), within(real_deferred)
    try:
        eng = pipeline.LookaheadFusionnet(mods, batch=1, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, lookahead=4)
        rec_stream.append(eng.streams[4])
        with torch.no_grad():
            eng.prime(*frame)
        eng.synchronize()
    finally:
        for name, fn in real.items():
            setattr(ops, name, fn)
        for sym, fn in real_native.items():
            setattr(L, sym, fn)
        ops.ConvLayer.run, ops.ConvLayer.run_deferred = real_run, real_deferred
    return mods, calls
