"""Records the native calls bench.py's default engine makes while it primes: used by tools/tc_bench.py to time each layer alone and
by tests/test_tc_reference.py to check each layer against an fp64 reference."""
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
    return name, id(a[1]), tuple(a[0][0].shape), bool(kw.get("defer_finish"))


def engine_calls(ops_recorded=("conv2d_tc",), height=None, width=None, device="cuda"):
    """Builds and primes bench.py's default engine (seed-7 weights, tensor-core backend with 1-term operands; bench.py's input
    size unless height / width are given) with every call of the named functions of dvmvs._ops ("conv2d_tc", "conv2d_halo",
    "expand_dwconv", "lstm_gates", "plane_sweep_tc") recorded: returns (mods, {key: (args, kwargs, ConvLayer or None, on the recurrent stage?)}).
    The recorded tensors are the engine's own buffers: their contents are whatever the engine left in them."""
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
        ops.ConvLayer.run, ops.ConvLayer.run_deferred = real_run, real_deferred
    return mods, calls
