"""Records the calls the depth engines make at each operating point bench.py reports (POINTS) and at the lookahead engine
configurations tools/pairnet_bench.py and tools/lookahead_cache_bench.py measure (ENGINE_POINTS): used by tools/tc_bench.py to
time each layer alone and by the fp64 reference tests (tests/test_tc_reference.py, tests/test_engine_coverage.py,
tests/test_sweep_reference.py) to check each call on the engine's own buffers, and to list every dvmvs_* entry point of the native
library the engine launches."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (REPO, os.path.join(REPO, "deep-video-mvs_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import numpy as np
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


def branch_of(fn):
    """runs fn, which makes one dvmvs_conv2d call; returns (conv2d_branch of that call, fn's result).  Counts the call's launches
    instead of profiling it: a process that profiles hundreds of calls stops receiving the profiler's kernel records."""
    from dvmvs import _native as N
    L = N.lib()
    real, seen = L.dvmvs_conv2d, []

    def spy(d, stream):
        before = L.dvmvs_kernel_launch_count()
        rc = real(d, stream)
        seen.append(conv2d_branch(d._obj, L.dvmvs_kernel_launch_count() - before))
        return rc
    L.dvmvs_conv2d = spy
    try:
        r = fn()
        torch.cuda.synchronize()
    finally:
        L.dvmvs_conv2d = real
    assert len(seen) == 1, "expected one dvmvs_conv2d call, saw %d" % len(seen)
    return seen[0], r


# bench.py's operating points, keyed by the JSON key each one is reported under ("value": the headline; the others are keys of
# "operating_points"): the engine that produces the number and its configuration.  Unset fields take bench.py's defaults
# (256x256, D = 64, M = 2, 1-term operands, no feature cache).
POINTS = {
    "value": dict(engine="lookahead", batch=1),
    "batched_8": dict(engine="pipelined", batch=8),
    "batched_32": dict(engine="pipelined", batch=32),
    "config_c3_320x256_96planes_4frames": dict(engine="lookahead", batch=1, height=256, width=320, n_depth_levels=96, n_measurement_frames=4),
    "operands_fp16_pairs_3_terms": dict(engine="lookahead", batch=1, terms=3),
    "pipelined_5_stages_no_lookahead": dict(engine="pipelined", batch=1),
    "feature_cache": dict(engine="pipelined", batch=1, feature_cache=8),
    "sequential_latency_ms_per_keyframe": dict(engine="graphed", batch=1),
    "script_sequence": dict(engine="script", batch=1),
}
# operating points bench.py reports that run none of the kernels above, with the test that covers them
NON_KERNEL_POINTS = {
    "tsdf_fusion": "tests/test_tsdf.py: TSDFVolume.integrate bit for bit against the reference's CPU fusion",
}


# The lookahead engines at the configurations tools/pairnet_bench.py and tools/lookahead_cache_bench.py measure, beyond bench.py's
# points: "pairnet" is LookaheadPairnet (pairnet modules: no LSTMFusion; the decoder runs over the whole group), "lookahead" is
# LookaheadFusionnet.  c1 (128x128, D = 32, M = 1) is the only input size whose 1/32 maps are 4x4 (bench.py's smallest are 8x8);
# the pairnet group batches (lookahead x batch, up to 64 keyframes and a 192-image trunk) are bench.py's largest or beyond; the
# feature cache size is lookahead_cache_bench.py's max(30, lookahead x (M + 1)).  (c2, batch 1, lookahead 1), pairnet_bench.py's
# smallest group at c2, has no row: its maps are 8x8 and larger and its batches those of bench.py's batch-1 points, which the
# replays run over POINTS; c1's smallest group is the one whose maps and batches no other configuration reaches.
C1 = dict(height=128, width=128, n_depth_levels=32, n_measurement_frames=1)
C2 = dict(height=256, width=256, n_depth_levels=64, n_measurement_frames=2)
C3 = dict(height=256, width=320, n_depth_levels=96, n_measurement_frames=4)
ENGINE_POINTS = {
    "pairnet_c1_b1_t1": dict(engine="pairnet", batch=1, lookahead=1, **C1),
    "pairnet_c1_b1_t8": dict(engine="pairnet", batch=1, lookahead=8, **C1),
    "pairnet_c1_b8_t8": dict(engine="pairnet", batch=8, lookahead=8, **C1),
    "pairnet_c1_b1_t8_cache": dict(engine="pairnet", batch=1, lookahead=8, feature_cache=30, **C1),
    "pairnet_c2_b1_t4": dict(engine="pairnet", batch=1, lookahead=4, **C2),
    "pairnet_c2_b1_t4_3terms": dict(engine="pairnet", batch=1, lookahead=4, terms=3, **C2),
    "pairnet_c2_b1_t4_cache": dict(engine="pairnet", batch=1, lookahead=4, feature_cache=30, **C2),
    "pairnet_c2_b8_t8": dict(engine="pairnet", batch=8, lookahead=8, **C2),
    "fusionnet_c2_t4_cache": dict(engine="lookahead", batch=1, lookahead=4, feature_cache=30, **C2),
    "fusionnet_c3_t4_cache": dict(engine="lookahead", batch=1, lookahead=4, feature_cache=30, **C3),
}


def point_config(point="value", height=None, width=None):
    """the full configuration of an operating point of POINTS or ENGINE_POINTS (bench.py's defaults filled in; height / width
    override the input size)"""
    import bench
    cfg = dict(engine="lookahead", batch=1, height=bench.H, width=bench.W, n_depth_levels=bench.D, n_measurement_frames=bench.M, terms=1,
               feature_cache=0, lookahead=4, n_stages=5)
    cfg.update(POINTS[point] if point in POINTS else ENGINE_POINTS[point])
    if height is not None:
        cfg["height"] = height
    if width is not None:
        cfg["width"] = width
    return cfg


def group_batch(cfg):
    """rows of one launch of the state-independent stages: lookahead x batch keyframes for the lookahead engines, the batch
    for the others"""
    return cfg["batch"] * (cfg["lookahead"] if cfg["engine"] in ("lookahead", "pairnet") else 1)


def decoder_batch(cfg):
    """the decoder's batch: pairnet decodes a whole group at once; fusionnet decodes each keyframe on its recurrent stage"""
    return group_batch(cfg) if cfg["engine"] == "pairnet" else cfg["batch"]


def last_stage(cfg):
    """what the engine's last stream runs: fusionnet's loop-carried (recurrent) stage, pairnet's decoder over the group"""
    return "decoder stage" if cfg["engine"] == "pairnet" else "recurrent stage"


def trunk_batch(cfg):
    """images per MnasNet trunk launch of the engine's graphs at this point: reference + measurement frames stacked over the
    batch (and over the lookahead group), the reference frames alone when the measurement features come from the cache, one
    image per pass in the script's call sequence"""
    if cfg["engine"] == "script":
        return cfg["batch"]
    per = 1 if cfg["feature_cache"] else cfg["n_measurement_frames"] + 1
    return per * group_batch(cfg)


def trunk_batches(cfg):
    """every batch the MnasNet trunk runs at this point: trunk_batch, and for a lookahead engine with a feature cache also the
    batch itself -- that engine runs the trunk eagerly, at the batch, on each measurement frame that missed the cache (the
    other engines run their misses at the batch of their graphs)"""
    batches = {trunk_batch(cfg)}
    if cfg["feature_cache"] and cfg["engine"] in ("lookahead", "pairnet"):
        batches.add(cfg["batch"])
    return batches


def batch_rows(B):
    """the batch rows a reference is computed for: every row up to 4, else the first two, the middle one and the last one.  Every
    replayed operation computes an output row from its own input row only, so a reference over these rows is exact for them."""
    return list(range(B)) if B <= 4 else sorted({0, 1, B // 2, B - 1})


def _stack(clips, t, M):
    """batched numpy inputs of keyframe t of every clip (bench.stack_frame for any number of measurement frames)"""
    f = [c["frames"][t] for c in clips]
    return (np.stack([c["images"][r] for c, (r, _) in zip(clips, f)]), np.stack([c["poses"][r] for c, (r, _) in zip(clips, f)]),
            [np.stack([c["images"][ms[m]] for c, (_, ms) in zip(clips, f)]) for m in range(M)],
            [np.stack([c["poses"][ms[m]] for c, (_, ms) in zip(clips, f)]) for m in range(M)], np.stack([c["K"] for c in clips]))


def build_modules(n_depth_levels, device, pairnet=False):
    """bench.py's module set, or pairnet's (dvmvs.pairnet.model: no LSTMFusion), with seed-7 synthetic weights; aggregator0 reads
    D + 32 channels, so the modules are built under Config.train_n_depth_levels = D as bench.py does for its c3 point"""
    from dvmvs.config import Config
    from dvmvs.fusionnet import model as fusionnet
    from dvmvs.pairnet import model as pairnet_model
    mm = pairnet_model if pairnet else fusionnet
    saved = Config.train_n_depth_levels
    Config.train_n_depth_levels = n_depth_levels
    try:
        mods = {"fe": mm.FeatureExtractor(), "fpn": mm.FeatureShrinker(), "cve": mm.CostVolumeEncoder(), "cvd": mm.CostVolumeDecoder()}
        if not pairnet:
            mods["lstm"] = fusionnet.LSTMFusion()
    finally:
        Config.train_n_depth_levels = saved
    for m in mods.values():
        shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes, seed=7).items()}, strict=True)
        m.to(device).eval()
    return mods


def _drive(cfg, mods, dev, frames, rec_stream):
    """runs the point's engine the way bench.py, tools/pairnet_bench.py and tools/lookahead_cache_bench.py do before their timed
    regions: prime() for the multi-stream engines (the feature-cache engines prime with unique frame ids: every measurement frame
    misses and runs the eager feature pass), two keyframes for the graphed engine and for the script's call sequence (the
    second one with recurrent state).  Returns the engine (None for the script's call sequence)."""
    from dvmvs import pipeline
    kw = dict(batch=cfg["batch"], height=cfg["height"], width=cfg["width"], n_measurement_frames=cfg["n_measurement_frames"],
              n_depth_levels=cfg["n_depth_levels"])
    with torch.no_grad():
        if cfg["engine"] == "script":
            st = pipeline.KeyframeState()
            for f in frames:
                _, st = pipeline.keyframe(mods, st, *f, n_depth_levels=cfg["n_depth_levels"], batch_features=False)
            torch.cuda.synchronize(dev)
            return None
        if cfg["engine"] == "graphed":
            eng = pipeline.GraphedFusionnet(mods, **kw)
            for f in frames:
                eng.step(*f)
            torch.cuda.synchronize(dev)
            return eng
        if cfg["engine"] in ("lookahead", "pairnet"):
            cls = pipeline.LookaheadPairnet if cfg["engine"] == "pairnet" else pipeline.LookaheadFusionnet
            eng = cls(mods, lookahead=cfg["lookahead"], feature_cache=cfg["feature_cache"], **kw)
        else:
            eng = pipeline.PipelinedFusionnet(mods, n_stages=cfg["n_stages"], feature_cache=cfg["feature_cache"], **kw)
        rec_stream.append(eng.streams[-1])
        eng.prime(*frames[0])
        eng.synchronize()
        return eng


def engine_calls(ops_recorded=("conv2d_tc",), height=None, width=None, device="cuda", native=None, point="value", engine=None):
    """Builds the engine of an operating point (POINTS[point] or ENGINE_POINTS[point]: seed-7 weights, tensor-core backend, the
    point's operand terms, batch, lookahead, feature cache, input size, D and M; height / width override the input size), runs
    it as its benchmark does before timing (_drive) with clip c in batch row c, and records every call of the named functions of
    dvmvs._ops ("conv2d_tc", "conv2d_halo", "expand_dwconv", "lstm_gates", "plane_sweep_tc", ...): returns
    (mods, {key: (args, kwargs, ConvLayer or None, on the engine's last stream (last_stage)?)}).
    Each call site keeps its LAST call -- the one of the steady-state graph the engine replays, with recurrent state where
    the site has one -- on the engine's own buffers: their contents are whatever the engine left in them.
    native: a dict filled with {dvmvs_* entry point: number of calls} of every native call made meanwhile, and for dvmvs_conv2d
    {"dvmvs_conv2d " + conv2d_branch: number of calls}.  engine: a list the driven engine is appended to."""
    cfg = point_config(point, height, width)
    ops.set_conv_backend("tc", terms=cfg["terms"], stride2=True)
    dev = torch.device(device, 0)
    H, W, M, B = cfg["height"], cfg["width"], cfg["n_measurement_frames"], cfg["batch"]
    mods = build_modules(cfg["n_depth_levels"], dev, pairnet=cfg["engine"] == "pairnet")
    clips = [synth.make_clip(c, 2, H, W, M) for c in range(B)]
    frames = []
    for t in range(2):
        ref, rpose, meas, mpose, K = _stack(clips, t, M)
        frames.append((torch.from_numpy(ref).to(dev), torch.from_numpy(rpose).to(dev), [torch.from_numpy(x).to(dev) for x in meas],
                       [torch.from_numpy(p).to(dev) for p in mpose], torch.from_numpy(K).to(dev)))
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
            on_rec = bool(rec_stream) and torch.cuda.current_stream(dev) == rec_stream[0]
            args = (list(a[0]),) + a[1:] if isinstance(a[0], list) else a
            r = real[name](*a, **kw)
            if kw.get("defer_finish") and r is None:
                return r                       # a deferred-finish launch that would not split declines and launches nothing
            calls.pop(key, None)               # the last call, in the order of the last calls
            calls[key] = (args, kw, current[-1] if current else None, on_rec)
            return r
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
        eng = _drive(cfg, mods, dev, frames, rec_stream)
        if engine is not None:
            engine.append(eng)
    finally:
        for name, fn in real.items():
            setattr(ops, name, fn)
        for sym, fn in real_native.items():
            setattr(L, sym, fn)
        ops.ConvLayer.run, ops.ConvLayer.run_deferred = real_run, real_deferred
    return mods, calls
