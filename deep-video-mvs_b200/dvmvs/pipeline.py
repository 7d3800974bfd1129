"""The per-keyframe call sequence of the reference's test drivers (fusionnet/run-testing.py:145-202,
pairnet/run-testing.py:139-164) as a function over the drop-in modules, for callers that do not want to copy
the script's loop body (bench.py, smoke test, examples).  It makes exactly the module / utils calls the script
makes, with the same keyword arguments."""
import os

import torch

from . import _native
from . import _ops as ops
from ._base import no_auto_graph
from .utils import (cost_volume_fusion, get_non_differentiable_rectangle_depth_estimation,
                    get_warp_grid_for_cost_volume_calculation)


class KeyframeState:
    """Recurrent state the caller carries between keyframes of one clip (run-testing.py:86-88)."""

    def __init__(self):
        self.lstm_state = None
        self.previous_depth = None
        self.previous_pose = None

    def reset(self):          # "TRACKING LOST" (run-testing.py:97-101)
        self.__init__()


def build_modules(weights, device="cuda", n_depth_levels=64, pairnet=False):
    """Constructs the modules, strict-loads `weights` (dict 'fe','fpn','cve'[,'lstm'],'cvd' -> state dict), eval()."""
    from .config import Config
    old = Config.train_n_depth_levels
    Config.train_n_depth_levels = n_depth_levels          # aggregator0 has D+32 inputs (fusionnet/model.py:170)
    try:
        if pairnet:
            from .pairnet import model as mm
        else:
            from .fusionnet import model as mm
        mods = {"fe": mm.FeatureExtractor(), "fpn": mm.FeatureShrinker(), "cve": mm.CostVolumeEncoder(), "cvd": mm.CostVolumeDecoder()}
        if not pairnet:
            mods["lstm"] = mm.LSTMFusion()
    finally:
        Config.train_n_depth_levels = old
    for tag, m in mods.items():
        m.load_state_dict(weights[tag], strict=True)
        m.to(device).eval()
    return mods


class FeatureCache:
    """SURVEY section 8 row f1: half-resolution FPN features of past reference frames, keyed by caller-supplied frame ids.

    The reference recomputes FeatureExtractor + FeatureShrinker for every measurement frame of every keyframe
    (run-testing.py:153-156, run-testing-online.py:159-162) although each measurement frame was the reference frame of an
    earlier keyframe (the keyframe buffer only holds past reference frames).  The modules are in eval mode, so those
    features are the same numbers; this cache keeps them in a fixed ring of device buffers (FIFO eviction, capacity =
    the keyframe buffer size, Config.test_keyframe_buffer_size) and hands them back.  Ids are explicit because the scripts
    re-upload the images as fresh tensors each keyframe: nothing on the device identifies a frame without a host sync.
    A miss is not an error -- the caller computes the features from the image and stores them.

    The ring is one device tensor `ring` of capacity + 1 entries (B, h, w, 32), so that a device index tensor can address
    it inside a CUDA graph (the lookahead engines store and gather whole groups with one indexed copy each).  Entry
    `capacity` is a sink no frame id owns: rows of an incomplete group that no keyframe filled store to it and gather from
    it.  Those engines reserve() entries at submit(); a reserved entry is pinned until unpin(), and FIFO eviction skips
    pinned entries."""

    def __init__(self, capacity=30):
        if capacity < 1:
            raise ValueError("FeatureCache capacity must be >= 1")
        self.capacity = int(capacity)
        self.sink = self.capacity
        self.ring = None                          # (capacity + 1, B, h, w, 32), allocated by allocate() or the first store
        self._index = {}                          # frame id -> ring index
        self._owner = [None] * self.capacity
        self._pinned = set()
        self.hits = 0
        self.misses = 0

    def allocate(self, entry_shape, device):
        """Allocates the ring for entries of shape (B, h, w, 32) on `device` (zeros: the sink gathers finite values)."""
        self.ring = torch.zeros((self.capacity + 1,) + tuple(entry_shape), dtype=torch.float32, device=device)

    def clear(self):
        self._index.clear()
        self._owner = [None] * self.capacity
        self._pinned.clear()

    def __contains__(self, frame_id):
        return frame_id in self._index

    def _entry(self, frame_id):
        """Ring index of `frame_id`; a new id takes a free entry or, with the ring full, evicts the oldest id (FIFO, in the
        order ids entered; a re-stored id keeps its age) whose entry no reservation pins."""
        idx = self._index.get(frame_id)
        if idx is None:
            if len(self._index) < self.capacity:
                idx = self._owner.index(None)
            else:
                victim = next((fid for fid, i in self._index.items() if i not in self._pinned), None)
                if victim is None:
                    raise RuntimeError("feature cache: every entry is pinned")
                idx = self._index.pop(victim)
            self._owner[idx] = frame_id
            self._index[frame_id] = idx
        return idx

    def lookup(self, frame_id):
        """Cached (B,32,h,w) API tensor (channels_last view of the ring entry) or None."""
        idx = self._index.get(frame_id)
        if idx is None:
            self.misses += 1
            return None
        self.hits += 1
        return self.ring[idx].permute(0, 3, 1, 2)

    def store(self, frame_id, half_features):
        """Copies (B,32,h,w) features into the ring on the current stream (a D2D copy; the ring outlives the caller's tensor)."""
        src = half_features.permute(0, 2, 3, 1)
        if self.ring is None:
            self.allocate(src.shape, src.device)
        elif self.ring.shape[1:] != src.shape or self.ring.device != src.device:
            raise ValueError("feature cache holds entries of shape %s on %s, got %s on %s"
                             % (tuple(self.ring.shape[1:]), self.ring.device, tuple(src.shape), src.device))
        idx = self._entry(frame_id)
        self.ring[idx].copy_(src)
        return idx

    def reserve(self, frame_id):
        """The ring entry `frame_id` is (or, if absent, will be) stored in, pinned until unpin(): no reservation or store
        evicts it before then.  Nothing is copied; the caller fills a new entry."""
        idx = self._entry(frame_id)
        self._pinned.add(idx)
        return idx

    def unpin(self):
        self._pinned.clear()


def _plane_sweep(f2, meas_half, ref_pose, meas_poses, full_K, min_depth, max_depth, n_depth_levels):
    """Fused plane-sweep cost volume of the reference frame's half-resolution features against the measurement frames'
    (run-testing.py:161-171), with the intrinsics halved to that resolution.  Returns (cost_volume, half_K)."""
    half_K = full_K.clone()
    half_K[:, 0:2, :] = half_K[:, 0:2, :] / 2.0
    cv = cost_volume_fusion(image1=f2, image2s=meas_half, pose1=ref_pose, pose2s=meas_poses, K=half_K, warp_grid=None,
                            min_depth=min_depth, max_depth=max_depth, n_depth_levels=n_depth_levels, device=f2.device,
                            dot_product=True)
    return cv, half_K


def feature_stage(mods, reference_image, reference_pose, measurement_images, measurement_poses, full_K,
                  min_depth=0.25, max_depth=20.0, n_depth_levels=64, batch_features=True, cache=None, reference_id=None,
                  measurement_ids=None):
    """First half of a keyframe -- everything that does not depend on the recurrent state: FeatureExtractor +
    FeatureShrinker on the reference and measurement images and the fused plane-sweep cost volume
    (run-testing.py:153-171).  Returns (f2, f4, f8, f16, cost_volume, half_K).

    With `cache` (FeatureCache) and frame ids, measurement frames whose half-resolution features are cached skip
    FeatureExtractor + FeatureShrinker (row f1); the reference frame's features are stored under `reference_id`."""
    B = reference_image.shape[0]
    if cache is not None:
        if measurement_ids is None or len(measurement_ids) != len(measurement_images):
            raise ValueError("feature cache: need one frame id per measurement image")
        meas_half = [cache.lookup(i) for i in measurement_ids]
        todo = [m for m, t in enumerate(meas_half) if t is None]
        stacked = torch.cat([reference_image] + [measurement_images[m] for m in todo], dim=0) if todo else reference_image
        a2, a4, a8, a16 = mods["fpn"](*mods["fe"](stacked))
        if todo:
            f2, f4, f8, f16 = ops.batch_slice(a2, 0, B), a4[:B], a8[:B], a16[:B]
        else:
            f2, f4, f8, f16 = a2, a4, a8, a16
        for n, m in enumerate(todo):
            meas_half[m] = ops.batch_slice(a2, (n + 1) * B, (n + 2) * B)
    elif batch_features and len(measurement_images) > 0:
        stacked = torch.cat([reference_image] + list(measurement_images), dim=0)
        a2, a4, a8, a16 = mods["fpn"](*mods["fe"](stacked))
        f2, f4, f8, f16 = ops.batch_slice(a2, 0, B), a4[:B], a8[:B], a16[:B]
        meas_half = [ops.batch_slice(a2, (m + 1) * B, (m + 2) * B) for m in range(len(measurement_images))]
    else:
        meas_half = []
        for im in measurement_images:
            half, _, _, _ = mods["fpn"](*mods["fe"](im))
            meas_half.append(half)
        f2, f4, f8, f16 = mods["fpn"](*mods["fe"](reference_image))
    cv, half_K = _plane_sweep(f2, meas_half, reference_pose, measurement_poses, full_K, min_depth, max_depth, n_depth_levels)
    if cache is not None:       # after the sweep: hits are views of ring entries that a store may evict and overwrite
        for m in todo:
            cache.store(measurement_ids[m], meas_half[m])
        if reference_id is not None:
            cache.store(reference_id, f2)
    return f2, f4, f8, f16, cv, half_K


def _stage_rec(mods, state, slot, enc, half_K):
    """The loop-carried stage: depth re-projection + ConvLSTM fusion (fusionnet only) and the decoder, from the cost-volume
    encoder's outputs `enc`.  `slot` holds ref_image, ref_pose and full_K, and optionally what an earlier stage prepared
    off the loop-carried critical path: ref_cl and lstm_K (_stage_side_inputs), input_gates (_stage_enc)."""
    s0, s1, s2, s3, bottom = enc
    reference_image, reference_pose, full_K = slot.get("ref_cl", slot["ref_image"]), slot["ref_pose"], slot["full_K"]
    B, _, H, W = reference_image.shape
    if "lstm" in mods:
        lstm_K = slot.get("lstm_K")
        if lstm_K is None:
            lstm_K = full_K.clone()
            lstm_K[:, 0:2, :] = lstm_K[:, 0:2, :] / 32.0
        if state.previous_depth is not None:
            de = get_non_differentiable_rectangle_depth_estimation(reference_pose_torch=reference_pose, measurement_pose_torch=state.previous_pose,
                                                                   previous_depth_torch=state.previous_depth, full_K_torch=full_K,
                                                                   half_K_torch=half_K, original_height=H, original_width=W)
            de = de[:, :, ::16, ::16].contiguous()      # == F.interpolate(scale_factor=1/16, mode='nearest') (run-testing.py:187-189)
        else:
            de = torch.zeros(size=(B, 1, H // 32, W // 32), device=reference_image.device)
        state.lstm_state = mods["lstm"](current_encoding=bottom, current_state=state.lstm_state, previous_pose=state.previous_pose,
                                        current_pose=reference_pose, estimated_current_depth=de, camera_matrix=lstm_K,
                                        input_gates=slot.get("input_gates"))
        bottom = state.lstm_state[0]
    pred = mods["cvd"](reference_image, s0, s1, s2, s3, bottom)[0]
    state.previous_depth = pred.view(B, 1, H, W)
    state.previous_pose = reference_pose
    return pred, state


def recurrent_stage(mods, state, features, reference_image, reference_pose, full_K):
    """Second half of a keyframe: cost-volume encoder, depth re-projection + ConvLSTM fusion (fusionnet only), decoder
    (run-testing.py:173-202).  `features` is feature_stage()'s return value.  Returns (depth (B,H,W), state)."""
    f2, f4, f8, f16, cv, half_K = features
    enc = mods["cve"](features_half=f2, features_quarter=f4, features_one_eight=f8, features_one_sixteen=f16, cost_volume=cv)
    return _stage_rec(mods, state, {"ref_image": reference_image, "ref_pose": reference_pose, "full_K": full_K}, enc, half_K)


def keyframe(mods, state, reference_image, reference_pose, measurement_images, measurement_poses, full_K,
             min_depth=0.25, max_depth=20.0, n_depth_levels=64, batch_features=True, cache=None, reference_id=None,
             measurement_ids=None):
    """One keyframe for B independent clips (tensors batched on dim 0, all CUDA).  With 'lstm' in mods this is the
    fusionnet loop body, without it the pairnet one.  Returns (depth (B,H,W), state).

    batch_features=True runs FeatureExtractor + FeatureShrinker ONCE over the reference and the M measurement images
    stacked on the batch axis (eval-mode BatchNorm: identical results, 1/(M+1) of the launches); False reproduces the
    script's M+1 separate passes (run-testing.py:153-159).  cache / reference_id / measurement_ids: see FeatureCache."""
    feats = feature_stage(mods, reference_image, reference_pose, measurement_images, measurement_poses, full_K, min_depth,
                          max_depth, n_depth_levels, batch_features, cache, reference_id, measurement_ids)
    return recurrent_stage(mods, state, feats, reference_image, reference_pose, full_K)


class _StaticState:
    """The recurrent state in static device buffers that the captured graphs of the loop-carried stage read and rewrite.
    The only code that knows the buffers' order: h, c, previous depth (B,1,H,W), previous pose."""

    def __init__(self):
        self.buffers = None       # allocated from the first recurrent result

    def allocate(self, state):
        self.buffers = (state.lstm_state[0].clone(), state.lstm_state[1].clone(), state.previous_depth.clone(),
                        state.previous_pose.clone())

    def keyframe_state(self, with_state):
        """A fresh KeyframeState; with_state: over views of the static buffers."""
        st = KeyframeState()
        if with_state:
            h, c, pd, pp = self.buffers
            st.lstm_state, st.previous_depth, st.previous_pose = (h, c), pd, pp
        return st

    def load(self, lstm_state, previous_depth, previous_pose):
        h, c, pd, pp = self.buffers
        with torch.no_grad():
            h.copy_(lstm_state[0])
            c.copy_(lstm_state[1])
            pd.copy_(previous_depth.reshape(pd.shape))
            pp.copy_(previous_pose)

    def write_back(self, state):
        """New recurrent state -> static buffers (read by the next replay)."""
        self.load(state.lstm_state, state.previous_depth, state.previous_pose)

    def snapshot(self):
        return None if self.buffers is None else [t.clone() for t in self.buffers]

    def restore(self, saved):
        if saved is not None:
            for dst, src in zip(self.buffers, saved):
                dst.copy_(src)


def _capture_graph(fn, stream, pdl=None, state=None, depth=None):
    """Warms `fn` up twice on `stream` (allocations, weight packing, function attributes), then captures it there.
    Returns (graph, result of the captured run, kernels of ours in the graph).

    pdl: None keeps the library's programmatic-dependent-launch default, False / True force it off / on for the
    warm-ups and the capture.  `state` (_StaticState) marks the loop-carried stage, whose fn returns (depth, KeyframeState):
    the graph then ends with the copy of the depth into `depth` and of the new state into the static buffers, which are
    allocated from the warm-up's result if need be; the state the buffers held before is put back afterwards."""
    saved = state.snapshot() if state is not None else None
    if pdl is not None:
        _native.lib().dvmvs_set_programmatic_launch(int(pdl))
    try:
        with torch.cuda.stream(stream), torch.no_grad(), no_auto_graph():
            for _ in range(2):
                res = fn()
        stream.synchronize()
        if state is not None and state.buffers is None:
            state.allocate(res[1])
        g = torch.cuda.CUDAGraph()
        n0 = _native.launch_count()
        with torch.no_grad(), torch.cuda.graph(g, stream=stream):
            res = fn()
            if state is not None:
                depth.copy_(res[0])
                state.write_back(res[1])
        n = _native.launch_count() - n0
    finally:
        if pdl is not None:
            _native.lib().dvmvs_set_programmatic_launch(-1)
    if state is not None:
        state.restore(saved)
    return g, res, n


def _take_inputs(slot, frame, reuse, first, last, device, out, hits=None, ring_index=None):
    """Consumes one keyframe's inputs on the caller's current stream, where they were produced: that stream waits for
    `reuse` (the event after which the static buffers of `slot` may be rewritten; None: no wait), copies the inputs into
    them and the engine's first stream is ordered after it.  So work the caller enqueues later on its stream runs after
    the copies: it may overwrite or free CUDA inputs, and pinned host inputs may be rewritten once that stream has passed
    this point.  A CUDA `out`, written on the last stream, is kept alive (caching-allocator wise) until that write has run.
    ring_index: (device buffer, host tensor) of a lookahead engine's feature-cache ring indices, copied with the inputs."""
    caller = torch.cuda.current_stream(device)
    if reuse is not None:
        caller.wait_event(reuse)
    _upload(slot, frame, hits)
    if ring_index is not None:
        ring_index[0].copy_(ring_index[1], non_blocking=True)
    first.wait_stream(caller)
    if out is not None and out.is_cuda:
        out.record_stream(last)


def _upload(slot, frame, hits=None):
    """Copies one keyframe's inputs (CPU-pinned or CUDA) into the static buffers of `slot` on the current stream.
    hits[m]: the feature cache holds measurement frame m, which then needs no image."""
    reference_image, reference_pose, measurement_images, measurement_poses, full_K = frame
    slot["ref_image"].copy_(reference_image, non_blocking=True)
    slot["ref_pose"].copy_(reference_pose, non_blocking=True)
    slot["full_K"].copy_(full_K, non_blocking=True)
    for m, (dst, src) in enumerate(zip(slot["meas_images"], measurement_images)):
        if hits is None or not hits[m]:
            dst.copy_(src, non_blocking=True)
    for dst, src in zip(slot["meas_poses"], measurement_poses):
        dst.copy_(src, non_blocking=True)


def _cache_hits(cache, M, measurement_images, reference_id, measurement_ids):
    """The frame-id rules of submit() for the engines with a feature cache, checked before anything is copied or launched:
    ids only with a cache, one id per measurement frame, and an image for every measurement frame the cache does not hold.
    Returns hits[m] (measurement frame m is cached), or None for an engine without a cache."""
    if cache is None:
        if reference_id is not None or measurement_ids is not None:
            raise ValueError("frame ids given but the engine was built without feature_cache")
        return None
    if measurement_ids is None or len(measurement_ids) != M:
        raise ValueError("feature cache: need %d measurement frame ids" % M)
    hits = [i in cache for i in measurement_ids]
    for m, hit in enumerate(hits):
        if not hit and measurement_images[m] is None:
            raise ValueError("feature cache miss for frame id %r and no image given" % (measurement_ids[m],))
    return hits


def _prime_ids(k, M):
    """Throw-away frame ids of prime()'s k-th keyframe: all misses, so that the miss path is exercised too."""
    return {"reference_id": ("prime", k), "measurement_ids": [("prime-m", k, m) for m in range(M)]}


def _load_state(self, lstm_state, previous_depth, previous_pose):
    """Continue a clip whose first keyframes ran elsewhere (e.g. through the module calls with fewer measurement frames):
    installs (h, c), the previous depth (B,1,H,W) and the previous pose as the recurrent state of the next submit().
    Needs the static state buffers, i.e. prime() or one earlier keyframe."""
    if self._static_state.buffers is None:
        raise RuntimeError("load_state: call prime() (or submit one keyframe) first")
    self.synchronize()
    self._static_state.load(lstm_state, previous_depth, previous_pose)
    torch.cuda.current_stream(self.device).synchronize()
    self._has_state = True


class GraphedFusionnet:
    """The keyframe loop body captured once into CUDA graphs (static shapes) and replayed: removes the ~300 host-side
    launches per keyframe.  Built from the same drop-in modules; two graphs are captured lazily -- keyframe without
    recurrent state (first frame / after reset) and steady state (hidden-state warp + depth re-projection on).

        eng = GraphedFusionnet(mods, batch=B, height=H, width=W, n_measurement_frames=M)
        depth = eng.step(ref_img, ref_pose, [meas_imgs], [meas_poses], full_K)      # CPU (pinned) or CUDA tensors

    step() copies the inputs into static device buffers on the current stream (H2D when they are host tensors),
    replays the graph and returns the static (B,H,W) depth buffer (valid until the next step)."""

    def __init__(self, mods, batch, height, width, n_measurement_frames, min_depth=0.25, max_depth=20.0, n_depth_levels=64,
                 device=None):
        self.mods, self.B, self.H, self.W, self.M = mods, batch, height, width, n_measurement_frames
        self.depth_args = (min_depth, max_depth, n_depth_levels)
        dev = device or next(mods["fe"].parameters()).device
        self.device = dev
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        self.slot = {"ref_image": z(batch, 3, height, width), "ref_pose": z(batch, 4, 4), "full_K": z(batch, 3, 3),
                     "meas_images": [z(batch, 3, height, width) for _ in range(n_measurement_frames)],
                     "meas_poses": [z(batch, 4, 4) for _ in range(n_measurement_frames)]}
        self.state = KeyframeState()
        self._graphs = {}
        self._capture_stream = None
        self.kernels_per_replay = {}
        self._static_state = _StaticState()
        self._out = z(batch, height, width)
        self._has_state = False

    def reset(self):
        self._has_state = False

    def _body(self, with_state):
        slot = self.slot
        return keyframe(self.mods, self._static_state.keyframe_state(with_state), slot["ref_image"], slot["ref_pose"],
                        slot["meas_images"], slot["meas_poses"], slot["full_K"], *self.depth_args)

    def _capture(self, with_state):
        if self._capture_stream is None:
            self._capture_stream = torch.cuda.Stream(device=self.device)
        s = self._capture_stream        # same stream for warm-up and capture: per-stream scratch is allocated outside the graph
        caller = torch.cuda.current_stream(self.device)
        s.wait_stream(caller)
        with torch.cuda.stream(s):      # the snapshot and the restore of the recurrent state around the warm-ups run on s too
            self._graphs[with_state], _, self.kernels_per_replay[with_state] = _capture_graph(
                lambda: self._body(with_state), s, None, self._static_state, self._out)
        caller.wait_stream(s)

    def step(self, reference_image, reference_pose, measurement_images, measurement_poses, full_K):
        if len(measurement_images) != self.M:
            raise ValueError("GraphedFusionnet was built for %d measurement frames, got %d" % (self.M, len(measurement_images)))
        frame = (reference_image, reference_pose, measurement_images, measurement_poses, full_K)
        with_state = self._has_state
        if with_state not in self._graphs:
            if with_state and self._static_state.buffers is None:
                raise RuntimeError("steady-state graph requested before any keyframe ran")
            _upload(self.slot, frame)
            self._capture(with_state)
        _upload(self.slot, frame)
        self._graphs[with_state].replay()
        self._has_state = True
        return self._out


def _stage_side_inputs(slot):
    """Small state-independent preparations the last stage would otherwise do on the loop-carried critical path: the
    channel-last copy of the reference image the decoder's refinement convolutions read, and the 1/32 intrinsics."""
    slot["ref_cl"] = ops.to_api(ops.to_nhwc(slot["ref_image"], "image"))      # (B,3,H,W) view with channels_last strides
    lstm_K = slot["full_K"].clone()
    lstm_K[:, 0:2, :] = lstm_K[:, 0:2, :] / 32.0
    slot["lstm_K"] = lstm_K


def _stacked_images(slot):
    """Reference + measurement images on the batch axis; the reference image alone when the measurement features come
    from the feature cache (slot["meas_half"], row f1)."""
    if slot.get("meas_half") is not None:
        return slot["ref_image"]
    return torch.cat([slot["ref_image"]] + list(slot["meas_images"]), dim=0)


def _stage_fe(mods, slot):
    """Stage 1 of 3: MnasNet trunk on the reference + measurement images stacked on the batch axis."""
    _stage_side_inputs(slot)
    return mods["fe"](_stacked_images(slot))


def _stage_fe_head(mods, slot):
    """MnasNet trunk up to layer3 (1/8 resolution) on the stacked images."""
    _stage_side_inputs(slot)
    return mods["fe"].forward_head(_stacked_images(slot))


def _stage_fe_tail(mods, slot, head):
    """MnasNet layers 4-5 (1/16, 1/32 resolution) from the head's outputs."""
    return mods["fe"].forward_tail(head)


def _sweep_from_pyramid(slot, pyramid, base, min_depth, max_depth, n_depth_levels):
    """Fused plane sweep of ONE keyframe from a feature pyramid whose batch axis stacks [reference, measurement 1..M] x B clips
    starting at row `base` (the lookahead engine's pyramid holds several keyframes)."""
    B = slot["ref_image"].shape[0]
    M = len(slot["meas_images"])
    a2, a4, a8, a16 = pyramid
    if slot.get("meas_half") is not None:         # feature cache: batch = the reference frames only
        f2, f4, f8, f16 = a2, a4, a8, a16
        meas_half = [t.permute(0, 3, 1, 2) for t in slot["meas_half"]]
        slot["ref_half"] = f2                     # the engine copies it into the cache ring after the stage's graph
    else:
        f2, f4, f8, f16 = ops.batch_slice(a2, base, base + B), a4[base:base + B], a8[base:base + B], a16[base:base + B]
        meas_half = [ops.batch_slice(a2, base + (m + 1) * B, base + (m + 2) * B) for m in range(M)]
    cv, half_K = _plane_sweep(f2, meas_half, slot["ref_pose"], slot["meas_poses"], slot["full_K"], min_depth, max_depth, n_depth_levels)
    return (f2, f4, f8, f16, cv), half_K


def _stage_sweep(mods, slot, fe_out, min_depth, max_depth, n_depth_levels):
    """Feature pyramid + fused plane sweep."""
    return _sweep_from_pyramid(slot, mods["fpn"](*fe_out), 0, min_depth, max_depth, n_depth_levels)


def _stage_enc(mods, slot, swept):
    """Cost-volume encoder (still independent of the recurrent state)."""
    (f2, f4, f8, f16, cv), half_K = swept
    enc = mods["cve"](features_half=f2, features_quarter=f4, features_one_eight=f8, features_one_sixteen=f16, cost_volume=cv)
    if "lstm" in mods:      # the input half of the ConvLSTM gate convolution does not depend on the recurrent state either
        slot["input_gates"] = mods["lstm"].lstm_cell.input_gates(enc[4])
    return enc, half_K


def _stage_mid(mods, slot, fe_out, min_depth, max_depth, n_depth_levels):
    """Feature pyramid, fused plane sweep, cost-volume encoder."""
    return _stage_enc(mods, slot, _stage_sweep(mods, slot, fe_out, min_depth, max_depth, n_depth_levels))


# PipelinedFusionnet's stages, each called as fn(engine, slot, output of the previous stage, recurrent state), and its plans.
# Only the last stage of a plan reads the recurrent state; everything before it is independent of the previous keyframe.
_STAGES = {
    "features": lambda e, slot, prev, st: feature_stage(e.mods, slot["ref_image"], slot["ref_pose"], slot["meas_images"],
                                                        slot["meas_poses"], slot["full_K"], *e.depth_args),
    "fe": lambda e, slot, prev, st: _stage_fe(e.mods, slot),
    "head": lambda e, slot, prev, st: _stage_fe_head(e.mods, slot),
    "tail": lambda e, slot, prev, st: _stage_fe_tail(e.mods, slot, prev),
    "mid": lambda e, slot, prev, st: _stage_mid(e.mods, slot, prev, *e.depth_args),
    "sweep": lambda e, slot, prev, st: _stage_sweep(e.mods, slot, prev, *e.depth_args),
    "enc": lambda e, slot, prev, st: _stage_enc(e.mods, slot, prev),
    "rec": lambda e, slot, prev, st: _stage_rec(e.mods, st, slot, *prev),
    "enc+rec": lambda e, slot, prev, st: recurrent_stage(e.mods, st, prev, slot["ref_image"], slot["ref_pose"], slot["full_K"]),
}
_PLANS = {2: ("features", "enc+rec"), 3: ("fe", "mid", "rec"), 4: ("head", "tail", "mid", "rec"),
          5: ("head", "tail", "sweep", "enc", "rec")}
_SWEEP_STAGES = ("features", "mid", "sweep")      # the stages that hold FPN + plane sweep


class PipelinedFusionnet:
    """Throughput engine for ONE clip (or B clips batched): consecutive keyframes are software-pipelined over CUDA streams.
    Only the last stage (depth re-projection, ConvLSTM, decoder) depends on the previous keyframe; everything before it
    -- n_stages=2: [FE + FPN + plane sweep | encoder + ConvLSTM + decoder]; n_stages=3 (default):
    [FE | FPN + plane sweep + encoder | ConvLSTM + decoder]; 4 and 5 split the MnasNet trunk at layer3 and (5) the
    encoder off the plane sweep -- runs ahead for the following keyframes on its own stream.
    Each (stage, slot) is a captured CUDA graph over n_stages-buffered static tensors.  Results are identical to
    GraphedFusionnet / keyframe(): the per-keyframe dataflow is unchanged, only independent work of neighbouring
    keyframes overlaps (tests/test_gpu_parity.py).

        eng = PipelinedFusionnet(mods, batch=B, height=H, width=W, n_measurement_frames=M)
        for frame in stream:  eng.submit(*frame, out=pinned_host_tensor_or_None)
        eng.synchronize()
    """

    def __init__(self, mods, batch, height, width, n_measurement_frames, min_depth=0.25, max_depth=20.0, n_depth_levels=64,
                 device=None, n_stages=3, feature_cache=0):
        if n_stages not in _PLANS:
            raise ValueError("n_stages must be 2, 3, 4 or 5")
        if feature_cache and n_stages < 3:
            raise ValueError("the feature cache needs n_stages >= 3 (feature pyramid + plane sweep in one stage)")
        self.mods, self.B, self.H, self.W, self.M = mods, batch, height, width, n_measurement_frames
        self.depth_args = (min_depth, max_depth, n_depth_levels)
        dev = device or next(mods["fe"].parameters()).device
        self.device = dev
        self.n_stages = n_stages
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        self.slots = []
        for _ in range(n_stages):
            self.slots.append({"ref_image": z(batch, 3, height, width), "ref_pose": z(batch, 4, 4), "full_K": z(batch, 3, 3),
                               "meas_images": [z(batch, 3, height, width) for _ in range(n_measurement_frames)],
                               "meas_poses": [z(batch, 4, 4) for _ in range(n_measurement_frames)],
                               "out": [None] * n_stages, "depth": z(batch, height, width),
                               "graph": [dict() for _ in range(n_stages)],
                               "done": [torch.cuda.Event() for _ in range(n_stages)]})
        # row f1: measurement features from a ring of past reference-frame features instead of M extra FE + FPN passes
        if feature_cache and feature_cache < n_measurement_frames + 1:
            raise ValueError("feature_cache capacity must be at least n_measurement_frames + 1")
        self.cache = FeatureCache(feature_cache) if feature_cache else None
        if self.cache is not None:
            for slot in self.slots:
                slot["meas_half"] = [z(batch, height // 2, width // 2, 32) for _ in range(n_measurement_frames)]
        self._plan = _PLANS[n_stages]
        self._sweep_stage = next(i for i, kind in enumerate(self._plan) if kind in _SWEEP_STAGES)
        # DVMVS_PIPE_PRIO=1 gives the last stage (the one carrying the loop dependence) a high-priority stream; measured
        # slower on the previous architecture, so it is off by default
        prio = os.environ.get("DVMVS_PIPE_PRIO", "0") == "1"
        self.streams = [torch.cuda.Stream(device=dev, priority=(-1 if (prio and i == n_stages - 1) else 0)) for i in range(n_stages)]
        # DVMVS_PIPE_REC_PDL=0: capture the last stage without programmatic dependent launch (its early-launched CTAs then do
        # not sit on SMs waiting for their predecessor while other stages could use them) -- experiment switch
        self._rec_pdl = os.environ.get("DVMVS_PIPE_REC_PDL", "1") == "1"
        # DVMVS_PIPE_PDL=1: capture the stages WITH programmatic dependent launch.  Off by default: with several stage graphs in
        # flight, early-launched CTAs that sit in griddepcontrol.wait hold shared memory and SM slots other stages' kernels
        # could use (measured slower with 5 stages on the previous architecture; a stage replayed alone gains a little from it)
        self._pdl = os.environ.get("DVMVS_PIPE_PDL", "0") == "1"
        if os.environ.get("DVMVS_PIPE_SERIAL") == "1":        # debugging aid: all stages on one stream (no overlap)
            self.streams = [self.streams[0]] * n_stages
        self.stream_a, self.stream_b = self.streams[0], self.streams[-1]      # first / last stage (timing hooks)
        self._static_state = _StaticState()
        self._has_state = False
        self.t = 0
        self._kernels = [0] * n_stages
        self.kernels_per_keyframe = 0

    def reset(self):
        """TRACKING LOST / new clip: drops the recurrent state (the feature cache is keyed by frame id and stays valid)."""
        self._has_state = False

    load_state = _load_state

    def _run_stage(self, i, slot, with_state):
        return _STAGES[self._plan[i]](self, slot, slot["out"][i - 1] if i > 0 else None, self._static_state.keyframe_state(with_state))

    def _capture(self, i, slot, with_state):
        last = i == self.n_stages - 1
        pdl_off = (not self._pdl) or (last and not self._rec_pdl)
        torch.cuda.synchronize(self.device)
        g, res, self._kernels[i] = _capture_graph(lambda: self._run_stage(i, slot, with_state), self.streams[i],
                                                  False if pdl_off else None, *((self._static_state, slot["depth"]) if last else ()))
        if not last:
            slot["out"][i] = res
        slot["graph"][i][with_state if last else False] = g
        torch.cuda.synchronize(self.device)

    # -- steady state ----------------------------------------------------------------------------------------------
    def submit(self, reference_image, reference_pose, measurement_images, measurement_poses, full_K, out=None,
               reference_id=None, measurement_ids=None):
        """Enqueue keyframe t (inputs CPU-pinned or CUDA).  If `out` (pinned host or CUDA tensor (B,H,W)) is given the
        depth is copied into it on the last stage's stream; otherwise read eng.depth_of(t) after synchronisation.

        The engine behaves as if it had consumed its inputs on the caller's current stream at the time of submit(): work
        the caller enqueues later on that stream may overwrite or free the CUDA inputs, and pinned host inputs may be
        rewritten once that stream has passed the submit() (e.g. after torch.cuda.current_stream().synchronize()).  That
        stream also waits, at submit(), until the slot keyframe t - n_stages used has left the pipeline.

        Engines built with feature_cache=N take frame ids: `measurement_ids[m]` names measurement frame m, `reference_id`
        the reference frame.  A measurement frame whose id is in the cache needs no image (pass None): its features are
        copied from the ring; on a miss the features are computed from the image (eagerly, on the sweep stage's stream)
        and cached.  The reference frame's features enter the ring under `reference_id`."""
        n, last = self.n_stages, self.n_stages - 1
        slot = self.slots[self.t % n]
        with_state = self._has_state
        hits = _cache_hits(self.cache, self.M, measurement_images, reference_id, measurement_ids)
        frame = (reference_image, reference_pose, measurement_images, measurement_poses, full_K)
        # slot reuse: keyframe t-n has left the pipeline
        _take_inputs(slot, frame, slot["done"][last], self.streams[0], self.streams[last], self.device, out, hits)
        slot["t"] = self.t
        for i in range(n):
            stream = self.streams[i]
            key = with_state if i == last else False
            with torch.cuda.stream(stream):
                if i > 0:
                    stream.wait_event(slot["done"][i - 1])
                if hits is not None and i == self._sweep_stage:
                    self._fill_measurement_features(slot, measurement_ids, hits)
                if key not in slot["graph"][i]:
                    self._capture(i, slot, with_state)
                slot["graph"][i][key].replay()
                if hits is not None and i == self._sweep_stage and reference_id is not None:
                    self.cache.store(reference_id, slot["ref_half"])
                if i == last and out is not None:
                    out.copy_(slot["depth"], non_blocking=True)
                slot["done"][i].record(stream)
        self._has_state = True
        self.kernels_per_keyframe = sum(self._kernels)
        self.t += 1
        return self.t - 1

    def _fill_measurement_features(self, slot, measurement_ids, hits):
        """Feature-cache engines, on the sweep stage's stream before its graph: slot["meas_half"][m] <- ring entry (hit) or
        <- FeatureShrinker(FeatureExtractor(image)) computed here and stored in the ring (miss)."""
        for m, hit in enumerate(hits):            # hits first: a miss's store may evict the oldest ring entry
            if hit:
                slot["meas_half"][m].copy_(self.cache.lookup(measurement_ids[m]).permute(0, 2, 3, 1))
        for m, hit in enumerate(hits):
            if not hit:
                self.cache.misses += 1
                with torch.no_grad():
                    half, _, _, _ = self.mods["fpn"](*self.mods["fe"](slot["meas_images"][m]))
                self.cache.store(measurement_ids[m], half)
                slot["meas_half"][m].copy_(half.permute(0, 2, 3, 1))

    def prime(self, reference_image, reference_pose, measurement_images, measurement_poses, full_K):
        """Captures every (stage, slot) graph -- including both variants of the last stage -- by running 2*n_stages throw-away
        keyframes, then resets the clip state.  Optional: submit() captures lazily; call this to keep the one-off
        captures out of a timed or latency-sensitive region."""
        for k in range(2 * self.n_stages):
            self.submit(reference_image, reference_pose, measurement_images, measurement_poses, full_K,
                        **(_prime_ids(k, self.M) if self.cache is not None else {}))
        self.synchronize()
        self.reset()
        if self.cache is not None:
            self.cache.clear()
            self.cache.hits = self.cache.misses = 0

    def depth_of(self, t):
        """The (B,H,W) depth buffer of keyframe t, valid after synchronisation until keyframe t + n_stages is submitted.
        Raises KeyError for a t its slot no longer (or not yet) holds."""
        slot = self.slots[t % self.n_stages]
        if slot.get("t") != t:
            raise KeyError("keyframe %r: its slot holds keyframe %r" % (t, slot.get("t")))
        return slot["depth"]

    def flush(self):
        """Nothing is ever held back by this engine (LookaheadFusionnet buffers keyframes; same call there launches them)."""

    def synchronize(self):
        for s in self.streams:
            s.synchronize()


def _group_buffers(T, B, H, W, M, device):
    """Input buffers of one group of T keyframes x B clips (TB = T * B rows) of a lookahead engine: the images stacked
    [reference block | measurement 1 block | ...], TB rows each, and the poses and intrinsics per row, sane until a keyframe
    overwrites them (identity poses, a valid K), so that the rows of an incomplete group always hold finite inputs."""
    TB = T * B
    images = torch.zeros(((M + 1) * TB, 3, H, W), dtype=torch.float32, device=device)
    K0 = torch.tensor([[float(W), 0.0, W / 2.0], [0.0, float(W), H / 2.0], [0.0, 0.0, 1.0]], device=device).repeat(TB, 1, 1)
    eye = lambda: torch.eye(4, dtype=torch.float32, device=device).repeat(TB, 1, 1)
    return {"images": images, "ref_image": images[:TB], "meas_images": [images[(m + 1) * TB:(m + 2) * TB] for m in range(M)],
            "ref_pose": eye(), "full_K": K0, "meas_poses": [eye() for _ in range(M)]}


def _keyframe_rows(grp, j, B):
    """Keyframe j's rows lo:hi of every input block of a group: the views _upload writes its inputs into."""
    lo, hi = j * B, (j + 1) * B
    return {"lo": lo, "hi": hi, "ref_image": grp["ref_image"][lo:hi], "meas_images": [mi[lo:hi] for mi in grp["meas_images"]],
            "ref_pose": grp["ref_pose"][lo:hi], "full_K": grp["full_K"][lo:hi], "meas_poses": [mp[lo:hi] for mp in grp["meas_poses"]]}


def _ring_buffers(grp, cache, T, B, H, W, M):
    """The feature-cache buffers of one group of a lookahead engine: `meas_half`, every keyframe's gathered measurement
    features in the [M][T][B] row order of the measurement image blocks (M views of TB channel-last rows), and `ring_index`,
    the ring entries the group's sweep stage addresses: row 0 the entry each keyframe's reference features are stored in,
    row 1 + m the entry measurement frame m is gathered from.  `ring_table` is its host copy, rewritten at each submit();
    columns no keyframe filled name the sink."""
    device = cache.ring.device
    grp["meas_half_rows"] = torch.zeros((M * T, B, H // 2, W // 2, 32), dtype=torch.float32, device=device)
    grp["meas_half"] = [grp["meas_half_rows"][m * T:(m + 1) * T].view(T * B, H // 2, W // 2, 32) for m in range(M)]
    grp["ring_index"] = torch.full((M + 1, T), cache.sink, dtype=torch.int64, device=device)
    grp["ring_table"] = torch.full((M + 1, T), cache.sink, dtype=torch.int64)
    grp["misses"] = []                    # (keyframe j, measurement m, ring entry) to compute at flush()


def _reserve_keyframe(cache, grp, j, reference_id, measurement_ids, hits):
    """Reserves (and pins) the ring entries keyframe j of the open group reads and stores, writes them into column j of the
    group's host index table, and counts the hits and misses.  Hits are pinned first, so that the entries taken for
    the misses and the reference frame cannot evict them.

    Why evicting here is safe: every ring write and every ring read runs on the sweep stage's stream, in group order --
    the miss stores flush() computes just before the sweep stage's graph, then that graph's store of the reference
    features and its gather of the measurement features.  An entry this reservation evicts can therefore still be read
    only by groups launched earlier, whose gathers precede this group's stores on that stream, or by this group, whose
    own entries are pinned until it is launched."""
    if j == 0:
        grp["ring_table"].fill_(cache.sink)
        grp["misses"] = []
    for want_hit in (True, False):
        for m, hit in enumerate(hits):
            if hit == want_hit:
                grp["ring_table"][1 + m, j] = idx = cache.reserve(measurement_ids[m])
                if not hit:
                    grp["misses"].append((j, m, idx))
    grp["ring_table"][0, j] = cache.sink if reference_id is None else cache.reserve(reference_id)
    cache.hits += sum(hits)
    cache.misses += len(hits) - sum(hits)
    return grp["ring_index"], grp["ring_table"].clone()


def _store_misses(mods, cache, grp, B):
    """The open group's missed measurement frames: FeatureShrinker(FeatureExtractor(image)) of each, eagerly on the current
    (the sweep stage's) stream, into its ring entry, before the sweep stage's graph gathers from the ring."""
    for j, m, idx in grp["misses"]:
        with torch.no_grad():
            half, _, _, _ = mods["fpn"](*mods["fe"](grp["meas_images"][m][j * B:(j + 1) * B]))
        cache.ring[idx].copy_(half.permute(0, 2, 3, 1))
    grp["misses"] = []


def _ring_store(grp, ring):
    """Each keyframe's half-resolution reference features (its B rows of the pyramid's a2) -> its ring entry."""
    a2 = grp["pyramid"][0]
    T = grp["ring_index"].shape[1]
    ring.index_copy_(0, grp["ring_index"][0], a2.permute(0, 2, 3, 1).reshape((T, -1) + tuple(ring.shape[2:])))


def _ring_gather(grp, ring):
    """Every keyframe's measurement features <- their ring entries, into the group's `meas_half` rows."""
    torch.index_select(ring, 0, grp["ring_index"][1:].reshape(-1), out=grp["meas_half_rows"])


def _ring_sweep(grp, ring, depth_args):
    """The sweep stage of a lookahead engine with a feature cache: store, gather, then the plane sweep."""
    _ring_store(grp, ring)
    _ring_gather(grp, ring)
    return _sweep_from_pyramid(grp, grp["pyramid"], 0, *depth_args)


def _group_head(mods, grp):
    """MnasNet trunk up to layer3 over all (M + 1) x TB images of a group -- the TB reference images only when the measurement
    features come from the feature cache -- after the side inputs of the later stages (channel-last reference images, 1/32
    intrinsics)."""
    _stage_side_inputs(grp)
    return mods["fe"].forward_head(grp["ref_image"] if "meas_half" in grp else grp["images"])


def _group_stages(mods, depth_args, cache=None):
    """(key, body) of the stages both lookahead engines run over a whole group, in stream order: trunk head | trunk tail +
    feature pyramid | plane sweep (each row with its own poses) | cost-volume encoder.  body(grp) reads the outputs earlier
    stages left in grp under their keys; its result is stored under `key`.  With a feature cache the plane-sweep stage also
    stores the reference features into the cache's ring and gathers the measurement features from it (_ring_sweep)."""
    if cache is None:
        sweep = lambda grp: _sweep_from_pyramid(grp, grp["pyramid"], 0, *depth_args)
    else:
        sweep = lambda grp: _ring_sweep(grp, cache.ring, depth_args)
    return [("head", lambda grp: _group_head(mods, grp)),
            ("pyramid", lambda grp: mods["fpn"](*mods["fe"].forward_tail(grp["head"]))),
            ("swept", sweep),
            ("enc", lambda grp: _stage_enc(mods, grp, grp["swept"]))]


def _group_decode(mods, grp):
    """Pairnet's decoder over a whole group: the (TB, H, W) depth, keyframe j's in rows j*B:(j+1)*B."""
    enc, _ = grp["enc"]
    return mods["cvd"](grp["ref_cl"], *enc)[0]


def _pairnet_group_stages(mods, depth_args, cache=None):
    """LookaheadPairnet's five stages: _group_stages, then the decoder over the group (no recurrent state to serialise on)."""
    return _group_stages(mods, depth_args, cache) + [("depth", lambda grp: _group_decode(mods, grp))]


def _lookahead_cache(feature_cache, T, B, H, W, M, device):
    """The feature cache of a lookahead engine (None for feature_cache=0), its ring allocated.  One open group pins at most
    T (M + 1) entries, so with at least that many a reservation always finds an entry to take."""
    if not feature_cache:
        return None
    if feature_cache < T * (M + 1):
        raise ValueError("feature_cache must be at least lookahead * (n_measurement_frames + 1) = %d, got %d"
                         % (T * (M + 1), feature_cache))
    cache = FeatureCache(feature_cache)
    cache.allocate((B, H // 2, W // 2, 32), device)
    return cache


class _LookaheadEngine:
    """What LookaheadFusionnet and LookaheadPairnet share.  submit() buffers keyframes into the open group of `lookahead`
    keyframes; flush() launches it: each of the engine's group stages (self.stages, (key, body) pairs) is one CUDA graph per
    group on its own stream, chained by the group's `done` events (done[i]: stream i has run its part of the group), then on
    the last stream, for each buffered keyframe in order, the engine's _keyframe_stage and the copy of the keyframe's depth
    into `out`.  done[4], recorded after that, is what the group's next first submit() waits for.  `kslots` hold each keyframe's rows of its
    group's inputs, its depth buffer and the graphs of its per-keyframe stage (none for pairnet)."""

    n_stages = 5
    _prime_rounds = 1                     # prime() submits _prime_rounds x n_groups x lookahead throw-away keyframes

    def __init__(self, stages, mods, batch, height, width, n_measurement_frames, min_depth, max_depth, n_depth_levels, device,
                 lookahead, n_groups, feature_cache, last_priority=0):
        """stages(mods, depth_args, cache): the engine's group stages.  last_priority: the last stream's priority."""
        if lookahead < 1 or n_groups < 2:
            raise ValueError("lookahead >= 1 and n_groups >= 2 required")
        self.mods, self.B, self.H, self.W, self.M = mods, batch, height, width, n_measurement_frames
        self.depth_args = (min_depth, max_depth, n_depth_levels)
        dev = device or next(mods["fe"].parameters()).device
        self.device = dev
        self.T, self.G = int(lookahead), int(n_groups)
        self.cache = _lookahead_cache(feature_cache, self.T, batch, height, width, n_measurement_frames, dev)
        self.stages = stages(mods, self.depth_args, self.cache)
        n = len(self.stages)
        self.groups, self.kslots = [], []
        for _ in range(self.G):
            grp = _group_buffers(self.T, batch, height, width, n_measurement_frames, dev)
            if self.cache is not None:
                _ring_buffers(grp, self.cache, self.T, batch, height, width, n_measurement_frames)
            grp.update({"graph": [None] * n, "done": [torch.cuda.Event() for _ in range(5)]})
            self.groups.append(grp)
            for j in range(self.T):
                self.kslots.append(dict(_keyframe_rows(grp, j, batch), graph=dict(),
                                        depth=torch.zeros(batch, height, width, dtype=torch.float32, device=dev)))
        self.streams = [torch.cuda.Stream(device=dev, priority=(last_priority if i == 4 else 0)) for i in range(5)]
        self.stream_a, self.stream_b = self.streams[0], self.streams[-1]
        self._has_state = False              # the next submitted keyframe continues a clip (read by the recurrent stage only)
        self._gi, self._fill = 0, 0          # group counter, keyframes buffered in the open group
        self._pending = []                   # (kslot index, with_state, out, t) of the open group
        self.t = 0
        self._kernels = [0] * 5
        self.kernels_per_keyframe = 0

    def _capture(self, fn, stream, pdl=False, *state):
        """_capture_graph on an otherwise idle device.  No PDL by default: it costs throughput with stages in flight (see
        PipelinedFusionnet)."""
        torch.cuda.synchronize(self.device)
        captured = _capture_graph(fn, stream, pdl, *state)
        torch.cuda.synchronize(self.device)
        return captured

    # -- steady state ---------------------------------------------------------------------------------------------------
    def submit(self, reference_image, reference_pose, measurement_images, measurement_poses, full_K, out=None,
               reference_id=None, measurement_ids=None):
        """Buffer keyframe t (inputs CPU-pinned or CUDA): its inputs are copied now, its group's stages are launched when the
        group of `lookahead` keyframes is complete (or at flush() / synchronize()).  If `out` (pinned host or CUDA tensor
        (B,H,W)) is given, the depth is copied into it on the last stream; otherwise read eng.depth_of(t).

        The engine behaves as if it had consumed its inputs on the caller's current stream at the time of submit(): work
        the caller enqueues later on that stream may overwrite or free the CUDA inputs, and pinned host inputs may be
        rewritten once that stream has passed the submit() (e.g. after torch.cuda.current_stream().synchronize()).  At the
        first submit() of a group that stream also waits until the group's previous use has finished.
        Engines built with feature_cache=N take frame ids as PipelinedFusionnet.submit does; every ValueError is raised
        before anything is copied."""
        hits = _cache_hits(self.cache, self.M, measurement_images, reference_id, measurement_ids)
        g = self._gi % self.G
        grp = self.groups[g]
        ki = g * self.T + self._fill
        frame = (reference_image, reference_pose, measurement_images, measurement_poses, full_K)
        ring_index = None if hits is None else _reserve_keyframe(self.cache, grp, self._fill, reference_id, measurement_ids, hits)
        # group reuse: all work of this group's previous use has finished reading its buffers
        _take_inputs(self.kslots[ki], frame, grp["done"][4] if self._fill == 0 else None, self.streams[0], self.streams[4],
                     self.device, out, hits, ring_index)
        self._pending.append((ki, self._has_state, out, self.t))
        self._has_state = True
        self._fill += 1
        self.t += 1
        if self._fill == self.T:
            self.flush()
        return self.t - 1

    def flush(self):
        """Launch the open group (complete or not): stream i runs group stage i, if the engine has one, over the group's
        buffers; the last stream then runs each buffered keyframe's per-keyframe stage and the copy of its depth into `out`,
        in order.  Rows no keyframe filled keep the finite inputs they held before; their results are not read.  Each stream
        is entered once and records one event: at small sizes the host's enqueue cost bounds the engine's rate."""
        if not self._pending:
            return
        grp = self.groups[self._gi % self.G]
        for i, stream in enumerate(self.streams):
            with torch.cuda.stream(stream):
                if i < len(self.stages):
                    key, body = self.stages[i]
                    if i > 0:
                        stream.wait_event(grp["done"][i - 1])
                    if i == 2 and self.cache is not None:
                        _store_misses(self.mods, self.cache, grp, self.B)
                    if grp["graph"][i] is None:
                        grp["graph"][i], grp[key], self._kernels[i] = self._capture(lambda: body(grp), stream)
                    grp["graph"][i].replay()
                if i == 4:
                    for ki, with_state, out, t in self._pending:
                        ks = self.kslots[ki]
                        ks["t"] = t
                        self._keyframe_stage(ks, grp, with_state)
                        if out is not None:
                            out.copy_(ks["depth"], non_blocking=True)
                grp["done"][i].record(stream)
        if self.cache is not None:
            self.cache.unpin()
        n = len(self.stages)          # a full group's share of the group stages' launches + the per-keyframe stage's
        self.kernels_per_keyframe = sum(self._kernels[:n]) / float(self.T) + sum(self._kernels[n:])
        self._pending = []
        self._fill = 0
        self._gi += 1

    def prime(self, reference_image, reference_pose, measurement_images, measurement_poses, full_K):
        """Captures every graph with throw-away keyframes (LookaheadFusionnet: 2 x n_groups x lookahead, so that the slot the
        next clip starts in has both variants of its recurrent stage; LookaheadPairnet: n_groups x lookahead), so that the
        one-off captures stay out of a timed or latency-sensitive region; then resets the clip state and clears the feature
        cache, whose throw-away ids missed."""
        for k in range(self._prime_rounds * self.G * self.T):
            self.submit(reference_image, reference_pose, measurement_images, measurement_poses, full_K,
                        **(_prime_ids(k, self.M) if self.cache is not None else {}))
        self.synchronize()
        self.reset()
        if self.cache is not None:
            self.cache.clear()
            self.cache.hits = self.cache.misses = 0

    def depth_of(self, t):
        """The (B,H,W) depth buffer of keyframe t, valid after synchronisation from the launch of its group (flush()) until
        the launch of the next keyframe in its slot.  Raises KeyError for a t no slot holds: stale, not yet submitted, or
        buffered in a group not launched yet."""
        for ks in self.kslots:
            if ks.get("t") == t:
                return ks["depth"]
        raise KeyError("keyframe %r: no keyframe slot holds its depth" % (t,))

    def synchronize(self):
        self.flush()
        for s in self.streams:
            s.synchronize()


class LookaheadFusionnet(_LookaheadEngine):
    """Throughput engine with everything that does NOT depend on the recurrent state batched over TIME: FeatureExtractor,
    FeatureShrinker, the plane sweep and the cost-volume encoder run once per group of `lookahead` consecutive keyframes
    (lookahead x B "clips", each with its own poses and its own M measurement frames) instead of once per keyframe; only the
    loop-carried stage (depth re-projection, ConvLSTM, decoder) runs keyframe by keyframe, on batch slices of the group's
    encoder outputs.  Every keyframe still gets all of its M + 1 feature passes, its own cost volume and its own encoder pass
    -- without feature_cache nothing is cached or skipped; the state-independent work is merely issued in
    batches the GPU runs far more efficiently than batches of one keyframe (at 8 x 8 .. 64 x 64 maps a single keyframe's
    kernels are one-tile CTAs and launch-bound).  Five streams as in PipelinedFusionnet: trunk head | trunk tail + pyramid |
    plane sweep | encoder | recurrent stage.

    Price: a keyframe's depth is available only after its group is complete (up to `lookahead` - 1 further submits) -- an
    offline / throughput engine, like the reference's run-testing.py loop over a recorded sequence.  submit() buffers; flush()
    (also called by synchronize()) launches an incomplete group.  Same per-sample arithmetic as the other engines; the only
    numerical difference is the split-K decision of a few convolutions, which depends on the batch (as with any batched run:
    <= 1 ulp of fp32 with 3-term operands, rounding flips of the fp16 operands in 1-term mode); the parity tests hold this
    engine to the same bounds against the oracle.

    feature_cache=N (row f1) keeps the half-resolution features of past reference frames in a ring of N entries (at least
    lookahead x (M + 1)) keyed by caller-supplied frame ids, as PipelinedFusionnet(feature_cache=N) does: the trunk and the
    feature pyramid then run over the group's reference images only, and the plane-sweep stage stores them into the ring and
    gathers every keyframe's measurement features from it.  submit() takes reference_id / measurement_ids; a measurement
    frame whose id the engine holds (`frame_id in eng.cache`, earlier keyframes of the open group included) needs no image
    (pass None), a miss is computed from its image at flush().  feature_cache=0 is the engine without a cache.

        eng = LookaheadFusionnet(mods, batch=B, height=H, width=W, n_measurement_frames=M, lookahead=4)
        for frame in stream:  eng.submit(*frame, out=pinned_host_tensor_or_None)
        eng.synchronize()
    """

    _prime_rounds = 2

    def __init__(self, mods, batch, height, width, n_measurement_frames, min_depth=0.25, max_depth=20.0, n_depth_levels=64,
                 device=None, lookahead=4, n_groups=3, feature_cache=0):
        # the recurrent stage's small kernels carry the loop dependence; on a high-priority stream their CTAs are dispatched
        # ahead of the queued CTAs of the batched stages' big grids (DVMVS_LA_PRIO=0: all streams equal)
        prio = os.environ.get("DVMVS_LA_PRIO", "1") == "1"
        super().__init__(_group_stages, mods, batch, height, width, n_measurement_frames, min_depth, max_depth, n_depth_levels,
                         device, lookahead, n_groups, feature_cache, last_priority=(-1 if prio else 0))
        # experiment switch, off: DVMVS_LA_REC_PDL=1 captures the recurrent stage's graph with programmatic dependent launch
        # (measured slower, as for the other stages)
        self._rec_pdl = os.environ.get("DVMVS_LA_REC_PDL", "0") == "1"
        self._static_state = _StaticState()

    def reset(self):
        """New clip / tracking lost: the next submitted keyframe starts without recurrent state (buffered keyframes keep theirs).
        The feature cache is keyed by frame id and stays."""
        self._has_state = False

    load_state = _load_state

    def _run_rec(self, ks, grp, with_state):
        lo, hi = ks["lo"], ks["hi"]
        enc, half_K = grp["enc"]
        view = {"ref_image": ks["ref_image"], "ref_pose": ks["ref_pose"], "full_K": ks["full_K"], "ref_cl": grp["ref_cl"][lo:hi],
                "lstm_K": grp["lstm_K"][lo:hi]}
        if grp.get("input_gates") is not None:
            view["input_gates"] = grp["input_gates"][lo:hi]
        return _stage_rec(self.mods, self._static_state.keyframe_state(with_state), view,
                          tuple(ops.batch_slice(e, lo, hi) for e in enc), half_K[lo:hi])

    def _keyframe_stage(self, ks, grp, with_state):
        """The recurrent stage of keyframe slot `ks` (its graph with or without state), after the group's encoder."""
        s4 = self.streams[4]
        s4.wait_event(grp["done"][3])
        if with_state not in ks["graph"]:
            ks["graph"][with_state], _, self._kernels[4] = self._capture(lambda: self._run_rec(ks, grp, with_state), s4,
                                                                         self._rec_pdl, self._static_state, ks["depth"])
        ks["graph"][with_state].replay()


class LookaheadPairnet(_LookaheadEngine):
    """LookaheadFusionnet's throughput engine for pairnet modules (build_modules(..., pairnet=True)).  Pairnet carries no state
    from one keyframe to the next, so the decoder runs batched over time too: every stage -- trunk head | trunk tail + feature
    pyramid | plane sweep | cost-volume encoder | decoder -- is one CUDA graph per group of `lookahead` x B keyframes, on its
    own stream, chained by per-group events.  Without feature_cache every keyframe gets all of its M + 1 feature passes.
    Same API as LookaheadFusionnet minus load_state, so a caller can swap one for the other:

        eng = LookaheadPairnet(mods, batch=B, height=H, width=W, n_measurement_frames=M, lookahead=4)
        for frame in stream:  eng.submit(*frame, out=pinned_host_tensor_or_None)
        eng.synchronize()

    Each batch row is computed on its own, so a keyframe's depth does not depend on its neighbours in the group; against
    keyframe() the results differ only by the split-K choice of a few convolutions, which depends on the batch.

    feature_cache=N: the feature cache of LookaheadFusionnet(feature_cache=N), with the same frame ids at submit().
    """

    def __init__(self, mods, batch, height, width, n_measurement_frames, min_depth=0.25, max_depth=20.0, n_depth_levels=64,
                 device=None, lookahead=4, n_groups=3, feature_cache=0):
        if "lstm" in mods:
            raise ValueError("LookaheadPairnet runs pairnet modules; fusionnet modules (with 'lstm') go to LookaheadFusionnet")
        # no loop-carried stage to favour: all streams at the same priority
        super().__init__(_pairnet_group_stages, mods, batch, height, width, n_measurement_frames, min_depth, max_depth,
                         n_depth_levels, device, lookahead, n_groups, feature_cache)

    def reset(self):
        """Does nothing: pairnet keyframes carry no state from one to the next, so there is no clip state to drop.  Kept so
        that code written for LookaheadFusionnet (reset() at a new clip or on tracking loss) runs unchanged."""

    def _keyframe_stage(self, ks, grp, with_state):
        """Keyframe slot `ks`'s rows of the group's depth, after the decoder's graph on the same stream."""
        ks["depth"].copy_(grp["depth"][ks["lo"]:ks["hi"]], non_blocking=True)


class OnlineFusionnet:
    """The loop body of fusionnet/run-testing-online.py:103-215 as an object: feed every incoming (pose, image) to push();
    it polls the keyframe buffer (dvmvs.keyframe_buffer.KeyframeBuffer, same selection as the script), and for a new
    keyframe runs one fusionnet keyframe with the selected measurement frames, carrying the recurrent state and resetting
    it on tracking loss (run-testing-online.py:106-113).

    Unlike the script it keys a FeatureCache with the buffer's frame ids (SURVEY section 8 row f1): a measurement frame
    that was a reference frame before is neither pre-processed nor pushed through FeatureExtractor + FeatureShrinker
    again.  Only the buffer's very first frame (stored without a prediction, response 0) ever misses.

        online = OnlineFusionnet(mods, full_K, preprocess=lambda raw: <(1,3,H,W) CUDA tensor>)
        depth = online.push(pose_4x4_numpy, raw_image)        # (1,H,W) CUDA tensor, or None when no keyframe was due

    `preprocess` maps whatever the caller stores in the buffer as "image" (a decoded frame, a file name, ...) to the
    network input; it is called for the reference frame and for cache misses only."""

    def __init__(self, mods, full_K, preprocess, n_measurement_frames=None, min_depth=0.25, max_depth=20.0, n_depth_levels=64,
                 buffer=None, cache_capacity=None):
        from .config import Config
        from .keyframe_buffer import KeyframeBuffer
        self.mods, self.preprocess = mods, preprocess
        self.device = next(mods["fe"].parameters()).device
        self.full_K = full_K.to(self.device).reshape(1, 3, 3).float()
        self.M = Config.test_n_measurement_frames if n_measurement_frames is None else int(n_measurement_frames)
        self.depth_args = (min_depth, max_depth, n_depth_levels)
        self.buffer = buffer if buffer is not None else KeyframeBuffer(
            buffer_size=Config.test_keyframe_buffer_size, keyframe_pose_distance=Config.test_keyframe_pose_distance,
            optimal_t_score=Config.test_optimal_t_measure, optimal_R_score=Config.test_optimal_R_measure, store_return_indices=False)
        self.cache = FeatureCache(cache_capacity or self.buffer.buffer.maxlen)
        self.state = KeyframeState()
        self.responses = []

    def _pose(self, pose):
        import numpy as np
        return torch.from_numpy(np.ascontiguousarray(pose, dtype=np.float32)).reshape(1, 4, 4).to(self.device)

    def push(self, pose, image):
        response = self.buffer.try_new_keyframe(pose, image)
        self.responses.append(response)
        if response == 3:                              # tracking lost: forget the recurrent state (run-testing-online.py:109-113)
            self.state.reset()
        if response != 1:
            return None
        reference_id = self.buffer.last_frame_id
        frames, ids = self.buffer.get_best_measurement_frames(self.M, with_ids=True)
        measurement_images = [None if i in self.cache else self.preprocess(f[1]) for f, i in zip(frames, ids)]
        measurement_poses = [self._pose(f[0]) for f in frames]
        with torch.no_grad():
            pred, self.state = keyframe(self.mods, self.state, self.preprocess(image), self._pose(pose), measurement_images,
                                        measurement_poses, self.full_K, *self.depth_args, cache=self.cache,
                                        reference_id=reference_id, measurement_ids=ids)
        return pred
