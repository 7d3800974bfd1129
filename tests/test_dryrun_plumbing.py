"""Host-logic smoke test without a GPU: with DVMVS_DRYRUN=1 the native entry points are replaced by no-op stubs, so the
whole Python side of a keyframe (module wiring, descriptor construction, shape bookkeeping, both conv backends, batched
and per-image feature passes) executes on CPU tensors.  Numerical results are meaningless; the test only checks that the
plumbing runs and produces correctly shaped outputs.  Runs in a subprocess because the switch is read at import time."""
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import sys, torch
sys.path.insert(0, %r); sys.path.insert(0, %r)
import synth_data as synth
from dvmvs import _ops as ops, pipeline
from oracle import dvmvs_oracle as oracle
H, W, D, M = 64, 96, 64, 2
shapes = oracle.state_dict_shapes(D)
w = {t: {k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes[t], seed=1).items()} for t in shapes}
clip = synth.make_clip(0, 2, H, W, M)
for backend in ("fp32", "tc"):
    ops.set_conv_backend(backend, terms=3, stride2=True)
    mods = pipeline.build_modules(w, device="cpu", n_depth_levels=D)
    for batch_features in (True, False):
        st = pipeline.KeyframeState()
        for ref_i, meas_i in clip["frames"]:
            T = torch.from_numpy
            pred, st = pipeline.keyframe(mods, st, T(clip["images"][ref_i])[None], T(clip["poses"][ref_i])[None],
                                         [T(clip["images"][j])[None] for j in meas_i], [T(clip["poses"][j])[None] for j in meas_i],
                                         T(clip["K"])[None], n_depth_levels=D, batch_features=batch_features)
            assert tuple(pred.shape) == (1, H, W), pred.shape
            assert tuple(st.lstm_state[0].shape) == (1, 512, H // 32, W // 32)
    # row f1: measurement features through the feature cache (hits skip FE + FPN; stores after the sweep)
    cache, st = pipeline.FeatureCache(capacity=M + 1), pipeline.KeyframeState()
    for ref_i, meas_i in clip["frames"]:
        T = torch.from_numpy
        pred, st = pipeline.keyframe(mods, st, T(clip["images"][ref_i])[None], T(clip["poses"][ref_i])[None],
                                     [T(clip["images"][j])[None] for j in meas_i], [T(clip["poses"][j])[None] for j in meas_i],
                                     T(clip["K"])[None], n_depth_levels=D, cache=cache, reference_id=ref_i, measurement_ids=meas_i)
        assert tuple(pred.shape) == (1, H, W)
    assert cache.misses == M and cache.hits == M, (cache.hits, cache.misses)      # keyframe 0: M misses; keyframe 1: M hits
    # the online loop: keyframe buffer -> feature cache -> keyframe(); poses 0.15 m apart so that every frame is a keyframe
    import numpy as np
    online = pipeline.OnlineFusionnet(mods, T(clip["K"]), preprocess=lambda i: T(clip["images"][i])[None], n_measurement_frames=M, n_depth_levels=D)
    outs = []
    for i in range(4):
        pose = np.eye(4)
        pose[0, 3] = 0.15 * i
        outs.append(online.push(pose, i))
    assert outs[0] is None and all(tuple(o.shape) == (1, H, W) for o in outs[1:]) and online.responses == [0, 1, 1, 1]
    assert online.cache.misses == 1 and online.cache.hits == 2 + 2
    assert online.push(np.full((4, 4), np.nan), 9) is None and online.responses[-1] == 5
    # the reference-named loss entry points over the fused loss kernels (stubbed here: shapes / bookkeeping only)
    from dvmvs import losses
    gt = torch.rand(2, H, W) + 0.5
    preds = [(torch.rand(2, H // s, W // s) + 0.5).requires_grad_(True) for s in (16, 8, 4, 2, 1)]
    class Recorder(losses.LossMeter):               # the stubbed kernels leave `sums` unwritten: record, do not divide
        def update(self, loss, count):
            self.sum, self.count = loss, count
    meters = [Recorder() for _ in range(4)]
    for training in (True, False):
        out = losses.update_losses(preds, [1, 1, 1, 1, 1], gt, training, *meters, loss_type="L1-inv")
        assert (torch.is_tensor(out) and out.dim() == 0) if training else out == 0
    assert len(losses.calculate_loss(gt, preds[-1])) == 5
    m = losses.LossMeter()
    m.update(6.0, 3)
    m.update(2.0, 1)
    assert (m.sum, m.count, m.avg, m.item_average, repr(m)) == (8.0, 4.0, 2.0, 2.0, "2.0000 (2.0000)")
    # the pipeline engine's stage functions (split MnasNet trunk, sweep / encoder split) compose to a keyframe
    T = torch.from_numpy
    ref_i, meas_i = clip["frames"][0]
    slot = {"ref_image": T(clip["images"][ref_i])[None], "ref_pose": T(clip["poses"][ref_i])[None], "full_K": T(clip["K"])[None],
            "meas_images": [T(clip["images"][j])[None] for j in meas_i], "meas_poses": [T(clip["poses"][j])[None] for j in meas_i]}
    fe = pipeline._stage_fe_tail(mods, slot, pipeline._stage_fe_head(mods, slot))
    assert [tuple(t.shape[1:]) for t in fe] == [(16, H // 2, W // 2), (24, H // 4, W // 4), (40, H // 8, W // 8), (96, H // 16, W // 16), (320, H // 32, W // 32)]
    enc, half_K = pipeline._stage_enc(mods, slot, pipeline._stage_sweep(mods, slot, fe, 0.25, 20.0, D))
    pred, _ = pipeline._stage_rec(mods, pipeline.KeyframeState(), slot, enc, half_K)
    assert tuple(pred.shape) == (1, H, W)
    # LookaheadFusionnet's composition: trunk / pyramid / sweep / encoder over a GROUP of keyframes (block layout: all reference
    # images, then all first measurement images, ...), recurrent stage per keyframe on batch slices of the group's outputs
    for terms in (1, 3):
        ops.set_conv_backend(backend, terms=terms, stride2=True)
        TB = len(clip["frames"])
        blocks = [[T(clip["images"][r])[None] for r, _ in clip["frames"]]] + [[T(clip["images"][ms[m]])[None] for _, ms in clip["frames"]] for m in range(M)]
        images = torch.cat([torch.cat(b, dim=0) for b in blocks], dim=0)
        grp = {"images": images, "ref_image": images[:TB], "meas_images": [images[(m + 1) * TB:(m + 2) * TB] for m in range(M)],
               "ref_pose": torch.cat([T(clip["poses"][r])[None] for r, _ in clip["frames"]]), "full_K": T(clip["K"])[None].repeat(TB, 1, 1),
               "meas_poses": [torch.cat([T(clip["poses"][ms[m]])[None] for _, ms in clip["frames"]]) for m in range(M)]}
        pipeline._stage_side_inputs(grp)
        pyramid = mods["fpn"](*mods["fe"].forward_tail(mods["fe"].forward_head(grp["images"])))
        assert pyramid[0].shape[0] == (M + 1) * TB
        enc, half_K = pipeline._stage_enc(mods, grp, pipeline._sweep_from_pyramid(grp, pyramid, 0, 0.25, 20.0, D))
        assert enc[4].shape[0] == TB and grp["input_gates"].shape[0] == TB
        st = pipeline.KeyframeState()
        for j in range(TB):
            sl = tuple(ops.batch_slice(e, j, j + 1) for e in enc)
            a = getattr(sl[0], "_dvmvs_act", None)
            if backend == "tc" and a is not None and a.pair is not None:
                assert (a.planes is not None) == (terms == 1), "stacked plane views travel with a batch slice only while no lo plane is read"
            view = {"ref_image": grp["ref_image"][j:j + 1], "ref_pose": grp["ref_pose"][j:j + 1], "full_K": grp["full_K"][j:j + 1],
                    "ref_cl": grp["ref_cl"][j:j + 1], "lstm_K": grp["lstm_K"][j:j + 1], "input_gates": grp["input_gates"][j:j + 1]}
            pred, st = pipeline._stage_rec(mods, st, view, sl, half_K[j:j + 1])
            assert tuple(pred.shape) == (1, H, W)
# pairnet: no ConvLSTM, the decoder reads the encoder's bottom and no recurrent state is carried
shapes = oracle.state_dict_shapes(D, with_lstm=False)
w = {t: {k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes[t], seed=1).items()} for t in shapes}
mods = pipeline.build_modules(w, device="cpu", n_depth_levels=D, pairnet=True)
pred, st = pipeline.keyframe(mods, pipeline.KeyframeState(), T(clip["images"][ref_i])[None], T(clip["poses"][ref_i])[None],
                             [T(clip["images"][j])[None] for j in meas_i], [T(clip["poses"][j])[None] for j in meas_i],
                             T(clip["K"])[None], n_depth_levels=D)
assert tuple(pred.shape) == (1, H, W) and st.lstm_state is None
print("dryrun ok")
"""


def test_keyframe_plumbing_runs_without_gpu():
    env = dict(os.environ, DVMVS_DRYRUN="1")
    code = SCRIPT % (REPO, os.path.join(REPO, "deep-video-mvs_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "dryrun ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
