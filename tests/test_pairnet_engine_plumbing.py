"""LookaheadPairnet's host logic without a GPU: with DVMVS_DRYRUN=1 (native entry points stubbed, see
test_dryrun_plumbing.py) one group is composed from the engine's exposed stage bodies, eagerly and without graphs, on CPU
tensors.  Checks where keyframe j's inputs land in every block of the group, the shapes each stage hands to the next, that
each keyframe's depth is read from its own rows, and the constructor's argument checks.  Depth values are meaningless here
(the stubs write nothing); the GPU side is tests/test_pairnet_engine.py.  Runs in a subprocess because the switch is read at
import time."""
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
H, W, D, M, T, B = 64, 96, 32, 2, 3, 2
shapes = oracle.state_dict_shapes(D, with_lstm=False)
w = {t: {k: torch.from_numpy(v) for k, v in synth.make_state_dict(shapes[t], seed=1).items()} for t in shapes}
clips = [synth.make_clip(3 + c, T, H, W, M) for c in range(B)]
TB = T * B

def frame(j):
    st = lambda pick: torch.stack([torch.from_numpy(pick(c)) for c in clips])
    ref = lambda c: c["frames"][j][0]
    meas = lambda c, m: c["frames"][j][1][m]
    return (st(lambda c: c["images"][ref(c)]), st(lambda c: c["poses"][ref(c)]), [st(lambda c: c["images"][meas(c, m)]) for m in range(M)],
            [st(lambda c: c["poses"][meas(c, m)]) for m in range(M)], st(lambda c: c["K"]))

frames = [frame(j) for j in range(T)]
for backend in ("fp32", "tc"):
    ops.set_conv_backend(backend, terms=1, stride2=True)
    mods = pipeline.build_modules(w, device="cpu", n_depth_levels=D, pairnet=True)
    grp = pipeline._group_buffers(T, B, H, W, M, "cpu")
    assert tuple(grp["images"].shape) == ((M + 1) * TB, 3, H, W)
    assert torch.equal(grp["ref_pose"], torch.eye(4).repeat(TB, 1, 1)) and float(grp["full_K"][:, 0, 0].min()) > 0
    rows = [pipeline._keyframe_rows(grp, j, B) for j in range(T)]
    for j in range(T):
        pipeline._upload(rows[j], frames[j])
    # keyframe j's rows in every block: reference block, measurement block m, poses, intrinsics
    for j, (ref, rpose, meas, mposes, K) in enumerate(frames):
        lo, hi = j * B, (j + 1) * B
        assert (rows[j]["lo"], rows[j]["hi"]) == (lo, hi)
        assert torch.equal(grp["images"][lo:hi], ref) and torch.equal(grp["ref_pose"][lo:hi], rpose) and torch.equal(grp["full_K"][lo:hi], K)
        for m in range(M):
            assert torch.equal(grp["images"][(m + 1) * TB + lo:(m + 1) * TB + hi], meas[m])
            assert torch.equal(grp["meas_poses"][m][lo:hi], mposes[m])
    # the five stages, composed from the bodies the engine captures, each reading what the earlier ones left in the group
    stages = pipeline._pairnet_group_stages(mods, (0.25, 20.0, D))
    assert [k for k, _ in stages] == ["head", "pyramid", "swept", "enc", "depth"]
    for key, body in stages:
        grp[key] = body(grp)
    assert tuple(grp["ref_cl"].shape) == (TB, 3, H, W)
    assert [t.shape[0] for t in grp["head"]] == [(M + 1) * TB] * len(grp["head"])
    assert [tuple(t.shape) for t in grp["pyramid"]] == [((M + 1) * TB, 32, H // s, W // s) for s in (2, 4, 8, 16)]
    (f2, f4, f8, f16, cv), half_K = grp["swept"]
    assert tuple(f2.shape) == (TB, 32, H // 2, W // 2) and tuple(cv.shape) == (TB, D, H // 2, W // 2) and tuple(half_K.shape) == (TB, 3, 3)
    enc, _ = grp["enc"]
    assert [t.shape[0] for t in enc] == [TB] * 5 and tuple(enc[4].shape) == (TB, 512, H // 32, W // 32)
    assert "input_gates" not in grp
    assert tuple(grp["depth"].shape) == (TB, H, W)
    # each keyframe's depth comes from its own rows: the engine copies grp["depth"][lo:hi] of its keyframe slot
    grp["depth"] = torch.arange(TB, dtype=torch.float32)[:, None, None].expand(TB, H, W).contiguous()
    for j in range(T):
        got = grp["depth"][rows[j]["lo"]:rows[j]["hi"]]
        assert torch.equal(got[:, 0, 0], torch.arange(j * B, (j + 1) * B, dtype=torch.float32)), (j, got[:, 0, 0])
# the constructor's argument checks (raised before any device is touched)
fus = pipeline.build_modules({t: {k: torch.from_numpy(v) for k, v in synth.make_state_dict(s, seed=1).items()}
                              for t, s in oracle.state_dict_shapes(D).items()}, device="cpu", n_depth_levels=D)
for bad, kw in ((fus, {}), (mods, {"lookahead": 0}), (mods, {"n_groups": 1})):
    try:
        pipeline.LookaheadPairnet(bad, batch=B, height=H, width=W, n_measurement_frames=M, n_depth_levels=D, **kw)
    except ValueError as e:
        print("ValueError:", e)
    else:
        raise AssertionError("no ValueError for " + repr(kw or "fusionnet modules"))
print("pairnet plumbing ok")
"""


def test_pairnet_engine_group_composes_without_gpu():
    env = dict(os.environ, DVMVS_DRYRUN="1")
    code = SCRIPT % (REPO, os.path.join(REPO, "deep-video-mvs_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "pairnet plumbing ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
