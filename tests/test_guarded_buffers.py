"""Every kernel, on its existing fp64 / oracle cases, with every operand and output in a guarded buffer (tests/guarded.py): the
existing tests are re-run unchanged under guard_allocations(), then verify() checks the fringes around every tensor, the inputs'
bytes and the split-K counters.  A masked read of a poisoned fringe or a skipped store shows up as NaN in the existing checks; a
store outside a tensor, a modified input or a counter left set shows up in verify().  Prints, per entry point, the cases run, the
tensors guarded and the fringe bytes verified.

On top of the case lists: bench.py's engine calls at the headline and batch-8 points replayed guarded, the lookahead engine's
batch-slice operands as rows of NaN-poisoned tensors, a sequence of split-K convolutions on one guarded workspace, the scalar
fall-backs of the staging, the fp32 plane sweep and the direct convolution on views 4 bytes off a 16-byte boundary, and the host's
refusal of misaligned pointers where a kernel vectorises."""
import ctypes
import inspect

import pytest
import torch

from tests import guarded as G
from tests.test_abi_coverage import EXEMPT, HOST_ONLY

DEV = "cuda"
gpu = pytest.mark.gpu

# exported symbol -> the test of this module that runs it guarded
GUARDED_TESTS = {
    "dvmvs_conv2d_tc": "test_conv2d_tc_cases_on_one_guarded_workspace",
    "dvmvs_split_planes": "test_fp32_and_staging_cases_guarded",
    "dvmvs_conv2d_halo": "test_halo_cases_guarded",
    "dvmvs_split_blocked": "test_halo_cases_guarded",
    "dvmvs_lstm_gates": "test_lstm_gate_cases_guarded",
    "dvmvs_lstm_gates_parts": "test_lstm_gate_cases_guarded",
    "dvmvs_expand_dwconv": "test_expand_dw_cases_guarded",
    "dvmvs_plane_sweep_tc": "test_sweep_cases_guarded",
    "dvmvs_plane_sweep_fused": "test_sweep_cases_guarded",
    "dvmvs_stem_conv": "test_fp32_and_staging_cases_guarded",
    "dvmvs_dwconv2d": "test_fp32_and_staging_cases_guarded",
    "dvmvs_conv2d": "test_fp32_and_staging_cases_guarded",
    "dvmvs_upsample2x": "test_fp32_and_staging_cases_guarded",
    "dvmvs_nchw_to_nhwc": "test_fp32_and_staging_cases_guarded",
    "dvmvs_nhwc_to_nchw": "test_fp32_and_staging_cases_guarded",
    "dvmvs_hidden_warp": "test_geometry_cases_guarded",
    "dvmvs_hidden_warp_backward": "test_geometry_cases_guarded",
    "dvmvs_depth_reproject": "test_geometry_cases_guarded",
    "dvmvs_plane_sweep_backward": "test_training_cases_guarded",
    "dvmvs_lstm_gates_backward": "test_training_cases_guarded",
    "dvmvs_depth_loss_forward": "test_training_cases_guarded",
    "dvmvs_depth_loss_backward": "test_training_cases_guarded",
    "dvmvs_tsdf_integrate": "test_tsdf_mesh_raycast_preprocess_cases_guarded",
    "dvmvs_mesh_count": "test_tsdf_mesh_raycast_preprocess_cases_guarded",
    "dvmvs_mesh_extract": "test_tsdf_mesh_raycast_preprocess_cases_guarded",
    "dvmvs_tsdf_raycast": "test_tsdf_mesh_raycast_preprocess_cases_guarded",
    "dvmvs_preprocess_rgb": "test_tsdf_mesh_raycast_preprocess_cases_guarded",
}


def unmapped(exported, tests=None):
    tests = GUARDED_TESTS if tests is None else tests
    return sorted(s for s in exported if s not in tests and s not in HOST_ONLY and s not in EXEMPT)


def test_every_exported_symbol_runs_guarded():
    from dvmvs import _native as N
    print()
    for s in N.EXPORTED_SYMBOLS:
        print("%-36s %s" % (s, GUARDED_TESTS.get(s) or ("host only" if s in HOST_ONLY else "EXEMPT: " + EXEMPT.get(s, "NOT GUARDED"))))
    assert not unmapped(N.EXPORTED_SYMBOLS), "exported entry points no guarded test runs: %s" % unmapped(N.EXPORTED_SYMBOLS)
    stale = sorted(set(GUARDED_TESTS) - set(N.EXPORTED_SYMBOLS))
    assert not stale, "mapped names the library does not export: %s" % stale
    assert not set(GUARDED_TESTS) & (HOST_ONLY | set(EXEMPT))
    assert all(callable(globals().get(t)) for t in GUARDED_TESTS.values())


def test_removing_a_guarded_entry_is_reported():
    from dvmvs import _native as N
    for s in ("dvmvs_conv2d_tc", "dvmvs_split_blocked", "dvmvs_mesh_extract"):
        assert unmapped(N.EXPORTED_SYMBOLS, {k: v for k, v in GUARDED_TESTS.items() if k != s}) == [s]


# ------------------------------------------------------------------------------------------------ running existing tests guarded
@pytest.fixture
def ops():
    from dvmvs import _ops
    old = (_ops._BACKEND, _ops._TC_TERMS_BASE, _ops._TC_STRIDE2)
    try:
        yield _ops
    finally:
        _ops.set_conv_backend(old[0], terms=old[1], stride2=old[2])


class Tally:
    """cases run, tensors guarded and fringe bytes verified under one heading"""

    def __init__(self, heading):
        self.heading, self.cases, self.skipped, self.tensors, self.fringe = heading, 0, 0, 0, 0

    def verify(self):
        torch.cuda.synchronize()
        self.tensors += len(G.REGISTRY.guards)
        self.fringe += G.REGISTRY.fringe_bytes_total()
        self.cases += 1
        G.verify()

    def report(self):
        print("\nguarded %-58s %4d cases %6d tensors %9.1f MiB of fringe verified%s" % (
            self.heading, self.cases, self.tensors, self.fringe / 2 ** 20, " (%d skipped)" % self.skipped if self.skipped else ""), flush=True)


def _param_sets(fn):
    """the parameter sets of an existing test's @pytest.mark.parametrize marks, as keyword dicts"""
    sets = [{}]
    for m in getattr(fn, "pytestmark", []):
        if m.name != "parametrize":
            continue
        names = [n.strip() for n in m.args[0].split(",")] if isinstance(m.args[0], str) else list(m.args[0])
        values = []
        for v in m.args[1]:
            v = v.values if type(v).__name__ == "ParameterSet" else (v if len(names) > 1 else (v,))
            values.append(dict(zip(names, v)))
        sets = [dict(s, **v) for s in sets for v in values]
    return sets


def _on_device_guarded(v):
    """what an operand factory returned, with every tensor a guarded input on the GPU (None, numbers and names unchanged)"""
    if isinstance(v, torch.Tensor):
        return G.guard_inputs(v.to(DEV), names=["operand %s" % (tuple(v.shape),)])
    if isinstance(v, (list, tuple)):
        return type(v)(_on_device_guarded(x) for x in v)
    if isinstance(v, dict):
        return {k: _on_device_guarded(x) for k, x in v.items()}
    return v


def rerun(tally, fn, fixtures=None, only=None, factories=()):
    """runs the existing test fn once per parameter set (only: a predicate on the set), each under its own guard_allocations() with
    fn's own module among the proxied ones -- so the buffers the test allocates for its direct C-ABI calls are guarded too -- and
    the operand factories (module, name) returning guarded GPU copies of what they build"""
    import sys
    fixtures = fixtures or {}
    wanted = inspect.signature(fn).parameters
    module = sys.modules[fn.__module__]
    for params in _param_sets(fn):
        if only is not None and not only(params):
            continue
        kw = dict(params, **{k: v for k, v in fixtures.items() if k in wanted})
        real = [(m, name, getattr(m, name)) for m, name in factories]
        for m, name, f in real:
            setattr(m, name, lambda *a, _f=f, **k: _on_device_guarded(_f(*a, **k)))
        try:
            with G.guard_allocations(modules=G.library_modules() + [module]):
                try:
                    fn(**kw)
                except pytest.skip.Exception:
                    tally.skipped += 1
                    continue
                except AssertionError as e:
                    raise AssertionError("%s%s: %s" % (fn.__name__, params, e)) from None
                tally.verify()
        finally:
            for m, name, f in real:
                setattr(m, name, f)


@pytest.fixture(autouse=True)
def ran_guarded(request):
    """after a guarded test: every entry point GUARDED_TESTS maps to it was called, and at least once with every device pointer
    inside a guarded buffer"""
    G.NATIVE.clear()
    yield
    if "gpu" not in request.keywords:
        return
    name = request.node.originalname
    for sym in sorted(s for s, t in GUARDED_TESTS.items() if t == name):
        rec = G.NATIVE.get(sym)
        assert rec is not None, "%s never called %s" % (name, sym)
        assert rec["guarded"] > 0, "%s: no call of %s ran on guarded buffers only (%d calls; %s)" % (name, sym, rec["calls"], rec["unguarded"])
    print("\nnative calls: " + ", ".join("%s %d/%d guarded" % (s.replace("dvmvs_", ""), r["guarded"], r["calls"]) for s, r in sorted(G.NATIVE.items())))


@gpu
@pytest.mark.parametrize("terms", [1, 3])
def test_conv2d_tc_cases_on_one_guarded_workspace(ops, terms):
    """TC_CASES (unsplit, then split-K), the deferred-finish parts and the deferred gate GEMM, one after another on ONE guarded
    workspace: every case within its fp64 bound, every fringe intact and the counters zero after each"""
    from tests import test_tc_reference as T
    t = Tally("conv2d_tc / split_planes terms=%d" % terms)
    seen = []
    real = T.NativeSpy.__exit__

    def spy_exit(self, *exc):
        seen.extend(l["ksplit"] for l in self.tc)
        return real(self, *exc)
    T.NativeSpy.__exit__ = spy_exit
    try:
        with G.guard_allocations() as g:
            ws = g.workspace
            for case in T.TC_CASES:
                T.test_conv2d_tc_vs_fp64_reference(ops, case, terms)
                t.verify()
            T.test_conv2d_tc_deferred_finish_parts(ops, terms)
            t.verify()
            T.test_lstm_deferred_gate_gemm_and_epilogue(ops, terms)
            t.verify()
            assert next(iter(ops._WORKSPACE.values())) is ws, "the calls did not use the guarded workspace"
    finally:
        T.NativeSpy.__exit__ = real
    assert len(set(seen)) >= 3 and 1 in seen, "split counts on the shared workspace: %s" % sorted(set(seen))
    print("\nsplit counts on the shared workspace: %s" % sorted(set(seen)))
    t.report()


@gpu
@pytest.mark.parametrize("terms", [1, 3])
def test_halo_cases_guarded(ops, terms, synth):
    from tests import test_halo_outputs as HO
    from tests import test_tc_reference as T
    t = Tally("conv2d_halo / split_blocked terms=%d" % terms)
    rerun(t, T.test_conv2d_halo_separate_sources_vs_fp64_reference, {"ops": ops, "terms": terms}, only=lambda p: p["terms"] == terms)
    rerun(t, HO.test_halo_output_flags, {"synth": synth}, only=lambda p: p["terms"] == terms)
    rerun(t, HO.test_split_blocked_hi_only_flag, {"synth": synth})
    t.report()


@gpu
def test_lstm_gate_cases_guarded(ops):
    from tests import test_tc_reference as T
    t = Tally("lstm_gates / lstm_gates_parts")
    rerun(t, T.test_lstm_gates_every_instantiation, {"ops": ops})
    rerun(t, T.test_lstm_gates_parts_form, {"ops": ops})
    t.report()


@gpu
def test_expand_dw_cases_guarded():
    from tests import test_expand_dw as E
    t = Tally("expand_dwconv")
    rerun(t, E.test_expand_dw_trunk_shapes)
    rerun(t, E.test_expand_dw_ragged_maps)
    t.report()


@gpu
def test_sweep_cases_guarded(ops):
    from tests import test_sweep_reference as S
    t = Tally("plane_sweep_tc (1, 3 terms) / fused / generic")
    rerun(t, S.test_sweep_kernels_vs_fp64_reference, {"ops": ops})
    t.report()


@gpu
def test_fp32_and_staging_cases_guarded(ops):
    from tests import test_fp32_reference as F
    t = Tally("conv2d / stem / dwconv / upsample2x / transposes / staging")
    for fn in (F.test_conv2d_vs_fp64_reference, F.test_stem_conv_vs_fp64_reference, F.test_dwconv_vs_fp64_reference,
               F.test_upsample2x_vs_fp64_reference, F.test_layout_transposes_exact, F.test_staging_bit_exact,
               F.test_staging_misaligned_view, F.test_concat_planes_three_sources_last_zero_fills, F.test_split_blocked_only_into_two_calls):
        rerun(t, fn, factories=[(F, "_randn")])
    t.report()


@gpu
def test_geometry_cases_guarded(synth):
    from tests import test_geometry_reference as GR
    t = Tally("hidden_warp / hidden_warp_backward / depth_reproject")
    rerun(t, GR.test_hidden_warp_vs_fp64_reference, factories=[(GR, "_t")])
    rerun(t, GR.test_depth_reproject_vs_fp64_reference, {"synth": synth})
    t.report()


@gpu
def test_training_cases_guarded():
    from tests import test_training_reference as TR
    t = Tally("plane_sweep_backward / lstm_gates_backward / depth_loss")
    rerun(t, TR.test_plane_sweep_backward_vs_fp64_reference)
    rerun(t, TR.test_plane_sweep_backward_same_buffer_twice_through_the_abi, factories=[(TR.R, "sweep_case")])
    rerun(t, TR.test_lstm_gates_backward_vs_fp64_reference, factories=[(TR.R, "lstm_case")])
    rerun(t, TR.test_depth_loss_vs_fp64_reference)
    t.report()


@gpu
def test_tsdf_mesh_raycast_preprocess_cases_guarded():
    from tests import test_gpu_parity as P
    from tests import test_mesh as ME
    from tests import test_raycast as RC
    from tests import test_tsdf as TS
    t = Tally("tsdf_integrate / mesh_count / mesh_extract / tsdf_raycast / preprocess_rgb")
    for fn in (TS.test_gpu_volume_equals_reference_goldens_bit_for_bit, ME.test_gpu_ragged_volume_equals_oracle,
               ME.test_gpu_volume_with_a_unit_dimension_has_an_empty_mesh, ME.test_gpu_integrated_golden_case_mesh_equals_oracle,
               RC.test_gpu_ragged_volume_equals_oracle, RC.test_gpu_volume_with_a_unit_dimension_gives_no_hits,
               RC.test_gpu_integrated_golden_case_renders_as_the_oracle, P.test_device_preprocessing_vs_cv2_host_path):
        rerun(t, fn)
    t.report()


# ------------------------------------------------------------------------------------------------ bench.py's engine calls
def _poisoned_rows(v, terms):
    """v (or every tensor in it) as rows of a NaN-poisoned larger tensor along its batch axis: (B,h,w,C) pairs on axis 0, stacked
    (2,B,...) planes and blocked (2,B,C/8,H,W,8) planes on axis 1 -- the stacked forms only for 1-term operands (3-term kernels
    find the lo plane at +B*h*w*C)"""
    if isinstance(v, torch.Tensor):
        if v.dtype == torch.float16 and v.dim() == 4:
            return G.row_slice_of_poisoned(v, 1, 1 + v.shape[0], 0)
        if v.dtype == torch.float16 and v.dim() >= 5 and terms == 1:
            return G.row_slice_of_poisoned(v, 1, 1 + v.shape[1], 1)
        return v
    if isinstance(v, (list, tuple)):
        return type(v)(_poisoned_rows(x, terms) for x in v)
    return v


@gpu
@pytest.mark.parametrize("point", ["value", "batched_8"])
def test_engine_calls_guarded(ops, point):
    """Every conv2d_tc, conv2d_halo, expand_dwconv, ConvLSTM gate and plane_sweep_tc call of bench.py's engine at this point,
    replayed on its recorded operands with every operand and output guarded: the layers against the fp64 reference (the
    helpers of test_every_benchmark_layer_vs_fp64_reference), the sweep bit for bit against its unguarded replay.  Then the
    sweep and every 1-term tensor-core and halo convolution again with their fp16 operands as rows of NaN-poisoned larger tensors
    (what batch_slice hands the lookahead engine's sweep, encoder and decoder: pair planes, stacked planes, blocked planes): bit for
    bit equal to the unguarded replay.  expand_dwconv is not re-run that way: it only runs in the feature trunk, on the trunk's own
    activations, never on a batch slice."""
    from tests import test_tc_reference as T
    from tools.engine_record import batch_rows, engine_calls, layer_names
    mods, calls = engine_calls(("conv2d_tc", "conv2d_halo", "expand_dwconv", "lstm_gates", "plane_sweep_tc"), point=point)
    names = layer_names(mods)
    gates_calls = [v for k, v in calls.items() if k[0] == "lstm_gates" and k[2]]
    t, ts = Tally("engine calls at %s" % point), Tally("engine calls at %s, batch slices of poisoned rows" % point)
    for key, (args, kw, lay, _) in calls.items():
        kind = key[0]
        if kind == "lstm_gates" and key[2]:
            continue
        layer = names.get(id(lay if lay is not None else (args[1] if len(args) > 1 else None)), kind)
        try:
            if kind == "plane_sweep_tc":
                with torch.no_grad():
                    plain = ops.plane_sweep_tc(*args, **kw).clone()
                    with G.guard_allocations():
                        out = ops.plane_sweep_tc(*args, **kw)
                        assert torch.equal(out, plain), "guarded sweep differs from the unguarded replay"
                        t.verify()
                    with G.guard_allocations():
                        out = ops.plane_sweep_tc(*_poisoned_rows(args, kw.get("terms", 3)), **kw)
                        assert torch.equal(out, plain), "sweep on poisoned rows differs from the unguarded replay"
                        ts.verify()
                continue
            if kind in ("conv2d_tc", "conv2d_halo") and not kw.get("defer_finish") and kw.get("terms", 3) == 1:
                with torch.no_grad():
                    plain = [None if x is None else x.clone() for x in getattr(ops, kind)(*args, **kw)]
                    with G.guard_allocations():
                        got = getattr(ops, kind)(_poisoned_rows(args[0], 1), *args[1:], **kw)
                        hi_only = not ops.lo_planes_needed()      # then no launch writes the lo plane of an fp16 output
                        for a, b in zip(got, plain):
                            if a is not None and a.dim() >= 5 and hi_only:
                                a, b = a[0], b[0]
                            assert (a is None) == (b is None) and (a is None or torch.equal(a, b)), \
                                "convolution on poisoned rows differs from the unguarded replay"
                        ts.verify()
            rows = torch.tensor(batch_rows(args[0][0].shape[1] if kind in ("conv2d_tc", "conv2d_halo") else
                                           (args[0].get_planes().shape[1] if kind == "expand_dwconv" else args[1].shape[0])), device=DEV)
            with G.guard_allocations(), T.NativeSpy() as spy:
                if kind == "conv2d_tc" and kw.get("defer_finish"):
                    T._replay_deferred(args, kw, lay, gates_calls[0], spy, rows)
                elif kind == "conv2d_tc":
                    T._replay_tc(args, kw, lay, spy, rows)
                elif kind == "conv2d_halo":
                    T._replay_halo(args, kw, lay, rows)
                elif kind == "expand_dwconv":
                    T._replay_expand(args, kw, rows)
                else:
                    T._replay_gates(args, rows)
                t.verify()
        except AssertionError as e:
            raise AssertionError("%s: %s %s: %s" % (point, layer, kind, e)) from None
    assert t.cases >= 40 and ts.cases >= 2, (t.cases, ts.cases)
    t.report()
    ts.report()


# ------------------------------------------------------------------------------------------------ unaligned storage offsets
def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


@gpu
def test_scalar_fallbacks_on_views_off_a_16_byte_boundary(ops):
    """the entry points whose host code routes a pointer that is not 16-byte aligned to a scalar path, on an input 4 bytes past a
    512-byte boundary: split_planes and split_blocked bit for bit equal to the aligned run, the fp32 plane sweep bit for bit equal
    to its generic kernel, the direct convolution (the depth head declines the pointer) within its fp64 bound"""
    from dvmvs import _native as N
    from tests import fp32_reference as FR
    from tests import test_fp32_reference as F
    from tests import test_sweep_reference as S
    from tools.engine_record import branch_of
    t = Tally("misaligned views: split_planes / split_blocked / plane_sweep_fused / conv2d")
    g = torch.Generator().manual_seed(11)
    with G.guard_allocations():
        for C, up in ((32, False), (24, True), (3, False)):
            x = torch.randn((2, 9, 7, C), generator=g).to(DEV)
            xa, xm = G.guard_inputs(x), G.guard_inputs(x, shift=4)
            assert xa.data_ptr() % 16 == 0 and xm.data_ptr() % 16 == 4
            assert torch.equal(_bits(ops.split_planes(xa, upsample=up)), _bits(ops.split_planes(xm, upsample=up)))
            assert torch.equal(_bits(ops.split_blocked([(xa, up)])), _bits(ops.split_blocked([(xm, up)])))
            t.verify()
        c = S.make_case("partial_tiles")
        f1, f2s = G.guard_inputs(c["f1"].to(DEV)), [G.guard_inputs(f.to(DEV)) for f in c["f2s"]]
        f1m, f2ms = G.guard_inputs(c["f1"].to(DEV), shift=4), [G.guard_inputs(f.to(DEV), shift=4) for f in c["f2s"]]
        args = (c["pose1"].to(DEV), [p.to(DEV) for p in c["pose2s"]], c["K"].to(DEV), S.MIN_DEPTH, S.MAX_DEPTH, c["D"])
        generic = ops.plane_sweep(f1, f2s, *args, force_generic=True)
        fused = ops.plane_sweep(f1m, f2ms, *args)
        assert torch.equal(_bits(generic), _bits(fused)), "fused sweep on misaligned features differs from the generic kernel"
        t.verify()
    with G.guard_allocations():
        case = next(k for k in F.CONV_CASES if k[0] == "head32_16x16_cin128_aux")
        xs, pc, _, _ = F._conv_case(ops, case)
        xm = G.guard_inputs(xs[0], shift=4)
        branch, (out, aux_out) = branch_of(lambda: ops.conv2d([(xm, N.SRC_DIRECT)], pc, aux=case[9]))
        assert branch.startswith("direct"), "the depth head accepted a misaligned source (%s)" % branch
        ref = FR.conv_reference([(F._nchw(xs[0]), False)], pc.weight, 1, pc.bias, None, 0, case[8], case[9],
                                chain=F.conv_chain(branch, pc.cin, [128], 3))
        F.check("misaligned head source, %s" % branch, F._nchw(out), ref.y, ref.bound)
        F.check("misaligned head source aux", F._nchw(aux_out), ref.aux, ref.aux_bound)
        t.verify()
    t.report()


# ------------------------------------------------------------------------------------------------ host alignment checks
def _refused(call, what):
    """call() must fail with RuntimeError naming the alignment, launching nothing"""
    from dvmvs import _native as N
    torch.cuda.synchronize()
    before = N.launch_count()
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        call()
    assert N.launch_count() == before, "%s: launched a kernel before refusing the pointer" % what


@gpu
def test_misaligned_pointers_are_refused_before_any_launch(ops):
    """dvmvs_conv2d_tc (bias, residual, fp32 / fp16-pair / blocked outputs), dvmvs_conv2d_halo (bias, residual, its three outputs) and
    dvmvs_hidden_warp_backward (grad_out, grad_h_in) vectorise through these pointers: a pointer 4 bytes off a 16-byte boundary is refused"""
    from dvmvs import _native as N
    ops.set_conv_backend("tc", terms=3)
    g = torch.Generator().manual_seed(5)
    B, H, W, cin, cout = 1, 8, 8, 32, 64
    x = torch.randn((B, H, W, cin), generator=g).to(DEV)
    pc = ops.PackedConv(torch.randn((cout, cin, 3, 3), generator=g).to(DEV) * 0.05, torch.randn(cout, generator=g).to(DEV), None)
    ptc = ops.PackedConvTC(pc, [cin], DEV)
    planes = ops.split_planes(x)
    buf = torch.zeros(2 * B * H * W * cout * 2 + 16, device=DEV)
    off = lambda n, dtype=torch.float32: buf.view(dtype)[4 // torch.empty((), dtype=dtype).element_size():][:n]
    res = off(B * H * W * cout).view(B, H, W, cout)
    blk = off(2 * B * H * W * cout, torch.float16).view(2, B, cout // 8, H, W, 8)
    _refused(lambda: ops.conv2d_tc([planes], ptc, residual=res, residual_mode=N.RES_SAME, allow_split=False), "conv2d_tc residual")
    _refused(lambda: ops.conv2d_tc([planes], ptc, blk_out=blk, allow_split=False), "conv2d_tc out_blk")
    bias = ptc.bias
    ptc.bias = off(cout)
    _refused(lambda: ops.conv2d_tc([planes], ptc, allow_split=False), "conv2d_tc bias")
    ptc.bias = bias

    def tc_with(field):
        d = N.ConvTcDesc()
        d.src_planes[0], d.src_channels[0], d.n_src = planes.data_ptr(), cin, 1
        d.w_hi, d.w_lo, d.w_rows, d.ktot, d.block_n, d.terms = ptc.w_hi.data_ptr(), ptc.w_lo.data_ptr(), ptc.rows, ptc.ktot, 64, 3
        d.B, d.Hin, d.Win, d.Cout, d.ksize, d.stride = B, H, W, cout, 3, 1
        d.out_f32 = d.out_planes = None
        setattr(d, field, buf.data_ptr() + 4)
        return lambda: N.check(N.lib().dvmvs_conv2d_tc(ctypes.byref(d), ops._stream()), "conv2d_tc")
    for field in ("out_f32", "out_planes"):
        _refused(tc_with(field), "conv2d_tc " + field)

    ph = ops.PackedConvHalo(pc, [cin], DEV)
    src = ops.split_blocked([(x, False)])

    def halo_with(field):
        d = N.ConvHaloDesc()
        d.src_blk[0], d.src_c8[0], d.n_src = src.data_ptr(), ph.src_c8[0], 1
        d.w_hi, d.w_lo, d.n_groups, d.kc, d.block_n, d.terms = ph.w_hi.data_ptr(), ph.w_lo.data_ptr(), ph.n_groups, ph.kc, ph.block_n, 3
        d.B, d.H, d.W, d.Cout, d.ksize, d.act = B, H, W, cout, 3, 0
        d.bias = ph.bias.data_ptr()
        d.out_f32 = buf.data_ptr() if field != "out_f32" else None
        setattr(d, field, buf.data_ptr() + 4)
        return lambda: N.check(N.lib().dvmvs_conv2d_halo(ctypes.byref(d), ops._stream()), "conv2d_halo")
    for field in ("bias", "residual", "out_f32", "out_blk", "out_nhwc"):
        _refused(halo_with(field), "conv2d_halo " + field)

    C = 32
    depth = torch.ones((1, 1, H, W), device=DEV)
    eye = torch.eye(4, device=DEV)[None]
    K = torch.tensor([[[W / 2, 0, W / 2], [0, H / 2, H / 2], [0, 0, 1]]], device=DEV)
    grad_in = torch.empty((1, H, W, C), device=DEV)
    gout = off(H * W * C).view(1, H, W, C)
    _refused(lambda: N.check(N.lib().dvmvs_hidden_warp_backward(gout.data_ptr(), depth.data_ptr(), eye.data_ptr(), eye.data_ptr(), K.data_ptr(),
                                                                 grad_in.data_ptr(), 1, C, H, W, 0.1, ops._stream()), "hidden_warp_backward"),
             "hidden_warp_backward grad_out")
    gout_aligned = torch.randn((1, H, W, C), generator=g).to(DEV)
    grad_in_off = off(H * W * C).view(1, H, W, C)
    _refused(lambda: N.check(N.lib().dvmvs_hidden_warp_backward(gout_aligned.data_ptr(), depth.data_ptr(), eye.data_ptr(), eye.data_ptr(),
                                                                 K.data_ptr(), grad_in_off.data_ptr(), 1, C, H, W, 0.1, ops._stream()),
                             "hidden_warp_backward"), "hidden_warp_backward grad_h_in")
