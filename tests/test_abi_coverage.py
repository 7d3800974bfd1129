"""Every entry point the native library exports is checked element-wise against fp64, or bit for bit against an oracle, by a named
test -- or is a host-only query, or carries a named exemption.  Runs without a GPU: it reads the export list and the test modules.

ABI_TESTS extends the engine's map (tests/test_engine_coverage.py ENTRY_TESTS, which covers what bench.py's engine launches) with the
training-step kernels, the TSDF fusion, mesh extraction and ray casting, and the device preprocessing; an exported symbol in none of
ABI_TESTS, HOST_ONLY and EXEMPT fails test_every_exported_symbol_is_covered."""
import importlib

from tests.test_engine_coverage import ENTRY_TESTS, HOST_ONLY as ENGINE_HOST_ONLY

ABI_TESTS = {k: v for k, v in ENTRY_TESTS.items() if " " not in k}      # the engine's map without its dvmvs_conv2d branches
ABI_TESTS.update({
    "dvmvs_plane_sweep_fused": "tests.test_sweep_reference::test_sweep_kernels_vs_fp64_reference",
    "dvmvs_hidden_warp_backward": "tests.test_geometry_reference::test_hidden_warp_vs_fp64_reference",
    "dvmvs_preprocess_rgb": "tests.test_gpu_parity::test_device_preprocessing_vs_cv2_host_path",
    "dvmvs_tsdf_integrate": "tests.test_tsdf::test_gpu_volume_equals_reference_goldens_bit_for_bit",
    "dvmvs_mesh_count": "tests.test_mesh::test_gpu_random_volume_equals_oracle",
    "dvmvs_mesh_extract": "tests.test_mesh::test_gpu_random_volume_equals_oracle",
    "dvmvs_tsdf_raycast": "tests.test_raycast::test_gpu_random_smooth_volume_equals_oracle",
    "dvmvs_plane_sweep_backward": "tests.test_training_reference::test_plane_sweep_backward_vs_fp64_reference",
    "dvmvs_lstm_gates_backward": "tests.test_training_reference::test_lstm_gates_backward_vs_fp64_reference",
    "dvmvs_depth_loss_forward": "tests.test_training_reference::test_depth_loss_vs_fp64_reference",
    "dvmvs_depth_loss_backward": "tests.test_training_reference::test_depth_loss_vs_fp64_reference",
})
HOST_ONLY = set(ENGINE_HOST_ONLY) | {
    "dvmvs_mesh_scratch_bytes",                 # scratch size of an extraction, computed on the host
    "dvmvs_plane_sweep_tc_set_timeline",        # registers a device buffer for timing stamps; launches nothing
}
EXEMPT = {
    "dvmvs_plane_sweep_fused_h16": "experimental, opt-in fp16-gather sweep (DVMVS_SWEEP_FP16=1); no default path launches it",
}


def unmapped(exported, tests=None):
    """the exported symbols that are neither mapped to a test nor host-only nor exempt"""
    tests = ABI_TESTS if tests is None else tests
    return sorted(s for s in exported if s not in tests and s not in HOST_ONLY and s not in EXEMPT)


def test_every_exported_symbol_is_covered():
    from dvmvs import _native as N
    print()
    for s in N.EXPORTED_SYMBOLS:
        print("%-36s %s" % (s, ABI_TESTS.get(s) or ("host only" if s in HOST_ONLY else "EXEMPT: " + EXEMPT.get(s, "NOT COVERED"))))
    assert not unmapped(N.EXPORTED_SYMBOLS), "exported entry points no test covers: %s" % unmapped(N.EXPORTED_SYMBOLS)
    assert not set(ABI_TESTS) & (HOST_ONLY | set(EXEMPT)) and not HOST_ONLY & set(EXEMPT)
    stale = sorted((set(ABI_TESTS) | HOST_ONLY | set(EXEMPT)) - set(N.EXPORTED_SYMBOLS))
    assert not stale, "mapped names the library does not export: %s" % stale


def test_removing_an_entry_is_reported():
    from dvmvs import _native as N
    for s in ("dvmvs_depth_loss_backward", "dvmvs_tsdf_raycast", "dvmvs_plane_sweep_tc"):
        dropped = {k: v for k, v in ABI_TESTS.items() if k != s}
        assert unmapped(N.EXPORTED_SYMBOLS, dropped) == [s]


def test_coverage_map_names_existing_tests():
    for entry, test in ABI_TESTS.items():
        mod, fn = test.split("::")
        assert callable(getattr(importlib.import_module(mod), fn, None)), "%s: %s does not exist" % (entry, test)
