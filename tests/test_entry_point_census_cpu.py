"""CPU: every entry point include/depthmap_b200.h declares is exercised by name in a test file that runs kernels (a GPU test
file, or test_cabi.py, which calls the loaded library's host entry points), or is listed below with the test that covers it
through a wrapper.  A name that only a CPU test mentions (a string in a fake library's trace, say) does not count: nothing ran
it.  A new entry point without a test fails here."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")

# entry points reached only through a Python wrapper or another entry point: name -> what covers it
INDIRECT = {
    "dm_device_name": "diagnostic string only; the library's exports are checked by test_cabi.py",
    "dm_normalize_u16": "core.normalize_prediction_batch, bit-exact against goldens and the oracle (test_gpu_parity.py)",
    "dm_normalize_u16_workspace_bytes": "sizes the workspace of dm_normalize_u16 (test_gpu_parity.py)",
    "dm_normalize_u16_outliers": "core.normalize_prediction_batch(clipdepth=True) (test_gpu_parity.py::test_normalize_outliers_clip_vs_oracle)",
    "dm_normalize_u16_outliers_workspace_bytes": "sizes the workspace of dm_normalize_u16_outliers (test_gpu_parity.py)",
    "dm_convert_to_i16_f64": "core.convert_to_i16_batch, through the funnel's 16-bit depth input (test_funnel_gpu.py)",
    "dm_stereo": "stereoimage_generation.create_stereoimages_batch, bit-exact against goldens (test_gpu_parity.py)",
    "dm_stereo_workspace_bytes": "sizes the workspace of dm_stereo (test_gpu_parity.py)",
    "dm_stereo_pack": "create_stereoimages_batch's packed modes (test_gpu_parity.py)",
    "dm_depth_to_nd64": "create_stereoimages_batch on non-u16 depth (test_gpu_parity.py::test_stereo_non_u16_depth_and_api_edges)",
    "dm_normalmap": "normalmap_generation.create_normalmap_batch, bit-exact against goldens (test_gpu_parity.py)",
    "dm_normalmap_workspace_bytes": "sizes the workspace of dm_normalmap (test_gpu_parity.py)",
    "dm_video_workspace_bytes": "video_mode.process_predictions_batch, bit-exact (test_video_gpu.py)",
    "dm_video_minmax": "video_mode.process_predictions_batch (test_video_gpu.py)",
    "dm_video_scale_f32": "video_mode.process_predictions_batch (test_video_gpu.py)",
    "dm_video_scale_f64": "video_mode.process_predictions_batch (test_video_gpu.py)",
    "dm_video_select_init": "video_mode.process_predictions_batch's percentile selection (test_video_gpu.py)",
    "dm_video_select_hist": "video_mode.process_predictions_batch's percentile selection (test_video_gpu.py)",
    "dm_video_select_pick": "video_mode.process_predictions_batch's percentile selection (test_video_gpu.py)",
    "dm_video_select_bounds": "video_mode.process_predictions_batch's percentile selection (test_video_gpu.py)",
    "dm_unet_first": "the merge U-Net at its only shape, 1024^2, held to 1e-4 (test_boost_gpu.py::test_merge_unet_vs_oracle)",
    "dm_unet_first_cols": "the merge U-Net (test_boost_gpu.py::test_merge_unet_vs_oracle)",
    "dm_unet_down_cols": "the merge U-Net (test_boost_gpu.py::test_merge_unet_vs_oracle)",
    "dm_unet_up_cols": "the merge U-Net (test_boost_gpu.py::test_merge_unet_vs_oracle)",
    "dm_unet_interleave": "the merge U-Net (test_boost_gpu.py::test_merge_unet_vs_oracle)",
    "dm_unet_final": "the merge U-Net (test_boost_gpu.py::test_merge_unet_vs_oracle)",
    "dm_unet_last": "the merge U-Net (test_boost_gpu.py::test_merge_unet_vs_oracle)",
    "dm_conv3x3_ex": "Ops.conv3x3 without a halo, the zero-padded conv of every fp16 engine (test_tiling_gpu.py::test_circular_conv3x3_vs_torch)",
    "dm_leres_stem_im2col": "the LeReS engine's stem on uint8 images (test_leres_gpu.py::test_leres_vs_oracle)",
    "dm_leres_stem_im2col_f32": "the LeReS stem on one float crop (test_boost_gpu.py::test_leres_on_float_crop_vs_oracle)",
    "dm_leres_stem_im2col_f32_batch": "the LeReS stem on BOOST's batched crops (test_boost_gpu.py::test_estimateboost_vs_oracle)",
}


def declared_entry_points():
    with open(os.path.join(ROOT, "include", "depthmap_b200.h")) as f:
        text = re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)
    return sorted(set(re.findall(r"\b(dm_\w+)\s*\(", text)))


def _test_sources():
    """the test files that run kernels: GPU test files (marked gpu), and test_cabi.py"""
    me = os.path.abspath(__file__)
    out = {}
    for name in sorted(os.listdir(TESTS)):
        path = os.path.join(TESTS, name)
        if name.endswith(".py") and os.path.abspath(path) != me:
            with open(path) as f:
                src = f.read()
            if re.search(r"\bpytest\.mark\.gpu\b", src) or name == "test_cabi.py":
                out[name] = src
    return out


def test_header_parses():
    names = declared_entry_points()
    assert len(names) > 80 and "dm_attention_small_f16" in names and "dm_boost_blend" in names, names


def test_every_entry_point_has_a_test():
    sources = _test_sources()
    missing = [n for n in declared_entry_points()
               if n not in INDIRECT and not any(re.search(r"\b" + n + r"\b", s) for s in sources.values())]
    assert not missing, f"entry points no test calls (add a test, or an INDIRECT entry naming the covering test): {missing}"


def test_indirect_table_is_current():
    """every INDIRECT name is still declared, and none of them has since gained a direct test (then it belongs there)"""
    declared = set(declared_entry_points())
    stale = sorted(set(INDIRECT) - declared)
    assert not stale, f"INDIRECT lists entry points the header no longer declares: {stale}"
    sources = _test_sources()
    direct = sorted(n for n in INDIRECT if any(re.search(r"\b" + n + r"\b", s) for s in sources.values()))
    assert not direct, f"INDIRECT entries that now have a direct test: {direct}"


def test_split_entry_points_are_called_directly():
    """the no_half (split) kernels are each called by name in a GPU test, not only reached through the network"""
    split = [n for n in declared_entry_points() if "split" in n or n == "dm_assemble_tokens_f32"]
    assert len(split) == 7, split
    sources = _test_sources()
    indirect = sorted(set(split) & set(INDIRECT))
    missing = [n for n in split if not any(re.search(r"\b" + n + r"\b", s) for s in sources.values())]
    assert not indirect and not missing, (indirect, missing)
