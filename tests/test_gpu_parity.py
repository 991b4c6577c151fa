"""GPU parity tests proper: the CUDA path (through the C-ABI) vs the oracle and the committed goldens.

Bit-exact bars (integer / byte outputs): uint16 depth given identical float32 prediction, uint8 stereo and normal map
given identical uint16 depth.
"""
import os

import numpy as np
import pytest

from golden.make_golden import FILLS, NORMAL_CASES, STEREO_CASES
from synth import noise_depth_u16, noise_rgb, synth_depth_u16, synth_rgb

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
MODES = ['left-right', 'red-cyan-anaglyph', 'top-bottom', 'cyan-red-reverseanaglyph']


@pytest.fixture(scope="module")
def gold():
    out = {}                                   # the vectors are split over files of less than 1 MB each
    for f in sorted(os.listdir(G)):
        if f.startswith("stereo_normal_golden_") and f.endswith(".npz"):
            out.update(np.load(os.path.join(G, f)))
    return out


def _u16_to_cuda(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).to(dev).view(torch.uint16)


# ----------------------------------------------------------------------------------------------------------------
# goldens (minted from the real reference)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["smooth", "noise", "black", "flat"])
@pytest.mark.parametrize("fill", FILLS)
def test_stereo_matches_reference_golden(cuda_device, gold, name, fill):
    from depthmap_b200.stereoimage_generation import create_stereoimages
    img, dep = gold[f"in_{name}_rgb"], gold[f"in_{name}_depth"]
    for ci, (div, sep, bal, ex) in enumerate(STEREO_CASES):
        res = create_stereoimages(img, dep, div, sep, MODES, bal, ex, fill)
        for m, r in zip(MODES, res):
            want = gold[f"stereo_{name}_{fill}_{ci}_{m}"]
            got = np.asarray(r)
            assert got.shape == want.shape
            assert np.array_equal(got, want), (name, fill, ci, m, int((got != want).sum()))
        # single-mode calls take the direct-pack kernel path
        for m in MODES:
            got = np.asarray(create_stereoimages(img, dep, div, sep, [m], bal, ex, fill)[0])
            assert np.array_equal(got, gold[f"stereo_{name}_{fill}_{ci}_{m}"]), (name, fill, ci, m, "single")


@pytest.mark.parametrize("name", ["smooth", "noise", "black"])
def test_normalmap_matches_reference_golden(cuda_device, gold, name):
    from depthmap_b200.normalmap_generation import create_normalmap
    dep = gold[f"in_{name}_depth"]
    for ci, (pb, sb, qb, inv) in enumerate(NORMAL_CASES):
        got = np.asarray(create_normalmap(dep, pb, sb, qb, inv))
        want = gold[f"normal_{name}_{ci}"]
        assert np.array_equal(got, want), (name, ci, int((got != want).sum()))


def test_normalize_matches_reference_golden(cuda_device):
    import torch
    from depthmap_b200.core import normalize_prediction_batch
    g = np.load(os.path.join(G, "normalize_golden.npz"))
    preds = torch.from_numpy(np.stack([g[f"pred_{i}"] for i in range(6)])).to(cuda_device)
    for inv in (False, True):
        for ci, (clip, far, near) in enumerate([(False, 0.0, 1.0), (True, 0.1, 0.8), (True, 0.0, 0.5)]):
            out = normalize_prediction_batch(preds, inv, clip, "Range", far, near).cpu().numpy()
            for i in range(6):
                assert np.array_equal(out[i], g[f"u16_{i}_{int(inv)}_{ci}"]), (i, inv, ci)


# ----------------------------------------------------------------------------------------------------------------
# oracle on fresh seeded inputs (sizes the oracle finishes in seconds), batched
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fill", FILLS)
@pytest.mark.parametrize("hw", [(40, 130), (33, 518), (17, 1), (5, 2), (16, 1031)])
def test_stereo_batch_vs_oracle(cuda_device, fill, hw):
    import torch
    from depthmap_b200.stereoimage_generation import create_stereoimages_batch
    from oracle import stereo as ost
    h, w = hw
    B = 3
    rgbs = [synth_rgb(h, w, 0), noise_rgb(h, w, 1), synth_rgb(h, w, 2)]
    deps = [synth_depth_u16(h, w, 0), noise_depth_u16(h, w, 1), synth_depth_u16(h, w, 2) // 7 + 100]
    rgbs[2][: h // 2, : w // 2] = 0
    rgb_t = torch.from_numpy(np.stack(rgbs)).to(cuda_device)
    dep_t = _u16_to_cuda(np.stack(deps), cuda_device)
    rng = np.random.default_rng(h * 1000 + w)
    for trial in range(3):
        div = float(rng.uniform(0.05, 15.0))
        sep = float(rng.uniform(-5, 5)) if trial else 0.0
        bal = float(rng.uniform(-1, 1)) if trial else 0.0
        ex = float(rng.choice([1.0, 2.0]))
        mode = MODES[trial % len(MODES)]
        got = create_stereoimages_batch(rgb_t, dep_t, div, sep, [mode], bal, ex, fill)[0].cpu().numpy()
        for b in range(B):
            with np.errstate(all="ignore"):
                want = ost.create_stereoimages(rgbs[b], deps[b], div, sep, [mode], bal, ex, fill, return_arrays=True)[0]
            assert np.array_equal(got[b], want), (fill, hw, b, div, sep, bal, ex, mode, int((got[b] != want).sum()))


def test_stereo_non_u16_depth_and_api_edges(cuda_device):
    from depthmap_b200.stereoimage_generation import create_stereoimages
    from oracle import stereo as ost
    img = noise_rgb(12, 40, 5)
    rng = np.random.default_rng(5)
    for dep in (rng.random((12, 40)).astype(np.float32), rng.random((12, 40)), rng.integers(0, 255, (12, 40)).astype(np.uint8)):
        for fill in ("naive", "polylines_sharp"):
            got = np.asarray(create_stereoimages(img, dep, 3.0, fill_technique=fill)[0])
            want = ost.create_stereoimages(img, dep, 3.0, fill_technique=fill, return_arrays=True)[0]
            assert np.array_equal(got, want), (dep.dtype, fill)
    dep = noise_depth_u16(12, 40, 1)
    assert create_stereoimages(img, dep, 2.5, modes=[]) == []
    with pytest.raises(Exception, match="Unknown mode"):
        create_stereoimages(img, dep, 2.5, modes=["sideways"])
    with pytest.raises(AssertionError):
        create_stereoimages(img, dep[:3], 2.5)
    assert create_stereoimages(img, dep, 2.5, modes="top-bottom")[0].size == (40, 24)


@pytest.mark.parametrize("hw", [(64, 64), (37, 518), (3, 5), (1, 9), (9, 1), (50, 2051), (40, 520), (16, 1032), (33, 8), (5, 512)])
def test_normalmap_batch_vs_oracle(cuda_device, hw):
    from depthmap_b200.normalmap_generation import create_normalmap_batch
    from oracle import normalmap as onm
    h, w = hw
    deps = [synth_depth_u16(h, w, 3), noise_depth_u16(h, w, 4), np.full((h, w), 777, np.uint16)]
    t = _u16_to_cuda(np.stack(deps), cuda_device)
    for (pb, sb, qb, inv) in [(None, 3, None, False), (None, 3, None, True), (None, 5, None, False), (None, None, None, True),
                              (3, 3, 3, False), (None, 31, None, False), (7, 1, None, False)]:
        got = create_normalmap_batch(t, pb, sb, qb, inv).cpu().numpy()
        for b in range(3):
            want = onm.create_normalmap(deps[b], pb, sb, qb, inv, return_array=True)
            assert np.array_equal(got[b], want), (hw, b, pb, sb, qb, inv, int((got[b] != want).sum()))


def test_normalmap_sobel3_full_2048_bit_exact(cuda_device):
    """Every pixel of two 2048^2 maps (smooth and noisy, both signs) through the fused Sobel-3 kernel against the oracle:
    8M+ pixels exercise the fp32-screen / fp64-detour decision of the fast path at its truncation boundaries."""
    from depthmap_b200.normalmap_generation import create_normalmap_batch
    from oracle import normalmap as onm
    deps = [synth_depth_u16(2048, 2048, 11), noise_depth_u16(2048, 2048, 12)]
    t = _u16_to_cuda(np.stack(deps), cuda_device)
    for inv in (False, True):
        got = create_normalmap_batch(t, None, 3, None, inv).cpu().numpy()
        for b in range(2):
            want = onm.create_normalmap(deps[b], None, 3, None, inv, return_array=True)
            assert np.array_equal(got[b], want), (b, inv, int((got[b] != want).sum()))


@pytest.mark.parametrize("hw", [(48, 64), (37, 518), (1, 1), (7, 3)])
def test_normalize_batch_vs_oracle(cuda_device, hw):
    import torch
    from depthmap_b200.core import normalize_prediction_batch
    from oracle import normalmap as onm
    h, w = hw
    rng = np.random.default_rng(h + w)
    preds = [(rng.standard_normal((h, w)) * 10 ** rng.uniform(-4, 4) + rng.uniform(-3, 3)).astype(np.float32) for _ in range(4)]
    preds.append(np.full((h, w), 1.5, np.float32))  # degenerate -> black
    t = torch.from_numpy(np.stack(preds)).to(cuda_device)
    for inv in (False, True):
        for (clip, far, near) in [(False, 0.0, 1.0), (True, 0.2, 0.7)]:
            got, flags = normalize_prediction_batch(t, inv, clip, "Range", far, near, return_flags=True)
            got = got.cpu().numpy()
            for b in range(len(preds)):
                want = onm.normalize_to_u16(preds[b], inv, clip, "Range", far, near)
                assert np.array_equal(got[b], want), (hw, b, inv, clip)
            assert int(flags[-1]) == 1


@pytest.mark.parametrize("hw", [(48, 64), (37, 518), (1, 1), (7, 3), (512, 512)])
def test_normalize_outliers_clip_vs_oracle(cuda_device, hw):
    """CLIPDEPTH_MODE 'Outliers' (src/core.py:200-202): np.percentile bounds from an exact radix select, float64 tail."""
    import warnings
    import torch
    from depthmap_b200.core import normalize_prediction_batch
    from oracle import normalmap as onm
    h, w = hw
    rng = np.random.default_rng(7 * h + w)
    preds = [(rng.standard_normal((h, w)) * 10 ** rng.uniform(-4, 4) + rng.uniform(-3, 3)).astype(np.float32) for _ in range(3)]
    preds.append(np.round(rng.standard_normal((h, w)) * 3).astype(np.float32))   # heavy ties (and +-0)
    preds.append(np.full((h, w), -2.5, np.float32))                              # degenerate -> black
    t = torch.from_numpy(np.stack(preds)).to(cuda_device)
    for inv in (False, True):
        for (far, near) in [(0.05, 0.95), (0.0, 1.0), (0.123456, 0.5), (0.5, 0.5), (0.999, 1.0)]:
            got = normalize_prediction_batch(t, inv, True, "Outliers", far, near).cpu().numpy()
            for b in range(len(preds)):
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")          # the collapsed-range case divides 0 by 0 in numpy
                    want = onm.normalize_to_u16(preds[b], inv, True, "Outliers", far, near)
                assert np.array_equal(got[b], want), (hw, b, inv, far, near, int((got[b] != want).sum()))


# ----------------------------------------------------------------------------------------------------------------
# BASELINE-size properties (no oracle at these sizes beyond one spot row block)
# ----------------------------------------------------------------------------------------------------------------
def test_fullsize_properties_2048(cuda_device):
    import torch
    from depthmap_b200.normalmap_generation import create_normalmap_batch
    from depthmap_b200.stereoimage_generation import create_stereoimages_batch
    from oracle import normalmap as onm
    from oracle import stereo as ost
    h = w = 2048
    rgb = synth_rgb(h, w, 0)
    dep = synth_depth_u16(h, w, 0)
    rgb_t = torch.from_numpy(rgb).to(cuda_device).unsqueeze(0)
    dep_t = _u16_to_cuda(dep, cuda_device).unsqueeze(0)
    # zero divergence: polylines must reproduce the source up to the reference's own 0.45/0.1 px blending
    for fill in FILLS:
        sbs = create_stereoimages_batch(rgb_t, dep_t, 2.5, 0.0, ['left-right'], 0.0, 1.0, fill)[0]
        ana = create_stereoimages_batch(rgb_t, dep_t, 2.5, 0.0, ['red-cyan-anaglyph'], 0.0, 1.0, fill)[0]
        # checksum-of-layouts: anaglyph == (R of left half, G,B of right half) of the SBS result
        L, R = sbs[0, :, :w], sbs[0, :, w:]
        assert torch.equal(ana[0, ..., 0], L[..., 0]) and torch.equal(ana[0, ..., 1:], R[..., 1:]), fill
        # rows are independent: a 16-row strip with the full image's depth range reproduces the same rows
        strip = slice(1000, 1016)
        d_strip = dep[strip].copy()
        d_strip[0, 0], d_strip[0, 1] = dep.min(), dep.max()
        want = ost.create_stereoimages(rgb[strip], d_strip, 2.5, 0.0, ['left-right'], 0.0, 1.0, fill, return_arrays=True)[0]
        got = sbs[0, strip].cpu().numpy()
        assert np.array_equal(got[1:], want[1:]), fill
    # balance extremes: an eye that the reference leaves untouched is the source image
    sbs = create_stereoimages_batch(rgb_t, dep_t, 2.5, 0.0, ['left-right'], -1.0, 1.0, 'polylines_sharp')[0]
    assert torch.equal(sbs[0, :, :w], rgb_t[0])
    n = create_normalmap_batch(dep_t)[0].cpu().numpy()
    want = onm.create_normalmap(dep[:64], return_array=True)
    assert np.array_equal(n[:63], want[:63])
    flat = create_normalmap_batch(torch.zeros_like(dep_t))[0]
    assert bool((flat == torch.tensor([128, 128, 255], dtype=torch.uint8, device=cuda_device)).all())
