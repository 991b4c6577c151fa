"""CPU: the C oracle reproduces the committed golden vectors (minted from the real reference by golden/make_golden.py)."""
import os

import numpy as np
import pytest

from oracle import normalmap as onm
from oracle import stereo as ost

G = os.path.join(os.path.dirname(__file__), "golden")
sys_path_ok = True
from golden.make_golden import FILLS, NORMAL_CASES, STEREO_CASES  # noqa: E402

MODES = ['left-right', 'red-cyan-anaglyph', 'top-bottom', 'cyan-red-reverseanaglyph']


@pytest.fixture(scope="module")
def gold():
    out = {}                                   # the vectors are split over files of less than 1 MB each
    for f in sorted(os.listdir(G)):
        if f.startswith("stereo_normal_golden_") and f.endswith(".npz"):
            out.update(np.load(os.path.join(G, f)))
    return out


@pytest.mark.parametrize("name", ["smooth", "noise", "black", "flat"])
@pytest.mark.parametrize("fill", FILLS)
def test_oracle_stereo_matches_golden(gold, name, fill):
    img, dep = gold[f"in_{name}_rgb"], gold[f"in_{name}_depth"]
    for ci, (div, sep, bal, ex) in enumerate(STEREO_CASES):
        with np.errstate(all="ignore"):
            res = ost.create_stereoimages(img, dep, div, sep, MODES, bal, ex, fill, return_arrays=True)
        for m, r in zip(MODES, res):
            assert np.array_equal(r, gold[f"stereo_{name}_{fill}_{ci}_{m}"]), (name, fill, ci, m)


@pytest.mark.parametrize("name", ["smooth", "noise", "black"])
def test_oracle_normalmap_matches_golden(gold, name):
    dep = gold[f"in_{name}_depth"]
    for ci, (pb, sb, qb, inv) in enumerate(NORMAL_CASES):
        r = onm.create_normalmap(dep, pb, sb, qb, inv, return_array=True)
        assert np.array_equal(r, gold[f"normal_{name}_{ci}"]), (name, ci)


def test_oracle_normalize_matches_golden():
    g = np.load(os.path.join(G, "normalize_golden.npz"))
    for i in range(6):
        raw = g[f"pred_{i}"]
        for inv in (False, True):
            for ci, (clip, far, near) in enumerate([(False, 0.0, 1.0), (True, 0.1, 0.8), (True, 0.0, 0.5)]):
                r = onm.normalize_to_u16(raw, inv, clip, "Range", far, near)
                assert np.array_equal(r, g[f"u16_{i}_{int(inv)}_{ci}"]), (i, inv, ci)


def test_oracle_degenerate_prediction_is_black():
    assert onm.normalize_to_u16(np.full((5, 7), 3.25, np.float32)).sum() == 0


def test_oracle_stereo_api_edges():
    img = np.zeros((4, 6, 3), np.uint8)
    dep = np.arange(24, dtype=np.uint16).reshape(4, 6)
    assert ost.create_stereoimages(img, dep, 2.5, modes=[]) == []
    with pytest.raises(Exception, match="Unknown mode"):
        ost.create_stereoimages(img, dep, 2.5, modes=["sideways"])
    with pytest.raises(AssertionError):
        ost.create_stereoimages(img, dep[:3], 2.5)
    out = ost.create_stereoimages(img, dep, 2.5, modes="left-right")
    assert out[0].size == (12, 4)


def test_zoedepth_oracle_path_runs_and_is_flip_symmetric():
    """D7 oracle end to end on the tiny structural configuration (beit_tiny core + metric head + pad / flip TTA): shape, range
    and the exact flip symmetry DepthModel.infer has by construction.  (The head and the TTA wrapper are pinned to the
    reference module in tests/test_oracle_pin.py; the BEiT core is parity-unpinned, see oracle/beit_dpt.py.)"""
    import torch
    from oracle import synth_weights, zoedepth
    from synth import synth_rgb
    core = synth_weights.make_beit_dpt_state_dict("beit_tiny", seed=3)
    feat = core["scratch.layer4_rn.weight"].shape[0]
    outc = core["scratch.output_conv.2.weight"].shape[0]
    sd = {("core.core." + k): v for k, v in core.items()}
    sd.update(synth_weights.make_zoedepth_head_state_dict(feat, outc, seed=4))
    rgb = synth_rgb(48, 64, 1)
    d, invert = zoedepth.get_raw_prediction(rgb, sd, net_w=64, net_h=64, core_name="beit_tiny")
    assert invert is True and d.shape == (48, 64) and d.dtype == np.float32
    assert np.isfinite(d).all() and (d > 0).all()
    d2, _ = zoedepth.get_raw_prediction(np.ascontiguousarray(rgb[:, ::-1]), sd, net_w=64, net_h=64, core_name="beit_tiny")
    assert np.allclose(d2[:, ::-1], d, rtol=0, atol=1e-6 * float(d.max()))
