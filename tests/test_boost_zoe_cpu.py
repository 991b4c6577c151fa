"""CPU: BOOST on ZoeDepth-NK (model type 9), the parts that need no GPU.

estimateboost's ZoeDepth branch (oracle.boost.estimateboost with tests/zoe_boost_oracle.py's estimate) is pinned against the
reference's own estimateboost(..., model_type=9, ...) with a stand-in ZoeDepth model whose infer_pil is a deterministic function of
the uint8 pixels PIL hands it and of the resizer size: equal patches and whole size, equal result.  That pins the R/B swap, the
wrap-around quantisation, the crop-size metric map and its use without normalisation.  What the reference computed is stored in
tests/golden/boost_zoe_pin.npz, so the test runs without the reference tree;
    DEPTHMAP_MINT_GOLDEN=1 python -m pytest tests/test_boost_zoe_cpu.py
recomputes it where the reference tree is present."""
import json
import os
import types

import numpy as np
import pytest

from oracle import ref_loader
from synth import synth_rgb

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "boost_zoe_pin.npz")
MINT = os.environ.get("DEPTHMAP_MINT_GOLDEN") == "1"
_stored = dict(np.load(GOLDEN)) if os.path.exists(GOLDEN) else {}
_minted = {}


def pinned(key, compute):
    """the reference's result for `key` (an array): the stored one, or, when minting, compute()"""
    if MINT:
        _minted[key] = np.asarray(compute())
        return _minted[key]
    if key not in _stored:
        pytest.fail(f"no stored reference result for {key}: mint {GOLDEN} with the reference tree present")
    return _stored[key]


def pinned_json(key, compute):
    return json.loads(str(pinned(key, lambda: np.asarray(json.dumps(compute())))))


@pytest.fixture(scope="module", autouse=True)
def _write_minted():
    yield
    if MINT and _minted:
        np.savez_compressed(GOLDEN, **dict(_stored, **_minted))


def _fake_infer(u8, msize):
    """stands for ZoeDepth's infer_pil at msize x msize: positive 'metric' values, not normalised, channel-asymmetric, and
    sensitive to every uint8 level (a wrapped overshoot changes it)"""
    import cv2
    x = u8.astype(np.float32) / 255.0
    g = cv2.blur(0.6 * x[..., 0] + 0.3 * x[..., 1] + 0.1 * x[..., 2], (5, 5))
    return (1.0 + 2.0 * g + 0.25 * np.sin(x[..., 0] * (msize / 64.0)) + 0.05 * x[..., 2]).astype(np.float32)


class _FakeZoe:
    """estimatezoedepth sets model.core.prep.resizer._Resize__width / __height, then calls model.infer_pil(PIL image)"""

    def __init__(self):
        self.core = types.SimpleNamespace(prep=types.SimpleNamespace(resizer=types.SimpleNamespace()))

    def infer_pil(self, img):
        r = self.core.prep.resizer
        assert r._Resize__width == r._Resize__height and img.mode == 'RGB'
        return _fake_infer(np.asarray(img), r._Resize__width)


class _FakePix2Pix:
    """stands for Pix2Pix4DepthModel: set_input / test / get_current_visuals (pix2pix/models/pix2pix4depth_model.py:96-116)"""

    def set_input(self, outer, inner):
        from oracle import pix2pix as op2p
        self.real_A = op2p.merge_input(outer, inner)

    def test(self):
        import torch
        o, i = self.real_A[:, :1], self.real_A[:, 1:]
        self.fake_B = torch.tanh(0.7 * o + 0.5 * i + 0.1 * o * i)

    def get_current_visuals(self):
        return {"fake_B": self.fake_B}


def _fake_merge(outer, inner):
    p = _FakePix2Pix()
    p.set_input(outer, inner)
    p.test()
    return p.fake_B.squeeze().numpy()


def _reference():
    import torch
    ref_loader.bootstrap()
    from src import depthmap_generation as dg
    dg.depthmap_device = torch.device("cpu")
    import skimage.measure as sm
    from oracle import boost
    sm.block_reduce = lambda img, block, func: boost.block_reduce_max(img, block[0])   # skimage is absent: zero-padded max pool
    dg.skimage = __import__("skimage")
    return dg


@pytest.mark.parametrize("hw,rmax,wraps", [((300, 420), 1600, True), ((520, 360), 1200, False)])
def test_estimateboost_zoe_equals_reference(hw, rmax, wraps):
    """estimateboost end to end for model type 9 (receptive field 384, patches at 768) with the stand-in networks: equal patch
    rects and whole size, estimate within 1e-6 relative.  In the first case some crop's cubic overshoot wraps in the quantisation."""
    import cv2
    from oracle import boost
    import zoe_boost_oracle as zbo
    img = cv2.cvtColor(synth_rgb(hw[0], hw[1], 12), cv2.COLOR_BGR2RGB) / 255.0
    key = f"estimateboost/9/{hw[0]}x{hw[1]}/{rmax}"

    def selection():
        dg = _reference()
        whole, scale = dg.calculateprocessingres(img, 384, 0.2, 3, rmax)
        factor = max(min(1, 4 * scale * whole / rmax), 0.2)
        a, b = boost.target_size(img.shape, whole, factor)
        big = cv2.resize(img, (b, a), interpolation=cv2.INTER_CUBIC)
        return [int(whole), [[int(v) for v in kv[1]["rect"]] for kv in dg.generatepatchs(big, 768, factor)]]
    want_sel = pinned_json(key + "/selection", selection)
    # stored as float32, every third row and column (file size)
    want = pinned(key + "/estimate", lambda: _reference().estimateboost(img.copy(), _FakeZoe(), 9, _FakePix2Pix(), rmax)[::3, ::3]
                  .astype(np.float32))
    info, crops, seen = {}, [], []
    estimate = zbo.estimate_fn(_fake_infer, crops)
    got = boost.estimateboost(img.copy(), 9, lambda crop, msize: seen.append(crop) or estimate(crop, msize), _fake_merge, rmax, info=info)
    assert info["whole_size"] == want_sel[0] and info["patches"] == want_sel[1] and len(info["patches"]) >= 1
    assert got.shape == hw and want.shape == ((hw[0] + 2) // 3, (hw[1] + 2) // 3)
    assert np.abs(got[::3, ::3] - want).max() <= 1e-6 * np.abs(want).max()
    assert [c.shape[:2] for _, c in crops] == [c.shape[:2] for c in seen]
    assert any(float(c.min()) < 0 or float(c.max()) * 255 >= 256 for c in seen) == wraps


def test_quantise_wraps_like_numpy():
    import zoe_boost_oracle as zbo
    v = np.array([0.0, 1.0, 260.1 / 255, -2.5 / 255, 254.99999 / 255, 1e-9])
    assert zbo.quantise(v).tolist() == [0, 255, 4, 254, 254, 0]


def test_boost_routing():
    """BoostPipeline takes ZoeDepth-NK (9) as a base network; 7, 8 and 12 are still refused, and so is no_half with 9 (no_half_route)"""
    from depthmap_b200.boost import BASE_NETWORKS, ESTIMATES, METRIC, BoostPipeline
    from depthmap_b200.depthmap_generation import no_half_route
    assert 9 in BASE_NETWORKS and ESTIMATES[9] == METRIC
    assert BoostPipeline(None, None, "cpu", 9).estimate == METRIC
    for t in (7, 8, 12):
        with pytest.raises(NotImplementedError):
            BoostPipeline(None, None, "cpu", t)
    for precision in ("autocast", "full"):
        with pytest.raises(NotImplementedError):
            no_half_route(9, True, precision)
