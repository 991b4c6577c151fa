"""CPU: BOOST on the MiDaS DPT base networks (model types 1-3), the parts that need no GPU.

oracle/midas_boost.py (estimatemidasBoost) and oracle/boost.py (estimateboost) are pinned against the reference's own functions
with cheap deterministic stand-in networks, and the engines' upper-bound net size against dmidas.transforms.Resize.get_size.
What the reference computed is stored in tests/golden/boost_midas_pin.npz, so these tests run without the reference tree;
    DEPTHMAP_MINT_GOLDEN=1 python -m pytest tests/test_boost_midas_cpu.py
recomputes it where the reference tree is present."""
import json
import os

import numpy as np
import pytest

from oracle import ref_loader
from synth import synth_rgb

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "boost_midas_pin.npz")
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


def _fake_midas():
    """stands for DPTDepthModel: estimatemidasBoost calls model.forward(normalised [1, 3, h, w]) -> [1, h, w]"""
    import torch
    import torch.nn.functional as F

    class FakeMidas(torch.nn.Module):
        def forward(self, x):
            g = x.mean(dim=1, keepdim=True)
            return (F.avg_pool2d(g, 9, 1, 4) + 0.25 * torch.sin(3.0 * x[:, :1]) + 0.1 * x[:, 2:3]).squeeze(1)

    return FakeMidas()


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


def _image(hw, seed):
    import cv2
    return cv2.cvtColor(synth_rgb(hw[0], hw[1], seed), cv2.COLOR_BGR2RGB) / 255.0


GRID = [(w, h, m) for m in (384, 500, 512, 1000, 1024, 1600) for (w, h) in
        ((512, 512), (300, 420), (420, 300), (1000, 37), (37, 1000), (1023, 1024), (777, 1601), (1601, 777), (250, 251), (96, 1500))]


def test_upper_bound_net_size_equals_reference():
    """DptBeitEngine's net size for BOOST (depthmap_generation.midas_boost_net_size) and the oracle's both equal
    Resize(m, m, keep_aspect_ratio, 32, 'upper_bound').get_size on a grid of crops; msize 500 / 1000 exercise the floor branch"""
    import cv2
    from depthmap_b200.depthmap_generation import midas_boost_net_size
    from oracle import midas_boost

    def compute():
        _reference()
        from dmidas.transforms import Resize
        return [[int(v) for v in Resize(m, m, resize_target=None, keep_aspect_ratio=True, ensure_multiple_of=32, resize_method="upper_bound",
                                        image_interpolation_method=cv2.INTER_CUBIC).get_size(w, h)] for w, h, m in GRID]
    want = pinned_json("net_size_grid", compute)
    got = [list(midas_boost_net_size(w, h, m)) for w, h, m in GRID]
    assert got == want
    assert [list(midas_boost.net_size(w, h, m)) for w, h, m in GRID] == want
    floors = [(w, h, m) for (w, h, m), (nw, nh) in zip(GRID, want) if max(nw, nh) < int(np.round(max(w * min(m / w, m / h), h * min(m / w, m / h)) / 32) * 32)]
    assert floors, "the grid never takes the floor branch"


@pytest.mark.parametrize("hw,rect,msize", [((300, 420), (0, 0, 420, 300), 512), ((300, 420), (40, 30, 250, 200), 1024), ((520, 360), (10, 20, 300, 480), 384)])
def test_estimatemidasboost_equals_reference(hw, rect, msize):
    from oracle import midas_boost
    img = _image(hw, 13)
    x, y, w, h = rect
    crop = np.ascontiguousarray(img[y:y + h, x:x + w])
    key = f"estimatemidasboost/{hw[0]}x{hw[1]}/{x},{y},{w},{h}/{msize}"
    # stored as float32, every third row and column (file size)
    want = pinned(key, lambda: _reference().estimatemidasBoost(crop.copy(), _fake_midas(), msize, msize)[::3, ::3].astype(np.float32))
    got = midas_boost.estimatemidasboost(crop, msize, _fake_midas())
    assert got.shape == (h, w) and want.shape == ((h + 2) // 3, (w + 2) // 3)
    assert np.abs(got[::3, ::3] - want).max() <= 1e-6 * np.abs(want).max()


@pytest.mark.parametrize("model_type", [1, 2])
@pytest.mark.parametrize("hw,rmax", [((300, 420), 1600), ((520, 360), 1200)])
def test_estimateboost_midas_equals_reference(model_type, hw, rmax):
    """estimateboost end to end for the MiDaS types (receptive field 512 / 384, patches at twice that) with the stand-in networks:
    equal patch rects and whole size, estimate within 1e-6 relative"""
    import cv2
    from oracle import boost, midas_boost
    img = _image(hw, 12)
    key = f"estimateboost/{model_type}/{hw[0]}x{hw[1]}/{rmax}"
    rf = boost.receptive_field(model_type)

    def selection():
        dg = _reference()
        whole, scale = dg.calculateprocessingres(img, rf, 0.2, 3, rmax)
        factor = max(min(1, 4 * scale * whole / rmax), 0.2)
        a, b = boost.target_size(img.shape, whole, factor)
        big = cv2.resize(img, (b, a), interpolation=cv2.INTER_CUBIC)
        return [int(whole), [[int(v) for v in kv[1]["rect"]] for kv in dg.generatepatchs(big, 2 * rf, factor)]]
    want_sel = pinned_json(key + "/selection", selection)
    # stored as float32, every third row and column (file size)
    want = pinned(key + "/estimate", lambda: _reference().estimateboost(img.copy(), _fake_midas(), model_type, _FakePix2Pix(), rmax)[::3, ::3]
                  .astype(np.float32))
    info = {}
    got = boost.estimateboost(img.copy(), model_type, midas_boost.estimate_fn(_fake_midas()), _fake_merge, rmax, info=info)
    assert info["whole_size"] == want_sel[0] and info["patches"] == want_sel[1] and len(info["patches"]) >= 1
    assert got.shape == hw and want.shape == ((hw[0] + 2) // 3, (hw[1] + 2) // 3)
    assert np.abs(got[::3, ::3] - want).max() <= 1e-6 * np.abs(want).max()


def test_constant_prediction_raises():
    from oracle import midas_boost
    with pytest.raises(ValueError):
        midas_boost.estimatemidasboost(np.full((40, 50, 3), 0.5), 384, lambda x: x[:, 0] * 0)
