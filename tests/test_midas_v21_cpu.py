"""CPU: MiDaS v2.1 (model type 5).  The fp32 oracle (oracle/midas_v21.py) against the reference's own MidasNet and estimatemidas,
the 'upper_bound' net size against the reference's Resize, the circular oracle against the reference module set circular, and the
engine's call sequence recorded against a fake library (test_engine_trace_cpu.py).

The reference builds MidasNet's encoder with torch.hub.load("facebookresearch/WSL-Images", "resnext101_32x8d_wsl"), which is
torchvision's ResNet(Bottleneck, [3, 4, 23, 3], groups=32, width_per_group=8): the reference module is built with that hub call
answered by torchvision.models.resnext101_32x8d(weights=None).  Its results are stored in tests/golden/midas_v21_pin.npz:

    DEPTHMAP_MINT_GOLDEN=1 python -m pytest tests/test_midas_v21_cpu.py      # rewrite them (reference tree present)
"""
from __future__ import annotations

import os
import re

import numpy as np
import pytest

from circular_oracle import circular_convs, padded_conv2d_modules, set_circular
from synth import synth_rgb
from test_engine_trace_cpu import fake  # noqa: F401  (fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "midas_v21_pin.npz")
MINT = os.environ.get("DEPTHMAP_MINT_GOLDEN") == "1"
_stored = dict(np.load(GOLDEN)) if os.path.exists(GOLDEN) else {}
_minted = {}
NETS = [(64, 64), (96, 64), (64, 128)]          # (net_w, net_h) of the network pins


def pinned(key, compute):
    """the reference's result for `key`: the stored one, or, when minting, compute()"""
    if MINT:
        _minted[key] = np.asarray(compute())
        return _minted[key]
    if key not in _stored:
        pytest.fail(f"no stored reference result for {key}: mint {GOLDEN} with the reference tree present")
    return _stored[key]


@pytest.fixture(scope="module", autouse=True)
def _write_minted():
    yield
    if MINT and _minted:
        np.savez_compressed(GOLDEN, **dict(_stored, **_minted))


@pytest.fixture(scope="module")
def sd():
    from oracle import midas_v21
    return midas_v21.make_state_dict(seed=1)


def _reference_model(sd, circular=False):
    """the reference's MidasNet(None) with the synthetic weights, loaded strictly but for the BatchNorm step counters"""
    from unittest import mock

    import torchvision
    from oracle import ref_loader
    ref_loader.bootstrap()
    with mock.patch("torch.hub.load", lambda *a, **k: torchvision.models.resnext101_32x8d(weights=None)):
        from dmidas.midas_net import MidasNet
        model = MidasNet(None).eval()
    res = model.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith("num_batches_tracked") for k in res.missing_keys)
    assert len(model.state_dict()) == 666
    return set_circular(model) if circular else model


def _x(net_w, net_h, seed=4):
    import torch
    return torch.randn(1, 3, net_h, net_w, generator=torch.Generator().manual_seed(seed))


def test_synthetic_state_dict_is_non_degenerate(sd):
    import torch
    from oracle import midas_v21
    with torch.no_grad():
        d = midas_v21.forward(sd, _x(64, 96))
    assert torch.isfinite(d).all() and d.min() > 0 and d.std() > 0.1 * d.mean(), (d.min(), d.mean(), d.std())


@pytest.mark.parametrize("net", NETS)
def test_oracle_network_equals_reference(sd, net):
    import torch
    from oracle import midas_v21

    def reference():
        with torch.no_grad():
            return _reference_model(sd)(_x(*net)).numpy()
    want = torch.from_numpy(pinned(f"network/{net[0]}x{net[1]}", reference))
    with torch.no_grad():
        got = midas_v21.forward(sd, _x(*net))
    assert got.shape == want.shape == (1, net[1], net[0])
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()


@pytest.mark.parametrize("hw,net", [((70, 90), (64, 64)), ((90, 70), (96, 64)), ((50, 120), (128, 64))])
def test_oracle_estimatemidas_equals_reference(sd, hw, net):
    """the reference's estimatemidas (fp32, depthmap_device = cpu, 'upper_bound', ImageNet NormalizeImage) on the float image
    get_raw_prediction hands it"""
    import cv2
    import torch
    from oracle import midas_v21
    rgb = synth_rgb(hw[0], hw[1], 7)
    img = cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0

    def reference():
        from oracle import ref_loader
        ref_loader.bootstrap()
        from dmidas.transforms import NormalizeImage
        from src import depthmap_generation as dg
        dg.depthmap_device = torch.device("cpu")
        norm = NormalizeImage(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
        return dg.estimatemidas(img, _reference_model(sd), net[0], net[1], "upper_bound", norm, True, False)
    want = pinned(f"estimate/{hw[0]}x{hw[1]}/{net[0]}x{net[1]}", reference)
    got, invert = midas_v21.get_raw_prediction(rgb, sd, net[0], net[1])
    assert invert is False and got.shape == want.shape == hw
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


SIZES = [(w, h) for w in (1, 31, 100, 383, 384, 385, 512, 1000, 4000) for h in (1, 17, 288, 384, 500, 3000)]
SIZE_NETS = [(384, 384), (384, 288), (512, 384), (256, 640)]


def test_net_size_equals_reference_resize():
    """the engine's net size against Resize(net_w, net_h, keep_aspect_ratio, multiple of 32, 'upper_bound').get_size; a side that
    rounds to 0 (an image too elongated for the net) raises ValueError instead of reaching cv2.resize"""
    from depthmap_b200.depthmap_generation import MidasV21Engine, midas_upper_bound_net_size
    from oracle import midas_v21

    def reference():
        import cv2
        from oracle import ref_loader
        ref_loader.bootstrap()
        from dmidas.transforms import Resize
        return [[Resize(nw, nh, resize_target=None, keep_aspect_ratio=True, ensure_multiple_of=32, resize_method="upper_bound",
                        image_interpolation_method=cv2.INTER_CUBIC).get_size(w, h) for (w, h) in SIZES] for nw, nh in SIZE_NETS]
    want = pinned("net_size", reference)
    zero = 0
    for ni, (nw, nh) in enumerate(SIZE_NETS):
        for si, (w, h) in enumerate(SIZES):
            ref = tuple(int(v) for v in want[ni][si])
            assert midas_upper_bound_net_size(w, h, nw, nh) == midas_v21.net_size(w, h, nw, nh) == ref, ((w, h), (nw, nh), ref)
            if min(ref) <= 0:
                zero += 1
                with pytest.raises(ValueError):
                    MidasV21Engine.net_size(None, w, h, nw, nh)
            else:
                assert MidasV21Engine.net_size(None, w, h, nw, nh) == ref
    assert zero > 0


def test_circular_oracle_equals_reference(sd):
    """tiling mode: the oracle with circular_convs against the reference module with every nn.Conv2d set circular; the number of
    padded convolutions a forward reaches is pinned too"""
    import torch
    from oracle import leres, midas_v21
    x = _x(96, 64, seed=5)

    def reference():
        model = _reference_model(sd, circular=True)
        n = [0]
        hooks = [m.register_forward_hook(lambda *a: n.__setitem__(0, n[0] + 1)) for m in padded_conv2d_modules(model)]
        with torch.no_grad():
            out = model(x.clone()).numpy()
        for h in hooks:
            h.remove()
        return [out, n[0]]
    want, count = pinned("circular/96x64", lambda: reference()[0]), int(pinned("circular/count", lambda: reference()[1]))
    with torch.no_grad(), circular_convs(midas_v21, leres) as c:
        got = midas_v21.forward(sd, x)
    with torch.no_grad():
        zero = midas_v21.forward(sd, x)
    want = torch.from_numpy(want)
    scale = want.abs().max().item()
    assert (got - want).abs().max().item() <= 1e-5 * scale
    assert (zero - want).abs().max().item() > 1e-3 * scale            # the padding mode matters on this input
    # stem + 33 grouped 3x3 + 4 layer_rn + 7 RCUs x 2 + 2 head convs
    assert c.padded == count == 1 + 33 + 4 + 14 + 2


# ---- the engine's call sequence against a fake library ------------------------------------------------------------------------
CIRCULAR = {"dm_conv3x3_circular_ex": "dm_conv3x3_ex", "dm_im2col_s2_circular_f16": "dm_im2col_s2_f16",
            "dm_midas_stem_im2col_circular": "dm_midas_stem_im2col",
            "dm_midas_stem_im2col_f32_crops_circular": "dm_midas_stem_im2col_f32_crops"}


def _relabel(calls):
    labels = {}

    def v(x):
        if isinstance(x, str) and re.fullmatch(r"(p|stream)\d+", x):
            return labels.setdefault(x, f"{x.rstrip('0123456789')}{len(labels)}")
        if isinstance(x, dict):
            return {k: v(y) for k, y in x.items()}
        return x
    return [[n, [v(a) for a in args]] for n, args in calls]


def _run(fake, sd, circular):
    import torch
    from depthmap_b200.depthmap_generation import MidasV21Engine
    start = len(fake.calls)
    eng = MidasV21Engine(sd, torch.device("cpu"), circular=circular)
    rgb = torch.from_numpy(np.stack([synth_rgb(100, 150, s) for s in range(2)]))
    out = eng.forward_batch(rgb, 384, 384)
    assert out.shape == (2, 100, 150)
    planar = torch.from_numpy(synth_rgb(300, 400, 3).transpose(2, 0, 1).astype(np.float32) / 255.0).contiguous()
    crops = eng.forward_crops(planar, [(0, 0, 200, 200), (100, 50, 200, 200), (300, 0, 100, 300)], 384)
    assert [tuple(c.shape) for c in crops] == [(200, 200), (200, 200), (300, 100)]
    return fake.calls[start:], eng.ops.launches


def test_engine_trace(fake, sd):
    """the engine's calls: the encoder is LeReS's (one call per layer), the decoder one conv per oracle convolution; with tiling on,
    the same sequence with the circular entry point at every padded convolution, one per padded convolution of the oracle"""
    zero, zl = _run(fake, sd, False)
    circ, cl = _run(fake, sd, True)
    assert zl == sum(k for _, _, k in zero)
    assert cl == sum(2 if n == "dm_conv3x3_circular_ex" else k for n, _, k in circ)
    forwards = sum(n.startswith("dm_midas_stem_im2col") for n, _, _ in zero)
    assert forwards == 3                          # the batch, then two net shapes among the crops
    assert not any(n in CIRCULAR.values() for n, _, _ in circ)
    mapped = [[CIRCULAR.get(n, n), args[:1] + args[2:] if n == "dm_conv3x3_circular_ex" else args] for n, args, _ in circ]
    assert _relabel(mapped) == _relabel([[n, a] for n, a, _ in zero])
    assert sum(n in CIRCULAR for n, _, _ in circ) == forwards * (1 + 33 + 4 + 14 + 2)
    names = [n for n, _, _ in zero]
    assert names.count("dm_midas_stem_im2col") == 1 and names.count("dm_midas_stem_im2col_f32_crops") == 2
    assert names.count("dm_resize_f32") == 1 and names.count("dm_boost_resize_cubic") == 3
    per = {k: names.count(k) / forwards for k in set(names) if not k.startswith(("dm_midas_stem", "dm_resize_f32", "dm_boost"))}
    # GEMMs: the stem, two 1x1s per bottleneck, the three strided 3x3s (on the strided im2col), four downsamples.  3x3 convs: 30
    # stride-1 grouped ones, 4 layer_rn, 7 RCUs x 2, 2 in the head
    assert per == {"dm_gemm_ex": 1 + 33 * 2 + 3 + 4, "dm_maxpool3x3s2_nhwc_f16": 1, "dm_im2col_s2_f16": 3, "dm_subsample2_nhwc_f16": 3,
                   "dm_conv3x3_ex": 30 + 4 + 14 + 2, "dm_resize_bilinear_nhwc_f16": 4, "dm_resize_bilinear_half_nhwc_f16": 1}, per


def test_missing_checkpoint_key_raises(fake, sd):
    import torch
    from depthmap_b200.depthmap_generation import MidasV21Engine
    bad = {k: v for k, v in sd.items() if k != "scratch.refinenet2.resConfUnit1.conv2.bias"}
    with pytest.raises(ValueError, match="scratch.refinenet2.resConfUnit1.conv2.bias"):
        MidasV21Engine(bad, torch.device("cpu"))
