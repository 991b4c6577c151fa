"""GPU: MiDaS v2.1 (model type 5).  The new kernels against float64 / torch restatements of their operations (tests/op_bars.py),
the engine against the fp32 oracle (oracle/midas_v21.py, pinned to the reference module by tests/test_midas_v21_cpu.py) under the
precision rule of tests/precision.py, whose yardstick is the same oracle run all-fp16 (the reference's GPU policy for this type is
`model.half()`, src/depthmap_generation.py:268-275), and the model through ModelHolder, the funnel, tiling mode and BOOST."""
import os
import subprocess
import sys

import numpy as np
import pytest

import op_bars
import precision
from circular_oracle import circular_convs
from synth import synth_rgb

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
CHAN_MAP = (2, 1, 0)


def _no_tf32():
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.fixture(scope="module")
def sd():
    from oracle import midas_v21
    return midas_v21.make_state_dict(seed=1)


def _consts():
    import ctypes
    return (ctypes.c_float * 3)(*MEAN), (ctypes.c_float * 3)(*STD), (ctypes.c_int * 3)(*CHAN_MAP)


# ---- kernels ------------------------------------------------------------------------------------------------------------------
def _stem_model(img, nh, nw, circular):
    """float64 [h, w, 3] image in its source channel order -> cv2 INTER_CUBIC to nh x nw (a copy at the same size), ImageNet
    normalise of channel map (2, 1, 0), 7x7 / 2 im2col with pad 3 (zeros or circular) -> [Ho*Wo, 147] ordered (ky, kx, c)"""
    import cv2
    x = img if img.shape[:2] == (nh, nw) else cv2.resize(img, (nw, nh), interpolation=cv2.INTER_CUBIC)
    x = (x[:, :, list(CHAN_MAP)] - np.array(MEAN)) / np.array(STD)
    x = np.pad(x, ((3, 3), (3, 3), (0, 0)), mode="wrap" if circular else "constant")
    ho, wo = (nh - 1) // 2 + 1, (nw - 1) // 2 + 1
    cols = np.empty((ho, wo, 7, 7, 3))
    for ky in range(7):
        for kx in range(7):
            cols[:, :, ky, kx] = x[ky:ky + 2 * ho:2, kx:kx + 2 * wo:2]
    return cols.reshape(ho * wo, 147)


@pytest.mark.parametrize("circular", [False, True])
@pytest.mark.parametrize("hw,net", [((97, 131), (64, 96)), ((64, 96), (64, 96)), ((40, 300), (32, 160))])
def test_stem_im2col_u8_vs_cv2(cuda_device, hw, net, circular):
    """dm_midas_stem_im2col / dm_midas_stem_im2col_circular: cubic resize (down, identity, up in one axis), normalise, channel map,
    im2col; columns 147..191 zero"""
    import torch
    from depthmap_b200 import _lib
    ops = _lib.Ops()
    B = 2
    imgs = [synth_rgb(hw[0], hw[1], 20 + i) for i in range(B)]
    nh, nw = net
    ho, wo = (nh - 1) // 2 + 1, (nw - 1) // 2 + 1
    cols = torch.full((B * ho * wo, 192), float("nan"), dtype=torch.float16, device=cuda_device)
    name = "dm_midas_stem_im2col_circular" if circular else "dm_midas_stem_im2col"
    ops.call(name, torch.from_numpy(np.stack(imgs)).to(cuda_device), B, hw[0], hw[1], nh, nw, *_consts(), cols)
    got = cols.cpu().double().numpy().reshape(B, ho * wo, 192)
    for i, img in enumerate(imgs):
        want = _stem_model(img.astype(np.float64) / 255.0, nh, nw, circular)
        bar = op_bars.check_f16(f"{name} {hw} -> {net} img{i}", got[i, :, :147], want)
        assert np.all(got[i, :, 147:] == 0)
        wrong = _stem_model(img.astype(np.float64) / 255.0, nh, nw, not circular)      # the other padding mode
        op_bars.teeth(f"{name}: the other padding", wrong, want, bar)


@pytest.mark.parametrize("circular", [False, True])
def test_stem_im2col_f32_crops_vs_cv2(cuda_device, circular):
    """dm_midas_stem_im2col_f32_crops / _circular: B crops of one planar fp32 image (values as they are), each resized to the net"""
    import torch
    from depthmap_b200 import _lib
    ops = _lib.Ops()
    rgb = synth_rgb(150, 220, 9)
    planar = torch.from_numpy(rgb.transpose(2, 0, 1).astype(np.float32) / 255.0).contiguous().to(cuda_device)
    rects = [(0, 0, 150, 150), (70, 30, 150, 120), (200, 0, 20, 150)]
    nh, nw = 64, 96
    ho, wo = (nh - 1) // 2 + 1, (nw - 1) // 2 + 1
    cols = torch.full((len(rects) * ho * wo, 192), float("nan"), dtype=torch.float16, device=cuda_device)
    r = torch.tensor(rects, dtype=torch.int32, device=cuda_device)
    name = "dm_midas_stem_im2col_f32_crops_circular" if circular else "dm_midas_stem_im2col_f32_crops"
    ops.call(name, planar, 150, 220, r, len(rects), nh, nw, *_consts(), cols)
    got = cols.cpu().double().numpy().reshape(len(rects), ho * wo, 192)
    img = planar.permute(1, 2, 0).cpu().double().numpy()
    for i, (x0, y0, w, h) in enumerate(rects):
        want = _stem_model(np.ascontiguousarray(img[y0:y0 + h, x0:x0 + w]), nh, nw, circular)
        bar = op_bars.check_f16(f"{name} crop {rects[i]}", got[i, :, :147], want)
        assert np.all(got[i, :, 147:] == 0)
        if i == 1:
            op_bars.teeth(f"{name}: the neighbouring crop", _stem_model(np.ascontiguousarray(img[y0:y0 + h, x0 + 1:x0 + w + 1]), nh, nw, circular),
                          want, bar)


@pytest.mark.parametrize("hw,out", [((12, 20), (24, 40)), ((7, 5), (14, 10)), ((9, 13), (5, 31))])
def test_resize_bilinear_half_vs_torch(cuda_device, hw, out):
    """dm_resize_bilinear_half_nhwc_f16 against F.interpolate(bilinear, align_corners=False) in float64; align_corners=True misses"""
    import torch
    import torch.nn.functional as F
    from depthmap_b200 import _lib
    ops = _lib.Ops()
    B, C = 2, 24
    x = torch.randn(B, hw[0], hw[1], C, generator=torch.Generator().manual_seed(3)).half()
    y = torch.empty(B, out[0], out[1], C, dtype=torch.float16, device=cuda_device)
    ops.call("dm_resize_bilinear_half_nhwc_f16", x.to(cuda_device), B, hw[0], hw[1], C, y, out[0], out[1])
    xd = x.double().permute(0, 3, 1, 2)
    want = F.interpolate(xd, size=out, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    bar = op_bars.check_f16(f"dm_resize_bilinear_half_nhwc_f16 {hw} -> {out}", y, want)
    op_bars.teeth("align_corners=True", F.interpolate(xd, size=out, mode="bilinear", align_corners=True).permute(0, 2, 3, 1), want, bar)


# ---- the engine ---------------------------------------------------------------------------------------------------------------
def _oracle(rgb, sd, net, dev, half=False):
    """estimatemidas on the GPU: fp32, or all-fp16 (precision.HalfView) for the reference-policy yardstick"""
    import cv2
    import torch
    import torch.nn.functional as F
    from oracle import midas_v21
    img = cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0
    x = midas_v21.preprocess(img, net[0], net[1]).to(dev)
    weights = precision.HalfView(sd, dev) if half else {k: v.to(dev) for k, v in sd.items()}
    with torch.no_grad():
        d = midas_v21.forward(weights, x.half() if half else x)
        d = F.interpolate(d.unsqueeze(1), size=img.shape[:2], mode="bicubic", align_corners=False)[0, 0].float()
    return d.cpu().numpy()


def _check(label, got, rgb, sd, net, dev):
    want = _oracle(rgb, sd, net, dev)
    ref16 = precision.norm_err(_oracle(rgb, sd, net, dev, half=True), want)
    return precision.check(label, got, want, ref16)


@pytest.mark.parametrize("hw,net", [((256, 256), (256, 256)), ((240, 320), (384, 384)), ((131, 197), (256, 192))])
def test_engine_vs_oracle(cuda_device, sd, hw, net):
    """B = 2: square, non-square (upper_bound: 384 x 288) and odd-sized images"""
    import torch
    from depthmap_b200.depthmap_generation import MidasV21Engine
    _no_tf32()
    eng = MidasV21Engine(sd, cuda_device)
    imgs = [synth_rgb(hw[0], hw[1], 40 + s) for s in range(2)]
    got = eng.forward_batch(torch.from_numpy(np.stack(imgs)).to(cuda_device), net[0], net[1]).cpu().numpy()
    assert got.shape == (2,) + hw and got.dtype == np.float32
    for i, img in enumerate(imgs):
        _check(f"midas_v21 {hw} net {net} img{i}", got[i], img, sd, net, cuda_device)


def test_graph_replay_is_bit_equal(cuda_device, sd):
    """the first call runs eagerly, the second captures a CUDA graph, the third replays it: all three bit-equal"""
    import torch
    from depthmap_b200.depthmap_generation import MidasV21Engine
    eng = MidasV21Engine(sd, cuda_device)
    rgb = torch.from_numpy(np.stack([synth_rgb(200, 300, s) for s in range(2)])).to(cuda_device)
    outs = [eng.forward_batch(rgb, 384, 384).clone() for _ in range(3)]
    assert eng._graphs._graphs, "no CUDA graph was captured"
    assert torch.isfinite(outs[0]).all() and float(outs[0].max() - outs[0].min()) > 0
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_modelholder_and_funnel(cuda_device, sd):
    """ensure_models(5): flat and {"model", "optimizer"} checkpoints, default net 384 x 384, invert False, resize mode
    'upper_bound'; core_generation_funnel with model_type=5 returns the holder's depth"""
    from PIL import Image
    from depthmap_b200 import core
    from depthmap_b200.depthmap_generation import MidasV21Engine, ModelHolder
    _no_tf32()
    assert ModelHolder.get_default_net_size(5) == [384, 384]
    img = synth_rgb(300, 400, 5)
    preds = []
    for ckpt in (sd, {"model": sd, "optimizer": {}}):
        mh = ModelHolder()
        mh.weights_provider = lambda t, c=ckpt: c
        mh.ensure_models(5, cuda_device, False)
        assert isinstance(mh.depth_model, MidasV21Engine) and mh.resize_mode == "upper_bound"
        pred, invert = mh.get_raw_prediction(Image.fromarray(img), 384, 384)
        assert invert is False and pred.shape == (300, 400) and pred.dtype == np.float32
        preds.append(pred)
        mh.unload_models()
    assert np.array_equal(preds[0], preds[1])
    _check("midas_v21 ModelHolder 384 net (300x400 image)", preds[0], img, sd, (384, 384), cuda_device)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: sd
    try:
        inp = dict(compute_device='GPU', model_type=5, net_width=384, net_height=384, boost=False, do_output_depth=True,
                   do_output_depth_prediction=True, gen_stereo=False, gen_normalmap=False)
        out = list(core.core_generation_funnel(None, [Image.fromarray(img)], None, None, inp, ops={}))
        assert [k for _, k, _ in out][:2] == ['depth_prediction', 'depth']
        assert np.array_equal(out[0][2], preds[0])
    finally:
        holder.unload_models()
        holder.weights_provider = None


def test_tiling_vs_circular_oracle(cuda_device, sd):
    """tiling mode through ModelHolder: every padded convolution circular, against the circular oracle (and its fp16 yardstick)"""
    from PIL import Image
    from depthmap_b200.depthmap_generation import ModelHolder
    from oracle import leres, midas_v21
    _no_tf32()
    img = synth_rgb(240, 320, 8)
    mh = ModelHolder()
    mh.weights_provider = lambda t: sd
    mh.ensure_models(5, cuda_device, False, tiling_mode=True)
    got, invert = mh.get_raw_prediction(Image.fromarray(img), 384, 384)
    mh.unload_models()
    with circular_convs(midas_v21, leres):
        want = _oracle(img, sd, (384, 384), cuda_device)
        ref16 = precision.norm_err(_oracle(img, sd, (384, 384), cuda_device, half=True), want)
    zero = _oracle(img, sd, (384, 384), cuda_device)
    assert precision.norm_err(zero, want)[0] > 1e-2          # the padding mode is visible on this input
    precision.check("midas_v21 tiling (240x320 image, 384 net)", got, want, ref16)


# ---- BOOST --------------------------------------------------------------------------------------------------------------------
def _oracle_forward(cuda_device, sd):
    import torch
    from oracle import midas_v21
    sdd = {k: v.to(cuda_device) for k, v in sd.items()}

    def forward(x):
        with torch.no_grad():
            return midas_v21.forward(sdd, x.to(cuda_device))
    return forward


def test_boost_vs_oracle(cuda_device, sd):
    """ensure_models(5, device, boost=True): pix2pix_model.run against oracle/boost.py's estimateboost with estimatemidasBoost
    around the fp32 oracle (the reference runs BOOST in fp32), at the bars of the LeReS BOOST tests"""
    import cv2
    from depthmap_b200.depthmap_generation import MidasV21Engine, ModelHolder
    from oracle import boost as ob, midas_boost, synth_weights
    from test_boost_midas_gpu import _merge_fn
    _no_tf32()
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    mh = ModelHolder()
    mh.weights_provider = lambda t: psd if t == "pix2pix" else sd
    mh.ensure_models(5, cuda_device, True)
    try:
        assert isinstance(mh.depth_model, MidasV21Engine) and mh.pix2pix_model is not None
        rgb = synth_rgb(300, 420, 12)
        info = {}
        got = mh.pix2pix_model.run(rgb, 1600, info=info)
        oinfo = {}
        want = ob.estimateboost(cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0, 5, midas_boost.estimate_fn(_oracle_forward(cuda_device, sd)),
                                _merge_fn(cuda_device, psd), 1600, info=oinfo)
        assert got.shape == want.shape == (300, 420) and got.dtype == np.float32
        assert info["rects"] == oinfo["patches"] and info["whole"] == oinfo["whole_size"] and len(info["rects"]) >= 1
        mx, mean = precision.norm_err(got, want)
        print(f"[precision] boost midas_v21 (300, 420) rmax 1600: {len(info['rects'])} patches, whole {info['whole']}, ours max {mx:.3e} "
              f"mean {mean:.3e} (reference policy: fp32)")
        assert mx < 3e-3 and mean < 6e-4, (mx, mean)
    finally:
        mh.unload_models()


def test_sharded_boost_type5_equals_single_rank(cuda_device):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29621", os.path.join(ROOT, "tools", "dist_check.py"), "--boost-model-type", "5"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "dist_check ok" in r.stdout and "boost_equal=True" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


@pytest.mark.parametrize("model_type", [4, 6, 11])
def test_unsupported_types_still_raise(cuda_device, model_type):
    from depthmap_b200.depthmap_generation import ModelHolder
    mh = ModelHolder()
    mh.weights_provider = lambda t: {}
    with pytest.raises(NotImplementedError):
        mh.ensure_models(model_type, cuda_device, False)
