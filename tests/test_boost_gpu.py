"""GPU: BOOST (SURVEY §8a row D9) — the merge U-Net and estimateboost on the sm_90a kernels against the oracle (oracle/pix2pix.py,
oracle/boost.py, oracle/leres.py; all three pinned to the reference in tests/test_oracle_pin.py).  The reference runs both networks
in fp32 when boost is on (src/depthmap_generation.py:268-275), so there is no fp16 yardstick: the merge network uses split-operand
(fp32-class) GEMMs and is held to 1e-4; the end-to-end result carries the fp16-operand LeReS forwards and is reported against
north_star's 1e-3 with the LeReS row's bar (tests/test_leres_gpu.py)."""
import numpy as np
import pytest

import precision
from synth import synth_rgb

pytestmark = pytest.mark.gpu


def _no_tf32():
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.mark.parametrize("split,kc,bar", [(True, 1024, 1e-4), (True, None, 1e-3), (False, None, 2e-2)])
def test_merge_unet_vs_oracle(cuda_device, split, kc, bar):
    import torch
    from depthmap_b200.boost import UnetMergeEngine
    from oracle import pix2pix as op2p, synth_weights
    _no_tf32()
    sd = synth_weights.make_pix2pix_state_dict(seed=1)
    eng = UnetMergeEngine(sd, cuda_device, split=split, kc=kc)
    rng = np.random.default_rng(5)
    yy, xx = np.mgrid[0:1024, 0:1024].astype(np.float32) / 1024
    outer = (np.sin(6 * xx) + yy + 0.05 * rng.standard_normal((1024, 1024))).astype(np.float32)
    inner = (outer * 0.7 + 0.3 * np.cos(9 * yy * xx) + 0.05 * rng.standard_normal((1024, 1024))).astype(np.float32)
    x = op2p.merge_input(outer, inner)                                  # [1, 2, 1024, 1024]
    with torch.no_grad():
        want = op2p.unet({k: v.to(cuda_device) for k, v in sd.items()}, x.to(cuda_device))[0, 0].cpu().numpy()
    got = eng.forward(x[0].permute(1, 2, 0).contiguous().to(cuda_device)).cpu().numpy()
    assert got.shape == want.shape == (1024, 1024) and np.abs(want).max() > 1e-2 and want.std() > 1e-3
    err = np.abs(got - want).max()
    print(f"[precision] merge unet_1024 split={split} kc={kc}: max abs err {err:.3e} (output in (-1, 1), std {want.std():.3f})")
    assert err < bar, err


def _oracle_fns(cuda_device, lsd, psd):
    import cv2
    import torch
    from oracle import leres, pix2pix as op2p
    lsd = {k: v.to(cuda_device) for k, v in lsd.items()}
    psd = {k: v.to(cuda_device) for k, v in psd.items()}

    def estimate(img, msize):
        with torch.no_grad():
            pred = leres.forward(lsd, leres.preprocess(img, msize, msize).to(cuda_device)).squeeze().cpu().numpy()
        return cv2.resize(pred, (img.shape[1], img.shape[0]), interpolation=cv2.INTER_CUBIC)

    def merge(outer, inner):
        with torch.no_grad():
            return op2p.unet(psd, op2p.merge_input(outer, inner).to(cuda_device))[0, 0].cpu().numpy()

    return estimate, merge


@pytest.mark.parametrize("hw,rmax", [((300, 420), 1600), ((400, 288), 1100)])
def test_estimateboost_vs_oracle(cuda_device, hw, rmax):
    import cv2
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import LeresEngine
    from oracle import boost as ob, synth_weights
    _no_tf32()
    lsd = synth_weights.make_leres_state_dict(seed=2)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    pipe = BoostPipeline(LeresEngine(lsd, cuda_device), UnetMergeEngine(psd, cuda_device), cuda_device, 0)
    rgb = synth_rgb(hw[0], hw[1], 12)
    info = {}
    got = pipe.run(rgb, rmax, info=info)
    estimate, merge = _oracle_fns(cuda_device, lsd, psd)
    oinfo = {}
    want = ob.estimateboost(cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0, 0, estimate, merge, rmax, info=oinfo)
    assert got.shape == want.shape == hw and got.dtype == np.float32
    assert info["rects"] == oinfo["patches"] and info["whole"] == oinfo["whole_size"] and len(info["rects"]) >= 1
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] boost res101 {hw} rmax {rmax}: {len(info['rects'])} patches, whole {info['whole']}, ours max {mx:.3e} mean {mean:.3e} "
          f"(reference policy: fp32)")
    assert mx < 3e-3 and mean < 6e-4, (mx, mean)


@pytest.mark.parametrize("net", [448, 896, 1120])
def test_leres_on_float_crop_vs_oracle(cuda_device, net):
    """the estimateleres call BOOST makes: a float crop of the work image, square net of 448 (receptive field), 896 (patches) or a
    whole-image size; result at the crop's size"""
    import torch
    from depthmap_b200.depthmap_generation import LeresEngine
    from oracle import leres, synth_weights
    _no_tf32()
    lsd = synth_weights.make_leres_state_dict(seed=2)
    eng = LeresEngine(lsd, cuda_device)
    rgb = synth_rgb(500, 640, 21)
    planar = torch.from_numpy((rgb.astype(np.float64) / 255.0).astype(np.float32).transpose(2, 0, 1).copy()).to(cuda_device)
    x, y, w, h = 37, 52, 411, 389
    got = eng.forward_batch(None, net, net, planar=(planar, (x, y, w, h)))[0].cpu().numpy()
    crop = (rgb.astype(np.float64) / 255.0)[y:y + h, x:x + w, ::-1]                    # estimateboost's channel order
    sd = {k: v.to(cuda_device) for k, v in lsd.items()}
    import cv2
    with torch.no_grad():
        pred = leres.forward(sd, leres.preprocess(np.ascontiguousarray(crop), net, net).to(cuda_device)).squeeze().cpu().numpy()
    want = cv2.resize(pred, (w, h), interpolation=cv2.INTER_CUBIC)
    assert got.shape == want.shape == (h, w)
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] leres res101 float crop {w}x{h} net {net}: ours max {mx:.3e} mean {mean:.3e} (reference policy: fp32)")
    assert mx < 3e-3 and mean < 6e-4, (mx, mean)


class _OracleDepthEngine:
    """Test double for the base network: estimateleres through the fp32 oracle, so that the test below isolates everything BOOST adds
    (resizes, merge network, normalisations, least-squares fit, mask blend) from the fp16-operand error of the LeReS forward."""

    def __init__(self, estimate, device):
        self.estimate, self.device = estimate, device

    def forward_batch(self, rgb, net_w, net_h=None, out_hw=None, planar=None):
        import torch
        img, (x, y, w, h) = planar
        crop = img[:, y:y + h, x:x + w].permute(1, 2, 0).cpu().numpy().astype(np.float64)[:, :, ::-1]      # the channel order estimateboost works in
        return torch.from_numpy(self.estimate(np.ascontiguousarray(crop), net_w)).to(self.device).unsqueeze(0)


def test_boost_glue_vs_oracle(cuda_device):
    import cv2
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from oracle import boost as ob, synth_weights
    _no_tf32()
    lsd = synth_weights.make_leres_state_dict(seed=2)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    estimate, merge = _oracle_fns(cuda_device, lsd, psd)
    pipe = BoostPipeline(_OracleDepthEngine(estimate, cuda_device), UnetMergeEngine(psd, cuda_device), cuda_device, 0)
    rgb = synth_rgb(300, 420, 12)
    got = pipe.run(rgb, 1600)
    want = ob.estimateboost(cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0, 0, estimate, merge, 1600)
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] boost glue (oracle base network, our merge network / resizes / fit / blend): max {mx:.3e} mean {mean:.3e}")
    assert mx < 5e-4 and mean < 5e-5, (mx, mean)


def test_modelholder_boost_api(cuda_device):
    """ensure_models(0, device, boost=True) + get_raw_prediction: net size ignored, float32 [H, W], invert = True (reference :375-403)"""
    from PIL import Image
    from depthmap_b200.depthmap_generation import ModelHolder
    from oracle import synth_weights
    lsd = synth_weights.make_leres_state_dict(seed=2)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    mh = ModelHolder()
    mh.weights_provider = lambda t: psd if t == "pix2pix" else lsd
    mh.update_settings(boost_rmax=1000)
    mh.ensure_models(0, cuda_device, True)
    assert mh.pix2pix_model is not None
    img = synth_rgb(256, 320, 4)
    pred, invert = mh.get_raw_prediction(Image.fromarray(img), 448, 448)
    assert invert is True and pred.shape == (256, 320) and pred.dtype == np.float32 and np.isfinite(pred).all()
    pred2, _ = mh.get_raw_prediction(Image.fromarray(img), 64, 64)
    assert np.array_equal(pred, pred2)
    with pytest.raises(NotImplementedError):
        mh.ensure_models(12, cuda_device, True)
    mh.unload_models()
    assert mh.pix2pix_model is None


def test_funnel_with_boost(cuda_device):
    """core_generation_funnel(..., BOOST=True, model type 0): the depth prediction the funnel yields is estimateboost's (not the plain
    LeReS forward), and the u16 depth / stereo that follow are computed from it (reference src/core.py:130,185-211)."""
    from PIL import Image
    from depthmap_b200 import core
    from oracle import synth_weights
    lsd = synth_weights.make_leres_state_dict(seed=2)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: psd if t == "pix2pix" else lsd
    try:
        img = synth_rgb(256, 320, 4)
        inp = dict(compute_device='GPU', model_type=0, net_width=448, net_height=448, boost=True, do_output_depth=True,
                   do_output_depth_prediction=True, gen_stereo=True, stereo_modes=['left-right'], gen_normalmap=False)
        out = list(core.core_generation_funnel(None, [Image.fromarray(img)], None, None, inp, ops={'boost_rmax': 1000}))
        assert [k for _, k, _ in out] == ['depth_prediction', 'depth', 'left-right']
        pred = out[0][2]
        direct = holder.pix2pix_model.run(img, 1000)
        assert pred.shape == (256, 320) and np.array_equal(pred, -direct)          # src/core.py:186-195: `out = -raw_prediction` for the "invert" models, and that is what is yielded
        plain = holder.depth_model.forward_batch(__import__("torch").from_numpy(img).to(cuda_device).unsqueeze(0), 448, 448)[0].cpu().numpy()
        assert np.abs(plain - direct).max() > 1e-3 * (plain.max() - plain.min())        # boost really ran
        assert out[1][2].size == (320, 256) and out[2][2].size == (640, 256)
    finally:
        holder.unload_models()
        holder.weights_provider = None
