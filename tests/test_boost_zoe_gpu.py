"""GPU: BOOST on ZoeDepth-NK (model type 9): the crop quantisation kernel, the pipeline glue, the engine end to end, ModelHolder and
the funnel, tiling mode, repeatability and the patch-parallel mode.

The reference's estimateboost hands ZoeDepth np.uint8(crop * 255) of its float64 work image (src/depthmap_generation.py:1062-1064)
and never halves the network under BOOST (:271), so the yardstick is oracle/boost.py driven by the fp32 oracle ZoeDepth-NK
(tests/zoe_boost_oracle.py) and the fp32 merge network, with the bars of tests/test_boost_midas_gpu.py.  The router takes an argmax
per forward: the weights and images below were probed with the oracle for logit margins, and every forward's route is asserted to
agree with the oracle's instead of loosening a bar."""
import os
import subprocess
import sys

import numpy as np
import pytest

import precision
import zoe_boost_oracle as zbo
from synth import synth_rgb
from test_zoe_gpu import make_zoe_state_dict

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 3       # make_zoe_state_dict('beit_tiny', SEED): every forward of the cases below routes to kitti, logit margins >= 0.05 (oracle)


def _no_tf32():
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _swapped(rgb):
    import cv2
    return cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0


def _merge_fn(cuda_device, psd):
    import torch
    from oracle import pix2pix as op2p
    psd = {k: v.to(cuda_device) for k, v in psd.items()}

    def merge(outer, inner):
        with torch.no_grad():
            return op2p.unet(psd, op2p.merge_input(outer, inner).to(cuda_device))[0, 0].cpu().numpy()
    return merge


def _quantise(planar, rects, h, w):
    import torch
    from depthmap_b200 import _lib as L
    r = torch.tensor(rects, dtype=torch.int32).to(planar.device)
    out = torch.full((len(rects), h, w, 3), 77, dtype=torch.uint8, device=planar.device)
    L.check(L.load().dm_boost_quantise_crops_u8(planar.data_ptr(), planar.shape[1], planar.shape[2], r.data_ptr(), len(rects), h, w,
                                                  out.data_ptr(), L.stream_ptr()), "dm_boost_quantise_crops_u8")
    torch.cuda.synchronize()
    return out.cpu().numpy()


# ---- the kernel --------------------------------------------------------------------------------------------------------------
def test_quantise_crops_u8_bit_exact(cuda_device):
    """dm_boost_quantise_crops_u8 equals np.uint8(np.float64(x) * 255) of the R/B-swapped crop bit for bit: values overshooting
    [0, 1] (wrap-around), values whose product lies within one ulp of an integer, square and border-clipped non-square crops"""
    import torch
    Hi, Wi = 123, 157
    rng = np.random.default_rng(5)
    img = rng.uniform(-0.2, 1.2, (3, Hi, Wi)).astype(np.float32)
    k = rng.integers(-3, 259, (3, Hi, Wi))
    exact = (k / 255.0).astype(np.float32)                            # x * 255 within an ulp or so of the integer k
    step = rng.integers(-1, 2, (3, Hi, Wi))
    near = np.where(step > 0, np.nextafter(exact, np.float32(np.inf)), np.where(step < 0, np.nextafter(exact, np.float32(-np.inf)), exact))
    sel = rng.random((3, Hi, Wi)) < 0.5
    img = np.where(sel, near, img).astype(np.float32)
    planar = torch.from_numpy(img).to(cuda_device)
    src = img[::-1].transpose(1, 2, 0).astype(np.float64)              # byte c from plane 2 - c
    with np.errstate(invalid="ignore"):
        want_all = np.uint8(src * 255)
    assert (np.abs(src * 255 - np.round(src * 255)) < 1e-4).sum() > 1000 and (src * 255 >= 256).any() and (src < 0).any()
    cases = [((64, 64), [(0, 0, 64, 64), (93, 59, 64, 64), (17, 40, 64, 64)]),
             ((37, 91), [(66, 0, 91, 37), (0, 86, 91, 37)]),                  # clipped at the right / bottom border
             ((123, 23), [(134, 0, 23, 123)]),
             ((1, 157), [(0, 122, 157, 1)])]
    for (h, w), rects in cases:
        got = _quantise(planar, rects, h, w)
        for i, (x, y, _, _) in enumerate(rects):
            assert np.array_equal(got[i], want_all[y:y + h, x:x + w]), ((h, w), rects[i])


def test_quantise_rejects_bad_shape(cuda_device):
    import torch
    planar = torch.zeros(3, 10, 12, dtype=torch.float32, device=cuda_device)
    with pytest.raises(ValueError):
        _quantise(planar, [(0, 0, 12, 11)], 11, 12)


# ---- the glue: BoostPipeline around an oracle-backed ZoeDepth --------------------------------------------------------------------
class _OracleZoe:
    """Test double for ZoeDepthNKEngine under BOOST: the pipeline's crop, quantised by dm_boost_quantise_crops_u8, through the fp32
    oracle ZoeDepth-NK at msize; isolates what BOOST adds from the fp16-operand error of the network"""

    def __init__(self, infer, device):
        self.infer, self.device = infer, device

    def forward_batch(self, rgb, net_w, net_h=None, out_hw=None, planar=None):
        import torch
        img, (x, y, w, h) = planar
        u8 = _quantise(img, [(x, y, w, h)], h, w)[0]
        return torch.from_numpy(self.infer(u8, net_w)).to(self.device).unsqueeze(0)


def test_boost_zoe_glue_vs_oracle(cuda_device):
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from oracle import boost as ob, synth_weights
    _no_tf32()
    sd = make_zoe_state_dict('beit_tiny', SEED)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    infer = zbo.nk_infer(sd, 'beit_tiny', cuda_device)
    pipe = BoostPipeline(_OracleZoe(infer, cuda_device), UnetMergeEngine(psd, cuda_device), cuda_device, 9)
    rgb = synth_rgb(300, 420, 12)
    got = pipe.run(rgb, 1600)
    want = ob.estimateboost(_swapped(rgb), 9, zbo.estimate_fn(infer), _merge_fn(cuda_device, psd), 1600)
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] boost glue, type 9 (oracle ZoeDepth-NK on our quantised crops; our merge network / resizes / fit / blend): "
          f"max {mx:.3e} mean {mean:.3e}")
    assert mx < 5e-4 and mean < 5e-5, (mx, mean)


# ---- end to end ------------------------------------------------------------------------------------------------------------------
def _record(eng, log):
    """wrap eng.forward_batch: every uint8 forward appends (msize, crop, (route of the crop, route of its flip)) per image"""
    orig = eng.forward_batch

    def forward_batch(rgb, net_w, net_h=None, out_hw=None, planar=None):
        out = orig(rgb, net_w, net_h, out_hw, planar)
        if planar is None:
            lg = eng._zbufs['logits'][:2 * rgb.shape[0], :2].cpu().numpy()
            name = lambda f: "nyu" if lg[f, 0] >= lg[f, 1] else "kitti"
            for b in range(rgb.shape[0]):
                log.append((net_w, rgb[b].cpu().numpy(), (name(2 * b), name(2 * b + 1))))
        return out
    eng.forward_batch = forward_batch


def _compare_crops(ours, theirs):
    """match every oracle estimate to one of ours (same msize and shape, fewest differing pixels) -> (pixels that differ, whether
    every route agrees); a differing pixel differs by one uint8 level (modulo 256: a wrapped overshoot)"""
    assert len(ours) == len(theirs), (len(ours), len(theirs))
    free = list(range(len(ours)))
    differ, routes_agree = 0, True
    for msize, crop, routes in theirs:
        cands = [i for i in free if ours[i][0] == msize and ours[i][1].shape == crop.shape]
        assert cands, (msize, crop.shape)
        best = min(cands, key=lambda i: int((ours[i][1] != crop).sum()))
        free.remove(best)
        d = np.abs(ours[best][1].astype(np.int32) - crop.astype(np.int32))
        assert np.minimum(d, 256 - d).max() <= 1, (msize, crop.shape)
        differ += int((d != 0).sum())
        routes_agree &= ours[best][2] == routes
    return differ, routes_agree


def _oracle_run(cuda_device, sd, psd, rgb, rmax):
    from oracle import boost as ob
    routes, crops, oinfo = [], [], {}
    want = ob.estimateboost(_swapped(rgb), 9, zbo.estimate_fn(zbo.nk_infer(sd, 'beit_tiny', cuda_device, routes), crops),
                            _merge_fn(cuda_device, psd), rmax, info=oinfo)
    theirs = [(m, c, (routes[2 * i][0], routes[2 * i + 1][0])) for i, (m, c) in enumerate(crops)]
    return want, oinfo, theirs, min(r[1] for r in routes)


def _check_e2e(label, got, info, ours, want, oinfo, theirs, margin):
    assert got.shape == want.shape and got.dtype == np.float32
    assert info["rects"] == oinfo["patches"] and info["whole"] == oinfo["whole_size"] and len(info["rects"]) >= 1
    differ, agree = _compare_crops(ours, theirs)
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] {label}: {len(info['rects'])} patches, whole {info['whole']}, {len(theirs)} estimates, {differ} crop pixels one "
          f"uint8 level off, smallest oracle route margin {margin:.3f}, ours max {mx:.3e} mean {mean:.3e} (reference policy: fp32)")
    assert agree, "a forward routed differently from the oracle"
    assert mx < 3e-3 and mean < 6e-4, (mx, mean)


@pytest.mark.parametrize("hw,rmax", [((300, 420), 1600), ((400, 288), 1100)])
def test_estimateboost_zoe_vs_oracle(cuda_device, hw, rmax):
    """ZoeDepthNKEngine (small BEiT core) under BoostPipeline against the oracle: identical patches and whole size, every route
    agreeing, within the BOOST bar; the first case's whole-image net passes 1024 (BEiT attention beyond the on-chip table, router
    attention over a large window)"""
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import ZoeDepthNKEngine
    from oracle import synth_weights
    _no_tf32()
    sd = make_zoe_state_dict('beit_tiny', SEED)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    eng = ZoeDepthNKEngine(sd, cuda_device, core_name='beit_tiny')
    ours, info = [], {}
    _record(eng, ours)
    got = BoostPipeline(eng, UnetMergeEngine(psd, cuda_device), cuda_device, 9).run(synth_rgb(hw[0], hw[1], 12), rmax, info=info)
    if rmax == 1600:
        assert max(m for m, _, _ in ours) > 1024
    want, oinfo, theirs, margin = _oracle_run(cuda_device, sd, psd, synth_rgb(hw[0], hw[1], 12), rmax)
    _check_e2e(f"boost zoedepth_nk tiny {hw} rmax {rmax}", got, info, ours, want, oinfo, theirs, margin)


def test_boost_zoe_tiling_vs_oracle(cuda_device):
    """tiling mode: circular convolutions in the ZoeDepth core, the merge network zero padded, against the oracle with circular
    convolutions in oracle/beit_dpt.py only"""
    from circular_oracle import circular_convs
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import ZoeDepthNKEngine
    from oracle import beit_dpt, synth_weights
    _no_tf32()
    sd = make_zoe_state_dict('beit_tiny', SEED)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    eng = ZoeDepthNKEngine(sd, cuda_device, core_name='beit_tiny', circular=True)
    ours, info = [], {}
    _record(eng, ours)
    rgb = synth_rgb(400, 288, 12)
    got = BoostPipeline(eng, UnetMergeEngine(psd, cuda_device), cuda_device, 9).run(rgb, 1100, info=info)
    with circular_convs(beit_dpt):
        want, oinfo, theirs, margin = _oracle_run(cuda_device, sd, psd, rgb, 1100)
    _check_e2e("tiling boost zoedepth_nk tiny (400, 288) rmax 1100", got, info, ours, want, oinfo, theirs, margin)


def test_boost_zoe_repeatable(cuda_device):
    """a second run() of the same image (the merge network then replays its captured graph, the engine reuses its buffer sets)
    is bit-identical to the first"""
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import ZoeDepthNKEngine
    from oracle import synth_weights
    eng = ZoeDepthNKEngine(make_zoe_state_dict('beit_tiny', SEED), cuda_device, core_name='beit_tiny')
    unet = UnetMergeEngine(synth_weights.make_pix2pix_state_dict(seed=1), cuda_device)
    pipe = BoostPipeline(eng, unet, cuda_device, 9)
    rgb = synth_rgb(300, 420, 12)
    a = pipe.run(rgb, 1600)
    sets = dict(eng._sets)
    b = pipe.run(rgb, 1600)
    assert unet._graphs._graphs and np.isfinite(a).all() and float(a.max() - a.min()) > 0
    assert np.array_equal(a, b)
    assert all(eng._sets.get(k) is v for k, v in sets.items()), "a buffer set was rebuilt"


# ---- ModelHolder and the funnel ----------------------------------------------------------------------------------------------------
def test_modelholder_and_funnel_boost_type9(cuda_device):
    """ensure_models(9, device, boost=True): ZoeDepth-NK (BEiT-L-384 core) + merge network; get_raw_prediction ignores the net size
    and returns invert = True (reference :402); the funnel's depth_prediction is pipeline.run's; 7 and 8 still refuse BOOST"""
    from PIL import Image
    from depthmap_b200 import core
    from depthmap_b200.depthmap_generation import ZoeDepthNKEngine
    from oracle import synth_weights
    sd = make_zoe_state_dict('beitl16_384', 3)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: psd if t == "pix2pix" else sd
    try:
        holder.update_settings(boost_rmax=1000)
        holder.ensure_models(9, cuda_device, True)
        assert isinstance(holder.depth_model, ZoeDepthNKEngine) and holder.pix2pix_model is not None
        img = synth_rgb(256, 320, 4)
        pred, invert = holder.get_raw_prediction(Image.fromarray(img), 384, 512)
        assert invert is True and pred.shape == (256, 320) and pred.dtype == np.float32 and np.isfinite(pred).all()
        pred2, _ = holder.get_raw_prediction(Image.fromarray(img), 64, 64)
        assert np.array_equal(pred, pred2)
        inp = dict(compute_device='GPU', model_type=9, net_width=384, net_height=512, boost=True, do_output_depth=True,
                   do_output_depth_prediction=True, gen_stereo=False, gen_normalmap=False)
        out = list(core.core_generation_funnel(None, [Image.fromarray(img)], None, None, inp, ops={'boost_rmax': 1000}))
        assert [k for _, k, _ in out][:2] == ['depth_prediction', 'depth']
        assert np.array_equal(out[0][2], -holder.pix2pix_model.run(img, 1000))      # the funnel negates an inverted prediction
        for t in (7, 8):
            with pytest.raises(NotImplementedError):
                holder.ensure_models(t, cuda_device, True)
    finally:
        holder.unload_models()
        holder.weights_provider = None


# ---- patch-parallel ----------------------------------------------------------------------------------------------------------------
def test_sharded_boost_type9_equals_single_rank(cuda_device):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29623", os.path.join(ROOT, "tools", "dist_check.py"), "--boost-model-type", "9"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "dist_check ok" in r.stdout and "boost_equal=True" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
