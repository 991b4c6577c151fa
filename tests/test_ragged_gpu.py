"""GPU: ragged batches.  Images of different pixel sizes that share one network input size run as one forward; every result
must equal, bit for bit, what the same image gets alone (B = 1):
  * each ragged pre- / post-processing entry point against its uniform twin run on each image alone, on odd sizes, with the
    circular and split variants, and a malformed descriptor refused before any launch;
  * each engine's forward_ragged against forward_batch of each image alone, on calls 1 to 3 (eager, capture, replay);
  * ModelHolder.get_raw_prediction_ragged (grouping by net size, input order, errors, BOOST) and the funnel."""
import ctypes

import numpy as np
import pytest
import torch
from PIL import Image

from synth import synth_rgb

pytestmark = pytest.mark.gpu

ODD = [(37, 53), (70, 98), (120, 90)]
MEAN, STD, CHAN = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225), (2, 1, 0)


def _c(vals, t=ctypes.c_float):
    return (t * 3)(*vals)


def _images(sizes, seed, dev):
    return [torch.from_numpy(synth_rgb(h, w, seed + i)).to(dev) for i, (h, w) in enumerate(sizes)]


def _packed(imgs, dev):
    from depthmap_b200 import _lib
    desc = _lib.Ragged([tuple(t.shape[:2]) for t in imgs], 3, dev)
    return torch.cat([t.reshape(-1) for t in imgs]), desc


@pytest.fixture()
def ops(cuda_device):
    from depthmap_b200 import _lib
    return _lib.Ops()


# ---- kernels -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("split", [0, 1])
def test_preprocess_patchify_ragged(ops, cuda_device, split):
    imgs = _images(ODD, 1, cuda_device)
    packed, desc = _packed(imgs, cuda_device)
    nh, nw, P, kpad = 56, 70, 14, 640
    rows = (nh // P) * (nw // P)
    wide = 3 if split else 1
    got = torch.full((len(imgs) * rows, wide * kpad), 7.0, dtype=torch.float16, device=cuda_device)
    ops.call("dm_preprocess_patchify_ragged", *desc.args(packed), nh, nw, P, _c(MEAN), _c(STD), _c(CHAN, ctypes.c_int), split, got, kpad)
    for i, t in enumerate(imgs):
        want = torch.full((rows, wide * kpad), 3.0, dtype=torch.float16, device=cuda_device)
        ops.call("dm_preprocess_patchify_split" if split else "dm_preprocess_patchify", t.unsqueeze(0), 1, t.shape[0], t.shape[1], nh, nw, P,
                 _c(MEAN), _c(STD), _c(CHAN, ctypes.c_int), want, kpad)
        assert torch.equal(got[i * rows:(i + 1) * rows], want), i


@pytest.mark.parametrize("ragged", ["dm_leres_stem_im2col_ragged", "dm_leres_stem_im2col_ragged_circular", "dm_midas_stem_im2col_ragged",
                                    "dm_midas_stem_im2col_ragged_circular"])
def test_stem_im2col_ragged(ops, cuda_device, ragged):
    uniform = ragged.replace("_ragged", "")                  # the uniform twin, e.g. dm_midas_stem_im2col_circular
    imgs = _images(ODD + [(64, 96)], 5, cuda_device)         # the last one at the net size: the resize is a copy
    packed, desc = _packed(imgs, cuda_device)
    nh, nw = 64, 96
    rows = ((nh - 1) // 2 + 1) * ((nw - 1) // 2 + 1)
    extra = () if "leres" in ragged else (_c(CHAN, ctypes.c_int),)
    got = torch.full((len(imgs) * rows, 192), 7.0, dtype=torch.float16, device=cuda_device)
    ops.call(ragged, *desc.args(packed), nh, nw, _c(MEAN), _c(STD), *extra, got)
    for i, t in enumerate(imgs):
        want = torch.empty(rows, 192, dtype=torch.float16, device=cuda_device)
        ops.call(uniform, t.unsqueeze(0), 1, t.shape[0], t.shape[1], nh, nw, _c(MEAN), _c(STD), *extra, want)
        assert torch.equal(got[i * rows:(i + 1) * rows], want), i


def test_zoe_preprocess_patchify_ragged(ops, cuda_device):
    from depthmap_b200.depthmap_generation import _zoe_pads
    imgs = _images(ODD, 9, cuda_device)
    packed, desc = _packed(imgs, cuda_device)
    nh, nw, P = 64, 96, 16
    kpad, rows = 3 * P * P, 2 * (nh // P) * (nw // P)
    got = torch.empty(len(imgs) * rows, kpad, dtype=torch.float16, device=cuda_device)
    ops.call("dm_zoe_preprocess_patchify_ragged", *desc.args(packed), nh, nw, P, got, kpad)
    for i, t in enumerate(imgs):
        H, W = t.shape[:2]
        want = torch.empty(rows, kpad, dtype=torch.float16, device=cuda_device)
        ops.call("dm_zoe_preprocess_patchify", t.unsqueeze(0), 1, H, W, *_zoe_pads(H, W), nh, nw, P, want, kpad)
        assert torch.equal(got[i * rows:(i + 1) * rows], want), i


@pytest.mark.parametrize("mode", [0, 1])
def test_resize_f32_ragged(ops, cuda_device, mode):
    from depthmap_b200 import _lib
    nh, nw = 48, 64
    sizes = ODD + [(nh, nw)]
    d = torch.randn(len(sizes), nh, nw, generator=torch.Generator().manual_seed(3)).to(cuda_device)
    layout = _lib.Ragged(sizes, 1, cuda_device)
    out = torch.full((layout.size,), 7.0, device=cuda_device)
    ops.call("dm_resize_f32_ragged", d, len(sizes), nh, nw, out, layout.size, layout.host.ctypes.data, layout.dev, mode)
    for i, (g, (h, w)) in enumerate(zip(layout.split(out), sizes)):
        want = torch.empty(1, h, w, device=cuda_device)
        ops.call("dm_resize_f32", d[i:i + 1], 1, nh, nw, want, h, w, mode)
        assert torch.equal(g, want[0]), i


def test_zoe_tta_combine_ragged(ops, cuda_device):
    from depthmap_b200 import _lib
    from depthmap_b200.depthmap_generation import _zoe_pads
    nh, nw = 96, 128
    sizes = ODD
    d = torch.rand(2 * len(sizes), nh, nw, generator=torch.Generator().manual_seed(4)).to(cuda_device)
    layout = _lib.Ragged(sizes, 1, cuda_device)
    out = torch.empty(layout.size, device=cuda_device)
    ops.call("dm_zoe_tta_combine_ragged", d, len(sizes), nh, nw, out, layout.size, layout.host.ctypes.data, layout.dev)
    for i, (g, (h, w)) in enumerate(zip(layout.split(out), sizes)):
        want = torch.empty(1, h, w, device=cuda_device)
        ops.call("dm_zoe_tta_combine", d[2 * i:2 * i + 2], 1, nh, nw, *_zoe_pads(h, w), h, w, want)
        assert torch.equal(g, want[0]), i


def test_malformed_descriptor_is_refused(ops, cuda_device):
    """offsets or sizes outside the buffer, or empty images, raise ValueError before any launch (the output stays untouched)"""
    from depthmap_b200 import _lib
    imgs = _images(ODD, 1, cuda_device)
    packed, desc = _packed(imgs, cuda_device)
    out = torch.full((3 * 20, 640), 7.0, dtype=torch.float16, device=cuda_device)
    for field, value in (("offset", desc.size), ("h", 0), ("w", -3), ("h", 10 ** 6), ("offset", -1)):
        bad = desc.host.copy()
        bad[1][field] = value
        with pytest.raises(ValueError):
            ops.call("dm_preprocess_patchify_ragged", packed, desc.size, bad.ctypes.data, desc.dev, desc.B, 56, 70, 14, _c(MEAN), _c(STD),
                     _c(CHAN, ctypes.c_int), 0, out, 640)
    layout = _lib.Ragged(ODD, 1, cuda_device)
    res = torch.empty(layout.size - 1, device=cuda_device)        # one float short
    with pytest.raises(ValueError):
        ops.call("dm_resize_f32_ragged", torch.zeros(3, 8, 8, device=cuda_device), 3, 8, 8, res, res.numel(), layout.host.ctypes.data,
                 layout.dev, 0)
    torch.cuda.synchronize()
    assert (out == 7.0).all()


# ---- engines -------------------------------------------------------------------------------------------------------
def _check_engine(eng, sizes, net_w, net_h=None, seed=11):
    """forward_ragged == forward_batch of each image alone, bit for bit, on calls 1 to 3 (eager, capture, replay)"""
    from depthmap_b200 import _lib
    dev = eng.device
    nets = {eng.net_size(w, h, net_w, net_h if net_h is not None else net_w) for h, w in sizes}
    assert len(nets) == 1 and len({s for s in sizes}) >= 2, (nets, sizes)
    imgs = _images(sizes, seed, dev)
    want = [eng.forward_batch(t.unsqueeze(0), net_w, net_h)[0].clone() for t in imgs]
    packed, desc = _packed(imgs, dev)
    layout = _lib.Ragged(sizes, 1, None)
    for call in range(3):
        got = layout.split(eng.forward_ragged(packed, desc, net_w, net_h))
        for i, (g, w) in enumerate(zip(got, want)):
            assert g.shape == w.shape and torch.equal(g, w), (call, i)


DAV2_SIZES = [(60, 80), (37, 53), (90, 120)]          # all at the 98 x 70 net of a 70 px request


@pytest.mark.parametrize("split, circular", [(False, False), (True, False), (False, True)])
def test_dav2_forward_ragged(cuda_device, split, circular):
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import synth_weights
    eng = DepthAnythingV2Engine(synth_weights.make_dav2_state_dict('vits', seed=1), 'vits', cuda_device, circular=circular, split=split)
    _check_engine(eng, DAV2_SIZES, 70)


@pytest.mark.parametrize("name", ["beit_tiny", "vit_tiny"])
def test_dpt_forward_ragged(cuda_device, name):
    from depthmap_b200.depthmap_generation import DptBeitEngine, DptVitEngine
    from oracle import synth_weights
    cls = DptBeitEngine if name == "beit_tiny" else DptVitEngine
    eng = cls(synth_weights.make_beit_dpt_state_dict(name, seed=2), name, cuda_device)
    _check_engine(eng, [(100, 130), (120, 160), (150, 200)], 96)


@pytest.mark.parametrize("circular", [False, True])
def test_leres_forward_ragged(cuda_device, circular):
    from depthmap_b200.depthmap_generation import LeresEngine
    from oracle import synth_weights
    eng = LeresEngine(synth_weights.make_leres_state_dict(seed=0), cuda_device, circular=circular)
    _check_engine(eng, [(60, 80), (37, 53), (64, 64)], 64)


@pytest.mark.parametrize("circular", [False, True])
def test_midas_v21_forward_ragged(cuda_device, circular):
    from depthmap_b200.depthmap_generation import MidasV21Engine
    from oracle import midas_v21
    eng = MidasV21Engine(midas_v21.make_state_dict(seed=1), cuda_device, circular=circular)
    _check_engine(eng, [(100, 150), (37, 53), (120, 180)], 384, 384)


def _zoe_sd(head):
    from oracle import synth_weights
    sd = {"core.core." + k: v for k, v in synth_weights.make_beit_dpt_state_dict('beit_tiny', seed=3).items()}
    sd.update(head)
    return sd


@pytest.mark.parametrize("variant", ["nk", "n", "k"])
def test_zoedepth_forward_ragged(cuda_device, variant):
    from depthmap_b200.depthmap_generation import ZoeDepthEngine, ZoeDepthNKEngine
    from oracle import beit_dpt, synth_weights
    from oracle import zoedepth_single as ozs
    feat = beit_dpt.CONFIGS['beit_tiny']['features']
    if variant == "nk":
        eng = ZoeDepthNKEngine(_zoe_sd(synth_weights.make_zoedepth_head_state_dict(feat_ch=feat, seed=100)), cuda_device, core_name='beit_tiny')
    else:
        eng = ZoeDepthEngine(_zoe_sd(ozs.make_zoedepth_single_head_state_dict(variant, feat_ch=feat, seed=100)), cuda_device, variant,
                             core_name='beit_tiny')
    _check_engine(eng, [(60, 80), (90, 120), (75, 100)], 96)


# ---- ModelHolder ---------------------------------------------------------------------------------------------------
@pytest.fixture()
def holder(cuda_device):
    from depthmap_b200.depthmap_generation import ModelHolder
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=2)
    mh = ModelHolder()
    mh.weights_provider = lambda t: sd
    mh.ensure_models(12, cuda_device, False)
    yield mh
    mh.unload_models()


def test_holder_ragged_two_net_sizes_in_order(holder, cuda_device):
    sizes = [(60, 80), (84, 70), (37, 53), (70, 84)]            # nets 98 x 70, 70 x 84, 98 x 70, 70 x 84
    assert holder.net_size(80, 60, 70, 70) == holder.net_size(53, 37, 70, 70) != holder.net_size(70, 84, 70, 70)
    imgs = _images(sizes, 21, cuda_device)
    got, invert = holder.get_raw_prediction_ragged(imgs, 70, 70)
    assert invert is False and len(got) == len(imgs)
    for i, t in enumerate(imgs):
        want, inv = holder.get_raw_prediction_batch(t.unsqueeze(0), 70, 70)
        assert got[i].dtype == torch.float32 and got[i].shape == sizes[i] and torch.equal(got[i], want[0]), i


def test_holder_ragged_rejects_bad_entries(holder, cuda_device):
    good = torch.zeros(40, 50, 3, dtype=torch.uint8, device=cuda_device)
    for bad in (torch.zeros(40, 50, 3, dtype=torch.float32, device=cuda_device), torch.zeros(40, 50, 4, dtype=torch.uint8, device=cuda_device),
                torch.zeros(40, 50, dtype=torch.uint8, device=cuda_device), np.zeros((40, 50, 3), np.uint8)):
        with pytest.raises(ValueError):
            holder.get_raw_prediction_ragged([good, bad], 70, 70)


def test_holder_ragged_with_boost_runs_the_pipeline(cuda_device):
    from depthmap_b200.depthmap_generation import ModelHolder
    from oracle import synth_weights
    weights = {0: synth_weights.make_leres_state_dict(seed=0), "pix2pix": synth_weights.make_pix2pix_state_dict(seed=0)}
    mh = ModelHolder()
    mh.weights_provider = lambda t: weights[t]
    mh.ensure_models(0, cuda_device, True)
    try:
        imgs = _images([(192, 256), (180, 200)], 31, cuda_device)     # large enough for BOOST's resolution search at 448
        got, invert = mh.get_raw_prediction_ragged(imgs, 448, 448)
        assert invert is True
        for g, t in zip(got, imgs):
            want = mh.pix2pix_model.run(t.cpu().numpy(), mh.boost_rmax, to_host=False)
            assert torch.equal(g, want)
    finally:
        mh.unload_models()


# ---- funnel --------------------------------------------------------------------------------------------------------
@pytest.fixture()
def funnel(cuda_device):
    from depthmap_b200 import core
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=2)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: sd
    yield core
    holder.unload_models()
    holder.weights_provider = None


def _opts(**kw):
    d = dict(compute_device='GPU', model_type=12, net_width=70, net_height=70, net_size_match=False, boost=False, do_output_depth=True,
             gen_stereo=True, stereo_modes=['left-right', 'red-cyan-anaglyph'], gen_normalmap=True, do_output_depth_prediction=True)
    d.update(kw)
    return d


def _as_bytes(out):
    return [(i, k, (v.mode, v.size, v.tobytes()) if isinstance(v, Image.Image) else (v.dtype, v.shape, v.tobytes())) for i, k, v in out]


def test_funnel_mixed_sizes_one_ragged_call_same_output(funnel, monkeypatch):
    core = funnel
    sizes = [(60, 80), (37, 53), (60, 80), (90, 120)]           # one net size, three pixel sizes, consecutive images differ
    imgs = [Image.fromarray(synth_rgb(h, w, 50 + i)) for i, (h, w) in enumerate(sizes)]
    holder = core.get_model_holder()
    calls = []
    ragged, batch = type(holder).get_raw_prediction_ragged, type(holder).get_raw_prediction_batch
    monkeypatch.setattr(type(holder), "get_raw_prediction_ragged", lambda s, im, nw, nh: calls.append(("ragged", len(im))) or ragged(s, im, nw, nh))
    monkeypatch.setattr(type(holder), "get_raw_prediction_batch", lambda s, rgb, nw, nh: calls.append(("batch", int(rgb.shape[0]))) or batch(s, rgb, nw, nh))
    got = _as_bytes(core.core_generation_funnel(None, imgs, None, None, _opts(), ops={}))
    assert calls == [("ragged", 4)]
    calls.clear()
    monkeypatch.setenv("DEPTHMAP_B200_MAX_BATCH", "1")
    want = _as_bytes(core.core_generation_funnel(None, imgs, None, None, _opts(), ops={}))
    assert calls == [("batch", 1)] * 4
    assert [(i, k) for i, k, _ in got] == [(i, k) for i, k, _ in want]
    assert got == want


def test_funnel_ragged_is_lazy_and_bounded(funnel, monkeypatch):
    core = funnel
    monkeypatch.setenv("DEPTHMAP_B200_MAX_BATCH", "2")
    sizes = [(60, 80), (37, 53), (90, 120), (45, 60), (60, 80)]
    imgs = [Image.fromarray(synth_rgb(h, w, 60 + i)) for i, (h, w) in enumerate(sizes)]
    holder = core.get_model_holder()
    calls = []
    ragged, batch = type(holder).get_raw_prediction_ragged, type(holder).get_raw_prediction_batch
    monkeypatch.setattr(type(holder), "get_raw_prediction_ragged", lambda s, im, nw, nh: calls.append(len(im)) or ragged(s, im, nw, nh))
    monkeypatch.setattr(type(holder), "get_raw_prediction_batch", lambda s, rgb, nw, nh: calls.append(int(rgb.shape[0])) or batch(s, rgb, nw, nh))
    gen = core.run_depthmap(None, imgs, None, None, _opts(gen_stereo=False, gen_normalmap=False, do_output_depth_prediction=False), ops={})
    first = next(gen)
    assert first[:2] == (0, 'depth') and calls == [2]           # only the first group has run
    rest = list(gen)
    assert calls == [2, 2, 1] and [i for i, _, _ in rest] == [1, 2, 3, 4]
