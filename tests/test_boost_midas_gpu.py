"""GPU: BOOST on the MiDaS DPT base networks (model types 1, 2, 3) and the relative-position attention that serves every BEiT window,
including BOOST's whole-image windows of up to 100 x 100 patches (SURVEY §8a rows D0 / D9).

The attention is held to the dense fp32 gather of the reference (test_attention_relpos_table's bar).  The reference runs the DPT in fp32 under BOOST
(src/depthmap_generation.py:268-275), so, as for LeReS under BOOST (tests/test_boost_gpu.py), the end-to-end bar is 3e-3 max /
6e-4 mean of the range against the fp32 oracle (oracle/midas_boost.py around oracle/beit_dpt.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import precision
from synth import synth_rgb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = {1: 'beitl16_512', 2: 'beitl16_384', 3: 'vitl16_384'}


def _no_tf32():
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


# ---- A: relative-position attention -----------------------------------------------------------------------------------
def _relpos_case(dev, B, gh, gw, H, seed=None):
    import torch
    N, C = gh * gw + 1, H * 64
    nrd = (2 * gh - 1) * (2 * gw - 1) + 3
    g = torch.Generator(device="cpu").manual_seed(seed if seed is not None else gh * 100 + gw)
    qkv = torch.randn(B * N, 3 * C, generator=g).half().to(dev)
    table = (torch.randn(nrd, H, generator=g) * 2).to(dev)
    tab_k = (table.t().contiguous() * 1.4426950408889634).float().contiguous()
    return qkv, table, tab_k, N, C, nrd


def _run_relpos(entry, dev, qkv, tab_k, B, gh, gw, H, N, C, nrd):
    import torch
    from depthmap_b200 import _lib as L
    lib = L.load()
    out = torch.full((B * N, C), float("nan"), dtype=torch.float16, device=dev)
    L.check(getattr(lib, entry)(qkv.data_ptr(), B, gh, gw, H, 0.125, tab_k.data_ptr(), nrd, out.data_ptr(), L.stream_ptr()), entry)
    torch.cuda.synchronize()
    return out


def _dense_ref_err(dev, out, qkv, table, B, gh, gw, H, N, C, qchunk=2048):
    """max |out - softmax(q k^T / 8 + bias) v| with the bias gathered from the table (gen_relative_position_index), fp32, per head and
    query chunk (a 100 x 100 window would need 6 GB per head for the whole [N, N] bias at once)"""
    import torch
    from oracle.beit_dpt import gen_relative_position_index
    idx = gen_relative_position_index((gh, gw)).to(dev)
    q, k, v = qkv.float().view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    err = 0.0
    got = out.float().view(B, N, H, 64).permute(0, 2, 1, 3)
    for h in range(H):
        for q0 in range(0, N, qchunk):
            rows = slice(q0, min(N, q0 + qchunk))
            bias = table[:, h][idx[rows].reshape(-1)].view(-1, N)
            s = (q[:, h, rows] * 0.125) @ k[:, h].transpose(-1, -2) + bias
            ref = s.softmax(-1) @ v[:, h]
            err = max(err, (got[:, h, rows] - ref).abs().max().item())
    return err


@pytest.mark.parametrize("B,gh,gw,H", [(1, 4, 4, 1), (2, 8, 6, 2), (2, 32, 32, 16), (1, 24, 24, 3), (1, 16, 16, 2), (2, 24, 16, 3),
                                        (1, 20, 32, 2), (1, 9, 48, 1), (1, 88, 88, 4), (1, 100, 100, 16), (1, 100, 74, 16), (1, 184, 184, 1)])
def test_attention_relpos_large_windows_vs_dense(cuda_device, B, gh, gw, H):
    """dm_attention_relpos_f16 with the table sub-windows streamed per key tile: the small grids, BOOST's whole-image windows
    (100 x 100 = a 157 KB table per head, more than the shared memory left beside the tiles; 100 x 74), and 184 x 184, whose key
    offsets pass 65535"""
    import torch
    qkv, table, tab_k, N, C, nrd = _relpos_case(cuda_device, B, gh, gw, H)
    out = _run_relpos("dm_attention_relpos_f16", cuda_device, qkv, tab_k, B, gh, gw, H, N, C, nrd)
    assert torch.isfinite(out.float()).all(), "some output rows were never written"
    err = _dense_ref_err(cuda_device, out, qkv, table, B, gh, gw, H, N, C)
    print(f"[precision] relpos {B}x{gh}x{gw} H{H}: max abs err {err:.3e}")
    assert err < 6e-3, (B, gh, gw, H, err)


def test_beit_large_512_net_1600_vs_oracle(cuda_device):
    """DptBeitEngine at BOOST's default whole-image limit (net 1600 x 1600, a 100 x 100 window): within the BEiT bar of the fp32
    oracle, and no [heads, N, N] tensor: the forward's peak device memory stays under 8 GB above what was allocated before"""
    import torch
    from depthmap_b200.depthmap_generation import DptBeitEngine
    from oracle import beit_dpt, synth_weights
    _no_tf32()
    name = 'beitl16_512'
    sd = synth_weights.make_beit_dpt_state_dict(name, seed=3)
    eng = DptBeitEngine(sd, name, cuda_device)
    img = synth_rgb(1600, 1600, 40)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    got = eng.forward_batch(torch.from_numpy(img).unsqueeze(0).to(cuda_device), 1600, 1600)[0].cpu().numpy()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"[memory] beitl16_512 net 1600: forward peak {peak / 2**30:.2f} GB above the weights")
    assert peak < 8 * 2**30, peak
    del eng
    torch.cuda.empty_cache()
    with torch.no_grad():      # get_raw_prediction on the GPU (net = image size, so its final resize is the identity)
        want = beit_dpt.forward({k: v.to(cuda_device) for k, v in sd.items()}, beit_dpt.preprocess(img, 1600, 1600).to(cuda_device), name)[0]
    want = want.cpu().numpy()
    ref16 = precision.reference_fp16_error('beit', img, sd, name, (1600, 1600), want, cuda_device)
    precision.check(f"{name} net 1600 (streamed relative-position table)", got, want, ref16)


def test_graph_net_1536_equals_eager(cuda_device, monkeypatch):
    """type 1 at net 1536 (a 96 x 96 window, whose whole table would not fit in shared memory) through the engine's CUDA graph
    (call 2 captures, call 3 replays): a result, bit-identical to the eager engine"""
    import torch
    from depthmap_b200.depthmap_generation import DptBeitEngine
    from oracle import synth_weights
    sd = synth_weights.make_beit_dpt_state_dict('beitl16_512', seed=3)
    rgb = torch.from_numpy(synth_rgb(1536, 1536, 41)).unsqueeze(0).to(cuda_device)
    monkeypatch.setenv("DEPTHMAP_B200_MODEL_GRAPH", "0")
    eager = DptBeitEngine(sd, 'beitl16_512', cuda_device)
    a = eager.forward_batch(rgb, 1536, 1536)
    del eager
    torch.cuda.empty_cache()
    monkeypatch.delenv("DEPTHMAP_B200_MODEL_GRAPH")
    eng = DptBeitEngine(sd, 'beitl16_512', cuda_device)
    assert torch.isfinite(a).all() and float(a.max() - a.min()) > 0
    for call in range(3):
        assert torch.equal(eng.forward_batch(rgb, 1536, 1536), a), call
    assert eng._graphs._graphs


# ---- B: pre-processing of float crops -----------------------------------------------------------------------------------
@pytest.mark.parametrize("rect,msize", [((0, 0, 512, 384), 512), ((37, 52, 300, 300), 512), ((10, 20, 700, 600), 384), ((5, 3, 640, 200), 1024)])
def test_patchify_f32_crops_vs_oracle(cuda_device, rect, msize):
    """dm_preprocess_patchify_f32_crops vs oracle.midas_boost.preprocess: identity (512 x 384 at msize 512), up-scale, down-scale and
    non-square crops; two crops of the same size at different origins in one launch, each checked against its own crop; within 1e-3
    on the fp16 operands"""
    import torch
    from depthmap_b200 import _lib as L
    from depthmap_b200.depthmap_generation import DptBeitEngine, midas_boost_net_size
    from oracle import midas_boost
    lib = L.load()
    rgb = synth_rgb(720, 800, 42)
    planar = torch.from_numpy((rgb.astype(np.float64) / 255.0).astype(np.float32).transpose(2, 0, 1).copy()).to(cuda_device)
    x, y, w, h = rect
    nw, nh = midas_boost_net_size(w, h, msize)
    assert (nw, nh) == midas_boost.net_size(w, h, msize)
    crops = [rect, (x + 13, y + 7, w, h)]                                      # same net shape, different origins
    rects = torch.tensor(crops, dtype=torch.int32).to(cuda_device)
    kpad = 768
    out = torch.full((2 * (nh // 16) * (nw // 16), kpad), float("nan"), dtype=torch.float16, device=cuda_device)
    m, s, c = (L.ctypes.c_float * 3)(*DptBeitEngine.BOOST_MEAN), (L.ctypes.c_float * 3)(*DptBeitEngine.BOOST_STD), (L.ctypes.c_int * 3)(*DptBeitEngine.CHAN_MAP)
    L.check(lib.dm_preprocess_patchify_f32_crops(planar.data_ptr(), 720, 800, rects.data_ptr(), 2, nh, nw, 16, m, s, c, out.data_ptr(), kpad, L.stream_ptr()))
    torch.cuda.synchronize()
    got = out.float().cpu()
    half = got.shape[0] // 2
    for i, (cx, cy, cw, ch) in enumerate(crops):
        crop = (rgb.astype(np.float64) / 255.0)[cy:cy + ch, cx:cx + cw, ::-1]     # estimateboost's channel order
        want = midas_boost.preprocess(np.ascontiguousarray(crop), msize)[0]       # [3, nh, nw]
        want = want.view(3, nh // 16, 16, nw // 16, 16).permute(1, 3, 0, 2, 4).reshape(-1, 768)
        err = (got[i * half:(i + 1) * half] - want).abs().max().item()
        assert err < 1e-3, (i, err)
    assert not torch.equal(got[:half], got[half:])


# ---- C / D: the engines and BoostPipeline -------------------------------------------------------------------------------
def _oracle_forward(cuda_device, sd, name):
    import torch
    from oracle import beit_dpt
    sdd = {k: v.to(cuda_device) for k, v in sd.items()}

    def forward(x):
        with torch.no_grad():
            return beit_dpt.forward(sdd, x.to(cuda_device), name)
    return forward


def _merge_fn(cuda_device, psd):
    import torch
    from oracle import pix2pix as op2p
    psd = {k: v.to(cuda_device) for k, v in psd.items()}

    def merge(outer, inner):
        with torch.no_grad():
            return op2p.unet(psd, op2p.merge_input(outer, inner).to(cuda_device))[0, 0].cpu().numpy()
    return merge


class _OracleMidas:
    """Test double for the DPT engine under BOOST: estimatemidasBoost's network and resize through the fp32 oracle (not normalised:
    the pipeline normalises), so that the glue test isolates what BOOST adds from the fp16-operand error of the network."""

    def __init__(self, forward, device, const=False):
        self.forward, self.device, self.const = forward, device, const

    def forward_batch(self, rgb, net_w, net_h=None, out_hw=None, planar=None):
        import cv2
        import torch
        from oracle import midas_boost
        img, (x, y, w, h) = planar
        crop = img[:, y:y + h, x:x + w].permute(1, 2, 0).cpu().numpy().astype(np.float64)[:, :, ::-1]
        if self.const:
            return torch.full((1, h, w), 0.5, dtype=torch.float32, device=self.device)
        with torch.no_grad():
            pred = self.forward(midas_boost.preprocess(np.ascontiguousarray(crop), net_w)).squeeze().cpu().numpy()
        return torch.from_numpy(cv2.resize(pred, (w, h), interpolation=cv2.INTER_CUBIC)).to(self.device).unsqueeze(0)


def test_boost_midas_glue_vs_oracle(cuda_device):
    import cv2
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from oracle import boost as ob, midas_boost, synth_weights
    _no_tf32()
    sd = synth_weights.make_beit_dpt_state_dict('beitl16_512', seed=3)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    fwd = _oracle_forward(cuda_device, sd, 'beitl16_512')
    pipe = BoostPipeline(_OracleMidas(fwd, cuda_device), UnetMergeEngine(psd, cuda_device), cuda_device, 1)
    rgb = synth_rgb(300, 420, 12)
    got = pipe.run(rgb, 1600)
    want = ob.estimateboost(cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0, 1, midas_boost.estimate_fn(fwd), _merge_fn(cuda_device, psd), 1600)
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] boost glue, type 1 (oracle DPT, our merge network / resizes / normalisations / fit / blend): max {mx:.3e} mean {mean:.3e}")
    assert mx < 5e-4 and mean < 5e-5, (mx, mean)


@pytest.mark.parametrize("model_type,hw,rmax", [(1, (300, 420), 1600), (2, (400, 288), 1100), (3, (300, 420), 1600)])
def test_estimateboost_midas_vs_oracle(cuda_device, model_type, hw, rmax):
    import cv2
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import DptBeitEngine, DptVitEngine
    from oracle import boost as ob, midas_boost, synth_weights
    _no_tf32()
    name = NAMES[model_type]
    sd = synth_weights.make_beit_dpt_state_dict(name, seed=3)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    eng = (DptVitEngine if model_type == 3 else DptBeitEngine)(sd, name, cuda_device)
    pipe = BoostPipeline(eng, UnetMergeEngine(psd, cuda_device), cuda_device, model_type)
    rgb = synth_rgb(hw[0], hw[1], 12)
    info = {}
    got = pipe.run(rgb, rmax, info=info)
    oinfo = {}
    want = ob.estimateboost(cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0, model_type, midas_boost.estimate_fn(_oracle_forward(cuda_device, sd, name)),
                            _merge_fn(cuda_device, psd), rmax, info=oinfo)
    assert got.shape == want.shape == hw and got.dtype == np.float32
    assert info["rects"] == oinfo["patches"] and info["whole"] == oinfo["whole_size"] and len(info["rects"]) >= 1
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] boost {name} {hw} rmax {rmax}: {len(info['rects'])} patches, whole {info['whole']}, ours max {mx:.3e} mean {mean:.3e} "
          f"(reference policy: fp32)")
    assert mx < 3e-3 and mean < 6e-4, (mx, mean)


def test_constant_prediction_raises(cuda_device):
    """estimatemidasBoost cannot normalise a constant prediction (the reference's next cv2.resize fails): ValueError"""
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from oracle import synth_weights
    pipe = BoostPipeline(_OracleMidas(None, cuda_device, const=True), UnetMergeEngine(synth_weights.make_pix2pix_state_dict(seed=1), cuda_device),
                         cuda_device, 1)
    with pytest.raises(ValueError):
        pipe.run(synth_rgb(256, 320, 4), 1000)


# ---- E: ModelHolder and the funnel --------------------------------------------------------------------------------------
def test_modelholder_and_funnel_boost_type1(cuda_device):
    """ensure_models(1, device, boost=True): op-level engine + merge network; get_raw_prediction ignores the net size and returns
    invert = False (reference :402); the funnel's depth_prediction is pipeline.run's; types 12-14 still refuse BOOST"""
    from PIL import Image
    from depthmap_b200 import core
    from depthmap_b200.depthmap_generation import DptBeitEngine
    from oracle import synth_weights
    sd = synth_weights.make_beit_dpt_state_dict('beitl16_512', seed=3)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: psd if t == "pix2pix" else sd
    try:
        holder.update_settings(boost_rmax=1000)
        holder.ensure_models(1, cuda_device, True)
        assert isinstance(holder.depth_model, DptBeitEngine) and holder.pix2pix_model is not None
        img = synth_rgb(256, 320, 4)
        pred, invert = holder.get_raw_prediction(Image.fromarray(img), 512, 512)
        assert invert is False and pred.shape == (256, 320) and pred.dtype == np.float32 and np.isfinite(pred).all()
        pred2, _ = holder.get_raw_prediction(Image.fromarray(img), 64, 64)
        assert np.array_equal(pred, pred2)
        inp = dict(compute_device='GPU', model_type=1, net_width=512, net_height=512, boost=True, do_output_depth=True,
                   do_output_depth_prediction=True, gen_stereo=False, gen_normalmap=False)
        out = list(core.core_generation_funnel(None, [Image.fromarray(img)], None, None, inp, ops={'boost_rmax': 1000}))
        assert [k for _, k, _ in out][:2] == ['depth_prediction', 'depth']
        assert np.array_equal(out[0][2], holder.pix2pix_model.run(img, 1000))
        with pytest.raises(NotImplementedError):
            holder.ensure_models(12, cuda_device, True)
    finally:
        holder.unload_models()
        holder.weights_provider = None


# ---- patch-parallel -----------------------------------------------------------------------------------------------------
def test_sharded_boost_type1_equals_single_rank(cuda_device):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29619", os.path.join(ROOT, "tools", "dist_check.py"), "--boost-model-type", "1"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "dist_check ok" in r.stdout and "boost_equal=True" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
