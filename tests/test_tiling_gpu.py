"""GPU: tiling mode (circular padding in every padded convolution of the depth networks) on the sm_90a kernels.

The kernels against fp32 torch (F.conv2d on F.pad(mode='circular')), the engines with circular=True against the circular oracle
(tests/circular_oracle.py around the fp32 functional oracles; pinned to the reference's modules in tests/test_tiling_cpu.py) at the
bar of tests/precision.py, whose fp16-policy yardstick is evaluated circularly as well, and the public surface: ModelHolder, the
funnel and BOOST."""
import numpy as np
import pytest

import precision
from circular_oracle import circular_convs
from synth import synth_rgb

pytestmark = pytest.mark.gpu


def _lib():
    from depthmap_b200 import _lib as L
    return L, L.load()


def _circ(x_nchw, p):
    import torch.nn.functional as F
    return F.pad(x_nchw, (p, p, p, p), mode="circular")


# ---- kernels -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C", [(2, 7, 5, 64), (1, 1, 9, 8), (1, 6, 1, 16), (3, 1, 1, 64), (1, 37, 45, 128)])
def test_halo_equals_circular_pad(cuda_device, B, H, W, C):
    import torch
    L, lib = _lib()
    x = torch.randn(B, H, W, C, generator=torch.Generator().manual_seed(1)).half().to(cuda_device)
    halo = torch.full((B, H + 2, W + 2, C), float("nan"), dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_circular_halo_f16(x.data_ptr(), B, H, W, C, halo.data_ptr(), L.stream_ptr()), "dm_circular_halo_f16")
    want = _circ(x.permute(0, 3, 1, 2).float(), 1).permute(0, 2, 3, 1).half()
    assert torch.equal(halo, want)


# (Cout, epilogue): Cout picks the tile (256 -> 64 x 256, 128 -> 128 x 128, 64 -> 128 x 64, 96 / 32 -> 128 x 32)
CONV_CASES = [(256, "store"), (128, "store"), (64, "store"), (96, "store"), (128, "resid"), (64, "f32"), (32, "head")]
SHAPES = [(2, 7, 5), (1, 1, 9), (1, 6, 1), (2, 3, 3), (1, 37, 45)]


@pytest.mark.parametrize("cout,epi", CONV_CASES)
@pytest.mark.parametrize("B,H,W", SHAPES)
def test_circular_conv3x3_vs_torch(cuda_device, cout, epi, B, H, W):
    """dm_conv3x3_circular_ex for each tile shape and epilogue at odd, 1-wide and sub-box sizes against fp32 torch; the zero-padded
    conv on the same operands is bit-identical to it away from the border and differs at the border"""
    import torch
    import torch.nn.functional as F
    L, _ = _lib()
    ops = L.Ops()
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + W + cout)
    cin = 64 if cout != 128 else 128
    x = torch.randn(B, H, W, cin, generator=g).half().to(cuda_device)
    w = (torch.randn(cout, cin, 3, 3, generator=g) / (3.0 * cin ** 0.5)).to(cuda_device)
    bias = (0.1 * torch.randn(cout, generator=g)).to(cuda_device)
    wt = w.half().permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()
    xf = x.permute(0, 3, 1, 2).float()
    conv = F.conv2d(_circ(xf, 1), w.half().float(), bias).permute(0, 2, 3, 1)          # [B, H, W, cout] fp32
    halo = torch.empty(B * (H + 2) * (W + 2) * cin + 7, dtype=torch.float16, device=cuda_device)
    M = B * H * W
    R = torch.randn(B, H, W, cout, generator=g).half().to(cuda_device)
    R2 = torch.randn(B, H, W, cout, generator=g).half().to(cuda_device)
    X0 = torch.randn(M, cout, generator=g).to(cuda_device)
    gamma = torch.randn(cout, generator=g).to(cuda_device)

    def run(halo_t):
        """-> (outputs, their fp32 expectation as a function of the conv result [B, H, W, cout])"""
        if epi == "store":
            C = torch.empty(B, H, W, cout, dtype=torch.float16, device=cuda_device)
            C2 = torch.empty_like(C)
            ops.conv3x3(x, B, H, W, cin, wt, cout, act=L.ACT_RELU, bias=bias, C=C, C2=C2, R=R, R2=R2, halo=halo_t)
            return [C, C2], lambda cv: [torch.relu(cv) + R.float() + R2.float(), torch.relu(torch.relu(cv) + R.float() + R2.float())]
        if epi == "resid":
            X = X0.clone()
            ops.conv3x3(x, B, H, W, cin, wt, cout, epi=L.EPI_RESID_F32, bias=bias, X=X, ldx=cout, gamma=gamma, halo=halo_t)
            return [X], lambda cv: [X0 + gamma * cv.reshape(M, cout)]
        if epi == "f32":
            X = torch.empty(M, cout, device=cuda_device)
            ops.conv3x3(x, B, H, W, cin, wt, cout, epi=L.EPI_STORE_F32, bias=bias, X=X, ldx=cout, halo=halo_t)
            return [X], lambda cv: [cv.reshape(M, cout)]
        X = torch.empty(M, device=cuda_device)
        ops.conv3x3(x, B, H, W, cin, wt, 32, epi=L.EPI_HEAD, act=L.ACT_RELU, bias=bias, X=X, gamma=gamma, head_b2=0.05, halo=halo_t)
        return [X], lambda cv: [torch.relu(torch.relu(cv).reshape(M, 32) @ gamma + 0.05)]

    n0 = ops.launches
    got, ref = run(halo)
    assert ops.launches - n0 == 2
    for gt, want in zip(got, ref(conv)):
        err = (gt.float().reshape(want.shape) - want).abs().max().item()
        assert err < 2e-2 * max(1.0, want.abs().max().item()), (epi, err)
    if epi == "resid":
        return
    zgot, zref = run(None)
    zero = F.conv2d(xf, w.half().float(), bias, padding=1).permute(0, 2, 3, 1)
    for a, z, wz in zip(got, zgot, zref(zero)):
        a, z = a.reshape(B, H, W, -1), z.reshape(B, H, W, -1)
        assert (z.float() - wz.reshape(z.shape)).abs().max().item() < 2e-2 * max(1.0, wz.abs().max().item())
        if H > 2 and W > 2:
            assert torch.equal(a[:, 1:-1, 1:-1], z[:, 1:-1, 1:-1])
        border = torch.ones(H, W, dtype=torch.bool, device=cuda_device)
        border[1:-1, 1:-1] = False
        assert (a[:, border] != z[:, border]).any()


def test_circular_conv_rejects_small_halo(cuda_device):
    import torch
    L, _ = _lib()
    x = torch.zeros(1, 4, 4, 64, dtype=torch.float16, device=cuda_device)
    wt = torch.zeros(64, 9 * 64, dtype=torch.float16, device=cuda_device)
    C = torch.empty_like(x)
    with pytest.raises(ValueError):
        L.Ops().conv3x3(x, 1, 4, 4, 64, wt, 64, C=C, halo=torch.empty(6 * 6 * 64 - 1, dtype=torch.float16, device=cuda_device))


@pytest.mark.parametrize("B,H,W,C", [(2, 37, 37, 64), (1, 1, 5, 64), (1, 6, 1, 128), (2, 7, 9, 64), (1, 2, 2, 64)])
def test_circular_im2col_s2_vs_torch(cuda_device, B, H, W, C):
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn(B, H, W, C, generator=g).half().to(cuda_device)
    w = (torch.randn(C, C, 3, 3, generator=g) * 0.05).half().to(cuda_device)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    cols = torch.empty(B * Ho * Wo, 9 * C, dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_im2col_s2_circular_f16(x.data_ptr(), B, H, W, C, cols.data_ptr(), L.stream_ptr()), "dm_im2col_s2_circular_f16")
    pad = _circ(x.permute(0, 3, 1, 2).float(), 1)
    want = F.unfold(pad, 3, stride=2).view(B, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 9 * C)
    assert torch.equal(cols.float(), want)                       # a gather: exact
    got = (cols.float() @ w.permute(0, 2, 3, 1).reshape(C, 9 * C).float().t()).view(B, Ho, Wo, C)
    ref = F.conv2d(pad, w.float(), stride=2).permute(0, 2, 3, 1)
    assert (got - ref).abs().max().item() < 1e-3


def _stem_cols_ref(net_input):
    """im2col of the 7x7 stride-2 circular-pad-3 stem on the network input [B, 3, h, w] -> [B*Ho*Wo, 147] ordered (ky, kx, c)"""
    import torch.nn.functional as F
    B, _, h, w = net_input.shape
    Ho, Wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return F.unfold(_circ(net_input, 3), 7, stride=2).view(B, 3, 49, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 147)


MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _normalise(t):
    import torch
    return (t - torch.tensor(MEAN).view(1, 3, 1, 1)) / torch.tensor(STD).view(1, 3, 1, 1)


@pytest.mark.parametrize("hw,net", [((64, 96), (64, 96)), ((70, 90), (64, 96)), ((40, 30), (32, 64))])
def test_circular_stem_uint8_vs_torch(cuda_device, hw, net):
    import ctypes
    import cv2
    import torch
    L, lib = _lib()
    B, (H, W), (nh, nw) = 2, hw, net
    imgs = [synth_rgb(H, W, 40 + i) for i in range(B)]
    rgb = torch.from_numpy(np.stack(imgs)).to(cuda_device)
    Ho, Wo = (nh - 1) // 2 + 1, (nw - 1) // 2 + 1
    cols = torch.empty(B * Ho * Wo, 192, dtype=torch.float16, device=cuda_device)
    m, s = (ctypes.c_float * 3)(*MEAN), (ctypes.c_float * 3)(*STD)
    L.check(lib.dm_leres_stem_im2col_circular(rgb.data_ptr(), B, H, W, nh, nw, m, s, cols.data_ptr(), L.stream_ptr()), "stem")
    inp = torch.stack([torch.from_numpy(cv2.resize(im.astype(np.float32) / 255.0, (nw, nh)).transpose(2, 0, 1).copy()) for im in imgs])
    want = _stem_cols_ref(_normalise(inp))
    torch.cuda.synchronize()
    assert (cols[:, :147].float().cpu() - want).abs().max().item() < 1e-2
    assert float(cols[:, 147:].abs().max()) == 0.0


def test_circular_stem_f32_crops_vs_torch(cuda_device):
    import ctypes
    import cv2
    import torch
    L, lib = _lib()
    Hi, Wi = 100, 120
    planar = torch.from_numpy(synth_rgb(Hi, Wi, 7).transpose(2, 0, 1).astype(np.float32) / 255.0).contiguous()
    rects = [(0, 0, 64, 64), (10, 20, 50, 70)]
    net = 64
    m, s = (ctypes.c_float * 3)(*MEAN), (ctypes.c_float * 3)(*STD)
    Ho = (net - 1) // 2 + 1
    pl = planar.to(cuda_device)

    def ref(rect):
        x0, y0, w, h = rect
        crop = planar[:, y0:y0 + h, x0:x0 + w].permute(1, 2, 0).numpy()
        return _stem_cols_ref(_normalise(torch.from_numpy(cv2.resize(crop, (net, net)).transpose(2, 0, 1).copy()).unsqueeze(0)))
    one = torch.empty(Ho * Ho, 192, dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_leres_stem_im2col_f32_circular(pl.data_ptr(), Hi, Wi, *rects[1], net, net, m, s, one.data_ptr(), L.stream_ptr()), "stem")
    r = torch.tensor(rects, dtype=torch.int32).to(cuda_device)
    batch = torch.empty(2 * Ho * Ho, 192, dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_leres_stem_im2col_f32_batch_circular(pl.data_ptr(), Hi, Wi, r.data_ptr(), 2, net, net, m, s, batch.data_ptr(), L.stream_ptr()),
            "stem batch")
    torch.cuda.synchronize()
    assert (one[:, :147].float().cpu() - ref(rects[1])).abs().max().item() < 1e-2
    assert torch.equal(batch[Ho * Ho:], one)
    assert (batch[:Ho * Ho, :147].float().cpu() - ref(rects[0])).abs().max().item() < 1e-2


# ---- engines against the circular oracle ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("encoder,hw,net", [("vits", (70, 98), 70), ("vitl", (84, 70), 70)])
def test_dav2_tiling_vs_oracle(cuda_device, encoder, hw, net):
    import torch
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import dav2 as odav2
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict(encoder, seed=1)
    eng = DepthAnythingV2Engine(sd, encoder, cuda_device, circular=True)
    imgs = [synth_rgb(hw[0], hw[1], s) for s in (3, 4)]
    got = eng.forward_batch(torch.from_numpy(np.stack(imgs)).to(cuda_device), net).cpu().numpy()
    zero = DepthAnythingV2Engine(sd, encoder, cuda_device).forward_batch(torch.from_numpy(np.stack(imgs)).to(cuda_device), net).cpu().numpy()
    for i, img in enumerate(imgs):
        with circular_convs(odav2):
            want, _ = odav2.get_raw_prediction(img, sd, encoder, net)
            ref16 = precision.reference_fp16_error('dav2', img, sd, encoder, net, want, cuda_device)
        precision.check(f"tiling dav2 {encoder} {hw} net {net} img{i}", got[i], want, ref16)
        assert precision.norm_err(zero[i], want)[0] > 1e-2          # the zero-padded engine is visibly different


def _dpt_check(cuda_device, cls, name, hw, net, B, seed):
    import torch
    from oracle import beit_dpt, synth_weights
    sd = synth_weights.make_beit_dpt_state_dict(name, seed=seed)
    eng = cls(sd, name, cuda_device, circular=True)
    imgs = [synth_rgb(hw[0], hw[1], 10 + s) for s in range(B)]
    got = eng.forward_batch(torch.from_numpy(np.stack(imgs)).to(cuda_device), net[0], net[1]).cpu().numpy()
    for i, img in enumerate(imgs):
        with circular_convs(beit_dpt):
            want, _ = beit_dpt.get_raw_prediction(img, sd, name, net[0], net[1])
            ref16 = precision.reference_fp16_error('beit', img, sd, name, net, want, cuda_device)
        precision.check(f"tiling {name} {hw} net {net} img{i}", got[i], want, ref16)


@pytest.mark.parametrize("name,hw,net,B", [("beit_tiny", (64, 96), (64, 64), 2), ("beit_tiny", (80, 50), (64, 64), 2),
                                           ("beitl16_512", (512, 512), (512, 512), 1)])
def test_beit_tiling_vs_oracle(cuda_device, name, hw, net, B):
    from depthmap_b200.depthmap_generation import DptBeitEngine
    _dpt_check(cuda_device, DptBeitEngine, name, hw, net, B, 3)


def test_vit_tiny_tiling_vs_oracle(cuda_device):
    from depthmap_b200.depthmap_generation import DptVitEngine
    _dpt_check(cuda_device, DptVitEngine, 'vit_tiny', (96, 128), (96, 96), 2, 5)


@pytest.mark.parametrize("hw,net", [((64, 96), (96, 64)), ((90, 70), (64, 96))])
def test_leres_tiling_vs_oracle(cuda_device, hw, net):
    import torch
    from depthmap_b200.depthmap_generation import LeresEngine
    from oracle import leres, synth_weights
    sd = synth_weights.make_leres_state_dict(seed=2)
    eng = LeresEngine(sd, cuda_device, circular=True)
    imgs = [synth_rgb(hw[0], hw[1], 60 + s) for s in range(2)]
    x = torch.from_numpy(np.stack(imgs)).to(cuda_device)
    got = eng.forward_batch(x, net[0], net[1]).cpu().numpy()
    again = [eng.forward_batch(x, net[0], net[1]).cpu().numpy() for _ in range(2)]      # eager, capture, replay of the CUDA graph
    for i, img in enumerate(imgs):
        with circular_convs(leres):
            want, _ = leres.get_raw_prediction(img, sd, net[0], net[1])
        mx, mean = precision.norm_err(got[i], want)
        print(f"[precision] tiling leres {hw} net {net} img{i}: ours max {mx:.3e} mean {mean:.3e} (reference policy: fp32)")
        assert mx < 3e-3 and mean < 6e-4, (mx, mean)
    assert all(np.array_equal(a, got) for a in again)


def _zoe_sd(variant, seed):
    if variant == "nk":
        from test_zoe_gpu import make_zoe_state_dict
        return make_zoe_state_dict('beit_tiny', seed)
    from test_zoedepth_n_k_gpu import make_state_dict
    return make_state_dict('beit_tiny', variant, seed)


@pytest.mark.parametrize("variant", ["nk", "n", "k"])
def test_zoedepth_tiling_vs_oracle(cuda_device, variant):
    import torch
    from depthmap_b200.depthmap_generation import ZoeDepthEngine, ZoeDepthNKEngine
    from oracle import beit_dpt
    from oracle import zoedepth as ozd
    from oracle import zoedepth_single as ozs
    from test_zoedepth_n_k_gpu import check_bar, reference_fp16_error_single
    seed, hw, net = 1, (96, 128), (64, 64)
    sd = _zoe_sd(variant, seed)
    eng = (ZoeDepthNKEngine(sd, cuda_device, core_name='beit_tiny', circular=True) if variant == "nk" else
           ZoeDepthEngine(sd, cuda_device, variant, core_name='beit_tiny', circular=True))
    imgs = [synth_rgb(hw[0], hw[1], 5 + s) for s in range(2)]
    got = eng.forward_batch(torch.from_numpy(np.stack(imgs)).to(cuda_device), net[0], net[1]).cpu().numpy()
    for i, img in enumerate(imgs):
        with circular_convs(beit_dpt):
            if variant == "nk":
                want, _ = ozd.get_raw_prediction(img, sd, net[0], net[1], core_name='beit_tiny')
                ref16 = precision.reference_fp16_error_zoe(img, sd, net[0], net[1], 'beit_tiny', want, cuda_device)
            else:
                want, _ = ozs.get_raw_prediction_single(img, sd, variant, net[0], net[1], core_name='beit_tiny')
                ref16 = reference_fp16_error_single(img, sd, variant, net[0], net[1], 'beit_tiny', want, cuda_device)
        label = f"tiling zoedepth_{variant} tiny {hw} net {net} img{i}"
        if variant == "k":
            check_bar(label, variant, got[i], want, ref16, tiny=True)
        else:
            # NK: the rule of tests/test_zoe_gpu.py.  N: its fixed bars (check_bar) sit at the fp16 noise level of this input's nearly
            # flat circular map (measured on an H100: mean 6.1e-4 against a 6e-4 bar, the all-fp16 evaluation 6.0e-4), so N is held to
            # the same fp16-policy rule
            precision.check(label, got[i], want, ref16, slack=1.5)


# ---- public surface ------------------------------------------------------------------------------------------------------------
def _served_state_dict(model_type):
    from oracle import synth_weights
    from oracle import zoedepth_single as ozs
    if model_type == 0:
        return synth_weights.make_leres_state_dict(seed=3)
    if model_type in (1, 2, 3):
        name = {1: 'beitl16_512', 2: 'beitl16_384', 3: 'vitl16_384'}[model_type]
        sd = synth_weights.make_beit_dpt_state_dict(name, seed=4)
        return {"model": sd, "optimizer": None}
    if model_type in (7, 8, 9):
        core = {"core.core." + k: v for k, v in synth_weights.make_beit_dpt_state_dict('beitl16_384', seed=4).items()}
        core.update(synth_weights.make_zoedepth_head_state_dict(feat_ch=256, seed=104) if model_type == 9 else
                    ozs.make_zoedepth_single_head_state_dict({7: 'n', 8: 'k'}[model_type], feat_ch=256, seed=104))
        return core
    return synth_weights.make_dav2_state_dict({12: 'vits', 13: 'vitb', 14: 'vitl'}[model_type], seed=4)


ENGINES = {0: "LeresEngine", 1: "DptBeitEngine", 2: "DptBeitEngine", 3: "DptVitEngine", 7: "ZoeDepthEngine", 8: "ZoeDepthEngine",
           9: "ZoeDepthNKEngine", 12: "DepthAnythingV2Engine", 13: "DepthAnythingV2Engine", 14: "DepthAnythingV2Engine"}


@pytest.mark.parametrize("model_type", sorted(ENGINES))
def test_model_holder_tiling_mode(cuda_device, model_type):
    """every served model type loads with tiling_mode=True on its op-level engine with circular padding, and predicts"""
    from PIL import Image
    from depthmap_b200.depthmap_generation import ModelHolder
    sd = _served_state_dict(model_type)
    mh = ModelHolder()
    mh.weights_provider = lambda t: sd
    try:
        mh.ensure_models(model_type, cuda_device, False, tiling_mode=True)
        assert type(mh.depth_model).__name__ == ENGINES[model_type] and mh.depth_model.circular is True and mh.tiling_mode is True
        w, h = (64, 64) if model_type in (0, 1, 2, 3, 7, 8, 9) else (70, 70)
        pred, invert = mh.get_raw_prediction(Image.fromarray(synth_rgb(h, w + 14, 6)), w, h)
        assert pred.shape == (h, w + 14) and pred.dtype == np.float32 and np.isfinite(pred).all()
        assert invert is (model_type in (0, 7, 8, 9))
        mh.ensure_models(model_type, cuda_device, False, tiling_mode=False)          # the flag changed: reloaded zero-padded
        assert getattr(mh.depth_model, "circular", False) is False and mh.tiling_mode is False
    finally:
        mh.unload_models()


def test_funnel_tiling_mode(cuda_device):
    """core_generation_funnel with tiling_mode on: Depth-Anything-V2 S through the circular engine equals the circular oracle"""
    from PIL import Image
    from depthmap_b200 import core
    from oracle import dav2 as odav2
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=2)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: sd
    img = synth_rgb(70, 98, 8)
    try:
        inp = dict(compute_device='GPU', model_type=12, net_width=70, net_height=70, net_size_match=False, boost=False, tiling_mode=True,
                   do_output_depth=True, gen_stereo=False, gen_normalmap=False, do_output_depth_prediction=True)
        out = list(core.core_generation_funnel(None, [Image.fromarray(img)], None, None, inp, ops={}))
        assert type(holder.depth_model).__name__ == "DepthAnythingV2Engine" and holder.depth_model.circular is True
        pred = out[0][2]
    finally:
        holder.unload_models()
        holder.weights_provider = None
    with circular_convs(odav2):
        want, _ = odav2.get_raw_prediction(img, sd, 'vits', 70)
        ref16 = precision.reference_fp16_error('dav2', img, sd, 'vits', 70, want, cuda_device)
    precision.check("tiling funnel dav2 vits", pred, want, ref16)


def test_boost_leres_tiling_vs_oracle(cuda_device):
    """BOOST (model type 0) with tiling: circular LeReS forwards and the usual zero-padded merge network, against oracle/boost.py
    driven by the circular LeReS oracle"""
    import cv2
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import LeresEngine
    from oracle import boost as ob, leres, synth_weights
    from test_boost_gpu import _no_tf32, _oracle_fns
    _no_tf32()
    lsd = synth_weights.make_leres_state_dict(seed=2)
    psd = synth_weights.make_pix2pix_state_dict(seed=1)
    pipe = BoostPipeline(LeresEngine(lsd, cuda_device, circular=True), UnetMergeEngine(psd, cuda_device), cuda_device, 0)
    rgb = synth_rgb(300, 420, 12)
    info = {}
    got = pipe.run(rgb, 1600, info=info)
    estimate, merge = _oracle_fns(cuda_device, lsd, psd)
    oinfo = {}
    with circular_convs(leres):
        want = ob.estimateboost(cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0, 0, estimate, merge, 1600, info=oinfo)
    assert got.shape == want.shape == (300, 420)
    assert info["rects"] == oinfo["patches"] and len(info["rects"]) >= 1
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] tiling boost res101 (300, 420): ours max {mx:.3e} mean {mean:.3e}")
    assert mx < 3e-3 and mean < 6e-4, (mx, mean)
