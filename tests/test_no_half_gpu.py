"""GPU: the split (fp32-class) path of `no_half` — kernels against fp64 references, Depth-Anything-V2 end to end against the fp32
oracle, and the ModelHolder / funnel routing.

Kernel bars: the split kernel's largest error against an fp64 evaluation of the same fp32 operands is within 8x of what fp32
arithmetic itself gives (torch in fp32, TF32 off), and (GEMM) at least 100x below the fp16 kernel's.  Network bars: normalised
max error <= 1e-4 and mean <= 1e-5 against the fp32 oracle, and >= 20x below the fp16 engine's error on the same input."""
import contextlib

import numpy as np
import pytest

import precision
from circular_oracle import circular_convs
from synth import synth_rgb

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def _no_tf32():
    import torch
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _split(x):
    """fp32 [..., n] -> split fp16 [..., 3n] = [hi | lo | hi]"""
    import torch
    hi = x.half()
    return torch.cat([hi, (x - hi.float()).half(), hi], dim=-1).contiguous()


def _unsplit(t):
    n = t.shape[-1] // 3
    return t[..., :n].double() + t[..., n:2 * n].double()


def _ops():
    from depthmap_b200 import _lib
    return _lib.Ops()


def _gelu64(x):
    import torch
    return 0.5 * x * (1 + torch.erf(x / np.sqrt(2.0)))


def _err(a, b):
    return float((a.double() - b.double()).abs().max())


# ---- split GEMM -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1024, 3072, 12288])
def test_split_gemm_vs_fp64(cuda_device, K):
    import torch
    from depthmap_b200 import _lib
    from depthmap_b200.depthmap_generation import split_weight
    g = torch.Generator(device=cuda_device).manual_seed(K)
    M, N = 301, 96                                             # odd M, an N tail past the 64-wide split tile
    A = torch.randn(M, K, device=cuda_device, generator=g)
    W = torch.randn(N, K, device=cuda_device, generator=g) * 0.02
    bias = torch.randn(N, device=cuda_device, generator=g) * 0.1
    ref = A.double() @ W.double().t() + bias.double()
    with _no_tf32():
        e32 = _err(A @ W.t() + bias, ref)
    ops = _ops()
    sw = split_weight(W)
    out = torch.empty(M, N, device=cuda_device)
    ops.gemm_split(_split(A), 3 * K, sw.t, 3 * K, sw.scale, M, N, 3 * K, epi=_lib.EPI_STORE_F32, bias=bias, X=out, ldx=N)
    C = torch.empty(M, 3 * N, dtype=torch.float16, device=cuda_device)
    ops.gemm_split(_split(A), 3 * K, sw.t, 3 * K, sw.scale, M, N, 3 * K, bias=bias, C=C, ldc=3 * N)
    o16 = torch.empty(M, N, device=cuda_device)
    ops.gemm(A.half(), K, W.half(), K, M, N, K, epi=_lib.EPI_STORE_F32, bias=bias, X=o16, ldx=N)
    torch.cuda.synchronize()
    e_split, e_store, e16 = _err(out, ref), _err(_unsplit(C), ref), _err(o16, ref)
    print(f"split gemm K={K}: split {e_split:.3g} (split store {e_store:.3g}), fp32 {e32:.3g}, fp16 {e16:.3g}")
    assert e_split <= 8 * e32 and e_store <= 8 * e32 + 2.0 ** -22 * float(ref.abs().max())
    assert e16 >= 100 * e_split
    assert torch.equal(C[:, :N], C[:, 2 * N:])


def test_split_gemm_epilogues_vs_fp64(cuda_device):
    """every split epilogue: bias + GELU / ReLU with the relu copy, split residuals, LayerScale into fp32, pixel shuffle, fused head"""
    import torch
    from depthmap_b200 import _lib
    from depthmap_b200.depthmap_generation import split_weight
    g = torch.Generator(device=cuda_device).manual_seed(7)
    M, K, N = 301, 1024, 96
    A = torch.randn(M, K, device=cuda_device, generator=g)
    W = torch.randn(N, K, device=cuda_device, generator=g) * 0.02
    bias = torch.randn(N, device=cuda_device, generator=g) * 0.1
    R, R2 = (torch.randn(M, N, device=cuda_device, generator=g) for _ in range(2))
    gamma = torch.rand(N, device=cuda_device, generator=g)
    ops, sw, As = _ops(), split_weight(W), _split(A)
    acc64 = A.double() @ W.double().t() + bias.double()
    with _no_tf32():
        acc32 = A @ W.t() + bias
    new = lambda n=N: torch.empty(M, 3 * n, dtype=torch.float16, device=cuda_device)
    cases = []
    # bias + GELU
    C = new()
    ops.gemm_split(As, 3 * K, sw.t, 3 * K, sw.scale, M, N, 3 * K, act=_lib.ACT_GELU, bias=bias, C=C, ldc=3 * N)
    cases.append(("gelu", lambda: _unsplit(C), _gelu64(acc64), torch.nn.functional.gelu(acc32)))
    # bias + ReLU, relu copy of (acc + bias + R + R2)
    C1, C2 = new(), new()
    ops.gemm_split(As, 3 * K, sw.t, 3 * K, sw.scale, M, N, 3 * K, bias=bias, C=C1, ldc=3 * N, C2=C2, R=_split(R), ldr=3 * N, R2=_split(R2), ldr2=3 * N)
    s64, s32 = acc64 + R.double() + R2.double(), acc32 + R + R2
    cases.append(("resid", lambda: _unsplit(C1), s64, s32))
    cases.append(("relu copy", lambda: _unsplit(C2), s64.clamp_min(0), s32.clamp_min(0)))
    C3 = new()
    ops.gemm_split(As, 3 * K, sw.t, 3 * K, sw.scale, M, N, 3 * K, act=_lib.ACT_RELU, bias=bias, C=C3, ldc=3 * N)
    cases.append(("relu", lambda: _unsplit(C3), acc64.clamp_min(0), acc32.clamp_min(0)))
    # LayerScale + residual into the fp32 stream
    X0 = torch.randn(M, N, device=cuda_device, generator=g)
    X = X0.clone()
    ops.gemm_split(As, 3 * K, sw.t, 3 * K, sw.scale, M, N, 3 * K, epi=_lib.EPI_RESID_F32, bias=bias, X=X, ldx=N, gamma=gamma)
    cases.append(("layerscale", lambda: X, X0.double() + gamma.double() * acc64, X0 + gamma * acc32))
    # pixel shuffle (ConvTranspose2d k = s = 2 on a 7 x 43 grid, cout 24)
    s, cout, gh, gw = 2, 24, 7, 43
    P = torch.empty(1, gh * s, gw * s, 3 * cout, dtype=torch.float16, device=cuda_device)
    ops.gemm_split(As, 3 * K, sw.t, 3 * K, sw.scale, M, N, 3 * K, epi=_lib.EPI_PIXSHUF, bias=bias, C=P, ps=(s, cout, gh, gw))
    shuf = lambda t: t.reshape(1, gh, gw, s, s, cout).permute(0, 1, 3, 2, 4, 5).reshape(1, gh * s, gw * s, cout)
    cases.append(("pixel shuffle", lambda: _unsplit(P), shuf(acc64), shuf(acc32)))
    # fused head: relu(relu(acc + b) . w2 + b2), N = 32
    Wh, bh = W[:32].contiguous(), bias[:32].contiguous()
    swh, w2 = split_weight(Wh), torch.rand(32, device=cuda_device, generator=g) - 0.5
    D = torch.empty(M, device=cuda_device)
    ops.gemm_split(As, 3 * K, swh.t, 3 * K, swh.scale, M, 32, 3 * K, epi=_lib.EPI_HEAD, act=_lib.ACT_RELU, bias=bh, X=D, gamma=w2, head_b2=0.05)
    cases.append(("head", lambda: D, (acc64[:, :32].clamp_min(0) @ w2.double() + 0.05).clamp_min(0),
                  (acc32[:, :32].clamp_min(0) @ w2 + 0.05).clamp_min(0)))
    torch.cuda.synchronize()
    for name, got, r64, r32 in cases:
        e, e32 = _err(got(), r64), _err(r32, r64)
        # a split store also rounds the result to hi + lo (2^-22 of its magnitude)
        floor = 2.0 ** -22 * float(r64.abs().max()) if name not in ("layerscale", "head") else 0.0
        print(f"split epilogue {name}: {e:.3g} (fp32 {e32:.3g})")
        assert e <= 8 * e32 + floor, (name, e, e32)


# ---- split conv3x3 --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("circular", [False, True])
def test_split_conv3x3_vs_fp64(cuda_device, circular):
    import torch
    import torch.nn.functional as F
    from depthmap_b200 import _lib
    from depthmap_b200.depthmap_generation import _conv_w, split_weight
    g = torch.Generator(device=cuda_device).manual_seed(3)
    B, H, W_, Cin, Cout = 2, 19, 37, 256, 64                  # K = 9 * 256 per output
    x = torch.randn(B, H, W_, Cin, device=cuda_device, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device=cuda_device, generator=g) * 0.02
    bias = torch.randn(Cout, device=cuda_device, generator=g) * 0.1
    pad = (lambda t: F.pad(t, (1, 1, 1, 1), mode="circular")) if circular else (lambda t: F.pad(t, (1, 1, 1, 1)))
    xc = x.permute(0, 3, 1, 2)
    ref = (F.conv2d(pad(xc.double()), w.double(), bias.double())).permute(0, 2, 3, 1)
    with _no_tf32():
        e32 = _err(F.conv2d(pad(xc), w, bias).permute(0, 2, 3, 1), ref)
    sw = split_weight(_conv_w(w, Cin, Cout, torch.float32), 9)
    out = torch.empty(B, H, W_, 3 * Cout, dtype=torch.float16, device=cuda_device)
    halo = torch.empty(B * (H + 2) * (W_ + 2) * 3 * Cin, dtype=torch.float16, device=cuda_device) if circular else None
    ops = _ops()
    ops.conv3x3_split(_split(x), B, H, W_, Cin, sw.t, sw.scale, Cout, bias=bias, C=out, halo=halo)
    o16 = torch.empty(B, H, W_, Cout, dtype=torch.float16, device=cuda_device)
    h16 = torch.empty(B * (H + 2) * (W_ + 2) * Cin, dtype=torch.float16, device=cuda_device) if circular else None
    ops.conv3x3(x.half().contiguous(), B, H, W_, Cin, _conv_w(w, Cin, Cout), Cout, bias=bias, C=o16, halo=h16)
    torch.cuda.synchronize()
    e, e16 = _err(_unsplit(out), ref), _err(o16, ref)
    print(f"split conv3x3 circular={circular}: {e:.3g}, fp32 {e32:.3g}, fp16 {e16:.3g}")
    assert e <= 8 * e32 + 2.0 ** -22 * float(ref.abs().max()) and e16 >= 100 * e
    with pytest.raises(ValueError):
        ops.conv3x3_split(_split(x), B, H, W_, Cin, sw.t, sw.scale, Cout, bias=bias, C=out,
                          halo=torch.empty(10, dtype=torch.float16, device=cuda_device))


# ---- split attention ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [2, 65, 1370, 5477])
@pytest.mark.parametrize("heads", [6, 16])
def test_split_attention_vs_fp64(cuda_device, N, heads):
    import torch
    g = torch.Generator(device=cuda_device).manual_seed(N + heads)
    B, C = 2, heads * 64
    qkv = torch.randn(B * N, 3 * C, device=cuda_device, generator=g)
    scale = 64 ** -0.5
    out = torch.empty(B * N, 3 * C, dtype=torch.float16, device=cuda_device)
    _ops().call("dm_attention_split", _split(qkv), B, N, heads, scale, out)
    torch.cuda.synchronize()
    got = _unsplit(out).reshape(B, N, heads, 64)
    q, k, v = qkv.reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    e = e32 = 0.0
    with _no_tf32():
        for b in range(B):
            for h in range(heads):
                r64 = torch.softmax(q[b, h].double() @ k[b, h].double().t() * scale, dim=-1) @ v[b, h].double()
                r32 = torch.softmax(q[b, h] @ k[b, h].t() * scale, dim=-1) @ v[b, h]
                e, e32 = max(e, _err(got[b, :, h], r64)), max(e32, _err(r32, r64))
    print(f"split attention N={N} heads={heads}: {e:.3g}, fp32 {e32:.3g}")
    assert e <= 8 * e32 + 2.0 ** -22 * float(v.abs().max()), (e, e32)


# ---- Depth-Anything-V2 end to end -----------------------------------------------------------------------------------------------------
def _oracle_gpu(img, sd, encoder, net, dev):
    """the fp32 oracle (oracle/dav2.py) on the GPU with TF32 off"""
    import torch
    import torch.nn.functional as F
    from oracle import dav2 as o
    sd_dev = {k: v.to(dev, torch.float32) for k, v in sd.items()}
    with torch.no_grad(), _no_tf32():
        x, (h, w) = o.preprocess(img, net)
        d = o.forward(sd_dev, x.to(dev), encoder)
        d = F.interpolate(d[:, None], (h, w), mode="bilinear", align_corners=True)[0, 0]
    return d.cpu().numpy()


def _check_net(label, got, got16, want):
    e_max, e_mean = precision.norm_err(got, want)
    f_max, f_mean = precision.norm_err(got16, want)
    print(f"{label}: split max {e_max:.3g} mean {e_mean:.3g}; fp16 engine max {f_max:.3g} mean {f_mean:.3g}")
    assert e_max <= 1e-4 and e_mean <= 1e-5, (label, e_max, e_mean)
    assert f_max >= 20 * e_max and f_mean >= 20 * e_mean, (label, f_max, e_max, f_mean, e_mean)


@pytest.mark.parametrize("encoder,hw,net", [("vits", (70, 98), 70), ("vits", (64, 64), 56), ("vits", (120, 90), 140), ("vitb", (84, 84), 84),
                                            ("vitl", (518, 518), 518)])
def test_dav2_split_vs_oracle(cuda_device, encoder, hw, net):
    import torch
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict(encoder, seed=1)
    imgs = [synth_rgb(hw[0], hw[1], s) for s in ((3, 4) if encoder != "vitl" else (3,))]
    batch = torch.from_numpy(np.stack(imgs)).to(cuda_device)
    got = DepthAnythingV2Engine(sd, encoder, cuda_device, split=True).forward_batch(batch, net).cpu().numpy()
    got16 = DepthAnythingV2Engine(sd, encoder, cuda_device).forward_batch(batch, net).cpu().numpy()
    for i, img in enumerate(imgs):
        _check_net(f"dav2 split {encoder} {hw} net {net} img{i}", got[i], got16[i], _oracle_gpu(img, sd, encoder, net, cuda_device))


def test_dav2_split_tiling_vs_circular_oracle(cuda_device):
    import torch
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import dav2 as odav2
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=1)
    imgs = [synth_rgb(70, 98, s) for s in (3, 4)]
    batch = torch.from_numpy(np.stack(imgs)).to(cuda_device)
    got = DepthAnythingV2Engine(sd, 'vits', cuda_device, circular=True, split=True).forward_batch(batch, 70).cpu().numpy()
    got16 = DepthAnythingV2Engine(sd, 'vits', cuda_device, circular=True).forward_batch(batch, 70).cpu().numpy()
    for i, img in enumerate(imgs):
        with circular_convs(odav2):
            want = _oracle_gpu(img, sd, 'vits', 70, cuda_device)
        _check_net(f"tiling dav2 split img{i}", got[i], got16[i], want)


# ---- ModelHolder / funnel -------------------------------------------------------------------------------------------------------------
def test_modelholder_no_half_dav2(cuda_device):
    import torch
    from PIL import Image
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine, ModelHolder
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=2)
    mh = ModelHolder()
    mh.weights_provider = lambda t: sd
    mh.update_settings(no_half=True, precision="autocast")
    mh.ensure_models(12, cuda_device, False)
    model = mh.depth_model
    assert isinstance(model, DepthAnythingV2Engine) and model.split
    img = synth_rgb(56, 84, 9)
    pred, invert = mh.get_raw_prediction(Image.fromarray(img), 56, 56)
    want = DepthAnythingV2Engine(sd, 'vits', cuda_device, split=True).forward_batch(torch.from_numpy(img[None]).to(cuda_device), 56)[0]
    assert invert is False and np.array_equal(pred, want.cpu().numpy())
    mh.update_settings(no_half=False)                       # read at load time only: no reload, as in the reference
    mh.ensure_models(12, cuda_device, False)
    assert mh.depth_model is model
    mh.unload_models()


def test_modelholder_no_half_unchanged_and_refused(cuda_device):
    import torch
    from oracle import midas_v21
    from oracle import synth_weights
    from depthmap_b200.depthmap_generation import ModelHolder
    rgb = torch.from_numpy(synth_rgb(96, 128, 5)[None]).to(cuda_device)
    weights = {1: lambda: synth_weights.make_beit_dpt_state_dict('beitl16_512', seed=1), 5: lambda: midas_v21.make_state_dict(seed=1)}
    for t, make in weights.items():
        sd = make()
        preds = []
        for no_half in (False, True):
            mh = ModelHolder()
            mh.weights_provider = lambda key, sd=sd: sd
            mh.update_settings(no_half=no_half, precision="autocast")
            mh.ensure_models(t, cuda_device, False)
            preds.append(mh.get_raw_prediction_batch(rgb, 128, 128)[0].clone())
            mh.unload_models()
        assert torch.equal(preds[0], preds[1]), t                # autocast MiDaS: no_half changes nothing, as in the reference
    for t, prec in ((8, "autocast"), (1, "full")):
        mh = ModelHolder()
        mh.update_settings(no_half=True, precision=prec)
        with pytest.raises(NotImplementedError, match=f"model type {t}"):
            mh.ensure_models(t, cuda_device, False)


def test_funnel_no_half(cuda_device):
    from PIL import Image
    from depthmap_b200 import core
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=2)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: sd
    try:
        rgbs = [synth_rgb(70, 98, 30 + i) for i in range(3)]
        inp = dict(compute_device='GPU', model_type=12, net_width=70, net_height=70, net_size_match=False, boost=False,
                   do_output_depth=True, do_output_depth_prediction=True, gen_stereo=False, gen_normalmap=False)
        out = list(core.core_generation_funnel(None, [Image.fromarray(x) for x in rgbs], None, None, inp, ops={'no_half': True}))
        assert holder.depth_model.split
        preds = [v for _, k, v in out if k == 'depth_prediction']
        assert len(preds) == 3
        for x, p in zip(rgbs, preds):
            want = _oracle_gpu(x, sd, 'vits', 70, cuda_device)
            assert precision.norm_err(p, want)[0] <= 1e-4
    finally:
        holder.unload_models()
        holder.weights_provider = None
        holder.update_settings(no_half=False)
