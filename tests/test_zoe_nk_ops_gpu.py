"""GPU: the ZoeDepth-NK head kernels (csrc/zoe_kernels.cu) one by one, each against a float64 restatement of its operation (the
pinned oracle's `_inv_attractor`, `_log_binom`, `infer` / `prep_for_midas` semantics), at the shapes ZoeDepthNKEngine sends
(nets that are multiples of 32, the batch doubled by the flip TTA, both routed heads in one batch) and at each kernel's edges.
Bars and the wrong-variant checks: tests/op_bars.py.  Also the router attention at every token count a net up to 2048^2 gives,
and the whole engine at a 1024 x 768 net, whose router sees more than 691 tokens."""
import math

import numpy as np
import pytest

from op_bars import check_exact, check_f16, check_f32, teeth

pytestmark = pytest.mark.gpu

NYU, KITTI = 0, 1


def _lib():
    import depthmap_b200._lib as L
    return L, L.load()


def _logits(heads, lld=32):
    """router logits [F, lld]: columns 0 / 1 pick `heads[f]`; None = an exact tie (torch.argmax takes index 0).  The other
    columns hold large values a wrong leading dimension would read."""
    import torch
    lg = torch.full((len(heads), lld), 9.0)
    for f, h in enumerate(heads):
        lg[f, :2] = torch.tensor([0.25, 0.25] if h is None else ([0.3, -0.2] if h == NYU else [0.1, 0.10001]))
    return lg


def _bilinear_ac(t, hw, dtype, align_corners=True):
    """NHWC -> NHWC bilinear resize at `dtype`"""
    import torch.nn.functional as F
    return F.interpolate(t.to(dtype).permute(0, 3, 1, 2), hw, mode="bilinear", align_corners=align_corners).permute(0, 2, 3, 1)


# ---- pre-processing ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,pad,net", [(1, 37, 53, None, (64, 96)), (2, 5, 7, (4, 6), (32, 64)), (2, 96, 128, None, (96, 128)),
                                           (1, 61, 40, (1, 0), (128, 64))])
def test_zoe_preprocess_patchify(cuda_device, B, H, W, pad, net):
    """/255 -> reflect pad -> flip of every odd forward -> bilinear align_corners=True -> (x - .5) / .5 -> 16 x 16 patches
    (F.unfold order).  Odd sizes, reflect padding at its limit (pad = H - 1, W - 1), non-square nets, B = 2."""
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    patch, kpad = 16, 768
    rng = np.random.default_rng(H * W + B)
    rgb = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    pad_h, pad_w = pad if pad is not None else (int(np.sqrt(H / 2) * 3.0), int(np.sqrt(W / 2) * 3.0))
    nh, nw = net
    rows = 2 * B * (nh // patch) * (nw // patch)
    out = torch.full((rows, kpad), float("nan"), dtype=torch.float16, device=cuda_device)
    rgb_d = torch.from_numpy(rgb).to(cuda_device)
    L.check(lib.dm_zoe_preprocess_patchify(rgb_d.data_ptr(), B, H, W, pad_h, pad_w, nh, nw, patch,
                                           out.data_ptr(), kpad, L.stream_ptr()), "dm_zoe_preprocess_patchify")
    torch.cuda.synchronize()

    def ref(flip=True, mode="reflect"):
        x = torch.from_numpy(rgb).double().permute(0, 3, 1, 2) / 255.0
        x = F.pad(x, (pad_w, pad_w, pad_h, pad_h), mode=mode)
        x = torch.stack([v for b in range(B) for v in (x[b], torch.flip(x[b], dims=[2]) if flip else x[b])])
        x = (F.interpolate(x, (nh, nw), mode="bilinear", align_corners=True) - 0.5) / 0.5
        return F.unfold(x, patch, stride=patch).transpose(1, 2).reshape(rows, 3 * patch * patch)
    want = ref()
    # the sampling coordinates are fp32 (sy * y): up to ~2e-5 pixel at these sizes, times a neighbour difference of up to 2
    u = check_f16(f"zoe_preprocess_patchify B{B} {H}x{W} pad {pad_h},{pad_w} net {nh}x{nw}", out.cpu(), want, floor=2.0 ** -3)
    teeth("patchify with the second forward not flipped", ref(flip=False), want, u)
    if pad_h or pad_w:
        teeth("patchify with replicate padding", ref(mode="replicate"), want, u)


# ---- router ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 13, 514])
def test_layernorm_post(cuda_device, rows):
    """x = LN(x) in place (fp32) and its fp16 copy; row counts that are not a multiple of the block's 8"""
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    g = torch.Generator().manual_seed(rows)
    x = torch.randn(rows, 128, generator=g) * 3 + 1
    w = 1 + 0.2 * torch.randn(128, generator=g)
    b = 0.2 * torch.randn(128, generator=g)
    xd = x.to(cuda_device)
    out = torch.full((rows + 8, 128), float("nan"), dtype=torch.float16, device=cuda_device)
    wd, bd = w.to(cuda_device), b.to(cuda_device)
    L.check(lib.dm_layernorm_post_f16(xd.data_ptr(), rows, 128, wd.data_ptr(), bd.data_ptr(), 1e-5,
                                      out.data_ptr(), L.stream_ptr()), "dm_layernorm_post_f16")
    torch.cuda.synchronize()

    def ln(stats_width=128):
        xx = x.double()
        mu = xx[:, :stats_width].mean(-1, keepdim=True)
        var = ((xx[:, :stats_width] - mu) ** 2).mean(-1, keepdim=True)
        return (xx - mu) / torch.sqrt(var + 1e-5) * w.double() + b.double()
    want = ln()
    got32, got16 = xd.cpu(), out.cpu()
    bar = check_f32(f"layernorm_post fp32 in place, {rows} rows", got32, want, F.layer_norm(x, (128,), w, b, 1e-5), 1e-6)
    check_exact("layernorm_post fp16 copy = fp16 of the fp32 result", got16[:rows], got32.half())
    check_f16("layernorm_post fp16 copy", got16[:rows], want)
    assert torch.isnan(got16[rows:].float()).all(), "rows past the end were written"
    teeth("layernorm_post with statistics over the first 64 channels", ln(64), want, bar)


@pytest.mark.parametrize("n", [4, 1024, 4 * (256 * 3 + 5)])
def test_cast_f32_f16(cuda_device, n):
    """round to nearest even, bit-exact against torch's .half(): overflow to inf, fp16 subnormals, ties"""
    import torch
    L, lib = _lib()
    x = torch.randn(n, generator=torch.Generator().manual_seed(n)) * 100
    x[:4] = torch.tensor([70000.0, 3e-6, 1.0 + 2.0 ** -11, -(1.0 + 3 * 2.0 ** -11)])
    out = torch.full((n,), float("nan"), dtype=torch.float16, device=cuda_device)
    xd = x.to(cuda_device)
    L.check(lib.dm_cast_f32_f16(xd.data_ptr(), n, out.data_ptr(), L.stream_ptr()), "dm_cast_f32_f16")
    torch.cuda.synchronize()
    check_exact(f"cast_f32_f16 n={n}", out.cpu(), x.half())
    assert float(x.half()[2]) == 1.0 and float(x.half()[3]) == -(1.0 + 4 * 2.0 ** -11)     # both ties really are ties (to even)


def _attention64(qkv, F_, S, heads, scale, keys=None):
    q, k, v = qkv.double().view(F_, S, 3, heads, 32).permute(2, 0, 3, 1, 4)
    if keys is not None:
        k, v = k[:, :, :keys], v[:, :, :keys]
    s = (q * scale) @ k.transpose(-1, -2)
    return (s.softmax(-1) @ v).transpose(1, 2).reshape(F_ * S, heads * 32), s


# 1 + cells of the 1/32 grid: 193 = 384 x 512, 257 = 512^2, 769 = 1024 x 768, 1025 = 1024^2; 691 / 692 bracket the token count the
# untiled kernel's shared memory (296 bytes per token) allowed
@pytest.mark.parametrize("S", [1, 2, 31, 32, 33, 166, 167, 193, 257, 691, 692, 769, 1025])
def test_attention_small(cuda_device, S):
    import torch
    L, lib = _lib()
    heads = 4
    scale = float(np.float32(1.0 / math.sqrt(32.0)))          # what the kernel receives (a C float)
    for F_ in (1, 2, 6):
        g = torch.Generator().manual_seed(S * 10 + F_)
        qkv = torch.randn(F_ * S, 3 * heads * 32, generator=g).half().to(cuda_device)
        out = torch.full((F_ * S, heads * 32), float("nan"), dtype=torch.float16, device=cuda_device)
        L.check(lib.dm_attention_small_f16(qkv.data_ptr(), F_, S, heads, scale, out.data_ptr(), L.stream_ptr()), "dm_attention_small_f16")
        torch.cuda.synchronize()
        want, _ = _attention64(qkv, F_, S, heads, scale)
        u = check_f16(f"attention_small F{F_} S{S}", out.cpu(), want.cpu())
        if S > 1:
            teeth("attention_small without the last key token", _attention64(qkv, F_, S, heads, scale, keys=S - 1)[0].cpu(), want.cpu(), u)


def test_attention_small_rising_scores(cuda_device):
    """keys grow along the sequence, so every row's running max rises from K / V tile to tile by a large factor: the online
    softmax must rescale its sum and accumulator each time"""
    import torch
    L, lib = _lib()
    F_, S, heads = 2, 769, 4
    scale = float(np.float32(1.0 / math.sqrt(32.0)))
    g = torch.Generator().manual_seed(7)
    qkv = torch.randn(F_ * S, 3, heads, 32, generator=g)
    qkv[:, 0] = qkv[:, 0].abs()
    qkv[:, 1] = qkv[:, 1].abs() * 0.2 + torch.linspace(0.0, 6.0, S).repeat(F_).view(F_ * S, 1, 1)
    qkv = qkv.reshape(F_ * S, 3 * heads * 32).half().to(cuda_device)
    out = torch.full((F_ * S, heads * 32), float("nan"), dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_attention_small_f16(qkv.data_ptr(), F_, S, heads, scale, out.data_ptr(), L.stream_ptr()), "dm_attention_small_f16")
    torch.cuda.synchronize()
    want, s = _attention64(qkv, F_, S, heads, scale)
    rise = (s.max(-1).values - s[..., :64].max(-1).values).cpu()
    assert float(rise.median()) > 16, float(rise.median())          # the scenario really does rescale
    check_f16("attention_small rising scores F2 S769", out.cpu(), want.cpu())


def test_attention_small_rejects_empty_shapes(cuda_device):
    """argument checks the host wrapper makes before any launch"""
    import torch
    L, lib = _lib()
    buf = torch.zeros(4, 384, dtype=torch.float16, device=cuda_device)
    for F_, S, heads in [(1, 0, 4), (0, 4, 4), (1, 4, 0)]:
        with pytest.raises(ValueError):
            L.check(lib.dm_attention_small_f16(buf.data_ptr(), F_, S, heads, 0.125, buf.data_ptr(), L.stream_ptr()), "dm_attention_small_f16")


# ---- seed bins ------------------------------------------------------------------------------------------------------------
def test_select_softplus(cuda_device):
    """F = 4 forwards routed [nyu, kitti, kitti, nyu], the last by an exact logit tie (index 0, as torch.argmax); seeds around
    F.softplus's threshold of 20"""
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    F_, n0, ld = 4, 37, 128
    heads = [NYU, KITTI, KITTI, NYU]
    g = torch.Generator().manual_seed(11)
    seed = torch.randn(F_ * n0, ld, generator=g) * 8
    edge = torch.tensor([19.5, 19.999998, 20.0, 20.000002, 20.5, -20.0, 0.0, 30.0, -90.0])
    seed[:, :9] = edge
    seed[:, 64:73] = edge
    lg = _logits([NYU, KITTI, KITTI, None])
    out = torch.full((F_ * n0, 64), float("nan"), device=cuda_device)
    sd_, lgd = seed.to(cuda_device), lg.to(cuda_device)
    L.check(lib.dm_zoe_select_softplus(sd_.data_ptr(), ld, lgd.data_ptr(), 32, F_, n0, out.data_ptr(),
                                       L.stream_ptr()), "dm_zoe_select_softplus")
    torch.cuda.synchronize()

    def pick(hs):
        return torch.cat([seed[f * n0:(f + 1) * n0, 64 * h:64 * h + 64] for f, h in enumerate(hs)])

    def softplus64(x):
        x = x.double()
        return torch.where(x > 20, x, torch.log1p(torch.exp(x)))
    want = softplus64(pick(heads))
    bar = check_f32("select_softplus", out.cpu(), want, F.softplus(pick(heads)), 1e-6 * float(want.abs().max()))
    teeth("select_softplus on the other head", softplus64(pick([1 - h for h in heads])), want, bar)
    teeth("select_softplus sending the tie to kitti", softplus64(pick([NYU, KITTI, KITTI, KITTI])), want, bar)


# ---- attractor levels -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Hs,Ws,H,W", [(6, 8, 12, 16), (1, 8, 5, 33), (6, 1, 12, 1), (1, 1, 3, 4), (6, 8, 1, 33), (12, 16, 6, 8)])
def test_resize_add_nhwc(cuda_device, Hs, Ws, H, W):
    """out = a + bilinear_align_corners(b_small); W = 33 at C = 128 is 528 threads per row (a partial block)"""
    import torch
    L, lib = _lib()
    B, C = 2, 128
    g = torch.Generator().manual_seed(Hs * 100 + Ws * 10 + H + W)
    a = torch.randn(B, H, W, C, generator=g).half()
    bs = torch.randn(B, Hs, Ws, C, generator=g).half()
    out = torch.full((B, H, W, C), float("nan"), dtype=torch.float16, device=cuda_device)
    ad, bsd = a.to(cuda_device), bs.to(cuda_device)
    L.check(lib.dm_resize_add_nhwc_f16(ad.data_ptr(), bsd.data_ptr(), B, Hs, Ws, C, out.data_ptr(), H, W,
                                       L.stream_ptr()), "dm_resize_add_nhwc_f16")
    torch.cuda.synchronize()
    want = a.double() + _bilinear_ac(bs, (H, W), torch.float64)
    # fp32 sampling coordinates and the fp32 sum: the floor leaves room for both next to the final rounding
    u = check_f16(f"resize_add_nhwc B{B} {Hs}x{Ws} -> {H}x{W}", out.cpu(), want, floor=2.0 ** -4)
    if (Hs > 1 and H > 1 and Hs != H) or (Ws > 1 and W > 1 and Ws != W):
        teeth("resize_add with align_corners=False", a.double() + _bilinear_ac(bs, (H, W), torch.float64, False), want, u)


def _attractor_ref(A, bprev, heads, H, W, dtype, align_corners=True):
    import torch
    import torch.nn.functional as F
    from oracle import zoedepth as ozd
    F_ = len(heads)
    b = _bilinear_ac(bprev, (H, W), dtype, align_corners)                                    # [F, H, W, 64]
    Af = A.view(F_, H, W, -1)
    a = F.softplus(torch.stack([Af[f, ..., 32 * h:32 * h + 16] for f, h in enumerate(heads)]).to(dtype))   # [F, H, W, 16]
    delta = torch.zeros_like(b)
    for i in range(16):
        delta += ozd._inv_attractor(a[..., i:i + 1] - b)
    return b + delta / 16


@pytest.mark.parametrize("Hp,Wp,H,W", [(6, 8, 12, 16), (3, 4, 7, 5), (1, 3, 1, 9), (12, 16, 12, 16)])
def test_zoe_attractor(cuda_device, Hp, Wp, H, W):
    """all 16 attractors of the routed head (columns head*32 .. +15 of A; the 16 unused columns of each head hold values a wrong
    offset would pick up), both heads in one batch of 4 forwards, b_prev bilinear from a different grid"""
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    heads = [NYU, KITTI, KITTI, NYU]
    F_ = len(heads)
    g = torch.Generator().manual_seed(Hp * Wp + H * W)
    A = torch.randn(F_ * H * W, 64, generator=g) * 1.5
    A[:, 16:32] += 6.0
    A[:, 48:64] += 6.0
    bprev = F.softplus(torch.randn(F_, Hp, Wp, 64, generator=g) * 1.5)
    out = torch.full((F_, H, W, 64), float("nan"), device=cuda_device)
    Ad, lgd, bpd = A.to(cuda_device), _logits(heads).to(cuda_device), bprev.to(cuda_device)
    L.check(lib.dm_zoe_attractor(Ad.data_ptr(), 64, lgd.data_ptr(), 32,
                                 bpd.data_ptr(), F_, Hp, Wp, H, W, out.data_ptr(), L.stream_ptr()), "dm_zoe_attractor")
    torch.cuda.synchronize()
    want = _attractor_ref(A, bprev, heads, H, W, torch.float64)
    bar = check_f32(f"zoe_attractor {Hp}x{Wp} -> {H}x{W}", out.cpu(), want, _attractor_ref(A, bprev, heads, H, W, torch.float32),
                    1e-6 * float(want.abs().max()))
    teeth("zoe_attractor on the other head", _attractor_ref(A, bprev, [1 - h for h in heads], H, W, torch.float64), want, bar)
    if (Hp, Wp) != (H, W) and H > 1 and W > 1:
        teeth("zoe_attractor with align_corners=False", _attractor_ref(A, bprev, heads, H, W, torch.float64, False), want, bar)


# ---- conditional log-binomial ---------------------------------------------------------------------------------------------
MIN_TEMP, MAX_TEMP = 0.0212, 50.0


def _clb_ref(t, heads, nh, nw, dtype, align_corners=True):
    """ConditionalLogBinomial (oracle `_conditional_log_binomial`) with mlp.0 split as the kernel takes it, then the expectation
    of the bilinearly up-sampled bin centres; returns (depth [F, nh, nw], temperature [F, nh, nw])"""
    import torch
    import torch.nn.functional as F
    from oracle import zoedepth as ozd
    hs = torch.tensor(heads)
    o = t['o32'].to(dtype)
    ze = torch.stack([t['ze'][f, ..., 64 * h:64 * h + 40] for f, h in enumerate(heads)])
    pre = torch.einsum('fyxc,fck->fyxk', o, t['wo'][hs].to(dtype)) + t['b0'][hs].to(dtype)[:, None, None, :] + \
        _bilinear_ac(ze, (nh, nw), dtype, align_corners)
    pt = torch.einsum('fyxk,fjk->fyxj', F.gelu(pre), t['w2'][hs].to(dtype)) + t['b2'][hs].to(dtype)[:, None, None, :]
    sp = F.softplus(pt) + 1e-4
    prob = sp[..., 0] / (sp[..., 0] + sp[..., 1])
    temp = (MAX_TEMP - MIN_TEMP) * (sp[..., 2] / (sp[..., 2] + sp[..., 3])) + MIN_TEMP
    k = torch.arange(64, dtype=dtype)
    y = ozd._log_binom(torch.tensor(63.0, dtype=dtype), k) + k * torch.log(torch.clamp(prob, 1e-4, 1))[..., None] + \
        (63 - k) * torch.log(torch.clamp(1 - prob, 1e-4, 1))[..., None]
    p = torch.softmax(y / temp[..., None], dim=-1)
    return (p * _bilinear_ac(t['bc'], (nh, nw), dtype, align_corners)).sum(-1), temp


@pytest.mark.parametrize("nh,nw,h3,w3", [(4, 96, 2, 48), (3, 129, 2, 33), (2, 384, 1, 96)])
def test_zoe_clb_final(cuda_device, nh, nw, h3, w3):
    """both heads in one batch, temperatures across [min_temp, max_temp], nw > 128 (a second, partial x-block), the bin
    centres and the bin embedding bilinear from a smaller grid"""
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    heads = [NYU, KITTI, KITTI, NYU]
    F_ = len(heads)
    g = torch.Generator().manual_seed(nh * nw + h3)
    w2 = torch.randn(2, 4, 40, generator=g) * 0.3
    w2[:, 2:] *= 4.0                                        # spreads ta / (ta + tb), i.e. the temperature, over its whole range
    t = dict(o32=torch.randn(F_, nh, nw, 32, generator=g).abs().half(), ze=torch.randn(F_, h3, w3, 128, generator=g) * 0.5,
             bc=torch.cumsum(F.softplus(torch.randn(F_, h3, w3, 64, generator=g)) * 0.15, dim=-1),
             wo=torch.randn(2, 32, 40, generator=g) * 0.3, b0=torch.randn(2, 40, generator=g) * 0.3, w2=w2,
             b2=torch.randn(2, 4, generator=g) * 0.5)
    d = {k: v.to(cuda_device) for k, v in t.items()}
    lgd = _logits(heads).to(cuda_device)
    out = torch.full((F_, nh, nw), float("nan"), device=cuda_device)
    L.check(lib.dm_zoe_clb_final(d['o32'].data_ptr(), 32, d['ze'].data_ptr(), 128, d['bc'].data_ptr(), lgd.data_ptr(),
                                 32, d['wo'].data_ptr(), d['b0'].data_ptr(), d['w2'].data_ptr(), d['b2'].data_ptr(), F_, nh, nw, h3, w3,
                                 MIN_TEMP, MAX_TEMP, out.data_ptr(), L.stream_ptr()), "dm_zoe_clb_final")
    torch.cuda.synchronize()
    want, temp = _clb_ref(t, heads, nh, nw, torch.float64)
    assert float(temp.min()) < 0.1 and float(temp.max()) > 45, (float(temp.min()), float(temp.max()))
    ev32, _ = _clb_ref(t, heads, nh, nw, torch.float32)
    bar = check_f32(f"zoe_clb_final {nh}x{nw} from {h3}x{w3}, temperature {float(temp.min()):.3f}..{float(temp.max()):.1f}", out.cpu(),
                    want, ev32, 1e-6 * float(want.abs().max()))
    teeth("zoe_clb_final on the other head", _clb_ref(t, [1 - h for h in heads], nh, nw, torch.float64)[0], want, bar)
    teeth("zoe_clb_final with align_corners=False", _clb_ref(t, heads, nh, nw, torch.float64, False)[0], want, bar)


# ---- TTA combine ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,pad,net", [(2, 40, 52, (6, 7), (52, 66)), (1, 50, 70, (0, 0), (32, 48)), (2, 20, 30, (3, 4), (64, 96)),
                                           (1, 37, 53, None, (64, 96))])
def test_zoe_tta_combine(cuda_device, B, H, W, pad, net):
    """bicubic (align_corners=False) from the net to the padded size, crop, average with the un-flipped prediction of the
    flipped forward: the same-size identity path (pad > 0), pad 0 with up-sampling, down-sampling, odd sizes"""
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    pad_h, pad_w = pad if pad is not None else (int(np.sqrt(H / 2) * 3.0), int(np.sqrt(W / 2) * 3.0))
    nh, nw = net
    Hp, Wp = H + 2 * pad_h, W + 2 * pad_w
    d = torch.randn(2 * B, nh, nw, generator=torch.Generator().manual_seed(H + W + nh)) + 3.0
    out = torch.full((B, H, W), float("nan"), device=cuda_device)
    dd = d.to(cuda_device)
    L.check(lib.dm_zoe_tta_combine(dd.data_ptr(), B, nh, nw, pad_h, pad_w, H, W, out.data_ptr(), L.stream_ptr()),
            "dm_zoe_tta_combine")
    torch.cuda.synchronize()

    def ref(dtype, flip=True, shift=0):
        up = d.to(dtype)[:, None]
        if (nh, nw) != (Hp, Wp):
            up = F.interpolate(up, (Hp, Wp), mode="bicubic", align_corners=False)
        up = up[:, 0]
        second = up[1::2].flip(-1) if flip else up[1::2]
        cols = torch.clamp(torch.arange(W) + pad_w + shift, max=Wp - 1)
        return (up[0::2, pad_h:pad_h + H, pad_w:pad_w + W] + second[:, pad_h:pad_h + H][..., cols]) / 2
    want = ref(torch.float64)
    bar = check_f32(f"zoe_tta_combine B{B} {H}x{W} pad {pad_h},{pad_w} net {nh}x{nw}", out.cpu(), want, ref(torch.float32),
                    1e-6 * float(want.abs().max()))
    teeth("tta_combine with the second forward not un-flipped", ref(torch.float64, flip=False), want, bar)
    teeth("tta_combine with the flip index off by one", ref(torch.float64, shift=1), want, bar)


# ---- the whole engine beyond 691 router tokens ----------------------------------------------------------------------------
def test_zoedepth_nk_1024x768_net(cuda_device):
    """ZoeDepth-NK (tiny BEiT core) at a 1024 x 768 net against the fp32 oracle under the network tests' precision rule.  The
    router sees 1 + 24 x 31 = 745 tokens here; the untiled router attention stopped at 691."""
    import torch
    import precision
    from depthmap_b200.depthmap_generation import ZoeDepthNKEngine, midas_net_size
    from oracle import zoedepth as ozd
    from synth import synth_rgb
    from test_zoe_gpu import make_zoe_state_dict
    H, W, net_w, net_h = 384, 512, 1024, 768
    pad_h, pad_w = int(np.sqrt(H / 2) * 3.0), int(np.sqrt(W / 2) * 3.0)
    nw, nh = midas_net_size(W + 2 * pad_w, H + 2 * pad_h, net_w, net_h)
    S = 1 + (nh // 32) * (nw // 32)
    assert S > 691, (nh, nw, S)
    sd = make_zoe_state_dict('beit_tiny', 3)
    eng = ZoeDepthNKEngine(sd, cuda_device, core_name='beit_tiny')
    img = synth_rgb(H, W, 5)
    got = eng.forward_batch(torch.from_numpy(img[None]).to(cuda_device), net_w, net_h).cpu().numpy()[0]
    want, invert = ozd.get_raw_prediction(img, sd, net_w, net_h, core_name='beit_tiny')
    assert invert is True and got.shape == want.shape == (H, W)
    ref16 = precision.reference_fp16_error_zoe(img, sd, net_w, net_h, 'beit_tiny', want, cuda_device)
    precision.check(f"zoedepth_nk tiny net {net_w}x{net_h} (S = {S})", got, want, ref16, slack=1.5)
