"""GPU: ViT / DPT building-block kernels vs plain PyTorch fp32 references of the same ops."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _lib():
    import depthmap_b200._lib as L
    return L, L.load()


@pytest.mark.parametrize("B,N,H", [(1, 128, 1), (2, 257, 2), (1, 1370, 6), (2, 1025, 16), (3, 577, 4)])
@pytest.mark.parametrize("with_bias", [False, True])
def test_attention(cuda_device, B, N, H, with_bias):
    import torch
    L, lib = _lib()
    C = H * 64
    g = torch.Generator(device="cpu").manual_seed(B * 100 + N + H)
    qkv = (torch.randn(B * N, 3 * C, generator=g)).half().to(cuda_device)
    scale = 0.125
    bias = None
    ld = (N + 127) // 128 * 128
    if with_bias:
        bias = torch.zeros(H, N, ld, dtype=torch.float16, device=cuda_device)
        bias[:, :, :N] = (torch.randn(H, N, N, generator=g) * 2).half().to(cuda_device)
    out = torch.empty(B * N, C, dtype=torch.float16, device=cuda_device)
    rc = lib.dm_attention_f16(qkv.data_ptr(), B, N, H, scale, bias.data_ptr() if with_bias else None, ld, out.data_ptr(), L.stream_ptr())
    L.check(rc, "dm_attention_f16")
    torch.cuda.synchronize()
    q, k, v = qkv.float().view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = (q * scale) @ k.transpose(-1, -2)
    if with_bias:
        s = s + bias[:, :, :N].float().unsqueeze(0)
    ref = (s.softmax(-1) @ v).transpose(1, 2).reshape(B * N, C)
    err = (out.float() - ref).abs().max().item()
    assert err < 6e-3, (B, N, H, with_bias, err)


@pytest.mark.parametrize("C", [384, 768, 1024])
def test_layernorm(cuda_device, C):
    import torch
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(C)
    B, T = 3, 50
    x = (torch.randn(B * T, C, generator=g) * 3 + 1).to(cuda_device)
    w = (1 + 0.1 * torch.randn(C, generator=g)).to(cuda_device)
    b = (0.1 * torch.randn(C, generator=g)).to(cuda_device)
    for drop in (0, 1):
        rows_out = B * (T - 1) if drop else B * T
        out = torch.zeros(rows_out, C, dtype=torch.float16, device=cuda_device)
        rc = lib.dm_layernorm_f16(x.data_ptr(), B * T, C, w.data_ptr(), b.data_ptr(), 1e-6, out.data_ptr(), T, drop, L.stream_ptr())
        L.check(rc, "dm_layernorm_f16")
        ref = torch.nn.functional.layer_norm(x, (C,), w, b, 1e-6)
        if drop:
            ref = ref.view(B, T, C)[:, 1:].reshape(-1, C)
        assert (out.float() - ref).abs().max().item() < 4e-3


def test_resize_bilinear_nhwc_and_f32(cuda_device):
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(1)
    x = torch.randn(2, 19, 23, 64, generator=g).half().to(cuda_device)
    for (ho, wo) in [(37, 37), (38, 46), (19, 23), (5, 100)]:
        out = torch.empty(2, ho, wo, 64, dtype=torch.float16, device=cuda_device)
        L.check(lib.dm_resize_bilinear_nhwc_f16(x.data_ptr(), 2, 19, 23, 64, out.data_ptr(), ho, wo, L.stream_ptr()))
        ref = F.interpolate(x.float().permute(0, 3, 1, 2), (ho, wo), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
        assert (out.float() - ref).abs().max().item() < 3e-3
    d = torch.randn(2, 30, 41, generator=g).to(cuda_device)
    for mode, kw in [(0, dict(mode="bilinear", align_corners=True)), (1, dict(mode="bicubic", align_corners=False))]:
        for (ho, wo) in [(30, 41), (64, 80), (17, 23)]:
            out = torch.empty(2, ho, wo, device=cuda_device)
            L.check(lib.dm_resize_f32(d.data_ptr(), 2, 30, 41, out.data_ptr(), ho, wo, mode, L.stream_ptr()))
            ref = F.interpolate(d[:, None], (ho, wo), **kw)[:, 0]
            assert (out - ref).abs().max().item() < 1e-4, (mode, ho, wo)


def test_preprocess_patchify_and_tokens(cuda_device):
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    rng = np.random.default_rng(0)
    B, H, W, patch = 2, 28, 42, 14
    img = torch.from_numpy(rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)).to(cuda_device)
    mean = (ctypes.c_float * 3)(0.485, 0.456, 0.406)
    std = (ctypes.c_float * 3)(0.229, 0.224, 0.225)
    cmap = (ctypes.c_int * 3)(2, 1, 0)
    kpad = 640
    gh, gw = H // patch, W // patch
    out = torch.full((B * gh * gw, kpad), 7.0, dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_preprocess_patchify(img.data_ptr(), B, H, W, H, W, patch, mean, std, cmap, out.data_ptr(), kpad, L.stream_ptr()))
    x = img.float()[..., [2, 1, 0]] / 255.0
    x = (x - torch.tensor([0.485, 0.456, 0.406], device=cuda_device)) / torch.tensor([0.229, 0.224, 0.225], device=cuda_device)
    x = x.permute(0, 3, 1, 2)  # B,3,H,W
    ref = F.unfold(x, kernel_size=patch, stride=patch).transpose(1, 2).reshape(B * gh * gw, 3 * patch * patch)
    assert (out[:, :588].float() - ref).abs().max().item() < 2e-3
    assert float(out[:, 588:].abs().max()) == 0.0
    # tokens
    C, Np = 128, gh * gw
    pe = torch.randn(B * Np, C, device=cuda_device).half()
    cls = torch.randn(C, device=cuda_device)
    pos = torch.randn(Np + 1, C, device=cuda_device)
    X = torch.empty(B, Np + 1, C, device=cuda_device)
    L.check(lib.dm_assemble_tokens(pe.data_ptr(), cls.data_ptr(), pos.data_ptr(), X.data_ptr(), B, Np, C, L.stream_ptr()))
    ref = torch.cat([cls.expand(B, 1, C), pe.float().view(B, Np, C)], 1) + pos
    assert (X - ref).abs().max().item() < 1e-6


def test_im2col_s2_matches_conv(cuda_device):
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(3)
    B, H, W, C, Co = 2, 37, 37, 64, 64
    x = torch.randn(B, H, W, C, generator=g).half().to(cuda_device)
    w = (torch.randn(Co, C, 3, 3, generator=g) * 0.05).half().to(cuda_device)
    Ho = Wo = 19
    cols = torch.empty(B * Ho * Wo, 9 * C, dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_im2col_s2_f16(x.data_ptr(), B, H, W, C, cols.data_ptr(), L.stream_ptr()))
    wt = w.permute(0, 2, 3, 1).reshape(Co, 9 * C)
    got = (cols.float() @ wt.float().t()).view(B, Ho, Wo, Co)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), stride=2, padding=1).permute(0, 2, 3, 1)
    assert (got - ref).abs().max().item() < 1e-3


@pytest.mark.parametrize("B,gh,gw,H", [(1, 4, 4, 1), (2, 8, 6, 2), (2, 32, 32, 16), (1, 24, 24, 3), (1, 16, 16, 2), (2, 24, 16, 3),
                                        (1, 20, 32, 2), (1, 9, 48, 1)])
@pytest.mark.parametrize("mode", ["table", "dense"])
def test_attention_relpos_table(cuda_device, B, gh, gw, H, mode):
    """BEiT relative-position bias vs the dense [H,N,N] gather of the reference, on every grid through both ways the engine
    has of applying it: "table" = generated inside the kernel from the per-head table in shared memory
    (dm_attention_relpos_f16), "dense" = the fp16 [H, N, ld] bias the engine builds for windows whose table does not fit
    on chip (dm_attention_f16 with a bias, as DptBeitEngine.dense_bias lays it out)."""
    import torch
    from oracle.beit_dpt import gen_relative_position_index
    L, lib = _lib()
    N, C = gh * gw + 1, H * 64
    nrd = (2 * gh - 1) * (2 * gw - 1) + 3
    g = torch.Generator(device="cpu").manual_seed(gh * 100 + gw)
    qkv = torch.randn(B * N, 3 * C, generator=g).half().to(cuda_device)
    table = (torch.randn(nrd, H, generator=g) * 2).to(cuda_device)
    idx = gen_relative_position_index((gh, gw)).to(cuda_device)
    bias = table[idx.view(-1)].view(N, N, H).permute(2, 0, 1)
    tab_k = (table.t().contiguous() * 1.4426950408889634).float().contiguous()
    out = torch.full((B * N, C), float("nan"), dtype=torch.float16, device=cuda_device)
    if mode == "table":
        L.check(lib.dm_attention_relpos_f16(qkv.data_ptr(), B, gh, gw, H, 0.125, tab_k.data_ptr(), nrd, out.data_ptr(), L.stream_ptr()))
    else:
        ld = (N + 127) // 128 * 128
        dense = torch.zeros(H, N, ld, dtype=torch.float16, device=cuda_device)
        dense[:, :, :N] = (tab_k / 1.4426950408889634)[:, idx.view(-1)].view(H, N, N).to(torch.float16)
        L.check(lib.dm_attention_f16(qkv.data_ptr(), B, N, H, 0.125, dense.data_ptr(), ld, out.data_ptr(), L.stream_ptr()))
        bias = dense[:, :, :N].float()                 # the reference adds the bias the kernel was given (rounded to fp16)
    torch.cuda.synchronize()
    q, k, v = qkv.float().view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = (q * 0.125) @ k.transpose(-1, -2) + bias.unsqueeze(0)
    ref = (s.softmax(-1) @ v).transpose(1, 2).reshape(B * N, C)
    assert torch.isfinite(out.float()).all(), "some output rows were never written"
    err = (out.float() - ref).abs().max().item()
    assert err < 6e-3, (B, gh, gw, H, err)


@pytest.mark.parametrize("N", [1025, 700])
def test_attention_rising_scores_force_rescale(cuda_device, N):
    """Keys grow along the sequence so the running row max rises by a large factor from tile to tile: exercises the
    online-softmax rescale (accumulated output and row sum scaled down by 2^(old max - new max) before each tile is added)."""
    import torch
    L, lib = _lib()
    B, H = 1, 2
    C = H * 64
    g = torch.Generator(device="cpu").manual_seed(N)
    qkv = torch.randn(B * N, 3, H, 64, generator=g)
    ramp = torch.linspace(0.0, 6.0, N).view(N, 1, 1)
    qkv[:, 0] = qkv[:, 0].abs()                       # positive queries ...
    qkv[:, 1] = qkv[:, 1].abs() * 0.2 + ramp          # ... against keys that keep growing
    qkv = qkv.reshape(B * N, 3 * C).half().to(cuda_device)
    out = torch.empty(B * N, C, dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_attention_f16(qkv.data_ptr(), B, N, H, 0.125, None, 0, out.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    q, k, v = qkv.float().view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = (q * 0.125) @ k.transpose(-1, -2)
    assert (s.max(-1).values - s[..., :128].max(-1).values).max().item() > 16        # the scenario really does rescale
    ref = (s.softmax(-1) @ v).transpose(1, 2).reshape(B * N, C)
    err = (out.float() - ref).abs().max().item()
    assert err < 6e-3, (N, err)
