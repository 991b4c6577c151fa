"""GPU: the LeReS / DPT helper kernels that only the network tests reached (csrc/leres_kernels.cu, csrc/vit_kernels.cu), each
against a float64 (or bit-exact) restatement of its operation at the shapes the engines send and at the kernels' own edges: grid
tails, 1-wide and 1-tall maps, odd sizes, B > 1.  Bars and the wrong-variant checks: tests/op_bars.py."""
import numpy as np
import pytest

from op_bars import check_exact, check_f16, check_f32, teeth

pytestmark = pytest.mark.gpu


def _lib():
    import depthmap_b200._lib as L
    return L, L.load()


@pytest.mark.parametrize("C", [8, 64])
@pytest.mark.parametrize("H,W", [(8, 8), (7, 9), (1, 5), (6, 1), (5, 130)])
def test_maxpool3x3s2(cuda_device, H, W, C):
    """F.max_pool2d(3, 2, padding 1) pads with -inf: on an all-negative map a zero-padded pool differs at every border output.
    W = 130, C = 64: Wo * C / 8 = 520 threads per row, a partial last block."""
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    B = 2
    g = torch.Generator().manual_seed(H * 1000 + W * 10 + C)
    x = (-0.1 - 4 * torch.rand(B, H, W, C, generator=g)).half()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xd = x.to(cuda_device)
    out = torch.full((B, Ho, Wo, C), float("nan"), dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_maxpool3x3s2_nhwc_f16(xd.data_ptr(), B, H, W, C, out.data_ptr(), L.stream_ptr()), "dm_maxpool3x3s2_nhwc_f16")
    torch.cuda.synchronize()
    xn = x.double().permute(0, 3, 1, 2)
    ref = F.max_pool2d(xn, 3, 2, 1).permute(0, 2, 3, 1)
    check_exact(f"maxpool B{B} {H}x{W}x{C}", out.cpu(), ref.half())
    zero_pad = F.max_pool2d(F.pad(xn, (1, 1, 1, 1), value=0.0), 3, 2, 0).permute(0, 2, 3, 1)
    teeth("maxpool with zero padding", zero_pad, ref, 0.0)


@pytest.mark.parametrize("H,W,C", [(8, 8, 64), (7, 9, 8), (1, 5, 64), (6, 1, 8), (9, 1030, 16)])
def test_subsample2(cuda_device, H, W, C):
    import torch
    L, lib = _lib()
    B = 2
    x = torch.randn(B, H, W, C, generator=torch.Generator().manual_seed(H + W + C)).half()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = torch.full((B, Ho, Wo, C), float("nan"), dtype=torch.float16, device=cuda_device)
    xd = x.to(cuda_device)
    L.check(lib.dm_subsample2_nhwc_f16(xd.data_ptr(), B, H, W, C, out.data_ptr(), L.stream_ptr()), "dm_subsample2_nhwc_f16")
    torch.cuda.synchronize()
    ref = x[:, ::2, ::2, :].contiguous()
    check_exact(f"subsample2 B{B} {H}x{W}x{C}", out.cpu(), ref)
    if H > 1 and W > 1:
        h, w = H // 2, W // 2
        teeth("subsample2 at the odd phase", x[:, 1::2, 1::2, :].float(), ref.float()[:, :h, :w], 0.0)


@pytest.mark.parametrize("n", [8, 8 * 256, 8 * (3 * 256 + 5)])
def test_add_f16(cuda_device, n):
    """bit-exact against torch's own fp16 a + b on CUDA (fp32 sum, one rounding), including sums that overflow to inf"""
    import torch
    L, lib = _lib()
    g = torch.Generator().manual_seed(n)
    a = (torch.randn(n, generator=g) * 4).half().to(cuda_device)
    b = (torch.randn(n, generator=g) * 4).half().to(cuda_device)
    a[:4] = torch.tensor([65504.0, -65504.0, 1e-7, 2.0 ** -24], dtype=torch.float16)
    b[:4] = torch.tensor([32.0, -32.0, 1e-7, 2.0 ** -24], dtype=torch.float16)
    out = torch.full_like(a, float("nan"))
    L.check(lib.dm_add_f16(a.data_ptr(), b.data_ptr(), out.data_ptr(), n, L.stream_ptr()), "dm_add_f16")
    want = a + b
    torch.cuda.synchronize()
    check_exact(f"add_f16 n={n}", out.cpu(), want.cpu())
    teeth("add_f16 with one operand dropped", a.cpu().float()[4:], want.cpu().float()[4:], 0.0)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("Hin,Win,Hout,Wout", [(30, 41, 64, 80), (30, 41, 17, 23), (1, 50, 1, 77), (12, 1, 40, 3), (24, 32, 24, 32)])
def test_resize_f32_ld(cuda_device, mode, Hin, Win, Hout, Wout):
    """channel 0 of an [pixels, 32] GEMM output (ld = 32), the other 31 channels holding different values: a wrong pixel stride
    reads them.  Mode 0 = bilinear align_corners=True, mode 1 = bicubic align_corners=False (A = -0.75)."""
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    B, ld = 2, 32
    g = torch.Generator().manual_seed(Hin * Win + Hout + mode)
    full = torch.randn(B, Hin, Win, ld, generator=g, dtype=torch.float64).float()
    full[..., 1:] += 5.0
    out = torch.full((B, Hout, Wout), float("nan"), device=cuda_device)
    fd = full.to(cuda_device)
    L.check(lib.dm_resize_f32_ld(fd.data_ptr(), ld, B, Hin, Win, out.data_ptr(), Hout, Wout, mode, L.stream_ptr()),
            "dm_resize_f32_ld")
    torch.cuda.synchronize()
    kw = dict(mode="bilinear", align_corners=True) if mode == 0 else dict(mode="bicubic", align_corners=False)

    def resize(t, **k):
        return F.interpolate(t[:, None], (Hout, Wout), **k)[:, 0]
    ch0 = full[..., 0]
    ref = resize(ch0.double(), **kw)
    bar = check_f32(f"resize_f32_ld mode {mode} {Hin}x{Win} -> {Hout}x{Wout}", out.cpu(), ref, resize(ch0, **kw), 1e-6)
    teeth("resize_f32_ld reading channel 1", resize(full[..., 1].double(), **kw), ref, bar)
    if (Hin, Win) != (Hout, Wout) and Hin > 1 and Win > 1:
        flipped = dict(kw, align_corners=not kw["align_corners"])
        teeth("resize_f32_ld with align_corners flipped", resize(ch0.double(), **flipped), ref, bar)


@pytest.mark.parametrize("C", [128, 384, 768, 1024])
@pytest.mark.parametrize("N", [2, 5])
def test_concat_readout(cuda_device, C, N):
    """row (b, p) = [x[b, 1 + p] | x[b, 0]] as fp16 (round to nearest); 2C > 1024 takes the block loop's second trip"""
    import torch
    L, lib = _lib()
    B = 3
    x = torch.randn(B, N, C, generator=torch.Generator().manual_seed(C + N)) * 3
    x[0, 0, :4] = torch.tensor([70000.0, -1e-8, 2.0 ** -25, 1.0 + 2.0 ** -11])       # overflow, underflow, ties
    out = torch.full((B * (N - 1), 2 * C), float("nan"), dtype=torch.float16, device=cuda_device)
    xd = x.to(cuda_device)
    L.check(lib.dm_concat_readout_f16(xd.data_ptr(), B, N, C, out.data_ptr(), L.stream_ptr()), "dm_concat_readout_f16")
    torch.cuda.synchronize()
    ref = torch.cat([x[:, 1:], x[:, :1].expand(B, N - 1, C)], dim=2).reshape(B * (N - 1), 2 * C).half()
    check_exact(f"concat_readout B{B} N{N} C{C}", out.cpu(), ref)
    swapped = torch.cat([x[:, :1].expand(B, N - 1, C), x[:, 1:]], dim=2).reshape(B * (N - 1), 2 * C).half()
    teeth("concat_readout with the halves swapped", swapped.float(), ref.float(), 0.0)


@pytest.mark.parametrize("drop", [0, 1])
def test_layernorm_f16_c128(cuda_device, drop):
    """C = 128, the width of the tiny test networks; 150 rows (not a multiple of the block's 8), drop_first removes token 0 of
    every image"""
    import torch
    L, lib = _lib()
    B, T, C = 3, 50, 128
    g = torch.Generator().manual_seed(128 + drop)
    x = torch.randn(B * T, C, generator=g) * 3 + 1
    w = 1 + 0.1 * torch.randn(C, generator=g)
    b = 0.1 * torch.randn(C, generator=g)
    rows_out = B * (T - 1) if drop else B * T
    out = torch.full((rows_out + 8, C), float("nan"), dtype=torch.float16, device=cuda_device)
    xd, wd, bd = x.to(cuda_device), w.to(cuda_device), b.to(cuda_device)
    L.check(lib.dm_layernorm_f16(xd.data_ptr(), B * T, C, wd.data_ptr(), bd.data_ptr(), 1e-6,
                                 out.data_ptr(), T, drop, L.stream_ptr()), "dm_layernorm_f16")
    torch.cuda.synchronize()
    out = out.cpu()
    assert torch.isnan(out[rows_out:].float()).all(), "rows past the output were written"

    def ln(xx, stats_width=C):
        xd = xx.double()
        mu = xd[:, :stats_width].mean(-1, keepdim=True)
        var = ((xd[:, :stats_width] - mu) ** 2).mean(-1, keepdim=True)
        return (xd - mu) / torch.sqrt(var + 1e-6) * w.double() + b.double()

    def select(y):
        return y.view(B, T, C)[:, 1:].reshape(-1, C) if drop else y
    ref = select(ln(x))
    u = check_f16(f"layernorm_f16 C=128 drop_first={drop}", out[:rows_out], ref)
    teeth("layernorm with statistics over the first 64 channels", select(ln(x, 64)), ref, u)
    if drop:
        teeth("layernorm dropping the last token instead of the first", ln(x).view(B, T, C)[:, :-1].reshape(-1, C), ref, u)
