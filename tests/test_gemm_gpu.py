"""GPU: wgmma GEMM / implicit-GEMM conv building blocks vs a plain PyTorch fp32 reference of the same op."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _lib():
    import depthmap_b200._lib as L
    return L, L.load()


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 128, 128), (128, 32, 64), (1000, 384, 256), (130, 64, 1024), (4100, 3072, 1024),
                                   (20000, 1024, 4096), (8300, 256, 256), (70, 256, 64)])
@pytest.mark.parametrize("mode", ["f32", "f16_bias_gelu"])
def test_gemm_f16(cuda_device, M, N, K, mode):
    import torch
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    A = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda_device)
    W = (torch.randn(N, K, generator=g) * 0.05).half().to(cuda_device)
    bias = torch.randn(N, generator=g).float().to(cuda_device)
    ref = A.float() @ W.float().t()
    if mode == "f32":
        C = torch.empty(M, N, dtype=torch.float32, device=cuda_device)
        rc = lib.dm_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, None, C.data_ptr(), N, M, N, K, 0, 1, L.stream_ptr())
        L.check(rc, "dm_gemm_f16")
        torch.cuda.synchronize()
        err = (C - ref).abs().max().item()
        assert err < 2e-3 * max(1.0, ref.abs().max().item()), (M, N, K, err)
    else:
        C = torch.empty(M, N, dtype=torch.float16, device=cuda_device)
        rc = lib.dm_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), C.data_ptr(), N, M, N, K, 1, 0, L.stream_ptr())
        L.check(rc, "dm_gemm_f16")
        torch.cuda.synchronize()
        want = torch.nn.functional.gelu(ref + bias)
        err = (C.float() - want).abs().max().item()
        assert err < 1e-2 * max(1.0, want.abs().max().item()), (M, N, K, err)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 8, 16, 64, 64), (2, 20, 37, 64, 32), (2, 19, 19, 128, 128), (1, 74, 74, 256, 256), (4, 148, 148, 256, 256)])
def test_conv3x3_f16(cuda_device, B, H, W, Cin, Cout):
    import torch
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(B + H + W + Cin)
    x = (torch.randn(B, H, W, Cin, generator=g) * 0.5).half().to(cuda_device)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05).half().to(cuda_device)
    bias = torch.randn(Cout, generator=g).float().to(cuda_device)
    wt = w.permute(0, 2, 3, 1).contiguous().reshape(Cout, 9 * Cin)  # (ky, kx, cin)
    out = torch.empty(B, H, W, Cout, dtype=torch.float16, device=cuda_device)
    rc = lib.dm_conv3x3_f16(x.data_ptr(), B, H, W, Cin, wt.data_ptr(), bias.data_ptr(), out.data_ptr(), Cout, 1, L.stream_ptr())
    L.check(rc, "dm_conv3x3_f16")
    torch.cuda.synchronize()
    ref = torch.relu(torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1)).permute(0, 2, 3, 1)
    err = (out.float() - ref).abs().max().item()
    assert err < 1e-2 * max(1.0, ref.abs().max().item()), err


def test_gemm_rejects_operands_the_epilogue_cannot_address(cuda_device):
    """The epilogue stores column pairs: an odd output pitch or an output that is not aligned to a pair is DM_E_INVALID,
    not a misaligned access inside the kernel."""
    import torch
    L, lib = _lib()
    M, N, K = 128, 64, 64
    A = torch.zeros(M, K, dtype=torch.float16, device=cuda_device)
    W = torch.zeros(N, K, dtype=torch.float16, device=cuda_device)
    C16 = torch.zeros(M * (N + 2) + 2, dtype=torch.float16, device=cuda_device)
    C32 = torch.zeros(M * (N + 2) + 2, dtype=torch.float32, device=cuda_device)
    for out, out_f32 in ((C16, 0), (C32, 1)):
        esz = out.element_size()
        assert lib.dm_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, None, out.data_ptr(), N + 2, M, N, K, 0, out_f32, L.stream_ptr()) == L.DM_OK
        assert lib.dm_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, None, out.data_ptr(), N + 1, M, N, K, 0, out_f32, L.stream_ptr()) == L.DM_E_INVALID
        assert lib.dm_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, None, out.data_ptr() + esz, N + 2, M, N, K, 0, out_f32, L.stream_ptr()) == L.DM_E_INVALID
    torch.cuda.synchronize()
