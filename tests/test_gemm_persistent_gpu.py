"""GPU: the persistent ping-pong wgmma GEMM / implicit-GEMM conv computes every output element independently of where it
falls in the tile schedule.

Every output element sums the same k-blocks and k-slices in the same order whatever the tile shape (64 x 256, 128 x 128,
128 x 64, 128 x 32), the CTA that owns it, the consumer warpgroup, or the tile's place in the CTA's sequence.  So a large call
must equal, bit for bit, smaller calls on row slices (different tile indices, CTAs and tile counts per CTA) and column slices
(different N, hence different tile shapes) of the same operands, for every epilogue.  A wrong tile index, a barrier-phase
slip across tiles or a ping-pong order that leaks into the arithmetic shows up here exactly.
"""
import ctypes

import pytest

pytestmark = pytest.mark.gpu

M_BIG = 32800                        # the flagship's token count (32 x 1025): 257 m-tiles of 128, a 32-row tail


def _lib():
    import depthmap_b200._lib as L
    return L, L.load()


def _rand(shape, seed, scale, dev, dtype):
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=dev) * scale).to(dtype)


class _Case:
    """operands of one epilogue; call(r0, r1, n0, n1) runs rows [r0, r1) x columns [n0, n1) as one GEMM into views of the outputs"""

    def __init__(self, epi, M, N, K, dev):
        import torch
        L, self.lib = _lib()
        self.L, self.epi, self.M, self.N, self.K = L, epi, M, N, K
        self.A = _rand((M, K), 1, 0.5, dev, torch.float16)
        self.W = _rand((N, K), 2, 0.05, dev, torch.float16)
        self.bias = _rand((N,), 3, 1.0, dev, torch.float32)
        self.gamma = _rand((N,), 4, 0.5, dev, torch.float32)
        self.R = _rand((M, N), 5, 1.0, dev, torch.float16)
        self.R2 = _rand((M, N), 6, 1.0, dev, torch.float16)
        self.X0 = _rand((M, N), 7, 1.0, dev, torch.float32)
        self.reset()

    def reset(self):
        import torch
        dev = self.A.device
        self.C = torch.zeros(self.M, self.N, dtype=torch.float16, device=dev)
        self.C2 = torch.zeros_like(self.C)
        self.X = self.X0.clone() if self.epi == "resid" else torch.zeros(self.M, self.N, dtype=torch.float32, device=dev)
        self.H = torch.zeros(self.M, dtype=torch.float32, device=dev)

    def desc(self, r0, r1, n0, n1):
        L, d = self.L, self.L.GemmDesc()
        d.M, d.N, d.K = r1 - r0, n1 - n0, self.K
        off16, off32 = (r0 * self.N + n0) * 2, (r0 * self.N + n0) * 4
        d.bias = self.bias.data_ptr() + 4 * n0
        if self.epi in ("f16_gelu_r", "f16_relu_r2_c2"):
            d.epi, d.C, d.ldc = L.EPI_STORE_F16, self.C.data_ptr() + off16, self.N
            d.R, d.ldr = self.R.data_ptr() + off16, self.N
            if self.epi == "f16_gelu_r":
                d.act = L.ACT_GELU
            else:
                d.act, d.C2, d.R2, d.ldr2 = L.ACT_RELU, self.C2.data_ptr() + off16, self.R2.data_ptr() + off16, self.N
        elif self.epi == "resid":
            d.epi, d.X, d.ldx, d.gamma = L.EPI_RESID_F32, self.X.data_ptr() + off32, self.N, self.gamma.data_ptr() + 4 * n0
        elif self.epi == "f32":
            d.epi, d.X, d.ldx = L.EPI_STORE_F32, self.X.data_ptr() + off32, self.N
        elif self.epi == "head":
            d.epi, d.act, d.X, d.gamma, d.head_b2 = L.EPI_HEAD, L.ACT_RELU, self.H.data_ptr() + 4 * r0, self.gamma.data_ptr(), 0.25
        return d

    def call(self, r0, r1, n0, n1, stream=None):
        L = self.L
        d = self.desc(r0, r1, n0, n1)
        s = L.stream_ptr() if stream is None else ctypes.c_void_p(stream.cuda_stream)
        A = self.A.data_ptr() + r0 * self.K * 2
        W = self.W.data_ptr() + n0 * self.K * 2
        L.check(self.lib.dm_gemm_ex(A, self.K, W, self.K, ctypes.byref(d), s), "dm_gemm_ex")

    def outputs(self):
        return {"f16_gelu_r": [self.C], "f16_relu_r2_c2": [self.C, self.C2], "resid": [self.X], "f32": [self.X], "head": [self.H]}[self.epi]


def _same(a, b):
    import torch
    return a.shape == b.shape and torch.equal(a.view(torch.int16 if a.element_size() == 2 else torch.int32),
                                              b.view(torch.int16 if b.element_size() == 2 else torch.int32))


# N = 3072 runs 64 x 256 tiles; its column slices run 128 x 128 (384), 128 x 64 (64 at an odd 64-offset) and 128 x 32 (96)
@pytest.mark.parametrize("epi,N", [("f16_gelu_r", 3072), ("f16_relu_r2_c2", 1024), ("resid", 1024), ("f32", 3072), ("head", 32)])
def test_rows_and_columns_are_position_independent(cuda_device, epi, N):
    import torch
    K = 1024 if epi != "head" else 256
    case = _Case(epi, M_BIG, N, K, cuda_device)
    case.call(0, M_BIG, 0, N)
    torch.cuda.synchronize()
    full = [t.clone() for t in case.outputs()]
    row_slices = [(0, 128), (64, 64 + 1000), (12345, 12345 + 4100), (M_BIG - 700, M_BIG), (1, 1 + 2 * 128 * 120 + 77)]
    col_slices = [] if N == 32 else [(256, 256 + 384), (N - 64 * 3, N - 64 * 2), (N - 96, N), (0, 256)]
    for r0, r1 in row_slices:
        case.reset()
        case.call(r0, r1, 0, N)
        torch.cuda.synchronize()
        for f, g in zip(full, case.outputs()):
            assert _same(f[r0:r1], g[r0:r1]), (epi, N, "rows", r0, r1)
    for n0, n1 in col_slices:
        case.reset()
        case.call(0, M_BIG, n0, n1)
        torch.cuda.synchronize()
        for f, g in zip(full, case.outputs()):
            assert _same(f[:, n0:n1], g[:, n0:n1]), (epi, N, "cols", n0, n1)


def test_pixel_shuffle_is_position_independent(cuda_device):
    """ConvTranspose k = s = 2 with 128 channels (N = 512, 64 x 256 tiles): a batch equals calls on image subsets"""
    import torch
    L, lib = _lib()
    nimg, h, w, s, cout, K = 146, 15, 15, 2, 128, 256
    N, M = s * s * cout, nimg * h * w
    A = _rand((M, K), 11, 0.5, cuda_device, torch.float16)
    W = _rand((N, K), 12, 0.05, cuda_device, torch.float16)
    bias = _rand((N,), 13, 1.0, cuda_device, torch.float32)

    def run(b0, b1, out):
        d = L.GemmDesc()
        d.M, d.N, d.K, d.epi, d.bias = (b1 - b0) * h * w, N, K, L.EPI_PIXSHUF, bias.data_ptr()
        d.C, d.ps_s, d.ps_cout, d.ps_h, d.ps_w = out[b0:].data_ptr(), s, cout, h, w
        L.check(lib.dm_gemm_ex(A.data_ptr() + b0 * h * w * K * 2, K, W.data_ptr(), K, ctypes.byref(d), L.stream_ptr()), "dm_gemm_ex")

    full = torch.zeros(nimg, s * h, s * w, cout, dtype=torch.float16, device=cuda_device)
    run(0, nimg, full)
    for b0, b1 in [(0, 1), (3, 40), (145, 146)]:
        part = torch.zeros_like(full)
        run(b0, b1, part)
        torch.cuda.synchronize()
        assert _same(full[b0:b1], part[b0:b1]), (b0, b1)
    ref = (A.float() @ W.float().t() + bias).view(nimg, h, w, s, s, cout).permute(0, 1, 3, 2, 4, 5).reshape(nimg, s * h, s * w, cout)
    assert (full.float() - ref).abs().max().item() < 1e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("M", [70, 1000, 4100, M_BIG])
@pytest.mark.parametrize("N", [256, 384, 3072])
def test_tile_shapes_match_fp32_reference(cuda_device, M, N):
    """N = 256 and 3072 run 64 x 256 tiles, N = 384 runs 128 x 128; tolerances as in test_gemm_gpu.py"""
    import torch
    L, lib = _lib()
    K = 1024
    A = _rand((M, K), M + N, 0.5, cuda_device, torch.float16)
    W = _rand((N, K), M + N + 1, 0.05, cuda_device, torch.float16)
    bias = _rand((N,), M + N + 2, 1.0, cuda_device, torch.float32)
    ref = A.float() @ W.float().t()
    C = torch.empty(M, N, dtype=torch.float32, device=cuda_device)
    L.check(lib.dm_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, None, C.data_ptr(), N, M, N, K, 0, 1, L.stream_ptr()), "dm_gemm_f16")
    torch.cuda.synchronize()
    assert (C - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())
    H = torch.empty(M, N, dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), H.data_ptr(), N, M, N, K, 1, 0, L.stream_ptr()), "dm_gemm_f16")
    torch.cuda.synchronize()
    want = torch.nn.functional.gelu(ref + bias)
    assert (H.float() - want).abs().max().item() < 1e-2 * max(1.0, want.abs().max().item())


def _conv(lib, L, x, wt, bias, Cout, relu, stream=None):
    import torch
    B, H, W, Cin = x.shape
    out = torch.zeros(B, H, W, Cout, dtype=torch.float16, device=x.device)
    s = L.stream_ptr() if stream is None else ctypes.c_void_p(stream.cuda_stream)
    L.check(lib.dm_conv3x3_f16(x.data_ptr(), B, H, W, Cin, wt.data_ptr(), bias.data_ptr(), out.data_ptr(), Cout, int(relu), s), "dm_conv3x3_f16")
    return out


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(3, 37, 53, 64, 256), (5, 45, 29, 128, 128), (7, 33, 35, 64, 64), (2, 131, 67, 64, 32),
                                            (1, 255, 257, 256, 256)])
def test_conv_odd_sizes_and_tile_counts(cuda_device, B, H, W, Cin, Cout):
    """odd H and W, tile counts that are not a multiple of the grid; the batch equals per-image calls bit for bit"""
    import torch
    L, lib = _lib()
    x = _rand((B, H, W, Cin), B + H + W, 0.5, cuda_device, torch.float16)
    w = _rand((Cout, Cin, 3, 3), Cin + Cout, 0.05, cuda_device, torch.float16)
    bias = _rand((Cout,), 5, 1.0, cuda_device, torch.float32)
    wt = w.permute(0, 2, 3, 1).contiguous().reshape(Cout, 9 * Cin)
    out = _conv(lib, L, x, wt, bias, Cout, True)
    torch.cuda.synchronize()
    ref = torch.relu(torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1)).permute(0, 2, 3, 1)
    assert (out.float() - ref).abs().max().item() < 1e-2 * max(1.0, ref.abs().max().item())
    for b in range(B):
        one = _conv(lib, L, x[b:b + 1].contiguous(), wt, bias, Cout, True)
        torch.cuda.synchronize()
        assert _same(out[b:b + 1], one), b


def test_graph_replay_equals_eager(cuda_device):
    import torch
    case = _Case("f16_gelu_r", 8300, 3072, 1024, cuda_device)
    case.call(0, case.M, 0, case.N)
    torch.cuda.synchronize()
    eager = case.C.clone()
    case.reset()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            case.call(0, case.M, 0, case.N)
    torch.cuda.synchronize()
    case.C.zero_()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    assert _same(eager, case.C)


def test_two_streams_concurrently(cuda_device):
    """two persistent calls of one SM-filling grid each, issued on two streams at once, as the BOOST merge U-Net issues its chunks"""
    import torch
    a = _Case("f32", 20000, 1024, 2048, cuda_device)
    b = _Case("f16_relu_r2_c2", 9000, 256, 3072, cuda_device)
    a.call(0, a.M, 0, a.N)
    b.call(0, b.M, 0, b.N)
    torch.cuda.synchronize()
    want = [t.clone() for t in a.outputs() + b.outputs()]
    a.reset()
    b.reset()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    for _ in range(3):
        a.call(0, a.M, 0, a.N, stream=s1)
        b.call(0, b.M, 0, b.N, stream=s2)
    torch.cuda.synchronize()
    for w, g in zip(want, a.outputs() + b.outputs()):
        assert _same(w, g)
