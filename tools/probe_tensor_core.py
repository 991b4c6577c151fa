"""Tool: two properties of the fp16 wgmma GEMM that decide how the split-operand (fp32-class) mode must be built
(csrc/boost_kernels.cu, depthmap_b200/boost.py): (1) are fp16 SUBNORMAL operands honoured or flushed; (2) how does the error of
the tensor core's own fp32 accumulation grow with the GEMM depth K (rounding grows like sqrt(K), alignment-truncation like K);
and (3) the same measurement on the split GEMM of no_half (dm_gemm_split_ex), whose promoted accumulation (csrc/gemm_wgmma.cu)
must keep the error at the level of fp32 arithmetic (torch.matmul in fp32, TF32 off) at any depth.
usage: python tools/probe_tensor_core.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from depthmap_b200 import _lib as L
    lib = L.load()
    dev = torch.device("cuda")

    def gemm(a, w):
        M, K = a.shape
        N = w.shape[0]
        out = torch.empty(M, N, dtype=torch.float32, device=dev)
        L.check(lib.dm_gemm_f16(a.data_ptr(), K, w.data_ptr(), K, None, out.data_ptr(), N, M, N, K, 0, 1, L.stream_ptr()), "dm_gemm_f16")
        torch.cuda.synchronize()
        return out

    K = 1024
    a = torch.full((128, K), 2.0 ** -20, dtype=torch.float16, device=dev)           # subnormal in fp16
    w = torch.ones(32, K, dtype=torch.float16, device=dev)
    print(f"subnormal A: got {gemm(a, w)[0, 0].item():.6e}, exact {K * 2.0 ** -20:.6e}")
    a = torch.ones(128, K, dtype=torch.float16, device=dev)
    w = torch.full((32, K), 2.0 ** -20, dtype=torch.float16, device=dev)
    print(f"subnormal W: got {gemm(a, w)[0, 0].item():.6e}, exact {K * 2.0 ** -20:.6e}")
    g = torch.Generator().manual_seed(0)
    for K in (64, 128, 256, 1024, 4096, 16384, 65536):
        a = (torch.rand(128, K, generator=g) + 0.5).half()
        w = (torch.rand(32, K, generator=g) + 0.5).half()
        exact = a.double() @ w.double().t()
        got = gemm(a.to(dev), w.to(dev)).cpu().double()
        rel = ((got - exact) / exact)
        print(f"K={K:6d} (all-positive products): mean rel err {rel.mean().item():+.3e}  max |rel| {rel.abs().max().item():.3e}   (2^-24 = 5.96e-8)")
    from depthmap_b200.depthmap_generation import split_weight
    ops = L.Ops()
    torch.backends.cuda.matmul.allow_tf32 = False
    for K in (1024, 4096, 16384, 65536):
        a = torch.rand(128, K, generator=g) + 0.5
        w = torch.rand(64, K, generator=g) + 0.5
        exact = a.double() @ w.double().t()
        hi = a.half()
        A = torch.cat([hi, (a - hi.float()).half(), hi], dim=1).to(dev)
        sw = split_weight(w.to(dev))
        out = torch.empty(128, 64, dtype=torch.float32, device=dev)
        ops.gemm_split(A, 3 * K, sw.t, 3 * K, sw.scale, 128, 64, 3 * K, epi=L.EPI_STORE_F32, X=out, ldx=64)
        torch.cuda.synchronize()
        rel = (out.cpu().double() - exact) / exact
        rel32 = ((a.to(dev) @ w.to(dev).t()).cpu().double() - exact) / exact
        print(f"split K={K:6d} (all-positive products): mean rel err {rel.mean().item():+.3e}  max |rel| {rel.abs().max().item():.3e}   "
              f"fp32 torch.matmul: mean {rel32.mean().item():+.3e}  max {rel32.abs().max().item():.3e}")


if __name__ == "__main__":
    main()
