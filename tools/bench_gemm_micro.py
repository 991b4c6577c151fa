"""Micro-benchmark of the wgmma GEMM / implicit-GEMM convolution at the shapes and epilogues of the flagship workload
(dpt_beit_large_512, batch 32, 512 x 512), against each shape's own roofline bound and cuBLAS at the same plain shape.

    python tools/bench_gemm_micro.py [--iters 20] [--only trunk|decoder]

It loads the library that DEPTHMAP_B200_LIB points to (default: the in-tree build), so two builds can be compared in one
session by running it twice.  The roofline bound of a shape is max(FLOP / 989 TFLOP/s, algorithmic bytes / 3.35 TB/s), the
H100 SXM data-sheet rates (dense fp16, 700 W); `share` is that bound over the measured time.  Bytes count every operand once:
A, W, the output and, for the residual epilogue, the fp32 residual stream read and written.
"""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import depthmap_b200._lib as L  # noqa: E402

PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
B = 32
TOKENS = B * 1025

# (name, M, N, K, epilogue): the four Linears of every BEiT-L block, in plain-store mode and with the epilogue they run with
TRUNK = [
    ("qkv", TOKENS, 3072, 1024, "bias"),
    ("proj", TOKENS, 1024, 1024, "resid"),
    ("fc1", TOKENS, 4096, 1024, "gelu"),
    ("fc2", TOKENS, 1024, 4096, "resid"),
]
# decoder: (name, H = W, Cin, Cout, epilogue) 3x3 convolutions at batch 32, and the 1x1 fusion out_conv GEMMs (K = 256)
CONVS = [
    ("rn0 / fusion 128^2", 128, 256, 256, "bias"),
    ("rn1 64^2", 64, 512, 256, "bias"),
    ("fusion 64^2", 64, 256, 256, "relu"),
    ("oc1 256^2", 256, 256, 128, "bias"),
    ("head 512^2", 512, 128, 32, "head"),
]
FUSION_1X1 = [("out_conv 1x1 128^2", B * 128 * 128, 256, 256, "bias"), ("out_conv 1x1 64^2", B * 64 * 64, 256, 256, "bias")]


def card_info():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the card name still identifies the run
        q = f"nvidia-smi unavailable ({e})"
    return f"{name} | power limit, max SM clock: {q}"


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def row(name, mode, flop, nbytes, ms, cublas_ms=None):
    bound = max(flop / PEAK_FLOPS, nbytes / PEAK_BW) * 1e3
    which = "math" if flop / PEAK_FLOPS >= nbytes / PEAK_BW else "HBM"
    cb = f"{flop / cublas_ms / 1e9:7.1f}" if cublas_ms else "      -"
    ratio = f"{cublas_ms / ms:5.2f}" if cublas_ms else "    -"
    print(f"{name:22s} {mode:6s} {ms:8.3f} {flop / ms / 1e9:8.1f} {bound:8.3f} {which:4s} {bound / ms:6.2f} {cb} {ratio}", flush=True)


def cublas(M, N, K, dev, iters):
    if 2 * M * K > (4 << 30):
        return None
    a = torch.randn(M, K, device=dev).half()
    w = torch.randn(N, K, device=dev).half()
    ms = timed(lambda: torch.matmul(a, w.t()), iters)
    del a, w
    return ms


def gemm_case(lib, dev, name, M, N, K, mode, iters, cublas_ms):
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g) * 0.5).half().to(dev)
    W = (torch.randn(N, K, generator=g) * 0.05).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    gamma = torch.full((N,), 0.1, device=dev)
    d = L.GemmDesc()
    d.M, d.N, d.K = M, N, K
    out_bytes = 2 * M * N
    if mode == "resid":
        X = torch.zeros(M, N, dtype=torch.float32, device=dev)
        d.epi, d.X, d.ldx, d.bias, d.gamma = L.EPI_RESID_F32, X.data_ptr(), N, bias.data_ptr(), gamma.data_ptr()
        out_bytes = 8 * M * N
    else:
        C = torch.empty(M, N, dtype=torch.float16, device=dev)
        d.epi, d.C, d.ldc = L.EPI_STORE_F16, C.data_ptr(), N
        if mode != "plain":
            d.bias = bias.data_ptr()
        d.act = {"plain": L.ACT_NONE, "bias": L.ACT_NONE, "gelu": L.ACT_GELU, "relu": L.ACT_RELU}[mode]
    ms = timed(lambda: L.check(lib.dm_gemm_ex(A.data_ptr(), K, W.data_ptr(), K, ctypes.byref(d), L.stream_ptr()), "dm_gemm_ex"), iters)
    row(name, mode, 2.0 * M * N * K, 2 * M * K + 2 * N * K + out_bytes, ms, cublas_ms)


def conv_case(lib, dev, name, H, Cin, Cout, mode, iters, cublas_ms):
    g = torch.Generator(device="cpu").manual_seed(H + Cin + Cout)
    x = (torch.randn(B, H, H, Cin, generator=g) * 0.5).half().to(dev)
    wt = (torch.randn(Cout, 9 * Cin, generator=g) * 0.05).half().to(dev)
    bias = torch.randn(Cout, generator=g).to(dev)
    M = B * H * H
    d = L.GemmDesc()
    d.N, d.bias = Cout, bias.data_ptr()
    if mode == "head":
        w2 = torch.randn(Cout, generator=g).to(dev)
        out = torch.empty(M, dtype=torch.float32, device=dev)
        d.epi, d.act, d.X, d.gamma, d.head_b2 = L.EPI_HEAD, L.ACT_RELU, out.data_ptr(), w2.data_ptr(), 0.1
        out_bytes = 4 * M
    else:
        out = torch.empty(B, H, H, Cout, dtype=torch.float16, device=dev)
        d.epi, d.C, d.ldc = L.EPI_STORE_F16, out.data_ptr(), Cout
        d.act = L.ACT_RELU if mode == "relu" else L.ACT_NONE
        out_bytes = 2 * M * Cout
    ms = timed(lambda: L.check(lib.dm_conv3x3_ex(x.data_ptr(), B, H, H, Cin, wt.data_ptr(), ctypes.byref(d), L.stream_ptr()), "dm_conv3x3_ex"),
               iters)
    row(name, mode, 2.0 * M * Cout * 9 * Cin, 2 * M * Cin + 2 * Cout * 9 * Cin + out_bytes, ms, cublas_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", choices=["trunk", "decoder"], default=None)
    ap.add_argument("--no-cublas", action="store_true")
    a = ap.parse_args()
    lib = L.load()
    dev = L.require_cuda()
    print(f"# {card_info()}")
    print(f"# library {os.path.abspath(L.LIB_PATH)}")
    print(f"{'shape':22s} {'mode':6s} {'ms':>8s} {'TFLOP/s':>8s} {'bound':>8s} {'by':4s} {'share':>6s} {'cuBLAS':>7s} {'x cuBLAS':>5s}")
    cub = (lambda M, N, K: None) if a.no_cublas else (lambda M, N, K: cublas(M, N, K, dev, a.iters))
    if a.only in (None, "trunk"):
        for name, M, N, K, mode in TRUNK:
            c = cub(M, N, K)
            gemm_case(lib, dev, f"{name} {M}x{N}x{K}", M, N, K, "plain", a.iters, c)
            gemm_case(lib, dev, f"{name} {M}x{N}x{K}", M, N, K, mode, a.iters, c)
            torch.cuda.empty_cache()
    if a.only in (None, "decoder"):
        for name, H, Cin, Cout, mode in CONVS:
            conv_case(lib, dev, f"{name} {Cin}->{Cout}", H, Cin, Cout, mode, a.iters, cub(B * H * H, Cout, 9 * Cin))
            torch.cuda.empty_cache()
        for name, M, N, K, mode in FUSION_1X1:
            gemm_case(lib, dev, name, M, N, K, mode, a.iters, cub(M, N, K))
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
