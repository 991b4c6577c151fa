"""Micro-benchmark of the wgmma GEMM: isolates main loop vs epilogue cost.  Prints TFLOP/s per configuration."""
import ctypes, os, sys
sys.path.insert(0, os.getcwd())
import torch
import depthmap_b200._lib as L
lib = L.load()
dev = torch.device('cuda')

def run(M, N, K, mode, iters=10):
    A = (torch.randn(M, K, device=dev) * 0.5).half()
    W = (torch.randn(N, K, device=dev) * 0.05).half()
    bias = torch.randn(N, device=dev)
    gamma = torch.ones(N, device=dev)
    d = L.GemmDesc()
    d.M, d.N, d.K = M, N, K
    C = torch.empty(M, N, dtype=torch.float16, device=dev)
    X = torch.zeros(M, N, dtype=torch.float32, device=dev) if mode in ('resid', 'f32') else None
    if mode == 'plain':
        d.epi, d.act, d.C, d.ldc = L.EPI_STORE_F16, 0, C.data_ptr(), N
    elif mode == 'bias':
        d.epi, d.act, d.C, d.ldc, d.bias = L.EPI_STORE_F16, 0, C.data_ptr(), N, bias.data_ptr()
    elif mode == 'gelu':
        d.epi, d.act, d.C, d.ldc, d.bias = L.EPI_STORE_F16, 1, C.data_ptr(), N, bias.data_ptr()
    elif mode == 'resid':
        d.epi, d.X, d.ldx, d.bias, d.gamma = L.EPI_RESID_F32, X.data_ptr(), N, bias.data_ptr(), gamma.data_ptr()
    elif mode == 'f32':
        d.epi, d.X, d.ldx = L.EPI_STORE_F32, X.data_ptr(), N
    def call():
        L.check(lib.dm_gemm_ex(A.data_ptr(), K, W.data_ptr(), K, ctypes.byref(d), L.stream_ptr()))
    for _ in range(3): call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): call()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print(f"M={M} N={N} K={K} {mode:6s} {ms:8.3f} ms {2.0*M*N*K/ms/1e9:8.1f} TFLOP/s", flush=True)

for (M, N, K) in [(32800, 4096, 1024), (32800, 1024, 4096), (32800, 3072, 1024), (32800, 1024, 1024)]:
    for mode in ['plain', 'bias', 'gelu', 'resid', 'f32']:
        run(M, N, K, mode)
a = torch.randn(8192, 8192, device=dev).half(); b = torch.randn(8192, 8192, device=dev).half()
for _ in range(3): torch.matmul(a, b)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(10): torch.matmul(a, b)
e1.record(); torch.cuda.synchronize()
print('cublas fp16 8192^3', 2 * 8192**3 / (e0.elapsed_time(e1) / 10) / 1e9, 'TFLOP/s')
a = torch.randn(32800, 1024, device=dev).half(); b = torch.randn(4096, 1024, device=dev).half()
for _ in range(3): torch.matmul(a, b.t())
torch.cuda.synchronize()
e0.record()
for _ in range(10): torch.matmul(a, b.t())
e1.record(); torch.cuda.synchronize()
print('cublas fp16 32800x4096x1024', 2 * 32800 * 4096 * 1024 / (e0.elapsed_time(e1) / 10) / 1e9, 'TFLOP/s')
