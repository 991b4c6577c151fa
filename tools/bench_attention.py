"""Tool: times the fused attention kernel alone on the two bench shapes (CUDA events, 20 launches after 3 warm-ups).
usage: python tools/bench_attention.py [beit|dav2|both]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    from depthmap_b200 import _lib as L
    lib = L.load()
    dev = torch.device("cuda")
    which = sys.argv[1] if len(sys.argv) > 1 else "both"
    H, C = 16, 1024
    g = torch.Generator(device="cpu").manual_seed(0)

    def run(name, fn, flops):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            fn()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / 20 * 1e3
        print(f"{name}: {us:.1f} us/launch  {flops / us * 1e-6:.1f} TFLOP/s")

    if which in ("beit", "both"):
        B, gh, gw = 32, 32, 32
        N = gh * gw + 1
        nrd = (2 * gh - 1) * (2 * gw - 1) + 3
        qkv = torch.randn(B * N, 3 * C, generator=g).half().to(dev)
        tab = (torch.randn(H, nrd, generator=g) * 2).float().to(dev).contiguous()
        out = torch.empty(B * N, C, dtype=torch.float16, device=dev)
        run("beit512 B=32 N=1025 relpos", lambda: L.check(lib.dm_attention_relpos_f16(
            qkv.data_ptr(), B, gh, gw, H, 0.125, tab.data_ptr(), nrd, out.data_ptr(), L.stream_ptr())),
            4.0 * B * H * N * N * 64)
    if which in ("dav2", "both"):
        B, N = 32, 1370
        qkv = torch.randn(B * N, 3 * C, generator=g).half().to(dev)
        out = torch.empty(B * N, C, dtype=torch.float16, device=dev)
        run("dav2 B=32 N=1370", lambda: L.check(lib.dm_attention_f16(qkv.data_ptr(), B, N, H, 0.125, None, 0, out.data_ptr(), L.stream_ptr())),
            4.0 * B * H * N * N * 64)


if __name__ == "__main__":
    main()
