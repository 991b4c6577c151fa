"""Depth-Anything-V2 S / B / L with no_half=False (fp16 operands) and no_half=True (the split fp32-class path), batch 32 at 518^2.

    python tools/bench_no_half.py [--batch 32] [--size 518] [--iters 3]

Prints one JSON line: per encoder, images/s of both paths (timed alternately in the same process, CUDA events around whole
forwards after a warm-up of each), their ratio, the split path's achieved tensor-pipe rate and the peak device memory of each path,
plus the card's name and power limit read in the same call.  The split rate counts the algorithmic MMA work the split kernels issue:
three times the fp16 GEMM / attention FLOPs of the network, computed from its shapes below (fp16_mma_flops)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def fp16_mma_flops(eng, nh, nw):
    """multiply-add FLOPs (2 per MAC) of every GEMM, convolution and attention product of one image's forward, at the padded
    shapes the kernels run (DepthAnythingV2Engine.run_network / run_head)"""
    cfg, P = eng.cfg, eng.PATCH
    C, depth = cfg['embed_dim'], cfg['depth']
    gh, gw = nh // P, nw // P
    Np, N = gh * gw, gh * gw + 1
    ocp, Fp, F2p = eng.ocp, eng.Fp, eng.F2p
    gemm = lambda m, n, k: 2.0 * m * n * k
    f = gemm(Np, C, eng.kpad)                                                     # patch embedding
    f += depth * (gemm(N, 3 * C, C) + gemm(N, C, C) + gemm(N, 4 * C, C) + gemm(N, C, 4 * C) + 2 * gemm(N, N, C))   # blocks
    sizes = [(gh * 4, gw * 4), (gh * 2, gw * 2), (gh, gw), ((gh - 1) // 2 + 1, (gw - 1) // 2 + 1)]
    px = [h * w for h, w in sizes]
    f += sum(gemm(Np, ocp[i], C) for i in range(4))                               # projects
    f += gemm(Np, 16 * ocp[0], ocp[0]) + gemm(Np, 4 * ocp[1], ocp[1]) + gemm(px[3], ocp[3], 9 * ocp[3])   # resize layers
    f += sum(gemm(px[i], Fp, 9 * ocp[i]) for i in range(4))                        # layer*_rn
    f += 2 * gemm(px[3], Fp, 9 * Fp) + gemm(px[3], Fp, Fp)                         # refinenet4: RCU2 + out_conv
    f += sum(4 * gemm(px[i], Fp, 9 * Fp) + gemm(px[i], Fp, Fp) for i in range(3))   # refinenet3..1
    f += gemm(4 * px[0], F2p, 9 * Fp) + gemm(nh * nw, 32, 9 * F2p)                 # output_conv1, output_conv2 (fused head)
    return f


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return name, power, clock


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=518)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--encoders", default="vits,vitb,vitl")
    a = ap.parse_args()
    import numpy as np
    import torch
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import synth_weights
    from synth import synth_rgb
    if not torch.cuda.is_available():
        raise SystemExit("bench_no_half: no CUDA device")
    dev = torch.device("cuda", 0)
    rgb = torch.from_numpy(np.stack([synth_rgb(a.size, a.size, i) for i in range(a.batch)])).to(dev)
    name, power, clock = card()
    out = {"tool": "bench_no_half", "gpu": name, "power_limit": power, "max_sm_clock": clock, "batch": a.batch, "size": a.size, "results": {}}
    for enc in a.encoders.split(","):
        sd = synth_weights.make_dav2_state_dict(enc, seed=0)
        engs, peak = {}, {}
        for k in ("fp16", "split"):                     # build + warm-up (allocations, module loads); each path's own peak memory
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            engs[k] = DepthAnythingV2Engine(sd, enc, dev, split=k == "split")
            engs[k].forward_batch(rgb, a.size)
            torch.cuda.synchronize()
            peak[k] = torch.cuda.max_memory_allocated(dev) - base
        del sd
        times = {k: [] for k in engs}
        for _ in range(a.iters):                        # alternate the two paths
            for k, e in engs.items():
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                e.forward_batch(rgb, a.size)
                t1.record()
                t1.synchronize()
                times[k].append(t0.elapsed_time(t1) / 1e3)
        nw, nh = engs["split"].net_size(a.size, a.size, a.size, a.size)
        flops = 3 * fp16_mma_flops(engs["split"], nh, nw) * a.batch
        best = {k: min(v) for k, v in times.items()}
        out["results"][enc] = {
            "fp16_images_per_s": round(a.batch / best["fp16"], 2), "split_images_per_s": round(a.batch / best["split"], 2),
            "split_cost_ratio": round(best["split"] / best["fp16"], 3),
            "split_tensor_tflops": round(flops / best["split"] / 1e12, 1),
            "fp16_peak_mem_gib": round(peak["fp16"] / 2 ** 30, 2), "split_peak_mem_gib": round(peak["split"] / 2 ** 30, 2),
            "times_s": {k: [round(t, 4) for t in v] for k, v in times.items()}}
        del engs
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
