"""Tool: the cost of tiling mode (circular padding in every padded convolution) on the op-level engines.  Prints JSON lines.
usage: python tools/bench_tiling.py [--steps K] [--warmup W] [--rounds R] [--configs beit512,dav2l518,leres448,zoe_nk768]

Per configuration, one engine with zero padding and one with circular padding (circular=True) on the same seeded synthetic weights
and images.  After `--warmup` forwards of each, `--rounds` rounds alternate the two, each round timing `--steps` forward_batch
calls between two CUDA events; images/s is the median over the rounds.  Configurations (images per step, image, net):
  beit512    DPT-BEiT-L 512 (model type 1): 32 x 512^2, net 512
  dav2l518   Depth-Anything-V2 ViT-L (type 14): 64 x 518^2, net 518
  leres448   LeReS res101 (type 0): 16 x 448^2, net 448 (from the second call on, its network replays a CUDA graph)
  zoe_nk768  ZoeDepth-NK (type 9): 32 x 768^2, UI default net (w 384, h 512), i.e. 64 DPT-BEiT-L-384 forwards at 512^2
The halo kernel (dm_circular_halo_f16) is timed on its own at the largest convolution input of beit512 (the head's
[32, 512, 512, 128] map), 20 launches: bytes read + written over time, against the H100 SXM data-sheet 3.35 TB/s.  The card's
name, power limit and maximum SM clock are read in the same run (read-only nvidia-smi query)."""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BYTES_PER_S = 3.35e12


def _engines(name, dev):
    """-> (zero-padded engine, circular engine, images per step, image side, net_w, net_h)"""
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine, DptBeitEngine, LeresEngine, ZoeDepthNKEngine
    from oracle import synth_weights
    if name == "beit512":
        sd = synth_weights.make_beit_dpt_state_dict('beitl16_512', seed=0)
        return DptBeitEngine(sd, 'beitl16_512', dev), DptBeitEngine(sd, 'beitl16_512', dev, circular=True), 32, 512, 512, 512
    if name == "dav2l518":
        sd = synth_weights.make_dav2_state_dict('vitl', seed=0)
        return DepthAnythingV2Engine(sd, 'vitl', dev), DepthAnythingV2Engine(sd, 'vitl', dev, circular=True), 64, 518, 518, 518
    if name == "leres448":
        sd = synth_weights.make_leres_state_dict(seed=0)
        return LeresEngine(sd, dev), LeresEngine(sd, dev, circular=True), 16, 448, 448, 448
    if name == "zoe_nk768":
        from bench_zoedepth import state_dict
        sd = state_dict(9)
        return ZoeDepthNKEngine(sd, dev), ZoeDepthNKEngine(sd, dev, circular=True), 32, 768, 384, 512
    raise ValueError(f"unknown configuration {name}")


def bench_config(name, dev, steps, warmup, rounds):
    import torch
    from bench import make_images
    from bench_zoedepth import time_ms
    off, on, B, side, net_w, net_h = _engines(name, dev)
    rgb = torch.from_numpy(make_images(B, side, side, 0)[0]).to(dev)
    runs = {"zero": lambda: off.forward_batch(rgb, net_w, net_h), "circular": lambda: on.forward_batch(rgb, net_w, net_h)}
    for fn in runs.values():
        for _ in range(max(1, warmup)):
            fn()
    torch.cuda.synchronize()
    rate = {k: [] for k in runs}
    for _ in range(rounds):
        for k, fn in runs.items():
            rate[k].append(B / (time_ms(fn, steps) / 1e3))
    rec = dict(config=name, images_per_step=B, image=f"{side}x{side}", net=f"{net_w}x{net_h}", steps=steps, rounds=rounds)
    for k, v in rate.items():
        rec[f"{k}_images_per_s"] = round(statistics.median(v), 2)
        rec[f"{k}_rounds"] = [round(x, 2) for x in v]
    rec["circular_over_zero"] = round(rec["circular_images_per_s"] / rec["zero_images_per_s"], 4)
    rec["circular_launches_per_step_extra"] = (on.ops.launches - off.ops.launches) // (warmup + rounds * steps)
    del off, on, runs
    torch.cuda.empty_cache()
    return rec


def bench_halo(dev, B=32, H=512, W=512, C=128):
    import torch
    from bench_zoedepth import time_ms
    from depthmap_b200 import _lib as L
    lib = L.load()
    x = torch.randn(B, H, W, C, device=dev).half()
    halo = torch.empty(B, H + 2, W + 2, C, dtype=torch.float16, device=dev)
    fn = lambda: L.check(lib.dm_circular_halo_f16(x.data_ptr(), B, H, W, C, halo.data_ptr(), L.stream_ptr()), "dm_circular_halo_f16")
    fn()
    torch.cuda.synchronize()
    ms = time_ms(fn, 20)
    nbytes = 2 * C * B * (H * W + (H + 2) * (W + 2))
    return dict(kernel="dm_circular_halo_f16", shape=[B, H, W, C], ms=round(ms, 4), bytes=nbytes, tb_per_s=round(nbytes / (ms / 1e3) / 1e12, 3),
                share_of_3_35_tb_per_s=round(nbytes / (ms / 1e3) / HBM_BYTES_PER_S, 3))


def main():
    import torch
    from bench_zoedepth import card
    arg = lambda k, d: sys.argv[sys.argv.index(k) + 1] if k in sys.argv else d
    steps, warmup, rounds = int(arg("--steps", 3)), int(arg("--warmup", 2)), int(arg("--rounds", 3))
    configs = arg("--configs", "beit512,dav2l518,leres448,zoe_nk768").split(",")
    if not torch.cuda.is_available():
        raise SystemExit("bench_tiling: no CUDA device; this tool measures on the GPU only")
    dev = torch.device("cuda")
    print(json.dumps(dict(card=card(torch.cuda.current_device()))), flush=True)
    print(json.dumps(bench_halo(dev)), flush=True)
    for name in configs:
        print(json.dumps(bench_config(name, dev, steps, warmup, rounds)), flush=True)


if __name__ == "__main__":
    main()
