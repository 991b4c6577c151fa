"""Tool: MiDaS v2.1 (model type 5) throughput on the op-level engine, against the same network in torch fp16.  Prints one JSON line.
usage: python tools/bench_midas_v21.py [--steps K] [--warmup W] [--rounds R] [--batch B]

Workloads (B images per step, seeded synthetic weights and images):
  net384      384 x 384 images, net 384 x 384
  net288x384  512 x 384 (w x h) images, whose 'upper_bound' net for 384 x 384 is 384 x 288
Per workload, after `--warmup` calls of each, `--rounds` rounds alternate the engine (uint8 images in, depth at the image size out:
pre-processing, network, bicubic resize; the network replays a CUDA graph) and the baseline (oracle/midas_v21.py's network with
fp16 weights and activations, the reference's GPU policy, channels_last, on the already pre-processed batch, plus the bicubic
resize), each round timing `--steps` calls between two CUDA events; the median over the rounds is reported.
FLOPs are counted by torch's FlopCounterMode on the oracle network on the meta device (2 per multiply-add):
  algorithmic  the network as written: 32-group 3x3 convolutions at their grouped cost
  executed     what the engine's tensor cores run: the grouped convolutions as block-diagonal dense filters
The card's name, power limit and maximum SM clock are read in the same run (read-only nvidia-smi query)."""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

WORKLOADS = {"net384": ((384, 384), (384, 384)), "net288x384": ((384, 512), (384, 384))}     # (image h, w), (net w, net h)


class _DenseGroups:
    """torch.nn.functional whose grouped conv2d runs as a dense one with block-diagonal filters (the engine's arithmetic)"""

    def __getattr__(self, name):
        import torch.nn.functional as F
        return getattr(F, name)

    def conv2d(self, x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
        import torch
        import torch.nn.functional as F
        if groups > 1:
            w = torch.empty(w.shape[0], w.shape[1] * groups, *w.shape[2:], dtype=w.dtype, device=w.device)
        return F.conv2d(x, w, b, stride, padding, dilation, 1)


def gflop_per_image(net_w, net_h, sd):
    """(algorithmic, executed) GFLOP of one network forward at net_w x net_h"""
    import torch
    from torch.utils.flop_counter import FlopCounterMode
    from oracle import leres, midas_v21
    meta = {k: v.to("meta") for k, v in sd.items()}
    x = torch.empty(1, 3, net_h, net_w, device="meta")
    out = []
    for dense in (False, True):
        saved = leres.F
        if dense:
            leres.F = _DenseGroups()
        try:
            with FlopCounterMode(display=False) as fc:
                midas_v21.forward(meta, x)
        finally:
            leres.F = saved
        out.append(fc.get_total_flops() / 1e9)
    return out


def bench_workload(name, eng, sd, sd16, B, steps, warmup, rounds, dev):
    import torch
    import torch.nn.functional as F
    from bench import make_images
    from bench_zoedepth import time_ms
    from depthmap_b200.depthmap_generation import midas_upper_bound_net_size
    from oracle import midas_v21
    (h, w), (net_w, net_h) = WORKLOADS[name]
    rgb = torch.from_numpy(make_images(B, h, w, 0)[0]).to(dev)
    nw, nh = midas_upper_bound_net_size(w, h, net_w, net_h)
    x = torch.randn(B, 3, nh, nw, generator=torch.Generator().manual_seed(0)).to(dev, torch.float16).contiguous(memory_format=torch.channels_last)

    def baseline():
        with torch.no_grad():
            d = midas_v21.forward(sd16, x)
            return F.interpolate(d.unsqueeze(1), size=(h, w), mode="bicubic", align_corners=False)
    runs = {"engine": lambda: eng.forward_batch(rgb, net_w, net_h), "torch_fp16": baseline}
    for fn in runs.values():
        for _ in range(max(1, warmup)):
            fn()
    torch.cuda.synchronize()
    rate = {k: [] for k in runs}
    for _ in range(rounds):
        for k, fn in runs.items():
            rate[k].append(B / (time_ms(fn, steps) / 1e3))
    alg, exe = gflop_per_image(nw, nh, sd)
    rec = dict(workload=name, images_per_step=B, image=f"{w}x{h}", net=f"{nw}x{nh}", algorithmic_gflop_per_image=round(alg, 1),
               executed_gflop_per_image=round(exe, 1))
    for k, v in rate.items():
        ips = statistics.median(v)
        rec[f"{k}_images_per_s"] = round(ips, 2)
        rec[f"{k}_rounds"] = [round(r, 2) for r in v]
        rec[f"{k}_algorithmic_tflop_per_s"] = round(ips * alg / 1e3, 1)
    rec["engine_executed_tflop_per_s"] = round(rec["engine_images_per_s"] * exe / 1e3, 1)
    rec["engine_over_torch_fp16"] = round(rec["engine_images_per_s"] / rec["torch_fp16_images_per_s"], 3)
    return rec


def main():
    import torch
    import precision
    from bench_zoedepth import card
    from depthmap_b200.depthmap_generation import MidasV21Engine
    from oracle import midas_v21
    arg = lambda k, d: sys.argv[sys.argv.index(k) + 1] if k in sys.argv else d
    steps, warmup, rounds, B = int(arg("--steps", 5)), int(arg("--warmup", 2)), int(arg("--rounds", 3)), int(arg("--batch", 32))
    if not torch.cuda.is_available():
        raise SystemExit("bench_midas_v21: no CUDA device; this tool measures on the GPU only")
    dev = torch.device("cuda")
    sd = midas_v21.make_state_dict(seed=0)
    eng = MidasV21Engine(sd, dev)
    sd16 = precision.HalfView(sd, dev)         # the oracle reads weights as .float(): fp16 tensors here
    rec = dict(tool="bench_midas_v21", card=card(torch.cuda.current_device()), steps=steps, warmup=warmup, rounds=rounds,
               workloads=[bench_workload(name, eng, sd, sd16, B, steps, warmup, rounds, dev) for name in WORKLOADS])
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
