"""Tool: BOOST on ZoeDepth-NK (model type 9) — wall time per image on a seeded synthetic 2048 x 2048 image at boost_rmax 1600,
with the real DPT-BEiT-L-384 core (seeded synthetic weights).  Prints one JSON line.
usage: python tools/bench_boost_zoe.py [--steps K]

Seconds per image: CUDA events around BoostPipeline.run with the control plane precomputed, after two untimed runs that warm
every shape.  Also the patch count, the whole-image size, the peak device memory of a run, the card's name and power limit (read
in the same run), and the algorithmic TFLOP of the base-network trunks the image needs: every ZoeDepth estimate is two forwards
(the crop and its flip) of 24 blocks of 24 N C^2 + 4 N^2 C (N tokens, C = 1024) at the net size of the crop with its reflect pad;
the DPT decoder, the ZoeDepth head and the merge network are not counted."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

RMAX = 1600


def trunk_flop(nh, nw, forwards, C=1024, depth=24):
    N = (nh // 16) * (nw // 16) + 1
    return forwards * depth * (24 * N * C * C + 4 * N * N * C)


def zoe_estimate_flop(w, h, msize):
    """one estimatezoedepth of a w x h crop at msize: the forward of the padded crop and of its flip"""
    from depthmap_b200.depthmap_generation import midas_net_size
    pad_h, pad_w = int(np.sqrt(h / 2) * 3.0), int(np.sqrt(w / 2) * 3.0)
    nw, nh = midas_net_size(w + 2 * pad_w, h + 2 * pad_h, msize, msize)
    return trunk_flop(nh, nw, 2)


def boost_trunk_flop(info, H, W):
    rf = info["rf"]
    total = sum(zoe_estimate_flop(W, H, m) for m in (rf, info["whole"]))
    for _, _, w, h in info["scaled_rects"]:
        total += sum(zoe_estimate_flop(w, h, m) for m in (rf, 2 * rf))
    return total


def main():
    import torch
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import ZoeDepthNKEngine
    from oracle import synth_weights
    from synth import synth_rgb
    from test_zoe_gpu import make_zoe_state_dict
    steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 2
    dev = torch.device("cuda")
    rec = {"card": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        rec["power_limit"] = q.stdout.strip()
    except Exception as e:  # noqa: BLE001 — the record says it could not be read
        rec["power_limit"] = f"unread ({e})"
    eng = ZoeDepthNKEngine(make_zoe_state_dict('beitl16_384', 3), dev)
    pipe = BoostPipeline(eng, UnetMergeEngine(synth_weights.make_pix2pix_state_dict(seed=1), dev), dev, 9)
    img = synth_rgb(2048, 2048, 7)
    info = {}
    pipe.run(img, RMAX, info=info, to_host=False)             # warm-up: every net shape, the merge-network graph
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    pipe.run(img, RMAX, precomputed=info, to_host=False)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        pipe.run(img, RMAX, precomputed=info, to_host=False)
    e1.record()
    torch.cuda.synchronize()
    sec = e0.elapsed_time(e1) / 1e3 / steps
    flop = boost_trunk_flop(info, 2048, 2048)
    rec["type9"] = dict(seconds_per_image=round(sec, 3), steps=steps, boost_rmax=RMAX, patches=len(info["scaled_rects"]),
                        whole_size=info["whole"], peak_memory_gb=round(peak / 2**30, 2), trunk_tflop=round(flop / 1e12, 2),
                        trunk_tflops_per_s=round(flop / sec / 1e12, 1))
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
