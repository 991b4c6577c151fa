"""Ragged batches against one forward per image, through the funnel.

    python tools/bench_ragged.py [--images 64] [--rounds 5] [--out results/bench_ragged.json]

Workload: core_generation_funnel on `--images` images cycling through four 4:3 sizes (640x480, 800x600, 1024x768, 1280x960, the
order rotated so that consecutive images always differ: the funnel's old pixel-size grouping runs them at B = 1).  Models:
Depth-Anything-V2-L at 518 (type 14), DPT-BEiT-L-512 (type 1) and LeReS (type 0), on seeded synthetic weights (speed does not
depend on the values).  For each model the ragged path (default batch bound) and DEPTHMAP_B200_MAX_BATCH=1 (one forward per
image, what the funnel did for this input before it grouped by network input size) run alternately, `--rounds` times each after
a warm-up of both; the median wall time of a whole funnel call (which ends in host copies, so the device is synchronised) is
reported with the card's name and power limit, read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SIZES = [(640, 480), (800, 600), (1024, 768), (1280, 960)]          # (width, height), all 4:3
MODELS = {14: ("dav2_vitl", 518, 518), 1: ("beitl16_512", 512, 512), 0: ("leres", 448, 448)}


def _weights(model_type):
    from oracle import synth_weights
    if model_type == 14:
        return synth_weights.make_dav2_state_dict('vitl', seed=0)
    if model_type == 1:
        return synth_weights.make_beit_dpt_state_dict('beitl16_512', seed=0)
    return synth_weights.make_leres_state_dict(seed=0)


def _card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return torch.cuda.get_device_name(), q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--models", default="14,1,0")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from PIL import Image
    from depthmap_b200 import core
    from synth import synth_rgb
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged needs a CUDA device")
    imgs = []
    for i in range(a.images):
        w, h = SIZES[(i + i // len(SIZES)) % len(SIZES)]
        imgs.append(Image.fromarray(synth_rgb(h, w, i)))
    assert all(imgs[i].size != imgs[i + 1].size for i in range(len(imgs) - 1))
    name, power = _card()
    result = dict(card=name, power_limit=power, images=a.images, sizes=SIZES, rounds=a.rounds, models={})
    holder = core.get_model_holder()
    for mt in map(int, a.models.split(",")):
        label, nw, nh = MODELS[mt]
        sd = _weights(mt)
        holder.unload_models()
        holder.weights_provider = lambda t, sd=sd: sd
        opts = dict(model_type=mt, net_width=nw, net_height=nh, boost=False, do_output_depth=True)

        def run(per_image):
            if per_image:
                os.environ["DEPTHMAP_B200_MAX_BATCH"] = "1"
            else:
                os.environ.pop("DEPTHMAP_B200_MAX_BATCH", None)
            t0 = time.perf_counter()
            n = sum(1 for _ in core.core_generation_funnel(None, imgs, None, None, opts, ops={}))
            torch.cuda.synchronize()
            assert n == len(imgs)
            return time.perf_counter() - t0

        run(False), run(True)                                   # warm-up: buffers, CUDA graphs, position tables
        times = {"ragged": [], "per_image": []}
        for _ in range(a.rounds):
            times["ragged"].append(run(False))
            times["per_image"].append(run(True))
        med = {k: statistics.median(v) for k, v in times.items()}
        result["models"][label] = dict(model_type=mt, net=[nw, nh], seconds=times, median_s=med,
                                       images_per_s={k: a.images / v for k, v in med.items()},
                                       speedup=med["per_image"] / med["ragged"])
        print(json.dumps({label: result["models"][label]["median_s"], "speedup": result["models"][label]["speedup"]}), flush=True)
        holder.unload_models()
        holder.weights_provider = None
        del sd
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
