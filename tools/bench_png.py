"""PNG files from the funnel: PIL on the host against encoding on the device.

    python tools/bench_png.py [--images 8] [--rounds 3] [--out results/bench_png.json]

Workload: `--images` synthetic 1920x1080 photos through Depth-Anything-V2-B (type 13, the funnel's default model) at net size
518 on seeded synthetic weights, with the default stereo modes (left-right, red-cyan-anaglyph) and a normal map: per image a
16-bit depth map, an SBS pair, an anaglyph and a normal map.  Two paths run alternately, `--rounds` times each after a warm-up
of both, and write every image file into a temporary directory:
  * pil: core_generation_funnel, then PIL's Image.save(format='png') of every yielded image (what backbone.save_image does);
  * gpu: core_generation_funnel_png, then the bytes written as they are.
Reported: the median images/s of each path, the device time of the encode kernels for one image's four outputs (CUDA events
around dm_png_encode on the funnel's output shapes), the total bytes of both paths' files, and the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return torch.cuda.get_device_name(), q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def _encode_ms(t, reps=10):
    """device milliseconds of one dm_png_encode of the batch t (kernels only, buffers allocated beforehand)"""
    import torch
    from depthmap_b200 import _lib
    L = _lib.load()
    C, bits = (1, 16) if t.dtype == torch.uint16 else (3, 8)
    B, H, W = (int(s) for s in t.shape[:3])
    bound = L.dm_png_encode_bound(H, W, C, bits)
    wsb = L.dm_png_encode_workspace_bytes(B, H, W, C, bits)
    out = torch.empty(B * bound, dtype=torch.uint8, device=t.device)
    off = torch.empty(B + 1, dtype=torch.int64, device=t.device)
    ws = torch.empty(wsb, dtype=torch.uint8, device=t.device)

    def call():
        _lib.check(L.dm_png_encode(t.data_ptr(), B, H, W, C, bits, 0, out.data_ptr(), out.numel(), off.data_ptr(), ws.data_ptr(), wsb,
                                   _lib.stream_ptr()), "dm_png_encode")
    call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    from PIL import Image
    from depthmap_b200 import core
    from oracle import synth_weights
    from synth import synth_rgb
    if not torch.cuda.is_available():
        raise SystemExit("bench_png needs a CUDA device")
    imgs = [Image.fromarray(synth_rgb(1080, 1920, i)) for i in range(a.images)]
    sd = synth_weights.make_dav2_state_dict('vitb', seed=0)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: sd
    opts = dict(model_type=13, net_width=518, net_height=518, boost=False, do_output_depth=True, gen_stereo=True,
                stereo_modes=["left-right", "red-cyan-anaglyph"], gen_normalmap=True)
    tmp = tempfile.mkdtemp(prefix="bench_png_")
    sizes = {}

    def run(path):
        d = os.path.join(tmp, path)
        shutil.rmtree(d, ignore_errors=True)
        os.makedirs(d)
        total = 0
        t0 = time.perf_counter()
        if path == "pil":
            for i, kind, im in core.core_generation_funnel(None, imgs, None, None, opts, ops={}):
                fn = os.path.join(d, f"{i:05}-{kind}.png")
                im.save(fn, format="png")
                total += os.path.getsize(fn)
        else:
            for i, kind, png in core.core_generation_funnel_png(None, imgs, None, None, opts, ops={}):
                with open(os.path.join(d, f"{i:05}-{kind}.png"), "wb") as f:
                    f.write(png)
                total += len(png)
        dt = time.perf_counter() - t0
        sizes[path] = total
        return dt

    try:
        run("pil"), run("gpu")                                       # warm-up: model buffers, CUDA graphs
        times = {"pil": [], "gpu": []}
        for _ in range(a.rounds):
            times["pil"].append(run("pil"))
            times["gpu"].append(run("gpu"))
        # the encode kernels on one image's outputs at the funnel's shapes, decoded back from the files just written
        d = os.path.join(tmp, "gpu")
        kinds = {"depth": None, "left-right": None, "red-cyan-anaglyph": None, "normalmap": None}
        for k in kinds:
            kinds[k] = torch.from_numpy(np.array(Image.open(os.path.join(d, f"00000-{k}.png")))).cuda().unsqueeze(0)
        enc_ms = {k: _encode_ms(t) for k, t in kinds.items()}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        holder.unload_models()
        holder.weights_provider = None
    name, power = _card()
    med = {k: statistics.median(v) for k, v in times.items()}
    result = dict(card=name, power_limit=power, images=a.images, size=[1920, 1080], model_type=13, rounds=a.rounds, seconds=times,
                  images_per_s={k: a.images / v for k, v in med.items()}, speedup=med["pil"] / med["gpu"],
                  encode_ms_per_image=enc_ms, encode_ms_per_image_total=sum(enc_ms.values()),
                  bytes={"pil": sizes["pil"], "gpu": sizes["gpu"]}, size_ratio=sizes["gpu"] / sizes["pil"])
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
