"""Tool: BOOST on the MiDaS DPT base networks — wall time per image on a synthetic 2048 x 2048 image for model types 1 and 2 (seeded
synthetic weights), and the relative-position attention at the windows it serves.  Prints one JSON line.
usage: python tools/bench_boost_midas.py [--steps K] [--types 1,2]

Per type: seconds per image (CUDA events around BoostPipeline.run with the control plane precomputed, after one untimed run that
warms every shape), patch count, whole-image size, and the algorithmic TFLOP of the base-network transformer trunks the image
needs (24 blocks of 24 N C^2 + 4 N^2 C, N tokens, C = 1024; the DPT decoder and the merge network are not counted) over that time.
Attention: one BEiT-L layer (16 heads) at the windows of bench.py's depth_beit512 (32 images at 32 x 32) and zoedepth_nk768 (64
forwards at 24 x 24) workloads, and at 88 x 88 and BOOST's 100 x 100 whole-image window (1 image); 20 launches per timing, the
timing repeated three times (min and max reported)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

NAMES = {1: 'beitl16_512', 2: 'beitl16_384'}


def trunk_flop(nh, nw, B=1, C=1024, depth=24):
    N = (nh // 16) * (nw // 16) + 1
    return B * depth * (24 * N * C * C + 4 * N * N * C)


def boost_trunk_flop(info, H, W, model_type):
    from depthmap_b200.depthmap_generation import midas_boost_net_size
    rf = info["rf"]
    total = 0
    for msize in (rf, info["whole"]):
        nw, nh = midas_boost_net_size(W, H, msize)
        total += trunk_flop(nh, nw)
    for x, y, w, h in info["scaled_rects"]:
        for msize in (rf, 2 * rf):
            nw, nh = midas_boost_net_size(w, h, msize)
            total += trunk_flop(nh, nw)
    return total


def time_ms(fn, n):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def attention_time(dev, B, gh, gw, H=16, n=20, repeats=3):
    import torch
    from depthmap_b200 import _lib as L
    lib = L.load()
    N, C = gh * gw + 1, H * 64
    nrd = (2 * gh - 1) * (2 * gw - 1) + 3
    g = torch.Generator(device="cpu").manual_seed(7)
    qkv = torch.randn(B * N, 3 * C, generator=g).half().to(dev)
    tab = (torch.randn(H, nrd, generator=g) * 2.885).to(dev)
    out = torch.empty(B * N, C, dtype=torch.float16, device=dev)
    run = lambda: L.check(lib.dm_attention_relpos_f16(qkv.data_ptr(), B, gh, gw, H, 0.125, tab.data_ptr(), nrd, out.data_ptr(), L.stream_ptr()),
                          "dm_attention_relpos_f16")
    ts = [time_ms(run, n) for _ in range(repeats)]
    flop = 4 * B * H * N * N * 64
    return dict(ms_min=round(min(ts), 4), ms_max=round(max(ts), 4), tflops=round(flop / min(ts) / 1e9, 1))


def main():
    import torch
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import DptBeitEngine
    from oracle import synth_weights
    from synth import synth_rgb
    steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 2
    types = [int(t) for t in sys.argv[sys.argv.index("--types") + 1].split(",")] if "--types" in sys.argv else [1, 2]
    dev = torch.device("cuda")
    rec = {"card": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        rec["power_limit"] = q.stdout.strip()
    except Exception as e:  # noqa: BLE001 — the record says it could not be read
        rec["power_limit"] = f"unread ({e})"
    rec["attention_relpos_16_heads"] = {
        "depth_beit512_32x32_B32": attention_time(dev, 32, 32, 32),
        "zoedepth_nk768_24x24_B64": attention_time(dev, 64, 24, 24),
        "88x88_B1": attention_time(dev, 1, 88, 88),
        "100x100_B1": attention_time(dev, 1, 100, 100),
    }
    unet = UnetMergeEngine(synth_weights.make_pix2pix_state_dict(seed=1), dev)
    img = synth_rgb(2048, 2048, 7)
    for t in types:
        eng = DptBeitEngine(synth_weights.make_beit_dpt_state_dict(NAMES[t], seed=3), NAMES[t], dev)
        pipe = BoostPipeline(eng, unet, dev, t)
        info = {}
        pipe.run(img, 1600, info=info, to_host=False)         # warm-up: every net shape, the merge-network graph
        pipe.run(img, 1600, precomputed=info, to_host=False)
        ms = time_ms(lambda: pipe.run(img, 1600, precomputed=info, to_host=False), steps)
        flop = boost_trunk_flop(info, 2048, 2048, t)
        rec[f"type{t}"] = dict(seconds_per_image=round(ms / 1e3, 3), patches=len(info["scaled_rects"]), whole_size=info["whole"],
                               trunk_tflop=round(flop / 1e12, 2), trunk_tflops_per_s=round(flop / (ms / 1e3) / 1e12, 1))
        del pipe, eng
        torch.cuda.empty_cache()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
