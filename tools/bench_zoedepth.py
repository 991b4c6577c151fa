"""Tool: ZoeDepth-N, ZoeDepth-K and ZoeDepth-NK (model types 7, 8, 9) in one run — images/s and the per-launch time of the head's
attractor and log-binomial kernels.  Prints one JSON line.
usage: python tools/bench_zoedepth.py [--steps K] [--warmup W] [--types 7,8,9]

Per type: 32 synthetic 768 x 768 images per step with the UI default net (w 384, h 512), i.e. 64 forwards of the DPT-BEiT-L-384
core at 512 x 512 (pad + flip TTA), seeded synthetic weights in the ZoeD_M12_{N,K,NK} layout.  One step (forward_batch) is
captured in a CUDA graph after `--warmup` eager steps and replayed `--steps` times between two CUDA events.  The kernels are
timed on their own on the buffers that step left, 20 launches per timing: the attractor of the largest level (refinenet1's
resolution) and the log-binomial at net resolution.  The card's name, power limit and maximum SM clock are read in the same run
(read-only nvidia-smi query)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

B, H, W, NET_W, NET_H = 32, 768, 768, 384, 512


def card(dev_index):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(dev_index)],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in q.stdout.strip().split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 — the record says it could not be read
        return dict(name=None, power_limit=f"unread ({e})", max_sm_clock=None)


def time_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def state_dict(model_type):
    from oracle import beit_dpt, synth_weights, zoedepth_single
    feat = beit_dpt.CONFIGS['beitl16_384']['features']
    sd = {"core.core." + k: v for k, v in synth_weights.make_beit_dpt_state_dict('beitl16_384', seed=0).items()}
    if model_type == 9:
        sd.update(synth_weights.make_zoedepth_head_state_dict(feat_ch=feat, seed=100, gain=1.5))
    else:
        sd.update(zoedepth_single.make_zoedepth_single_head_state_dict({7: 'n', 8: 'k'}[model_type], feat_ch=feat, seed=100, gain=1.5))
    return sd


def head_kernels(eng, model_type):
    """(attractor, log-binomial) launches of the last forward, re-issued on its buffers."""
    from depthmap_b200 import _lib as L
    from depthmap_b200.depthmap_generation import ZOE_CONFIG, ZOE_SINGLE_CONFIG
    lib, zb, st = eng.ops.L, eng._zbufs, L.stream_ptr
    Fn, nh, nw = eng._zbuf_key
    (h2, w2), (h3, w3) = zb['levels'][2], zb['levels'][3]
    bprev, bnew = zb['bnew'][2], zb['bnew'][3]
    if model_type == 9:
        lg = zb['logits']
        we, wo, b0, w2c, b2c = eng.z['clb']
        att = lambda: L.check(lib.dm_zoe_attractor(zb['A'][3].data_ptr(), 64, lg.data_ptr(), 32, bprev.data_ptr(), Fn, h2, w2, h3, w3,
                                                   bnew.data_ptr(), st()), "dm_zoe_attractor")
        clb = lambda: L.check(lib.dm_zoe_clb_final(zb['o32'].data_ptr(), 32, zb['ze'].data_ptr(), 128, bnew.data_ptr(), lg.data_ptr(), 32,
                                                   wo.data_ptr(), b0.data_ptr(), w2c.data_ptr(), b2c.data_ptr(), Fn, nh, nw, h3, w3,
                                                   ZOE_CONFIG['min_temp'], ZOE_CONFIG['max_temp'], zb['d'].data_ptr(), st()), "dm_zoe_clb_final")
        return att, clb
    c = ZOE_SINGLE_CONFIG
    we, wo, b0, w2c, b2c = eng.z['clb']
    normed = int(eng.normed)
    att = lambda: L.check(lib.dm_zoe_attractor_single(zb['A'][3].data_ptr(), 32, c['n_attractors'][3], normed, bprev.data_ptr(), Fn, h2, w2,
                                                      h3, w3, normed, c['min_depth'], c['max_depth'], bnew.data_ptr(), st()),
                          "dm_zoe_attractor_single")
    clb = lambda: L.check(lib.dm_zoe_clb_single(zb['o32'].data_ptr(), 32, zb['ze'].data_ptr(), 128, bnew.data_ptr(), wo.data_ptr(), b0.data_ptr(),
                                                w2c.data_ptr(), b2c.data_ptr(), eng.w['oc3_w'].data_ptr(), eng.oc3_b, Fn, nh, nw, h3, w3,
                                                c['min_temp'], c['max_temp'], zb['d'].data_ptr(), st()), "dm_zoe_clb_single")
    return att, clb


def main():
    import torch
    from bench import make_images
    from depthmap_b200.depthmap_generation import ZoeDepthEngine, ZoeDepthNKEngine
    arg = lambda k, d: sys.argv[sys.argv.index(k) + 1] if k in sys.argv else d
    steps, warmup = int(arg("--steps", 5)), int(arg("--warmup", 2))
    types = [int(t) for t in arg("--types", "7,8,9").split(",")]
    dev = torch.device("cuda")
    rec = dict(card=card(torch.cuda.current_device()), images_per_step=B, image=f"{H}x{W}", net=f"{NET_W}x{NET_H} (UI default) -> 512x512",
               steps=steps, warmup=warmup)
    rgb = torch.from_numpy(make_images(B, H, W, 0)[0]).to(dev)
    for t in types:
        sd = state_dict(t)
        eng = ZoeDepthNKEngine(sd, dev) if t == 9 else ZoeDepthEngine(sd, dev, {7: 'n', 8: 'k'}[t])
        del sd
        for _ in range(max(1, warmup)):
            eng.forward_batch(rgb, NET_W, NET_H)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            eng.forward_batch(rgb, NET_W, NET_H)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            eng.forward_batch(rgb, NET_W, NET_H)
        g.replay()
        torch.cuda.synchronize()
        ms = time_ms(g.replay, steps)
        att, clb = head_kernels(eng, t)
        att(), clb()
        torch.cuda.synchronize()
        rec[f"type{t}"] = dict(images_per_s=round(B / (ms / 1e3), 1), ms_per_step=round(ms, 2),
                               attractor_last_level_ms=round(time_ms(att, 20), 4), log_binomial_ms=round(time_ms(clb, 20), 4))
        del g, eng
        torch.cuda.empty_cache()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
