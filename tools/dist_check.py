"""torchrun tool: the N-rank sharded + gathered result equals the 1-rank result BIT FOR BIT (SURVEY.md §4 / §8e).
Every rank builds the same model (seeded synthetic weights), takes its contiguous slice of the same batch, runs
depth -> u16 -> stereo -> normal map, all-gathers the finished tensors over NCCL and compares with the whole batch computed
locally.   python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tools/dist_check.py [--boost-model-type T]
--boost-model-type: the BOOST base network, 0 = LeReS res101 (default), 1 = DPT-BEiT-L 512, 2 = DPT-BEiT-L 384, 3 = DPT-Large 384,
5 = MiDaS v2.1, 9 = ZoeDepth-NK (on the small 'beit_tiny' core)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import datetime
    import numpy as np
    import torch
    import torch.distributed as dist
    from depthmap_b200.core import normalize_prediction_batch
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from depthmap_b200.dist import all_gather_batch, shard_range
    from depthmap_b200.normalmap_generation import create_normalmap_batch
    from depthmap_b200.stereoimage_generation import create_stereoimages_batch
    from oracle import synth_weights
    from synth import synth_rgb
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(minutes=5))
    n = 2 * world + 1                                   # uneven shards on purpose
    rgb = torch.from_numpy(np.stack([synth_rgb(84, 112, 300 + i) for i in range(n)])).to(dev)
    model = DepthAnythingV2Engine(synth_weights.make_dav2_state_dict('vits', seed=1), 'vits', dev)

    def pipeline(x):
        pred = model.forward_batch(x, 84, 84)
        depth = normalize_prediction_batch(pred, False)
        sbs = create_stereoimages_batch(x, depth, 2.5, 0.0, ['left-right'], 0.0, 1.0, 'polylines_sharp')[0]
        return depth, sbs, create_normalmap_batch(depth)

    lo, hi = shard_range(n, rank, world)
    mine = pipeline(rgb[lo:hi].contiguous())
    gathered = [all_gather_batch(t, n) for t in mine]
    whole = pipeline(rgb)
    ok = all(torch.equal(g.view(torch.uint8), w.view(torch.uint8)) for g, w in zip(gathered, whole))
    # BOOST (SURVEY 8e, BASELINE configs[4]): ONE image, its patches dealt to the ranks, the fitted patches exchanged with one
    # all-gather, every rank replays the blend: must equal the single-rank result bit for bit
    boost_note = ""
    if os.environ.get("DIST_CHECK_BOOST", "1") != "0":
        from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
        from depthmap_b200.depthmap_generation import DptBeitEngine, DptVitEngine, LeresEngine, MidasV21Engine, ZoeDepthNKEngine
        from oracle import midas_v21
        t = int(sys.argv[sys.argv.index("--boost-model-type") + 1]) if "--boost-model-type" in sys.argv else 0
        if t == 0:
            base = LeresEngine(synth_weights.make_leres_state_dict(seed=2), dev)
        elif t == 5:
            base = MidasV21Engine(midas_v21.make_state_dict(seed=1), dev)
        elif t == 9:
            from test_zoe_gpu import make_zoe_state_dict
            base = ZoeDepthNKEngine(make_zoe_state_dict('beit_tiny', 1), dev, core_name='beit_tiny')
        else:
            name = {1: 'beitl16_512', 2: 'beitl16_384', 3: 'vitl16_384'}[t]
            base = (DptVitEngine if t == 3 else DptBeitEngine)(synth_weights.make_beit_dpt_state_dict(name, seed=3), name, dev)
        pipe = BoostPipeline(base, UnetMergeEngine(synth_weights.make_pix2pix_state_dict(seed=1), dev), dev, t)
        img = synth_rgb(300, 420, 12)
        info = {}
        sharded = pipe.run(img, 1600, group=dist.group.WORLD, info=info)
        single = pipe.run(img, 1600)
        same = np.array_equal(sharded, single)
        ok = ok and same
        boost_note = f" boost_model_type={t} boost_patches={len(info['rects'])} boost_equal={same}"
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(f"dist_check {'ok' if flag.item() == 1 else 'MISMATCH'} world={world} images={n}{boost_note} nccl={'.'.join(map(str, torch.cuda.nccl.version()))}", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1 else 1)


if __name__ == "__main__":
    main()
