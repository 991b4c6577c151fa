"""Tool: where the time of one BOOST image goes — CUDA-event timings of the pieces (LeReS at the three net sizes on a float crop,
the merge U-Net, the glue kernels), each as used by boost.BoostPipeline (graph replays after the second call).
usage: python tools/bench_boost_parts.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import numpy as np
    import torch
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import LeresEngine
    from oracle import synth_weights
    dev = torch.device("cuda")
    leres = LeresEngine(synth_weights.make_leres_state_dict(seed=2), dev)
    unet = UnetMergeEngine(synth_weights.make_pix2pix_state_dict(seed=1), dev)
    pipe = BoostPipeline(leres, unet, dev, 0)
    img = torch.rand(3, 2048, 2048, device=dev)

    def timeit(name, fn, n=10):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        print(f"{name:58s} {e0.elapsed_time(e1) / n:8.3f} ms")

    for net in (448, 896, 1568):
        timeit(f"LeReS forward, float crop 600x600 -> net {net}", lambda: leres.forward_batch(None, net, net, planar=(img, (100, 100, 600, 600))))
    a = torch.rand(1024, 1024, device=dev)
    b = torch.rand(1024, 1024, device=dev)
    x2 = torch.rand(1024, 1024, 2, device=dev) * 2 - 1
    timeit("merge U-Net forward (split operands, K chunks of 1024)", lambda: unet.forward(x2))
    os.environ["X"] = "1"
    timeit("merge input (2 min-max + normalise) + U-Net", lambda: pipe._merge(a, b))
    timeit("double estimate of a 600x600 crop (448 + 896 + merge + post)", lambda: pipe.double_estimate(img, (100, 100, 600, 600), 448, 896))
    base = torch.rand(2048, 2048, device=dev)
    timeit("one patch: double estimate + merge with base + fit sums", lambda: pipe.fitted_patch(img, base, (100, 100, 600, 600), 448))
    upd = base.clone()
    mapped, sums = pipe.fitted_patch(img, base, (100, 100, 600, 600), 448)
    timeit("blend of a 600x600 patch", lambda: pipe.blend(upd, mapped, sums, (100, 100, 600, 600)))
    timeit("cubic resize 3 x 2048^2 -> 3 x 3136^2", lambda: pipe._cubic(img.data_ptr(), 2048, 2048, 2048, 3136, 3136, planes=3, src_plane=2048 * 2048))
    # eager (no graph) for comparison
    unet2 = UnetMergeEngine(synth_weights.make_pix2pix_state_dict(seed=1), dev)
    unet2._graphs.enabled = False
    timeit("merge U-Net forward, eager launches", lambda: unet2.forward(x2), n=5)


if __name__ == "__main__":
    main()
