"""Tool for ncu: one eager step of a bench workload between cudaProfilerStart / Stop (use `ncu --profile-from-start off`).
The ViT / DPT engines' CUDA graph is disabled so that every kernel is an individual launch.
usage: DEPTHMAP_B200_MODEL_GRAPH=0 python tools/profile_step.py [depth_beit512|dav2_stereo|stereo2048] [batch]"""
import os
import sys

os.environ.setdefault("DEPTHMAP_B200_MODEL_GRAPH", "0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    import bench
    name = sys.argv[1] if len(sys.argv) > 1 else "depth_beit512"
    cls = bench.WORKLOADS[name]
    if len(sys.argv) > 2:
        cls.B = int(sys.argv[2])
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    wl = cls(dev, 0)
    for _ in range(2):
        wl.step_resident(False)
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStart()
    wl.step_resident(False)
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStop()
    print("profiled one step of", name, "B =", wl.B)


if __name__ == "__main__":
    main()
