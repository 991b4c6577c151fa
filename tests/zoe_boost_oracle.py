"""Test infrastructure: singleestimate's ZoeDepth branch (src/depthmap_generation.py:1062-1064) as the `estimate` callable of
oracle.boost.estimateboost, whose driver is the same for every base network.

    estimatezoedepth(Image.fromarray(np.uint8(img * 255)).convert('RGB'), model, msize, msize)

img is the float64 crop of the R/B-swapped image get_raw_prediction made (:381); np.uint8 of a float64 truncates toward zero and
keeps the low 8 bits (x86-64), so a cubic overshoot wraps.  estimatezoedepth (:443-452) sets the resizer to msize x msize and runs
infer_pil: metric depth at the crop's size, not normalised.  The network is a parameter: `infer(u8 [h, w, 3], msize) -> float32
[h, w]` (nk_infer: the fp32 oracle ZoeDepth-NK)."""
from __future__ import annotations

import numpy as np


def quantise(img):
    """np.uint8(img * 255), as singleestimate hands the crop to PIL"""
    with np.errstate(invalid="ignore"):
        return np.uint8(np.asarray(img, dtype=np.float64) * 255)


def estimate_fn(infer, crops=None):
    """estimate(img, msize) for oracle.boost.estimateboost; `crops` collects (msize, uint8 crop) per call"""
    def estimate(img, msize):
        u8 = quantise(img)
        if crops is not None:
            crops.append((msize, u8))
        return infer(u8, msize)
    return estimate


def nk_infer(sd, core_name, device=None, routes=None):
    """infer(u8, msize): oracle/zoedepth.py's ZoeDepth-NK with the resizer at msize x msize (DepthModel.infer_pil: pad + flip
    augmentation), on `device` (default CPU).  `routes` collects (head name, |logit margin|) per forward: the crop, then its flip."""
    import torch
    from oracle import beit_dpt
    from oracle import zoedepth as ozd
    move = (lambda t: t.to(device)) if device is not None else (lambda t: t)
    core_sd = {k[len("core.core."):]: move(v) for k, v in sd.items() if k.startswith("core.core.")}
    head_sd = {k: move(v) for k, v in sd.items() if not k.startswith("core.")}

    def infer(u8, msize):
        def model_fn(x):
            _, feats = beit_dpt.forward(core_sd, ozd.prep_for_midas(x, msize, msize), core_name, return_features=True)
            depth, logits, name = ozd.metric_head(feats, head_sd)
            if routes is not None:
                routes.append((name, float((logits[0, 0] - logits[0, 1]).abs())))
            return depth
        x = move(torch.from_numpy(np.ascontiguousarray(u8)).permute(2, 0, 1).float().div(255.0).unsqueeze(0))    # ToTensor
        with torch.no_grad():
            return ozd.infer(model_fn, x, pad_input=True, with_flip_aug=True).squeeze().cpu().numpy()
    return infer
