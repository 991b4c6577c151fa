"""ORACLE (test infrastructure only — the product never imports this): numpy / cv2 restatement of estimatemidasBoost, the
singleestimate BOOST makes for the MiDaS base networks (model types 1-6; SURVEY.md §8a row D9).

Follows /root/reference/src/depthmap_generation.py:1180-1220 and dmidas/transforms.py:48-231:
  Resize(msize, msize, keep_aspect_ratio, ensure_multiple_of=32, resize_method="upper_bound", INTER_CUBIC) on the float64 crop,
  NormalizeImage(ImageNet mean / std), PrepareForNet (CHW float32); the network's prediction resized back to the crop with
  cv2 INTER_CUBIC and min-max normalised.  The crop keeps the channel order estimateboost hands it (the BGR-swapped image of :381).
The network is a parameter: `forward(x [1, 3, h, w] float32 tensor) -> [1, h, w]` stands for model.forward.  Use
`estimate_fn(forward)` as oracle.boost.estimateboost's `estimate`.  Pinned by tests/test_boost_midas_cpu.py against the reference
function itself."""
from __future__ import annotations

import numpy as np

MEAN = np.array([0.485, 0.456, 0.406])
STD = np.array([0.229, 0.224, 0.225])


def _constrain(x, multiple_of, max_val):
    """Resize.constrain_to_multiple_of with max_val (dmidas/transforms.py:94-104)"""
    y = int(np.round(x / multiple_of) * multiple_of)
    if y > max_val:
        y = int(np.floor(x / multiple_of) * multiple_of)
    return y


def net_size(width, height, msize, multiple_of=32):
    """Resize.get_size, 'upper_bound' with keep_aspect_ratio (transforms.py:106-160) -> (width, height)"""
    scale_h, scale_w = msize / height, msize / width
    if scale_w < scale_h:
        scale_h = scale_w
    else:
        scale_w = scale_h
    return _constrain(scale_w * width, multiple_of, msize), _constrain(scale_h * height, multiple_of, msize)


def preprocess(img, msize):
    """float [h, w, 3] crop -> float32 tensor [1, 3, nh, nw] (the transform of :1182-1198)"""
    import cv2
    import torch
    w, h = net_size(img.shape[1], img.shape[0], msize)
    x = cv2.resize(img, (w, h), interpolation=cv2.INTER_CUBIC)
    x = (x - MEAN) / STD
    return torch.from_numpy(np.ascontiguousarray(np.transpose(x, (2, 0, 1))).astype(np.float32)).unsqueeze(0)


def estimatemidasboost(img, msize, forward):
    """-> float32 [h, w] in [0, 1].  Where the reference would return the scalar 0 (max - min <= float64 eps) and fail at the next
    cv2.resize, this raises ValueError."""
    import cv2
    import torch
    with torch.no_grad():
        pred = forward(preprocess(img, msize)).squeeze().cpu().numpy()
    pred = cv2.resize(pred, (img.shape[1], img.shape[0]), interpolation=cv2.INTER_CUBIC)
    lo, hi = pred.min(), pred.max()
    if not hi - lo > np.finfo("float").eps:
        raise ValueError("constant prediction")
    return (pred - lo) / (hi - lo)


def estimate_fn(forward):
    """estimate(img, msize) for oracle.boost.estimateboost (model types 1-3)"""
    return lambda img, msize: estimatemidasboost(img, msize, forward)
