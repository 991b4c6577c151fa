"""Normal maps on H100 — drop-in for the reference's ``src/normalmap_generation.py``.

``create_normalmap`` keeps the reference signature and return type (PIL RGB, 8-bit); ``create_normalmap_batch`` is the
additive batched device face.  Compute = ``dm_normalmap`` (csrc/normalmap.cu).
"""
from __future__ import annotations

import numpy as np
from PIL import Image

from . import _lib


def _k(v):
    return int(v) if v is not None and v > 0 else 0


def create_normalmap_batch(depth, pre_blur=None, sobel_gradient=3, post_blur=None, invert=False):
    """depth: uint16 CUDA tensor [B,H,W] -> uint8 CUDA tensor [B,H,W,3]."""
    import torch
    _lib.require_cuda()
    if depth.dtype != torch.uint16:
        raise NotImplementedError("depthmap_b200 normal map expects a uint16 depth map (the funnel's img_output)")
    depth = depth.contiguous()
    B, H, W = depth.shape
    L = _lib.load()
    out = torch.empty((B, H, W, 3), dtype=torch.uint8, device=depth.device)
    pk, sk, qk = _k(pre_blur), _k(sobel_gradient), _k(post_blur)
    ws_bytes = L.dm_normalmap_workspace_bytes(B, H, W, pk, sk, qk)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=depth.device)
    rc = L.dm_normalmap(depth.data_ptr(), B, H, W, pk, sk, qk, 1 if invert else 0, out.data_ptr(), ws.data_ptr(),
                        ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "dm_normalmap")
    return out


def create_normalmap(depthmap, pre_blur=None, sobel_gradient=3, post_blur=None, invert=False):
    """Generates normalmaps — same contract as the reference (src/normalmap_generation.py:5-56).

    :param depthmap: depthmap that will be used to generate normalmap (uint16, as produced by the funnel)
    :param pre_blur: apply gaussian blur before taking gradient, None / -1 for disable, otherwise kernel size
    :param sobel_gradient: use Sobel gradient, None for regular gradient, otherwise kernel size
    :param post_blur: apply gaussian blur after taking gradient, None / -1 for disable, otherwise kernel size
    :param invert: depthmap will be inverted before calculating normalmap
    """
    import torch
    dev = _lib.require_cuda()
    d = np.asarray(depthmap)
    if d.dtype != np.uint16:
        raise NotImplementedError("depthmap_b200 normal map expects a uint16 depth map (the funnel's img_output)")
    t = torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).to(dev).view(torch.uint16).unsqueeze(0)
    out = create_normalmap_batch(t, pre_blur, sobel_gradient, post_blur, invert)
    return Image.fromarray(out[0].cpu().numpy())
