"""Stereo pair generation on H100 — drop-in for the reference's ``src/stereoimage_generation.py``.

``create_stereoimages`` keeps the reference signature, argument meaning, return type (list of PIL RGB images) and
error behaviour (src/stereoimage_generation.py:13-74); the per-row warp + gap-fill + packing runs in the
``dm_stereo`` CUDA kernel (csrc/stereo.cu).  ``create_stereoimages_batch`` is the additive batched face used by the
batched funnel and the bench: device tensors in, device tensors out, no host synchronisation.
"""
from __future__ import annotations

import ctypes

import numpy as np
from PIL import Image

from . import _lib

_MODES = ('left-right', 'right-left', 'top-bottom', 'bottom-top', 'red-cyan-anaglyph', 'left-only', 'only-right',
          'cyan-red-reverseanaglyph')


def _eye_setup(divergence, separation, stereo_balance, W):
    """src/stereoimage_generation.py:43-50 and :82-83 — per-eye (div_px, sep_px, mode), evaluated in Python floats."""
    balance = (stereo_balance + 1) / 2
    eyes = []
    # left eye: +divergence * balance, -separation ; right eye: -divergence * (1 - balance), +separation
    for identity, div, sep in ((balance < 0.001, +1 * divergence * balance, -1 * separation),
                               (balance > 0.999, -1 * divergence * (1 - balance), separation)):
        div_px = (div / 100.0) * W
        sep_px = (sep / 100.0) * W
        eyes.append((float(div_px), float(sep_px), _lib.DM_EYE_IDENTITY if identity else _lib.DM_EYE_WARP))
    return eyes


def _launch(rgb, depth, depth_kind, eyes, exponent, fill, pack, red_eye, out0, out1, strides):
    import torch
    L = _lib.load()
    B, H, W, _ = rgb.shape
    p = _lib.StereoParams()
    for e in range(2):
        p.div_px[e], p.sep_px[e], p.eye_mode[e] = eyes[e]
        p.dst_row_stride[e], p.dst_img_stride[e] = strides[e]
    p.exponent = float(exponent)
    p.fill = fill
    p.pack = pack
    p.anaglyph_red_eye = red_eye
    p.depth_kind = depth_kind
    ws_bytes = L.dm_stereo_workspace_bytes(B, H, W)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=rgb.device)
    rc = L.dm_stereo(rgb.data_ptr(), depth.data_ptr(), B, H, W, ctypes.byref(p),
                     out0.data_ptr() if out0 is not None else None, out1.data_ptr() if out1 is not None else None,
                     ws.data_ptr(), ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "dm_stereo")


def _prepare_depth(depth, poly):
    """uint16 goes to the fused device path; anything else is normalised like numpy would (:79-81) into float64 by
    dm_depth_to_nd64 (float32 / float64 / integer maps; float16 maps, which numpy would normalise in float16, are widened first)."""
    import torch
    if depth.dtype == torch.uint16:
        return depth.contiguous(), _lib.DM_DEPTH_U16, None
    B = depth.shape[0]
    if depth.dtype == torch.float32:
        d, code = depth.contiguous(), 0
    elif depth.dtype == torch.float64:
        d, code = depth.contiguous(), 1
    elif depth.dtype in (torch.float16, torch.bfloat16):
        mn = depth.reshape(B, -1).min(dim=1).values.view(B, 1, 1)
        mx = depth.reshape(B, -1).max(dim=1).values.view(B, 1, 1)
        return ((depth - mn) / (mx - mn)).to(torch.float64).contiguous(), _lib.DM_DEPTH_ND64, (mx == mn).view(B)
    else:
        d, code = depth.to(torch.int64).contiguous(), 2
    n = d[0].numel()
    nd = torch.empty(d.shape, dtype=torch.float64, device=d.device)
    flat = torch.empty(B, dtype=torch.int32, device=d.device)
    _lib.check(_lib.load().dm_depth_to_nd64(d.data_ptr(), code, B, n, nd.data_ptr(), flat.data_ptr(), _lib.stream_ptr()), "dm_depth_to_nd64")
    return nd, _lib.DM_DEPTH_ND64, flat.bool()


def create_stereoimages_batch(rgb, depth, divergence, separation=0.0, modes=None, stereo_balance=0.0,
                              stereo_offset_exponent=1.0, fill_technique='polylines_sharp'):
    """Batched device face.  rgb: uint8 CUDA tensor [B,H,W,3]; depth: CUDA tensor [B,H,W] (uint16 = fast path).
    Returns one uint8 CUDA tensor per requested mode ([B,H,2W,3], [B,2H,W,3] or [B,H,W,3])."""
    import torch
    if modes is None:
        modes = ['left-right']
    if not isinstance(modes, list):
        modes = [modes]
    if len(modes) == 0:
        return []
    _lib.require_cuda()
    if rgb.dim() != 4 or rgb.shape[-1] != 3 or rgb.dtype != torch.uint8:
        raise NotImplementedError("depthmap_b200 stereo expects uint8 RGB images [B,H,W,3]")
    assert tuple(rgb.shape[1:3]) == tuple(depth.shape[1:3]), 'Depthmap and the image must have the same size'
    if fill_technique not in _lib.DM_FILL:
        # the reference's apply_stereo_divergence falls through and np.hstack then fails on None (:85-92)
        raise ValueError(f"unknown fill_technique {fill_technique!r}")
    rgb = rgb.contiguous()
    B, H, W, _ = rgb.shape
    fill = _lib.DM_FILL[fill_technique]
    poly = fill >= 3
    dep, kind, flat = _prepare_depth(depth, poly)
    eyes = _eye_setup(divergence, separation, stereo_balance, W)
    dev = rgb.device

    def eyes_for(need_left, need_right):
        e = list(eyes)
        if not need_left:
            e[0] = (e[0][0], e[0][1], _lib.DM_EYE_SKIP)
        if not need_right:
            e[1] = (e[1][0], e[1][1], _lib.DM_EYE_SKIP)
        return e

    def fix_flat(t_left, t_right):
        # non-uint16 depth with max == min: nd is NaN everywhere; reference output pinned by the oracle
        if flat is None or not bool(flat.any()):
            return
        for t, (divp, sepp, mode) in ((t_left, eyes[0]), (t_right, eyes[1])):
            if t is None or mode != _lib.DM_EYE_WARP:
                continue
            fill_val = rgb[:, :, :1, :].expand(-1, -1, W, -1) if poly else torch.zeros_like(rgb)
            t[flat] = fill_val[flat]

    results = []
    single = len(modes) == 1
    sbs = None  # [B,H,2W,3] left | right, computed once when several modes are requested

    def get_sbs():
        nonlocal sbs
        if sbs is None:
            sbs = torch.empty((B, H, 2 * W, 3), dtype=torch.uint8, device=dev)
            _launch(rgb, dep, kind, eyes, stereo_offset_exponent, fill, _lib.DM_PACK_STRIDED, 0,
                    sbs, sbs[:, :, W:, :], [(2 * W * 3, H * 2 * W * 3)] * 2)
            fix_flat(sbs[:, :, :W, :], sbs[:, :, W:, :])
        return sbs

    for mode in modes:
        if mode not in _MODES:
            raise Exception('Unknown mode')
        if not single or flat is not None and bool(flat.any()):
            s = get_sbs()                       # eyes computed once; every mode is one dm_stereo_pack pass over the pair
            code = _MODES.index(mode)
            oh, ow = (2 * H if code in (2, 3) else H), (2 * W if code in (0, 1) else W)
            out = torch.empty((B, oh, ow, 3), dtype=torch.uint8, device=dev)
            _lib.check(_lib.load().dm_stereo_pack(s.data_ptr(), B, H, W, code, out.data_ptr(), _lib.stream_ptr()), "dm_stereo_pack")
            results.append(out)
            continue
        # single mode: the kernel writes the packed layout directly (compulsory traffic only)
        if mode in ('left-right', 'right-left'):
            out = torch.empty((B, H, 2 * W, 3), dtype=torch.uint8, device=dev)
            l_off, r_off = (0, W) if mode == 'left-right' else (W, 0)
            _launch(rgb, dep, kind, eyes, stereo_offset_exponent, fill, _lib.DM_PACK_STRIDED, 0,
                    out[:, :, l_off:, :], out[:, :, r_off:, :], [(2 * W * 3, H * 2 * W * 3)] * 2)
        elif mode in ('top-bottom', 'bottom-top'):
            out = torch.empty((B, 2 * H, W, 3), dtype=torch.uint8, device=dev)
            l_off, r_off = (0, H) if mode == 'top-bottom' else (H, 0)
            _launch(rgb, dep, kind, eyes, stereo_offset_exponent, fill, _lib.DM_PACK_STRIDED, 0,
                    out[:, l_off:, :, :], out[:, r_off:, :, :], [(W * 3, 2 * H * W * 3)] * 2)
        elif mode in ('red-cyan-anaglyph', 'cyan-red-reverseanaglyph'):
            out = torch.empty((B, H, W, 3), dtype=torch.uint8, device=dev)
            _launch(rgb, dep, kind, eyes, stereo_offset_exponent, fill, _lib.DM_PACK_ANAGLYPH,
                    0 if mode == 'red-cyan-anaglyph' else 1, out, None, [(W * 3, H * W * 3)] * 2)
        else:
            out = torch.empty((B, H, W, 3), dtype=torch.uint8, device=dev)
            left = mode == 'left-only'
            _launch(rgb, dep, kind, eyes_for(left, not left), stereo_offset_exponent, fill, _lib.DM_PACK_STRIDED, 0,
                    out if left else None, None if left else out, [(W * 3, H * W * 3)] * 2)
        results.append(out)
    return results


def create_stereoimages(original_image, depthmap, divergence, separation=0.0, modes=None,
                        stereo_balance=0.0, stereo_offset_exponent=1.0, fill_technique='polylines_sharp'):
    """Creates stereoscopic images — same contract as the reference (src/stereoimage_generation.py:13-74).

    :param original_image: PIL image or ndarray [H,W,3] uint8
    :param depthmap: depth map of the same size, white = near; uint16 (funnel output) or any numeric dtype
    :param float divergence: 3D effect in percent of the image width
    :param float separation: extra horizontal shift of the two halves in percent
    :param list modes: any of 'left-right', 'right-left', 'top-bottom', 'bottom-top', 'red-cyan-anaglyph',
      'left-only', 'only-right', 'cyan-red-reverseanaglyph' (default ['left-right'])
    :param float stereo_balance: split of the divergence between the eyes, in [-1, 1]
    :param float stereo_offset_exponent: 1 or 2 in the UI
    :param str fill_technique: 'none', 'naive', 'naive_interpolating', 'polylines_soft', 'polylines_sharp'
    :return: list of PIL RGB images, one per mode
    """
    import torch
    if modes is None:
        modes = ['left-right']
    if not isinstance(modes, list):
        modes = [modes]
    if len(modes) == 0:
        return []
    dev = _lib.require_cuda()
    img = np.asarray(original_image)
    dep = np.asarray(depthmap)
    assert img.shape[:2] == dep.shape, 'Depthmap and the image must have the same size'
    if img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.uint8:
        raise NotImplementedError("depthmap_b200 stereo expects uint8 RGB images [H,W,3]")
    rgb_t = torch.from_numpy(np.ascontiguousarray(img)).to(dev, non_blocking=True).unsqueeze(0)
    if dep.dtype == np.uint16:
        dep_t = torch.from_numpy(np.ascontiguousarray(dep).view(np.int16)).to(dev, non_blocking=True).view(torch.uint16)
    elif dep.dtype == np.uint32 or dep.dtype == np.uint64:
        dep_t = torch.from_numpy(dep.astype(np.int64)).to(dev)
    else:
        dep_t = torch.from_numpy(np.ascontiguousarray(dep)).to(dev)
    outs = create_stereoimages_batch(rgb_t, dep_t.unsqueeze(0), divergence, separation, modes, stereo_balance,
                                     stereo_offset_exponent, fill_technique)
    return [Image.fromarray(o[0].cpu().numpy()) for o in outs]
