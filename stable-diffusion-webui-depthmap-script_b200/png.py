"""PNG files of device images: the host receives finished, compressed files instead of raw pixels to save with PIL.

``encode_png_batch`` runs dm_png_encode (csrc/png_encode.cu): per-row PNG filtering, deflate in independent 32 KiB segments (one CTA
each) and the PNG container, all on the device, then one device -> host copy of the packed files.  Files are lossless and depend
only on their image.  There is no CPU fallback.
"""
from __future__ import annotations

from . import _lib


def _check_image_batch(t):
    import torch
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError("encode_png_batch: expected a CUDA tensor")
    if t.dtype == torch.uint16 and t.dim() == 3:
        return 1, 16
    if t.dtype == torch.uint8 and t.dim() == 4 and t.shape[3] == 3:
        return 3, 8
    raise ValueError(f"encode_png_batch: expected uint16 [B,H,W] or uint8 [B,H,W,3], got {t.dtype} {tuple(t.shape)}")


def encode_png_batch(t, invert=False) -> list:
    """uint16 [B,H,W] (16-bit greyscale) or uint8 [B,H,W,3] (RGB) CUDA tensor -> B PNG files (bytes).  invert (uint16 only)
    writes np.bitwise_not of the depth, as OUTPUT_DEPTH_INVERT does."""
    import torch
    C, bits = _check_image_batch(t)
    if invert and bits != 16:
        raise ValueError("encode_png_batch: invert applies to uint16 depth only")
    B, H, W = (int(s) for s in t.shape[:3])
    if min(B, H, W) <= 0:
        raise ValueError(f"encode_png_batch: empty batch or image {tuple(t.shape)}")
    t = t.contiguous()
    L = _lib.load()
    bound = L.dm_png_encode_bound(H, W, C, bits)
    ws_bytes = L.dm_png_encode_workspace_bytes(B, H, W, C, bits)
    out = torch.empty(B * bound, dtype=torch.uint8, device=t.device)
    offsets = torch.empty(B + 1, dtype=torch.int64, device=t.device)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=t.device)
    rc = L.dm_png_encode(t.data_ptr(), B, H, W, C, bits, _lib.DM_PNG_INVERT if invert else 0, out.data_ptr(), out.numel(),
                         offsets.data_ptr(), ws.data_ptr(), ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "dm_png_encode")
    off = offsets.cpu().tolist()
    data = out[:off[-1]].cpu().numpy().tobytes()
    return [data[off[i]:off[i + 1]] for i in range(B)]


def combine_depth_rgb(rgb, depth, horizontal=True, invert=False):
    """OUTPUT_DEPTH_COMBINE on the device: uint8 [B,H,W,3] and uint16 [B,H,W] -> uint8 [B,H,2W,3] (horizontal) or [B,2H,W,3],
    the image next to depth >> 8 on all three channels (np.bitwise_not of the depth first when invert) — what
    np.concatenate((rgb, convert_i16_to_rgb(depth, rgb)), axis) gives."""
    import torch
    if not (isinstance(rgb, torch.Tensor) and isinstance(depth, torch.Tensor) and rgb.is_cuda and depth.is_cuda):
        raise ValueError("combine_depth_rgb: expected CUDA tensors")
    if rgb.dtype != torch.uint8 or rgb.dim() != 4 or rgb.shape[3] != 3 or depth.dtype != torch.uint16 or tuple(depth.shape) != tuple(rgb.shape[:3]):
        raise ValueError(f"combine_depth_rgb: expected uint8 [B,H,W,3] and uint16 [B,H,W], got {tuple(rgb.shape)} and {tuple(depth.shape)}")
    B, H, W = (int(s) for s in depth.shape)
    out = torch.empty((B, H, 2 * W, 3) if horizontal else (B, 2 * H, W, 3), dtype=torch.uint8, device=rgb.device)
    rgb, depth = rgb.contiguous(), depth.contiguous()
    _lib.check(_lib.load().dm_depth_combine_rgb(rgb.data_ptr(), depth.data_ptr(), B, H, W, 1 if horizontal else 0, 1 if invert else 0,
                                                out.data_ptr(), _lib.stream_ptr()), "dm_depth_combine_rgb")
    return out
