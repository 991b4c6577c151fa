"""Video mode's cross-frame depth normalisation on H100 — drop-in for ``process_predicitons`` of the reference's
``src/video_mode.py:103-128`` (the misspelt name is the reference's), SURVEY.md §8(f) rank 1.

``process_predicitons(predictions, smoothening)`` keeps the reference's contract: a list of float32 [H,W] raw predictions in,
a list of normalised frames out (float32 for 'none', float64 for 'experimental', untouched for anything else), bit for bit
what numpy gives.  ``process_predictions_batch`` is the device form; with ``group`` set the frames of the clip are sharded
over the ranks of a torch.distributed group (rank r holds the contiguous global frames [first, first + N_local)) and the only
traffic is an all-reduce of two floats ('none') or of four 256-bin histograms per radix pass plus a two-frame halo exchange
('experimental').  No CPU fallback: the kernels are in csrc/normalize.cu behind include/depthmap_b200.h."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib


def percentile_ranks(n, percents, dtype=np.float32):
    """np.percentile(a, percents) with a.size == n, a.dtype == dtype, method 'linear': per percentile the two 0-based ranks it
    reads and the float64 interpolation weight — numpy's own expressions (numpy/lib/_function_base_impl.py: percentile divides
    by `a.dtype.type(100)` for floating arrays, then _quantile's virtual index / gamma), same order of operations."""
    q = np.true_divide(np.asanyarray(percents, dtype=np.float64), np.dtype(dtype).type(100))
    virtual = (n - 1) * q
    previous = np.floor(virtual).astype(np.intp)
    nxt = previous + 1
    above = virtual >= n - 1
    previous[above] = -1
    nxt[above] = -1
    below = virtual < 0
    previous[below] = 0
    nxt[below] = 0
    gamma = np.asanyarray(virtual - previous, dtype=virtual.dtype)
    return [(int(p) % n, int(x) % n, float(g)) for p, x, g in zip(previous, nxt, gamma)]


def process_predictions_batch(frames, smoothening='none', group=None, first=0, n_total=None, halo=None):
    """frames: float32 CUDA tensor [N_local, H, W] = global frames [first, first + N_local) of a clip of n_total frames.
    halo: for 'experimental' with a group, (frames before [<=2,H,W], frames after [<=2,H,W]) already exchanged by the caller,
    or None to have this function exchange them (all_gather of the boundary frames).  Returns the normalised local frames."""
    import torch
    _lib.require_cuda()
    if smoothening not in ('none', 'experimental'):
        return frames
    if frames.dtype != torch.float32 or frames.dim() != 3:
        raise ValueError("frames must be a float32 tensor [N, H, W]")
    L = _lib.load()
    frames = frames.contiguous()
    N, H, W = frames.shape
    hw = H * W
    n_total = N if n_total is None else int(n_total)
    dev = frames.device
    st = _lib.stream_ptr
    ws_bytes = L.dm_video_workspace_bytes()
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    dist = None
    if group is not None:
        import torch.distributed as dist
    if smoothening == 'none':
        lohi = torch.empty(2, dtype=torch.float32, device=dev)
        _lib.check(L.dm_video_minmax(frames.data_ptr(), N * hw, lohi.data_ptr(), ws.data_ptr(), ws_bytes, st()), "dm_video_minmax")
        if dist is not None:      # the path's one exchange: global min / max
            dist.all_reduce(lohi[0:1], op=dist.ReduceOp.MIN, group=group)
            dist.all_reduce(lohi[1:2], op=dist.ReduceOp.MAX, group=group)
        out = torch.empty_like(frames)
        _lib.check(L.dm_video_scale_f32(frames.data_ptr(), N * hw, lohi.data_ptr(), out.data_ptr(), st()), "dm_video_scale_f32")
        return out
    # 'experimental': bounds from the blended stack
    local, base = frames, first
    if dist is not None and n_total > N:
        if halo is None:
            halo = exchange_halo(frames, group, first, n_total)
        before, after = halo
        local = torch.cat([before, frames, after], dim=0).contiguous()
        base = first - before.shape[0]
    blended = torch.empty_like(frames)
    _lib.check(L.dm_video_blend(local.data_ptr(), hw, base, local.shape[0], n_total, first, N, blended.data_ptr(), st()), "dm_video_blend")
    (p0, n0, g0), (p1, n1, g1) = percentile_ranks(n_total * hw, [0.5, 99.5], np.float32)
    ranks = (ctypes.c_longlong * 4)(p0, n0, p1, n1)
    _lib.check(L.dm_video_select_init(ws.data_ptr(), ranks, st()), "dm_video_select_init")
    hist = ws[32:32 + 4096].view(torch.int32)
    for p in range(4):
        _lib.check(L.dm_video_select_hist(blended.data_ptr(), N * hw, p, ws.data_ptr(), st()), "dm_video_select_hist")
        if dist is not None:
            dist.all_reduce(hist, op=dist.ReduceOp.SUM, group=group)
        _lib.check(L.dm_video_select_pick(ws.data_ptr(), p, st()), "dm_video_select_pick")
    ab = torch.empty(2, dtype=torch.float64, device=dev)
    _lib.check(L.dm_video_select_bounds(ws.data_ptr(), g0, g1, ab.data_ptr(), st()), "dm_video_select_bounds")
    out = torch.empty((N, H, W), dtype=torch.float64, device=dev)
    _lib.check(L.dm_video_scale_f64(frames.data_ptr(), N * hw, ab.data_ptr(), out.data_ptr(), st()), "dm_video_scale_f64")
    return out


def halo_plan(first, n_local, n_total):
    """Global indices of the (at most two) frames a rank needs before and after its own block for the 5-tap blend."""
    before = [g for g in (first - 2, first - 1) if g >= 0]
    after = [g for g in (first + n_local, first + n_local + 1) if g <= n_total - 1]
    return before, after


def exchange_halo(frames, group, first, n_total):
    """All ranks publish their first two and last two frames; each rank keeps the ones adjacent to its block.  (An all_gather
    of 4 frames per rank: the blocks are contiguous and ordered by rank, so neighbours are enough, but blocks shorter than two
    frames make the neighbour's neighbour necessary — gathering is simpler than chasing that.)"""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    N, H, W = frames.shape
    edge = torch.zeros(4, H, W, dtype=frames.dtype, device=frames.device)
    idx = torch.full((4,), -1, dtype=torch.int64, device=frames.device)
    for slot, j in enumerate((0, 1, N - 2, N - 1)):
        if 0 <= j < N:
            edge[slot] = frames[j]
            idx[slot] = first + j
    edges = [torch.empty_like(edge) for _ in range(world)]
    idxs = [torch.empty_like(idx) for _ in range(world)]
    dist.all_gather(edges, edge, group=group)
    dist.all_gather(idxs, idx, group=group)
    have = {}
    for e, ix in zip(edges, idxs):
        for slot, g in enumerate(ix.tolist()):
            if g >= 0:
                have[g] = e[slot]
    before_i, after_i = halo_plan(first, N, n_total)
    empty = frames[:0]
    before = torch.stack([have[g] for g in before_i]) if before_i else empty
    after = torch.stack([have[g] for g in after_i]) if after_i else empty
    return before, after


def process_predicitons(predictions, smoothening='none'):
    """Reference contract (src/video_mode.py:103-128): list of float32 [H,W] arrays -> list of normalised arrays."""
    import torch
    if smoothening not in ('none', 'experimental'):
        return predictions
    dev = _lib.require_cuda()
    stack = np.stack([np.asarray(p) for p in predictions])
    if stack.dtype != np.float32:
        raise NotImplementedError("depthmap_b200 video normalisation expects float32 predictions (what get_raw_prediction returns)")
    out = process_predictions_batch(torch.from_numpy(stack).to(dev), smoothening).cpu().numpy()
    return [out[i] for i in range(out.shape[0])]
