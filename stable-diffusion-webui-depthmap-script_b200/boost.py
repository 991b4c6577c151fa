"""BOOST ("Boosting Monocular Depth"): estimateboost and the pix2pix merge network on the sm_90a kernels (SURVEY.md §8a row D9,
§8e patch-parallel).

reference: src/depthmap_generation.py:774-941 (estimateboost), :944-953 (generatemask), :969-1024 (calculateprocessingres),
:1028-1050 (doubleestimate), :1070-1177 (generatepatchs / applyGridpatch / adaptiveselection), :673-718 (ImageandPatchs);
pix2pix/models/networks.py:444-543 (UnetGenerator 'unet_1024', norm 'none'), pix2pix/models/pix2pix4depth_model.py:96-116.

Split of work.  The CONTROL PLANE stays on the host exactly as in the reference, because its results are integers that must not
move: the R_x resolution search and the patch selection look only at the RGB image (Sobel gradients, thresholds, an integral
image) and run through the same cv2 calls.  Every PIXEL of the depth result is produced on the GPU: the float image and its two
cubic resizes, the base-network forwards on crops (LeReS, model type 0: csrc/boost_kernels.cu leres_stem_im2col_f32; the MiDaS DPT
models 1-3 and MiDaS v2.1 (5) through estimatemidasBoost, :1180-1220: csrc/vit_kernels.cu preprocess_patchify_f32_crops or
csrc/midas_kernels.cu midas_stem_im2col_f32_crops, then the per-call min-max normalisation at crop size; ZoeDepth-NK (9) through
estimatezoedepth on np.uint8(crop * 255), :1062-1064: csrc/boost_kernels.cu quantise_crops_u8, then the ZoeDepth forward with its
pad + flip augmentation, metric depth at crop size), the cubic resizes to and from the
1024^2 merge resolution, the merge U-Net (split-operand fp32-class GEMMs), min-max normalisations, the degree-1 least-squares fit
(fp64 sums) and the Gaussian-mask blend; one device->host copy at the end.

Patch-parallel (§8e): the network work of a patch depends only on the base estimate; with a torch.distributed group the patches
are dealt round-robin to the ranks, the fitted 1024^2 patches are exchanged with ONE all-gather, and every rank applies the
(order-dependent) blend itself."""
from __future__ import annotations

import contextlib
import math

import numpy as np

from . import _lib

PIX2PIX_SIZE = 1024
MASK_SIZE = 3000


# ---------------------------------------------------------------------------------------------------------------------
# control plane (host, integers): which resolutions, which patches
# ---------------------------------------------------------------------------------------------------------------------
def receptive_field(model_type: int) -> int:
    """reference :777-786"""
    return {0: 448, 1: 512, 11: 518, 12: 518, 13: 518, 14: 518}.get(model_type, 384)


def _edge_strength(img):
    """|d/dy| + |d/dx| (Sobel 3) of the luma the reference uses (:956-958 weights, applied to whatever channel order it is handed)"""
    import cv2
    luma = np.dot(img[..., :3], [0.2989, 0.5870, 0.1140])
    return np.abs(cv2.Sobel(luma, cv2.CV_64F, 0, 1, ksize=3)) + np.abs(cv2.Sobel(luma, cv2.CV_64F, 1, 0, ksize=3))


def _max_pool_zero_padded(a, n):
    """what skimage.measure.block_reduce(a, (n, n), np.max) returns (reference :961-966)"""
    rows, cols = -(-a.shape[0] // n), -(-a.shape[1] // n)
    padded = np.zeros((rows * n, cols * n), a.dtype)
    padded[:a.shape[0], :a.shape[1]] = a
    return padded.reshape(rows, n, cols, n).max(axis=(1, 3))


def processing_resolution(img, basesize, confidence, scale_threshold, whole_size_threshold):
    """calculateprocessingres (:969-1024): the largest resolution at which at most `confidence` of the pixels are farther than
    half a receptive field from any edge, and the edge density at a quarter of the receptive field.  Both cv2.resize calls are
    bilinear: the reference passes its interpolation flag in the `dst` position."""
    import cv2
    unit = 32
    side = int(min(img.shape[0:2]))
    edges = cv2.resize(_edge_strength(img), (side, side))
    cut = edges.min() + 0.4 * (edges.max() - edges.min())
    edges = np.where(edges >= cut, 1.0, 0.0)
    reach = np.ones((int(basesize / unit), int(basesize / unit)), float)
    reach_quarter = np.ones((int(basesize / (4 * unit)), int(basesize / (4 * unit))), float)
    limit = min(whole_size_threshold, scale_threshold * max(img.shape[:2]))
    best = basesize / unit
    coarse = None
    for p in range(int(basesize / unit), int(limit / unit), int(basesize / (2 * unit))):
        coarse = cv2.resize(_max_pool_zero_padded(edges, int(np.floor(edges.shape[0] / p))), (p, p))
        coarse = np.where(coarse >= 0.5, 1.0, 0.0)
        if (1 - cv2.dilate(coarse, reach, iterations=1)).mean() > confidence:
            break
        best = p
    if coarse is None:
        raise ValueError("boost: the size limit leaves no resolution to search (whole_size_threshold too small for this model)")
    return int(best * unit), cv2.dilate(coarse, reach_quarter, iterations=1).mean()


def select_patches(img, base_size, factor):
    """generatepatchs + applyGridpatch + adaptiveselection (:1070-1165) -> list of [x, y, w, h], largest first (stable)."""
    import cv2
    g = _edge_strength(img)
    g[g < g[g > 0].mean()] = 0
    mean_density = g.sum() / g.size
    table = cv2.integral(g)
    rows, cols = table.shape

    def density(x, y, w, h):
        return (table[y + h, x + w] - table[y, x + w] - table[y + h, x] + table[y, x]) / (w * h)

    half = int(round(base_size / 2))
    stride = int(round(half * 0.75))
    grow = int(32 / factor)
    kept = []
    for cx in range(half, img.shape[1] - half, stride):            # columns outermost, as the reference enumerates its grid
        for cy in range(half, img.shape[0] - half, stride):
            x, y, w, h = cx - half, cy - half, 2 * half, 2 * half
            if density(x, y, w, h) < mean_density:
                continue
            tx, ty, tw, th = x, y, w, h
            while True:                                            # enlarge while the patch stays at least as dense as the image
                tx, ty, tw, th = tx - int(grow / 2), ty - int(grow / 2), tw + grow, th + grow
                if tx < 0 or ty < 0 or ty + th >= rows or tx + tw >= cols or density(tx, ty, tw, th) < mean_density:
                    break
                x, y, w, h = tx, ty, tw, th
            kept.append([x, y, w, h])
    return sorted(kept, key=lambda r: r[2], reverse=True)


def mask_profile(n=MASK_SIZE):
    """generatemask (:944-953) is separable: a box with a 15 % margin blurred by a Gaussian (sigma n/16, kernel 2*ceil(2*sigma)+1) and
    min-max normalised is the outer product of this 1-D profile with itself (the margin exceeds the kernel radius, so min = 0)."""
    sigma = int(n / 16)
    k = int(2 * math.ceil(2 * sigma) + 1)
    t = np.arange(k, dtype=np.float64) - (k - 1) / 2
    kern = np.exp(-(t * t) / (2.0 * sigma * sigma))
    kern /= kern.sum()
    box = np.zeros(n, np.float64)
    box[int(0.15 * n):n - int(0.15 * n)] = 1
    prof = np.convolve(box, kern, mode="same")
    return (prof / prof.max()).astype(np.float32)


def plan(img_f64, model_type, whole_size_threshold):
    """Everything estimateboost decides before it touches a depth value. img_f64: what get_raw_prediction hands over (:381)."""
    import cv2
    rf = receptive_field(model_type)
    H, W = img_f64.shape[:2]
    whole, patch_scale = processing_resolution(img_f64, rf, 0.2, 3, whole_size_threshold)
    factor = max(min(1, 4 * patch_scale * whole / whole_size_threshold), 0.2)
    if H > W:
        a, b = 2 * whole, round(2 * whole * W / H)
    else:
        a, b = round(2 * whole * H / W), 2 * whole
    a, b = int(round(a / factor)), int(round(b / factor))
    big = cv2.resize(img_f64, (b, a), interpolation=cv2.INTER_CUBIC)
    rects = select_patches(big, 2 * rf, factor)
    scale = H / a
    work = (round(a * scale), round(b * scale))                       # rows, cols of the image the patches are cut from (:685)
    scaled = []
    for r in rects:                                                   # :700-703, then clipped the way numpy slicing clips a crop
        x, y, w, h = np.round(np.array(r) * scale).astype(int).tolist()
        scaled.append([x, y, min(w, work[1] - x), min(h, work[0] - y)])
    return dict(rf=rf, whole=whole, patch_scale=patch_scale, factor=factor, target=(a, b), work=work, rects=rects, scaled_rects=scaled)


# ---------------------------------------------------------------------------------------------------------------------
# merge network
# ---------------------------------------------------------------------------------------------------------------------
class UnetMergeEngine:
    """pix2pix `unet_1024` generator (2 -> 1 channels, 10 levels, norm 'none'): down = [LeakyReLU(0.2), Conv 4x4/2], up = [ReLU,
    ConvTranspose 4x4/2] with skip concatenation, tanh at the end (pix2pix/models/networks.py:444-543).  Activations stay fp32 NHWC;
    every convolution is column building (activation fused into the gather) + the wgmma GEMM with fp32 output.  With
    split=True (default: the reference runs this network in fp32) operands are hi + lo fp16 pairs and the GEMM depth is tripled."""

    CH = [(2, 64), (64, 128), (128, 256), (256, 512)] + [(512, 512)] * 6      # (in, out) of the down conv at depth d

    KC = 1024      # GEMM depth per launch in split mode; the chunks' partial products are added in fp32 by dm_sum_chunks_f32, see _gemms

    def __init__(self, state_dict, device, split=True, kc=KC):
        import torch
        self.device, self.split, self.kc = device, bool(split), kc
        self.copies = 3 if split else 1
        self.ops = _lib.Ops()
        sd = {k[7:] if k.startswith("module.") else k: v for k, v in state_dict.items()}
        self.down, self.up = [], []
        prefix = "model."
        for d in range(10):
            if d == 0:
                kd, ku, child = prefix + "model.0.weight", prefix + "model.3.weight", prefix + "model.1."
            elif d == 9:
                kd, ku, child = prefix + "model.1.weight", prefix + "model.3.weight", None
            else:
                kd, ku, child = prefix + "model.1.weight", prefix + "model.5.weight", prefix + "model.3."
            wd = sd[kd].detach().float().to(device)                      # [Cout, Cin, 4, 4]
            assert tuple(wd.shape[:2]) == (self.CH[d][1], self.CH[d][0]), (kd, wd.shape)
            m = wd.permute(0, 2, 3, 1).reshape(wd.shape[0], -1)            # columns (ky, kx, cin)
            if d == 0:
                m = torch.nn.functional.pad(m, (0, 32))
            self.down.append(self._operand(m))
            wu = sd[ku].detach().float().to(device)                      # [Cin_total, Cout, 4, 4]
            cout = wu.shape[1]
            per_parity = []
            for a in (0, 1):
                for b in (0, 1):
                    ky, kx = ((1, 3), (0, 2))[a], ((1, 3), (0, 2))[b]
                    taps = [wu[:, :, ky[ty], kx[tx]].t() for ty in (0, 1) for tx in (0, 1)]      # each [Cout, Cin_total]
                    m = torch.stack(taps, dim=1).reshape(cout, -1)                              # columns (ty, tx, cin)
                    if cout < 32:
                        m = torch.nn.functional.pad(m, (0, 0, 0, 32 - cout))
                    per_parity.append(self._operand(m))
            self.up.append((per_parity, cout))
            if d == 0:
                self.bias = float(sd[prefix + "model.3.bias"].detach().float().item())
                # the two ends of the network as direct fp32 kernels (split mode): 2 -> 64 conv and (64 + 64) -> 1 transposed conv
                self.first_w = wd.permute(0, 2, 3, 1).reshape(64, 32).contiguous()
                par = []
                for a in (0, 1):
                    for b in (0, 1):
                        ky, kx = ((1, 3), (0, 2))[a], ((1, 3), (0, 2))[b]
                        par.append(torch.stack([wu[:, 0, ky[ty], kx[tx]] for ty in (0, 1) for tx in (0, 1)], dim=0))     # [4 taps, Cin_total]
                self.last_w = torch.stack(par, dim=0).contiguous()                                                    # [4, 4, 128]
            prefix = child
        self._bufs = {}
        # every call has the same shapes: after one eager call (allocations) the ~600 launches of a forward are captured into a CUDA
        # graph and replayed
        self._graphs = _lib.GraphCache(self.ops, "DEPTHMAP_B200_UNET_GRAPH", "merge-net")
        self._streams = [torch.cuda.Stream(device=device) for _ in range(8)] if self.split else []

    def _operand(self, m):
        """-> (fp16 operand [N, K * copies], fp32 [N] output scale).  Split mode scales the filter bank by a power of two first so
        that the low halves of the weights are normal fp16 numbers (a trained filter of 1e-2 has a low half of 2e-6, a subnormal),
        and hands the inverse back as the epilogue's per-column factor."""
        import torch
        if not self.split:
            return m.half().contiguous(), None
        k = int(math.floor(math.log2(1024.0 / max(float(m.abs().max()), 1e-30))))
        m = m * (2.0 ** k)
        hi = m.half()
        lo = (m - hi.float()).half()
        return torch.cat([hi, hi, lo], dim=1).contiguous(), torch.full((m.shape[0],), 2.0 ** -k, dtype=torch.float32, device=m.device)

    def _gemms(self, jobs):
        """jobs: [(cols [M, K] fp16, K, operand, M, N, out [M, N] fp32)] — the GEMMs of one layer (one for a convolution, the four parities
        of a transposed one).  out = cols @ W^T.
        Split mode cuts the tripled depth into chunks of `kc`: the tensor core's own fp32 accumulator aligns and TRUNCATES partial sums, a
        bias that grows linearly with the number of K steps (tools/probe_tensor_core.py), so every chunk is accumulated on its own and
        the chunks are added in a fixed order by a rounding fp32 adder (dm_sum_chunks_f32, which also undoes the filter pre-scale).
        The chunk GEMMs of a layer are independent (deep levels: a handful of CTAs each, ~20 us of latency): they are issued round-robin
        on side streams — concurrent branches of the captured graph — and joined before the reduction."""
        import torch
        if not self.split:
            for cols, K, (w, _), M, N, out in jobs:
                self.ops.gemm(cols, K, w, K, M, N, K, epi=_lib.EPI_STORE_F32, X=out, ldx=N)
            return
        main = torch.cuda.current_stream()
        launches = []
        for ji, (cols, K, (w, gamma), M, N, out) in enumerate(jobs):
            kc = self.kc or K
            chunks = [(k0, min(kc, K - k0)) for k0 in range(0, K, kc)]
            ws = self._buf(f"ws{ji}", (len(chunks), M, N), torch.float32)
            for ci, (k0, kk) in enumerate(chunks):
                launches.append((cols, K, w, M, N, k0, kk, ws[ci]))
            jobs[ji] = (ws, len(chunks), M, N, gamma, out)
        streams = self._streams[:min(len(self._streams), len(launches))] if len(launches) > 1 else []
        for s_ in streams:
            s_.wait_stream(main)
        for li, (cols, K, w, M, N, k0, kk, dst) in enumerate(launches):
            with torch.cuda.stream(streams[li % len(streams)]) if streams else contextlib.nullcontext():
                self.ops.gemm(cols[:, k0:], K, w[:, k0:], K, M, N, kk, epi=_lib.EPI_STORE_F32, X=dst, ldx=N)
        for s_ in streams:
            main.wait_stream(s_)
        for ws, n, M, N, gamma, out in jobs:
            self.ops.call("dm_sum_chunks_f32", ws, n, M * N, N, gamma, out)

    def _buf(self, name, shape, dtype):
        import torch
        n = int(np.prod(shape))
        t = self._bufs.get(name)
        if t is None or t.numel() < n or t.dtype != dtype:
            t = torch.empty(n, dtype=dtype, device=self.device)
            self._bufs[name] = t
        return t[:n].view(*shape)

    def forward(self, x2):
        """x2: fp32 CUDA [1024, 1024, 2] (real_A as NHWC) -> fp32 CUDA [1024, 1024] in (-1, 1)"""
        return self._graphs.run(tuple(x2.shape), self._forward, x2, copy_out=True)

    def _forward(self, x2):
        import torch
        ops, cp = self.ops, self.copies
        S = int(x2.shape[0])
        assert x2.shape == (S, S, 2) and S % 1024 == 0 and x2.dtype == torch.float32
        h = []
        for d in range(10):
            Hin = S >> d
            cin, cout = self.CH[d]
            M = (Hin // 2) ** 2
            K = (64 if d == 0 else 16 * cin) * cp
            if d == 0 and self.split:
                out = self._buf("h0", (M, cout), torch.float32)
                ops.call("dm_unet_first", x2, Hin, Hin, self.first_w, out)
                h.append(out)
                continue
            cols = self._buf("cols", (M, K), torch.float16)
            if d == 0:
                ops.call("dm_unet_first_cols", x2, Hin, Hin, cols, int(self.split))
            else:
                ops.call("dm_unet_down_cols", h[d - 1], Hin, Hin, cin, cols, int(self.split))
            out = self._buf(f"h{d}", (M, cout), torch.float32)
            self._gemms([(cols, K, self.down[d], M, cout, out)])
            h.append(out)
        u, cu = None, 0
        for d in range(9, -1, -1):
            Hs = S >> (d + 1)
            M = Hs * Hs
            c1 = self.CH[d][1]
            if d == 0 and self.split:
                out = torch.empty(2 * Hs, 2 * Hs, dtype=torch.float32, device=self.device)
                ops.call("dm_unet_last", h[0], c1, u, cu, Hs, Hs, self.last_w, self.bias, out)
                break
            K = 4 * (c1 + cu) * cp
            cols = self._buf("cols", (4, M, K), torch.float16)
            ops.call("dm_unet_up_cols", h[d], c1, u, cu, Hs, Hs, cols, int(self.split))
            weights, cout = self.up[d]
            N = max(cout, 32)
            tmp = self._buf("tmp", (4, M, N), torch.float32)
            self._gemms([(cols[par], K, weights[par], M, N, tmp[par]) for par in range(4)])
            if d > 0:
                u = self._buf(f"u{d}", (2 * Hs, 2 * Hs, cout), torch.float32)
                ops.call("dm_unet_interleave", tmp, Hs, Hs, N, cout, u)
                cu = cout
            else:
                out = torch.empty(2 * Hs, 2 * Hs, dtype=torch.float32, device=self.device)
                ops.call("dm_unet_final", tmp, Hs, Hs, N, self.bias, out)
        return out


# ---------------------------------------------------------------------------------------------------------------------
# data plane
# ---------------------------------------------------------------------------------------------------------------------
# How singleestimate (:1053-1066) hands each base network's map to doubleestimate:
#   NET_SIZE    LeReS res101 (0): estimateleres' map, at net size from forward_crops, cubic-resized back to the crop
#   NORMALISED  DPT-BEiT-L 512 / 384, DPT-Large 384, MiDaS v2.1 (1, 2, 3, 5): estimatemidasBoost's map at crop size, min-max
#               normalised (a constant map is flagged)
#   METRIC      ZoeDepth-NK (9): estimatezoedepth's metric depth at crop size, used as is
NET_SIZE, NORMALISED, METRIC = "net size", "normalised", "metric"
ESTIMATES = {0: NET_SIZE, 1: NORMALISED, 2: NORMALISED, 3: NORMALISED, 5: NORMALISED, 9: METRIC}
BASE_NETWORKS = tuple(ESTIMATES)


class BoostPipeline:
    """estimateboost for one image on one GPU (or one rank of a patch-parallel group)."""

    def __init__(self, depth_engine, merge_engine, device, model_type=0):
        import torch
        if model_type not in BASE_NETWORKS:
            raise NotImplementedError(f"boost is built for the base networks LeReS res101 (model type 0), the MiDaS models (1, 2, 3, 5) "
                                      f"and ZoeDepth-NK (9), not model type {model_type}")
        self.depth, self.merge, self.device, self.model_type = depth_engine, merge_engine, device, model_type
        self.estimate = ESTIMATES[model_type]
        self.ops = _lib.Ops()
        self.P = int(self.ops.L.dm_boost_partials())
        self.profile = torch.from_numpy(mask_profile()).to(device)
        self._degenerate = torch.zeros(1, dtype=torch.int32, device=device)

    # -- small device helpers ---------------------------------------------------------------------------------------
    def _cubic(self, src, pitch, hin, win, hout, wout, planes=1, src_plane=0, out=None):
        import torch
        if out is None:
            out = torch.empty((planes, hout, wout) if planes > 1 else (hout, wout), dtype=torch.float32, device=self.device)
        self.ops.call("dm_boost_resize_cubic", src, pitch, src_plane, hin, win, out, wout, hout * wout, hout, wout, planes)
        return out

    def _minmax(self, x):
        import torch
        p = torch.empty(self.P * 2, dtype=torch.float32, device=self.device)
        self.ops.call("dm_boost_minmax", x, x.numel(), p)
        return p

    def _merge(self, outer, inner):
        """Pix2Pix4DepthModel.set_input + test: two [1024, 1024] estimates -> fake_B"""
        import torch
        n = outer.numel()
        x2 = torch.empty(PIX2PIX_SIZE, PIX2PIX_SIZE, 2, dtype=torch.float32, device=self.device)
        po, pi = self._minmax(outer), self._minmax(inner)
        self.ops.call("dm_boost_merge_input", outer, inner, n, po, pi, x2)
        return self.merge.forward(x2)

    def _post(self, t, normalise):
        import torch
        out = torch.empty_like(t)
        p = self._minmax(t) if normalise else None
        self.ops.call("dm_boost_post", t, t.numel(), p, int(normalise), out)
        return out

    def _normalise_estimate(self, est):
        """estimatemidasBoost's tail (:1212-1220): (p - min) / (max - min) of the crop-size prediction; a constant prediction is
        flagged on the device and reported by run() (the reference returns a scalar there and its next cv2.resize fails)"""
        import torch
        out = torch.empty_like(est)
        p = self._minmax(est)
        self.ops.call("dm_boost_minmax_normalise", est, est.numel(), p, out, self._degenerate)
        return out

    def _estimate_1024(self, planar, rect, msize):
        """singleestimate on a crop (LeReS at msize x msize or the DPT at its upper-bound net size, cubic back to the crop size;
        min-max normalised for the DPT; ZoeDepth's metric map at the crop size as it is) followed by the cubic resize to 1024^2"""
        est = self.depth.forward_batch(None, msize, msize, planar=(planar, rect))[0]
        if self.estimate == NORMALISED:
            est = self._normalise_estimate(est)
        return self._cubic(est.data_ptr(), rect[2], rect[3], rect[2], PIX2PIX_SIZE, PIX2PIX_SIZE)

    def double_estimate(self, planar, rect, size1, size2):
        """doubleestimate (:1028-1050) -> [1024, 1024], min-max normalised"""
        low = self._estimate_1024(planar, rect, size1)
        high = self._estimate_1024(planar, rect, size2)
        return self._post(self._merge(low, high), True)

    PATCH_BATCH = 8      # crops per base-network forward in the patch loop (LeReS 896 net: ~1.5 GB per crop; BEiT-L 1024 net: ~1 GB)

    def fitted_patches(self, work_img, base, rects, rf):
        """fitted_patch for a list of patches with the base network BATCHED over the crops (all patches use the same two net sizes);
        yields (mapped, sums) in the order of `rects`.  Engines without `forward_crops` (test doubles) go one by one."""
        if not hasattr(self.depth, "forward_crops") or self.PATCH_BATCH <= 1:
            for rect in rects:
                yield self.fitted_patch(work_img, base, rect, rf)
            return
        for c0 in range(0, len(rects), self.PATCH_BATCH):
            chunk = rects[c0:c0 + self.PATCH_BATCH]
            low = self.depth.forward_crops(work_img, chunk, rf)
            high = self.depth.forward_crops(work_img, chunk, 2 * rf)
            for k, rect in enumerate(chunk):
                x, y, w, h = rect
                ests = []
                for net, src in ((rf, low[k]), (2 * rf, high[k])):      # the crop-size map (ESTIMATES), then cubic to 1024^2 (doubleestimate)
                    if self.estimate == NORMALISED:
                        at_crop = self._normalise_estimate(src)
                    elif self.estimate == NET_SIZE:
                        at_crop = self._cubic(src.data_ptr(), net, net, net, h, w)
                    else:
                        at_crop = src
                    ests.append(self._cubic(at_crop.data_ptr(), w, h, w, PIX2PIX_SIZE, PIX2PIX_SIZE))
                est = self._post(self._merge(ests[0], ests[1]), True)
                yield self.fitted_patch(work_img, base, rect, rf, est=est)

    def fitted_patch(self, work_img, base, rect, rf, est=None):
        """the network part of one patch: -> (mapped [1024, 1024], fit partial sums); independent of every other patch"""
        import torch
        x, y, w, h = rect
        if est is None:
            est = self.double_estimate(work_img, rect, rf, 2 * rf)
        pitch = int(base.shape[1])
        base1024 = self._cubic(base.data_ptr() + 4 * (y * pitch + x), pitch, h, w, PIX2PIX_SIZE, PIX2PIX_SIZE)
        mapped = self._post(self._merge(base1024, est), False)
        sums = torch.empty(self.P * 4, dtype=torch.float64, device=self.device)
        self.ops.call("dm_boost_fit_sums", mapped, base1024, mapped.numel(), sums)
        return mapped, sums

    def blend(self, updated, mapped, sums, rect):
        x, y, w, h = rect
        self.ops.call("dm_boost_blend", mapped, PIX2PIX_SIZE, sums, self.profile, MASK_SIZE, updated, int(updated.shape[1]), x, y, w, h)

    # -- the whole thing ----------------------------------------------------------------------------------------------
    def run(self, rgb_u8, whole_size_threshold, group=None, info=None, precomputed=None, to_host=True):
        """rgb_u8: numpy uint8 [H, W, 3] (the PIL image) -> numpy float32 [H, W] (what estimateboost returns).
        precomputed: a previous call's `info` for the same image (skips the host control plane: bench's resident-input measurement);
        to_host=False returns the CUDA tensor."""
        import cv2
        import torch
        rgb_u8 = np.array(rgb_u8, dtype=np.uint8, order='C', copy=True)      # PIL hands out read-only buffers
        H, W = rgb_u8.shape[:2]
        self._degenerate.zero_()
        if precomputed is None:
            swapped = cv2.cvtColor(rgb_u8, cv2.COLOR_BGR2RGB) / 255.0        # the image the reference's control plane sees (:381)
            p = plan(swapped, self.model_type, whole_size_threshold)
        else:
            p = precomputed
        if info is not None:
            info.update(p)
        rf = p["rf"]
        dev_rgb = torch.from_numpy(rgb_u8).to(self.device)
        img = torch.empty(3, H, W, dtype=torch.float32, device=self.device)
        self.ops.call("dm_boost_u8_to_planar", dev_rgb, H, W, img)
        whole = self.double_estimate(img, (0, 0, W, H), rf, p["whole"])
        a, b = p["target"]
        big = self._cubic(img.data_ptr(), W, H, W, a, b, planes=3, src_plane=H * W)
        wh, ww = p["work"]
        work = self._cubic(big.data_ptr(), b, a, b, wh, ww, planes=3, src_plane=a * b)
        base = self._cubic(whole.data_ptr(), PIX2PIX_SIZE, PIX2PIX_SIZE, PIX2PIX_SIZE, wh, ww)
        updated = base.clone()
        rects = p["scaled_rects"]
        world, rank = (group.size(), group.rank()) if group is not None else (1, 0)
        if world == 1 or not rects:         # no patch selected (flat or small image): the result is the resized whole-image estimate
            for rect, (mapped, sums) in zip(rects, self.fitted_patches(work, base, rects, rf)):
                self.blend(updated, mapped, sums, rect)
        else:
            from .dist import all_gather_round_robin
            mine = list(range(rank, len(rects), world))
            got = list(self.fitted_patches(work, base, [rects[i] for i in mine], rf))
            loc_m = torch.stack([m.view(-1) for m, _ in got]) if got else torch.zeros(0, PIX2PIX_SIZE * PIX2PIX_SIZE, dtype=torch.float32, device=self.device)
            loc_s = torch.stack([q for _, q in got]) if got else torch.zeros(0, self.P * 4, dtype=torch.float64, device=self.device)
            all_m = all_gather_round_robin(loc_m, len(rects), group)          # the path's one exchange: the fitted patches ...
            all_s = all_gather_round_robin(loc_s, len(rects), group)          # ... and their five fp64 sums
            for i, rect in enumerate(rects):                                # the blend is order dependent: every rank replays it in order
                self.blend(updated, all_m[i].view(PIX2PIX_SIZE, PIX2PIX_SIZE), all_s[i], rect)
        out = self._cubic(updated.data_ptr(), ww, wh, ww, H, W)
        if self.estimate == NORMALISED and int(self._degenerate.item()):
            raise ValueError("boost: the base network returned a constant depth map for a crop (estimatemidasBoost cannot normalise it)")
        return out.cpu().numpy() if to_host else out
