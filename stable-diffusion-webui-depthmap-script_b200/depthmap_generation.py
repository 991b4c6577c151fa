"""Depth estimation on H100 — drop-in for the hot-path part of the reference's ``src/depthmap_generation.py``.

``ModelHolder`` keeps the reference's public methods and attributes (src/depthmap_generation.py:40-403):
``update_settings``, ``ensure_models``, ``load_models``, ``get_default_net_size``, ``offload``, ``reload``,
``unload_models``, ``get_raw_prediction(input, net_width, net_height) -> (float32 [H,W], invert)``, plus the additive
``get_raw_prediction_batch`` (uint8 CUDA batch in, float32 CUDA batch out, no host sync) used by the batched funnel and
the bench.  The network forward is a sequence of C-ABI calls (wgmma GEMM / implicit-GEMM conv / fused attention /
LayerNorm / resize kernels, include/depthmap_b200.h); PyTorch only owns device memory and the stream.

Implemented model types: 0 (LeReS res101), 1, 2 (MiDaS 3.1 DPT-BEiT-L 512 / 384), 3 (MiDaS 3.0 DPT-Large 384), 5 (MiDaS v2.1,
ResNeXt-101 MidasNet), 7, 8, 9 (ZoeDepth-N, -K, -NK) and 12, 13, 14 (Depth-Anything-V2 S/B/L).  Others raise NotImplementedError naming the type.
Weights: a state_dict in the upstream checkpoint layout (``depth_anything_v2_vit{s,b,l}.pth``), packed once at load
into the kernels' layout (fp16 GEMM operands, (ky,kx,cin)-ordered conv filters, ConvTranspose as GEMM + pixel shuffle).
Tiling mode (``tiling_mode``, src/depthmap_generation.py:251-260) makes every padded Conv2d of the depth network pad
circularly: the engines' ``circular=True`` runs those convolutions through the circular conv / im2col / stem entry points.
"""
from __future__ import annotations

import ctypes
import functools
import gc
import math
import os

import numpy as np

from . import _lib

DAV2_CONFIGS = {
    'vits': dict(embed_dim=384, depth=12, heads=6, features=64, out_channels=[48, 96, 192, 384], layers=[2, 5, 8, 11]),
    'vitb': dict(embed_dim=768, depth=12, heads=12, features=128, out_channels=[96, 192, 384, 768], layers=[2, 5, 8, 11]),
    'vitl': dict(embed_dim=1024, depth=24, heads=16, features=256, out_channels=[256, 512, 1024, 1024], layers=[4, 11, 17, 23]),
}


def _ru(x, m):
    return (x + m - 1) // m * m


def _constrain_to_multiple_of(x, multiple_of, min_val=0, max_val=None):
    y = int(np.round(x / multiple_of) * multiple_of)
    if max_val is not None and y > max_val:
        y = int(np.floor(x / multiple_of) * multiple_of)
    if y < min_val:
        y = int(np.ceil(x / multiple_of) * multiple_of)
    return y


def dav2_net_size(width, height, target, multiple_of=14):
    """Resize(keep_aspect_ratio, lower_bound, multiple of 14) of the reference (util/transform.py:61-104)."""
    sh, sw = target / height, target / width
    if sw > sh:
        sh = sw
    else:
        sw = sh
    return (_constrain_to_multiple_of(sw * width, multiple_of, min_val=target),
            _constrain_to_multiple_of(sh * height, multiple_of, min_val=target))


# ---- the kernels' weight layout: zero-padded [N, K] matrices (fp16, or fp32 for split_weight), (ky, kx, cin) 3x3 filters, fp32
# bias vectors.  Every engine packs its checkpoint through these three.
def _mat(m, rows=None, cols=None, dtype=None):
    """[N, ...] (flattened to [N, K]) -> [rows, cols] fp16 (unless `dtype`), zero padded"""
    import torch
    dtype = dtype or torch.float16
    m = m.reshape(m.shape[0], -1)
    t = torch.zeros(rows or m.shape[0], cols or m.shape[1], dtype=dtype, device=m.device)
    t[:m.shape[0], :m.shape[1]] = m.to(dtype)
    return t


def _conv_w(w, cin_pad=None, cout_pad=None, dtype=None, groups=1):
    """[Cout, Cin/groups, 3, 3] -> [cout_pad, 9*cin_pad] fp16 (unless `dtype`), K ordered (ky, kx, cin), zero padded; the groups
    become diagonal blocks of a dense filter"""
    import torch
    dtype = dtype or torch.float16
    co, cig = w.shape[:2]
    cin_pad, cout_pad, cog = cin_pad or cig * groups, cout_pad or co, co // groups
    t = torch.zeros(cout_pad, 3, 3, cin_pad, dtype=dtype, device=w.device)
    wp = w.permute(0, 2, 3, 1).to(dtype)
    for g in range(groups):
        t[g * cog:(g + 1) * cog, :, :, g * cig:(g + 1) * cig] = wp[g * cog:(g + 1) * cog]
    return t.reshape(cout_pad, 9 * cin_pad).contiguous()


def _vec(b, n=None):
    """[n] fp32, zero padded"""
    import torch
    t = torch.zeros(n or b.numel(), dtype=torch.float32, device=b.device)
    t[:b.numel()] = b.float().reshape(-1)
    return t


def _ragged_net_size(engine, desc, net_w, net_h):
    """the one network input size of a ragged batch (desc: _lib.Ragged of its images); ValueError if the images do not share one"""
    net_h = net_h if net_h is not None else net_w
    nets = {engine.net_size(w, h, net_w, net_h) for h, w in desc.sizes}
    if len(nets) != 1:
        raise ValueError(f"a ragged batch must share one network input size; these images map to {sorted(nets)}")
    return nets.pop()


def _resize_ragged(engine, d, B, nh, nw, desc, mode):
    """the final resize of a ragged batch: d fp32 [B, nh, nw] -> packed fp32, image i at desc.sizes[i] (layout _lib.Ragged(sizes, 1))"""
    import torch
    out_desc = _lib.Ragged(desc.sizes, 1, engine.device)
    out = torch.empty(out_desc.size, dtype=torch.float32, device=engine.device)
    engine.ops.call("dm_resize_f32_ragged", d, B, nh, nw, out, out_desc.size, out_desc.host.ctypes.data, out_desc.dev, mode)
    return out


class SplitWeight:
    """A GEMM / conv operand of the split (fp32-class) path: `t` fp16 [N, 3K], `scale` fp32 [N] (see split_weight)."""

    def __init__(self, t, scale):
        self.t, self.scale = t, scale


def split_weight(m, groups=1):
    """fp32 [N, K] -> SplitWeight for dm_gemm_split_ex / dm_conv3x3_split_ex.  Row n is pre-scaled by 2^e[n], the power of two
    that brings its largest magnitude into [1024, 2048), so that the low halves of the weights are normal fp16 numbers (a trained
    weight of 1e-2 has a low half near 2e-6, a subnormal); scale = 2^-e[n] undoes it in the epilogue.  The K columns are `groups`
    runs (the taps of a 3x3 filter), each packed [w_hi | w_hi | w_lo] against the activations' [a_hi | a_lo | a_hi]."""
    import torch
    m = m.float()
    N, K = m.shape
    amax = m.abs().amax(dim=1)
    e = torch.where(amax > 0, torch.floor(torch.log2(1024.0 / amax.clamp_min(1e-30))), torch.zeros_like(amax)).clamp(-100, 100)
    ms = m * torch.exp2(e)[:, None]
    hi = ms.half()
    lo = (ms - hi.float()).half()
    g = lambda t: t.reshape(N, groups, K // groups)
    return SplitWeight(torch.cat([g(hi), g(hi), g(lo)], dim=2).reshape(N, 3 * K).contiguous(), torch.exp2(-e).contiguous())


class DepthAnythingV2Engine:
    """Depth-Anything-V2 (DINOv2 ViT + DPT head) forward on the sm_90a kernels.

    Mirrors DepthAnythingV2.forward / DPTHead.forward / DINOv2.get_intermediate_layers of the reference
    (ddepth_anything_v2/depth_anything_v2/dpt.py:117-184, dinov2.py:297-321) plus image2tensor (dpt.py:196-221) and the
    final resize of estimatedepthanything_v2 (src/depthmap_generation.py:548-559).  Also the base of DptBeitEngine: the
    two families share the ViT block sequence and the whole DPT decoder and differ only in the hooks below.
    circular=True: tiling mode, every padded convolution (the decoder's 3x3 convs and the reassemble stage's stride-2 one) pads
    circularly.
    split=True: the fp32-class path of no_half.  Every GEMM / convolution operand is a split tensor (fp16 hi + lo, 3x the width,
    gemm_wgmma.cu) against split weights, with promoted fp32 accumulation; the residual stream, LayerNorm statistics and softmax
    are fp32.  Only Depth-Anything-V2 itself has it (SUPPORTS_SPLIT)."""

    PATCH = 14
    MEAN = (0.485, 0.456, 0.406)
    STD = (0.229, 0.224, 0.225)
    # the reference swaps R/B three times before the network sees the image (src/depthmap_generation.py:381,550; dpt.py:213):
    # network channel c carries source channel 2-c
    CHAN_MAP = (2, 1, 0)
    FINAL_RESIZE_MODE = 0  # bilinear, align_corners=True (src/depthmap_generation.py:558)
    CONFIGS = DAV2_CONFIGS
    SUPPORTS_SPLIT = True
    NEEDS_READOUT = False       # the features come through the final LayerNorm (emit_feature), not a readout projection

    def __init__(self, state_dict, encoder, device, circular=False, split=False):
        import torch
        if split and not type(self).SUPPORTS_SPLIT:
            raise NotImplementedError(f"{type(self).__name__} has no split (no_half) path; it is implemented for Depth-Anything-V2 only")
        self.cfg = self.CONFIGS[encoder]
        self.encoder = encoder
        self.device = device
        self.circular = circular
        self.split = bool(split)
        self.ops = _lib.Ops()
        self._buf_key = None
        self._bufs = {}
        self._pos_cache = {}
        # from the second call on at a given (B, net size) the launches of run_network + run_head replay from a CUDA graph
        self._graphs = _lib.GraphCache(self.ops, "DEPTHMAP_B200_MODEL_GRAPH", type(self).__name__)
        self._pack(state_dict)

    # ---- weight packing --------------------------------------------------------------------------------------------
    def _pack(self, sd):
        """sd in Depth-Anything-V2's checkpoint layout, which the MiDaS DPT engines map theirs to (_MidasDptEngine._pack).  Without
        POS_EMBED there is no 'pretrained.pos_embed', with NEEDS_READOUT no final 'pretrained.norm'."""
        import torch
        dev = self.device
        cfg = self.cfg
        C, Fch, oc = cfg['embed_dim'], cfg['features'], cfg['out_channels']
        # GEMM / conv operands: fp16, or (split) built in fp32 and packed by split_weight; `groups` = the taps of a 3x3 filter
        wdt = torch.float32 if self.split else torch.float16
        op = (lambda t, groups=1: split_weight(t, groups)) if self.split else (lambda t, groups=1: t)
        key = lambda k: sd[k].detach().to(dev)
        mat = lambda k, rows=None, cols=None: op(_mat(key(k), rows, cols, wdt))
        conv_w = lambda k, ci, co: op(_conv_w(key(k), ci, co, wdt), 9)
        vec = lambda k, n=None: _vec(key(k), n)
        w = {}
        self.kpad = _ru(sd['pretrained.patch_embed.proj.weight'][0].numel(), 64)
        w['pe_w'], w['pe_b'] = mat('pretrained.patch_embed.proj.weight', cols=self.kpad), vec('pretrained.patch_embed.proj.bias')
        w['cls'] = vec('pretrained.cls_token')
        self._pos_embed = vec('pretrained.pos_embed').view_as(sd['pretrained.pos_embed']) if self.POS_EMBED else None
        blocks = []
        for i in range(cfg['depth']):
            p = f'pretrained.blocks.{i}.'
            blocks.append(dict(
                ln1_w=vec(p + 'norm1.weight'), ln1_b=vec(p + 'norm1.bias'),
                qkv_w=mat(p + 'attn.qkv.weight'), qkv_b=vec(p + 'attn.qkv.bias'),
                proj_w=mat(p + 'attn.proj.weight'), proj_b=vec(p + 'attn.proj.bias'), ls1=vec(p + 'ls1.gamma'),
                ln2_w=vec(p + 'norm2.weight'), ln2_b=vec(p + 'norm2.bias'),
                fc1_w=mat(p + 'mlp.fc1.weight'), fc1_b=vec(p + 'mlp.fc1.bias'),
                fc2_w=mat(p + 'mlp.fc2.weight'), fc2_b=vec(p + 'mlp.fc2.bias'), ls2=vec(p + 'ls2.gamma')))
        w['blocks'] = blocks
        if not self.NEEDS_READOUT:
            w['norm_w'], w['norm_b'] = vec('pretrained.norm.weight'), vec('pretrained.norm.bias')
        # ---- DPT head; channel counts padded to multiples of 64 with zero weights (ViT-S/B have 48/96-wide maps) ----
        self.ocp = [_ru(c, 64) for c in oc]
        self.Fp = _ru(Fch, 64)
        self.F2p = _ru(Fch // 2, 64)
        h = 'depth_head.'
        for i in range(4):
            w[f'proj{i}_w'], w[f'proj{i}_b'] = mat(h + f'projects.{i}.weight', self.ocp[i]), vec(h + f'projects.{i}.bias', self.ocp[i])
        for i, s in ((0, 4), (1, 2)):  # ConvTranspose2d(k = s): W[(i,j,co), ci] = w[ci, co, i, j]
            wt = key(h + f'resize_layers.{i}.weight')  # [ci, co, s, s]
            t = torch.zeros(s, s, self.ocp[i], self.ocp[i], dtype=wdt, device=dev)
            t[:, :, :oc[i], :oc[i]] = wt.permute(2, 3, 1, 0).to(wdt)
            w[f'up{i}_w'] = op(t.reshape(s * s * self.ocp[i], self.ocp[i]).contiguous())
            w[f'up{i}_b'] = vec(h + f'resize_layers.{i}.bias', self.ocp[i]).repeat(s * s).contiguous()
        w['down3_w'] = conv_w(h + 'resize_layers.3.weight', self.ocp[3], self.ocp[3])
        w['down3_b'] = vec(h + 'resize_layers.3.bias', self.ocp[3])
        for i in range(4):
            w[f'rn{i}_w'] = conv_w(h + f'scratch.layer{i + 1}_rn.weight', self.ocp[i], self.Fp)
        for i in range(1, 5):
            r = h + f'scratch.refinenet{i}.'
            w[f'rf{i}_out_w'] = mat(r + 'out_conv.weight', self.Fp, self.Fp)
            w[f'rf{i}_out_b'] = vec(r + 'out_conv.bias', self.Fp)
            for u in (1, 2):
                for cv in (1, 2):
                    k = r + f'resConfUnit{u}.conv{cv}.'
                    if k + 'weight' in sd:
                        w[f'rf{i}_u{u}c{cv}_w'], w[f'rf{i}_u{u}c{cv}_b'] = conv_w(k + 'weight', self.Fp, self.Fp), vec(k + 'bias', self.Fp)
        w['oc1_w'], w['oc1_b'] = conv_w(h + 'scratch.output_conv1.weight', self.Fp, self.F2p), vec(h + 'scratch.output_conv1.bias', self.F2p)
        w['oc2_w'], w['oc2_b'] = conv_w(h + 'scratch.output_conv2.0.weight', self.F2p, 32), vec(h + 'scratch.output_conv2.0.bias')
        w['oc3_w'] = vec(h + 'scratch.output_conv2.2.weight')
        self.oc3_b = float(sd[h + 'scratch.output_conv2.2.bias'].detach().float().reshape(-1)[0])
        self.w = w

    POS_EMBED = "dm_dinov2_pos_embed"    # interpolate_pos_encoding (dinov2.py:179-210); identity for the native 37x37 grid

    def _pos(self, gh, gw):
        """the position embedding resized to a gh x gw grid by the host routine POS_EMBED.  Setup-time, cached."""
        import torch
        key = (gh, gw)
        if key not in self._pos_cache:
            pe = self._pos_embed
            C = pe.shape[-1]
            N = pe.shape[1] - 1
            n = int(round(math.sqrt(N)))
            # host arithmetic in float32 and torch's operation order (csrc/pos_tables.cu)
            src = np.ascontiguousarray(pe.reshape(N + 1, C).cpu().numpy(), dtype=np.float32)
            dst = np.empty((gh * gw + 1, C), dtype=np.float32)
            _lib.check(getattr(self.ops.L, self.POS_EMBED)(src.ctypes.data, n, C, gh, gw, dst.ctypes.data), self.POS_EMBED)
            self._pos_cache[key] = torch.from_numpy(dst).to(self.device)
        return self._pos_cache[key]

    # ---- activation buffers ----------------------------------------------------------------------------------------
    def _buffers(self, B, nh, nw):
        import torch
        key = (B, nh, nw)
        if self._buf_key == key:
            return self._bufs
        # the graphs read and write the buffers about to be freed.  Their key is the buffers' key, so at most one shape has
        # graphs at a time; the resolution tables they read (_pos, rel_tables) are only evicted when a new resolution arrives,
        # which always lands here first.
        self._graphs.clear()
        self._bufs = {}
        self._buf_key = None
        dev = self.device
        C, Fp = self.cfg['embed_dim'], self.Fp
        gh, gw = nh // self.PATCH, nw // self.PATCH
        Np, N = gh * gw, gh * gw + 1
        # split: every fp16 activation is a split tensor of 3x the width; the patch embedding is fp32 (the token assembly adds
        # the class token and position embedding to it in fp32)
        wide = 3 if self.split else 1
        h16 = lambda *s: torch.empty(*s[:-1], wide * s[-1], dtype=torch.float16, device=dev)
        b = {}
        b['patches'] = h16(B * Np, self.kpad)
        b['pe'] = torch.empty(B * Np, C, dtype=torch.float32, device=dev) if wide == 3 else h16(B * Np, C)
        b['x'] = torch.empty(B * N, C, dtype=torch.float32, device=dev)
        b['h'] = h16(B * N, C)
        b['qkv'] = h16(B * N, 3 * C)
        b['att'] = h16(B * N, C)
        b['mlp'] = h16(B * N, 4 * C)
        b['feat'] = [h16(B * Np, C) for _ in range(4)]
        b['cat'] = h16(B * Np, 2 * C) if self.NEEDS_READOUT else None
        sizes = [(gh * 4, gw * 4), (gh * 2, gw * 2), (gh, gw), ((gh - 1) // 2 + 1, (gw - 1) // 2 + 1)]
        b['sizes'] = sizes
        b['p'] = [h16(B * Np, self.ocp[i]) for i in range(4)]
        b['r'] = [h16(B, sizes[0][0], sizes[0][1], self.ocp[0]), h16(B, sizes[1][0], sizes[1][1], self.ocp[1]), None,
                  h16(B, sizes[3][0], sizes[3][1], self.ocp[3])]
        b['cols3'] = h16(B * sizes[3][0] * sizes[3][1], 9 * self.ocp[3])
        b['l'] = [h16(B, s[0], s[1], Fp) for s in sizes]
        b['lr'] = [h16(B, s[0], s[1], Fp) for s in sizes]
        for i in range(4):
            s = sizes[i]
            b[f't{i}'] = h16(B, s[0], s[1], Fp)      # relu(conv1(.)) scratch
            b[f'o{i}'] = h16(B, s[0], s[1], Fp)      # fused sum
            b[f'or{i}'] = h16(B, s[0], s[1], Fp)     # relu copy
            b[f'u{i}'] = h16(B, s[0], s[1], Fp)      # RCU2 output
        up = [sizes[2], sizes[1], sizes[0], (sizes[0][0] * 2, sizes[0][1] * 2)]  # target size of refinenet4..1
        b['up_sizes'] = up
        b['v'] = [h16(B, s[0], s[1], Fp) for s in (sizes[3], sizes[2], sizes[1], sizes[0])]   # out_conv output, before the up-sample
        b['path'] = [h16(B, s[0], s[1], Fp) for s in up]   # refinenet output (up-sampled)
        b['oc1'] = h16(B, up[3][0], up[3][1], self.F2p)
        b['oc1u'] = h16(B, nh, nw, self.F2p)
        b['d'] = torch.empty(B, nh, nw, dtype=torch.float32, device=dev)
        # circular padding: the halo copy of a 3x3 convolution's input, sized for the largest one
        convs = [(s, c) for s, c in zip(sizes, self.ocp)] + [(s, Fp) for s in sizes] + [(up[3], Fp), ((nh, nw), self.F2p)]
        b['halo'] = h16(max(B * (h + 2) * (w + 2) * c for (h, w), c in convs)) if self.circular else None
        self._head_buffers(b, B, nh, nw)
        self._bufs, self._buf_key = b, key
        return b

    def _head_buffers(self, b, B, nh, nw):
        """hook: a head's own buffers, added to `b` (kept and replaced with the rest)"""

    # ---- model-family hooks ------------------------------------------------------------------------------------------
    def net_size(self, W, H, net_w, net_h):
        return dav2_net_size(W, H, net_w)  # estimatedepthanything_v2 passes w as input_size (:552)

    def attention(self, i, b, B, N, heads, C, gh, gw):
        if self.split:
            self.ops.call("dm_attention_split", b['qkv'], B, N, heads, (C // heads) ** -0.5, b['att'])
            return
        self.ops.call("dm_attention_f16", b['qkv'], B, N, heads, (C // heads) ** -0.5, None, 0, b['att'])

    def emit_feature(self, b, fi, B, N, C):
        """get_intermediate_layers(norm=True) without the class token (dinov2.py:297-321)."""
        self.ops.call(self._ln, b['x'], B * N, C, self.w['norm_w'], self.w['norm_b'], 1e-6, b['feat'][fi], N, 1)

    # ---- kernel calls of the two paths (split: the same layer on split operands, see split_weight) -----------------------
    @property
    def _ln(self):
        return "dm_layernorm_split" if self.split else "dm_layernorm_f16"

    @property
    def _resize(self):
        return "dm_resize_bilinear_nhwc_split" if self.split else "dm_resize_bilinear_nhwc_f16"

    def _gemm(self, A, lda, W, ldw, M, N, K, **kw):
        """ops.gemm, or its split form: depths and pitches of the split operands are 3x the logical ones (ldx is fp32's)"""
        if not self.split:
            return self.ops.gemm(A, lda, W, ldw, M, N, K, **kw)
        if 'ldc' in kw:
            kw['ldc'] *= 3
        self.ops.gemm_split(A, 3 * lda, W.t, 3 * ldw, W.scale, M, N, 3 * K, **kw)

    def _conv(self, x, B, H, W_, Cin, Wt, Cout, **kw):
        if not self.split:
            return self.ops.conv3x3(x, B, H, W_, Cin, Wt, Cout, **kw)
        self.ops.conv3x3_split(x, B, H, W_, Cin, Wt.t, Wt.scale, Cout, **kw)

    # ---- forward ---------------------------------------------------------------------------------------------------
    def forward_batch(self, rgb, net_w, net_h=None, out_hw=None):
        """rgb: uint8 CUDA [B,H,W,3] -> float32 CUDA [B,H,W] raw prediction (what the reference's estimate* returns)."""
        import torch
        B, H, W, _ = rgb.shape
        nw, nh = self.net_size(W, H, net_w, net_h if net_h is not None else net_w)
        P_ = self.PATCH
        b = self._buffers(B, nh, nw)
        # image2tensor; the kernel zero-fills the patch matrix's K padding first, if it has any
        self.ops.call("dm_preprocess_patchify_split" if self.split else "dm_preprocess_patchify", rgb, B, H, W, nh, nw, P_,
                      (ctypes.c_float * 3)(*self.MEAN), (ctypes.c_float * 3)(*self.STD), (ctypes.c_int * 3)(*self.CHAN_MAP), b['patches'],
                      self.kpad, launches=1 + (self.kpad > 3 * P_ * P_))
        d = self._graphs.run((B, nh, nw), lambda: self._network(b, B, nh, nw))
        oh, ow = out_hw if out_hw is not None else (H, W)
        out = torch.empty(B, oh, ow, dtype=torch.float32, device=self.device)
        self.ops.call("dm_resize_f32", d, B, nh, nw, out, oh, ow, self.FINAL_RESIZE_MODE)
        return out

    def forward_ragged(self, packed, desc, net_w, net_h=None):
        """Ragged batch: uint8 CUDA images packed back to back (desc: their _lib.Ragged, unit 3) that share one net size -> fp32 CUDA
        predictions packed the same way (_lib.Ragged(desc.sizes, 1)).  Image i's prediction equals forward_batch of that image alone:
        only the pre-processing and the final resize see the image sizes, and the network runs under the uniform batch's graph key."""
        nw, nh = _ragged_net_size(self, desc, net_w, net_h)
        B, P_ = desc.B, self.PATCH
        b = self._buffers(B, nh, nw)
        self.ops.call("dm_preprocess_patchify_ragged", *desc.args(packed), nh, nw, P_, (ctypes.c_float * 3)(*self.MEAN),
                      (ctypes.c_float * 3)(*self.STD), (ctypes.c_int * 3)(*self.CHAN_MAP), int(self.split), b['patches'], self.kpad,
                      launches=1 + (self.kpad > 3 * P_ * P_))
        d = self._graphs.run((B, nh, nw), lambda: self._network(b, B, nh, nw))
        return _resize_ragged(self, d, B, nh, nw, desc, self.FINAL_RESIZE_MODE)

    def _network(self, b, B, nh, nw):
        """patch matrix in b['patches'] -> the net-size prediction b['d']"""
        self.run_network(b, B, nh, nw)
        return self.run_head(b, B, nh, nw)

    def run_network(self, b, B, nh, nw):
        """patch embedding -> transformer blocks -> reassemble -> fusion blocks; leaves refinenet1's output in b['path'][3]
        (and layer4_rn / refinenet4..2 in b['l'][3] / b['path'][0..2], which the ZoeDepth head reads)."""
        ops, w, cfg = self.ops, self.w, self.cfg
        C, heads, Fp = cfg['embed_dim'], cfg['heads'], self.Fp
        P_ = self.PATCH
        gh, gw = nh // P_, nw // P_
        Np, N = gh * gw, gh * gw + 1
        # patch embedding + tokens
        if self.split:
            self._gemm(b['patches'], self.kpad, w['pe_w'], self.kpad, B * Np, C, self.kpad, epi=_lib.EPI_STORE_F32, bias=w['pe_b'], X=b['pe'], ldx=C)
        else:
            ops.gemm(b['patches'], self.kpad, w['pe_w'], self.kpad, B * Np, C, self.kpad, bias=w['pe_b'], C=b['pe'], ldc=C)
        ops.call("dm_assemble_tokens_f32" if self.split else "dm_assemble_tokens", b['pe'], w['cls'],
                 self._pos(gh, gw) if self.POS_EMBED else None, b['x'], B, Np, C)
        rows = B * N
        fi = 0
        for i, blk in enumerate(w['blocks']):
            ops.call(self._ln, b['x'], rows, C, blk['ln1_w'], blk['ln1_b'], 1e-6, b['h'], 1, 0)
            self._gemm(b['h'], C, blk['qkv_w'], C, rows, 3 * C, C, bias=blk['qkv_b'], C=b['qkv'], ldc=3 * C)
            self.attention(i, b, B, N, heads, C, gh, gw)
            self._gemm(b['att'], C, blk['proj_w'], C, rows, C, C, epi=_lib.EPI_RESID_F32, bias=blk['proj_b'], X=b['x'], ldx=C, gamma=blk['ls1'])
            ops.call(self._ln, b['x'], rows, C, blk['ln2_w'], blk['ln2_b'], 1e-6, b['h'], 1, 0)
            self._gemm(b['h'], C, blk['fc1_w'], C, rows, 4 * C, C, act=_lib.ACT_GELU, bias=blk['fc1_b'], C=b['mlp'], ldc=4 * C)
            self._gemm(b['mlp'], 4 * C, blk['fc2_w'], 4 * C, rows, C, 4 * C, epi=_lib.EPI_RESID_F32, bias=blk['fc2_b'], X=b['x'], ldx=C, gamma=blk['ls2'])
            if i in cfg['layers']:
                self.emit_feature(b, fi, B, N, C)
                fi += 1
        # ---- DPT head (dpt.py:117-150) ----
        sizes = b['sizes']
        for i in range(4):
            self._gemm(b['feat'][i], C, w[f'proj{i}_w'], C, B * Np, self.ocp[i], C, bias=w[f'proj{i}_b'], C=b['p'][i], ldc=self.ocp[i])
        self._gemm(b['p'][0], self.ocp[0], w['up0_w'], self.ocp[0], B * Np, 16 * self.ocp[0], self.ocp[0], epi=_lib.EPI_PIXSHUF, bias=w['up0_b'],
                   C=b['r'][0], ps=(4, self.ocp[0], gh, gw))
        self._gemm(b['p'][1], self.ocp[1], w['up1_w'], self.ocp[1], B * Np, 4 * self.ocp[1], self.ocp[1], epi=_lib.EPI_PIXSHUF, bias=w['up1_b'],
                   C=b['r'][1], ps=(2, self.ocp[1], gh, gw))
        r2 = b['p'][2]
        # the im2col is channel-agnostic: on a split tensor it gathers 3x the channels, which down3_w's per-tap split layout matches
        ops.call("dm_im2col_s2_circular_f16" if self.circular else "dm_im2col_s2_f16", b['p'][3], B, gh, gw,
                 self.ocp[3] * (3 if self.split else 1), b['cols3'])
        self._gemm(b['cols3'], 9 * self.ocp[3], w['down3_w'], 9 * self.ocp[3], B * sizes[3][0] * sizes[3][1], self.ocp[3], 9 * self.ocp[3],
                   bias=w['down3_b'], C=b['r'][3], ldc=self.ocp[3])
        rs = [b['r'][0], b['r'][1], r2, b['r'][3]]
        for i in range(4):  # layer{i}_rn (no bias) -> l_i and relu(l_i)
            self._conv(rs[i], B, sizes[i][0], sizes[i][1], self.ocp[i], w[f'rn{i}_w'], Fp, C=b['l'][i], C2=b['lr'][i], halo=b['halo'])
        # refinenet4: resConfUnit2(l4) -> resize -> out_conv.  The 1x1 out_conv (+ bias) commutes with the bilinear
        # interpolation (a per-pixel channel mix against per-channel spatial weights that sum to one), so it runs BEFORE the
        # up-sample: a quarter of the MACs and no full-resolution intermediate (dmidas/blocks.py:425-437 has it after).
        s3 = sizes[3]
        self._conv(b['lr'][3], B, s3[0], s3[1], Fp, w['rf4_u2c1_w'], Fp, act=_lib.ACT_RELU, bias=w['rf4_u2c1_b'], C=b['t3'], halo=b['halo'])
        self._conv(b['t3'], B, s3[0], s3[1], Fp, w['rf4_u2c2_w'], Fp, bias=w['rf4_u2c2_b'], C=b['u3'], R=b['l'][3], halo=b['halo'])
        up = b['up_sizes']
        self._gemm(b['u3'], Fp, w['rf4_out_w'], Fp, B * s3[0] * s3[1], Fp, Fp, bias=w['rf4_out_b'], C=b['v'][0], ldc=Fp)
        ops.call(self._resize, b['v'][0], B, s3[0], s3[1], Fp, b['path'][0], up[0][0], up[0][1])
        # refinenet3, 2, 1: output = path + RCU1(l_i); output = RCU2(output); out_conv; resize (commuted, see above)
        for step, (li, rf) in enumerate(((2, 3), (1, 2), (0, 1))):
            s = sizes[li]
            path = b['path'][step]
            self._conv(b['lr'][li], B, s[0], s[1], Fp, w[f'rf{rf}_u1c1_w'], Fp, act=_lib.ACT_RELU, bias=w[f'rf{rf}_u1c1_b'], C=b[f't{li}'],
                        halo=b['halo'])
            self._conv(b[f't{li}'], B, s[0], s[1], Fp, w[f'rf{rf}_u1c2_w'], Fp, bias=w[f'rf{rf}_u1c2_b'], C=b[f'o{li}'], C2=b[f'or{li}'],
                        R=b['l'][li], R2=path, halo=b['halo'])
            self._conv(b[f'or{li}'], B, s[0], s[1], Fp, w[f'rf{rf}_u2c1_w'], Fp, act=_lib.ACT_RELU, bias=w[f'rf{rf}_u2c1_b'], C=b[f't{li}'],
                        halo=b['halo'])
            self._conv(b[f't{li}'], B, s[0], s[1], Fp, w[f'rf{rf}_u2c2_w'], Fp, bias=w[f'rf{rf}_u2c2_b'], C=b[f'u{li}'], R=b[f'o{li}'], halo=b['halo'])
            t = up[step + 1]
            self._gemm(b[f'u{li}'], Fp, w[f'rf{rf}_out_w'], Fp, B * s[0] * s[1], Fp, Fp, bias=w[f'rf{rf}_out_b'], C=b['v'][step + 1], ldc=Fp)
            ops.call(self._resize, b['v'][step + 1], B, s[0], s[1], Fp, b['path'][step + 1], t[0], t[1])

    def run_output_conv1(self, b, B, nh, nw):
        """output_conv's first 3x3 conv (dpt.py:139-150 / dpt_depth.py:150-158) and the resize to the net size -> b['oc1u']"""
        t = b['up_sizes'][3]
        self._conv(b['path'][3], B, t[0], t[1], self.Fp, self.w['oc1_w'], self.F2p, bias=self.w['oc1_b'], C=b['oc1'], halo=b['halo'])
        self.ops.call(self._resize, b['oc1'], B, t[0], t[1], self.F2p, b['oc1u'], nh, nw)

    def run_head(self, b, B, nh, nw):
        """output_conv -> the net-size prediction [B, nh, nw] (a pooled buffer, valid until the next forward at this shape)."""
        w = self.w
        self.run_output_conv1(b, B, nh, nw)
        # conv3x3 -> ReLU -> conv1x1 -> ReLU (+ the outer F.relu, idempotent) fused into one epilogue
        self._conv(b['oc1u'], B, nh, nw, self.F2p, w['oc2_w'], 32, epi=_lib.EPI_HEAD, act=_lib.ACT_RELU, bias=w['oc2_b'], X=b['d'],
                    gamma=w['oc3_w'], head_b2=self.oc3_b, halo=b['halo'])
        return b['d']

    def to(self, device):
        return self

BEIT_CONFIGS = {
    'beitl16_512': dict(embed_dim=1024, depth=24, heads=16, features=256, out_channels=[256, 512, 1024, 1024],
                        layers=[5, 11, 17, 23], window=32),
    'beitl16_384': dict(embed_dim=1024, depth=24, heads=16, features=256, out_channels=[256, 512, 1024, 1024],
                        layers=[5, 11, 17, 23], window=24),
    'beit_tiny': dict(embed_dim=128, depth=4, heads=2, features=64, out_channels=[64, 64, 128, 128],
                      layers=[0, 1, 2, 3], window=4),  # structural test configuration
}


def midas_net_size(width, height, net_w, net_h, multiple_of=32):
    """Resize(keep_aspect_ratio, 'minimal', multiple of 32) of the reference (dmidas/transforms.py:61-104)."""
    sh, sw = net_h / height, net_w / width
    if abs(1 - sw) < abs(1 - sh):
        sh = sw
    else:
        sw = sh
    return _constrain_to_multiple_of(sw * width, multiple_of), _constrain_to_multiple_of(sh * height, multiple_of)


def midas_upper_bound_net_size(width, height, net_w, net_h, multiple_of=32):
    """Resize(net_w, net_h, keep_aspect_ratio, 'upper_bound', multiple of 32) (dmidas/transforms.py:94-160): scale by the smaller of
    the two ratios, so the net fits inside net_w x net_h with the image's aspect; a side that rounds past its bound is floored
    instead, and may become 0 for a very elongated image."""
    sh, sw = net_h / height, net_w / width
    if sw < sh:
        sh = sw
    else:
        sw = sh
    return (_constrain_to_multiple_of(sw * width, multiple_of, max_val=net_w),
            _constrain_to_multiple_of(sh * height, multiple_of, max_val=net_h))


def midas_boost_net_size(width, height, msize, multiple_of=32):
    """Resize(msize, msize, keep_aspect_ratio, 'upper_bound', multiple of 32) of estimatemidasBoost (src/depthmap_generation.py:1183-1192):
    the largest net inside msize x msize with the crop's aspect."""
    return midas_upper_bound_net_size(width, height, msize, msize, multiple_of)


def _check_rects(rects, hi, wi):
    """BOOST's crops (x0, y0, w, h) must lie inside the wi x hi image"""
    for x0, y0, w, h in rects:
        if x0 < 0 or y0 < 0 or w <= 0 or h <= 0 or x0 + w > wi or y0 + h > hi:
            raise ValueError(f"crop {(x0, y0, w, h)} outside the {wi}x{hi} image")


def _check_planar(planar):
    """BOOST's planar image: a contiguous fp32 [3, Hi, Wi] tensor -> (Hi, Wi)"""
    import torch
    if planar.dtype != torch.float32 or planar.dim() != 3 or planar.shape[0] != 3 or not planar.is_contiguous():
        raise ValueError("planar must be a contiguous float32 tensor [3, H, W]")
    return int(planar.shape[1]), int(planar.shape[2])


def _midas_crop_groups(planar, rects, msize):
    """estimatemidasBoost's crops (x0, y0, w, h) of one planar fp32 image [3, Hi, Wi] -> (Hi, Wi, {(nh, nw): [crop indices]}): each
    crop at its upper-bound net size for msize.  Crops clipped at the image border are not square, hence the grouping."""
    hi, wi = _check_planar(planar)
    _check_rects(rects, hi, wi)
    groups = {}
    for k, (x0, y0, w, h) in enumerate(rects):
        nw, nh = midas_boost_net_size(w, h, msize)
        if nw <= 0 or nh <= 0:
            raise ValueError(f"crop {w}x{h} is too elongated for a net of at most {msize} px")
        groups.setdefault((nh, nw), []).append(k)
    return hi, wi, groups


class _MidasBoost:
    """BOOST on a MiDaS network (estimatemidasBoost, src/depthmap_generation.py:1180-1220): forward_batch(None, msize, msize,
    planar=(img, rect)) -> _forward_crop, and forward_crops(img, rects, msize), on float crops of a planar fp32 image: upper-bound net
    size (midas_boost_net_size), ImageNet mean / std, the channel order of the crop unchanged (network channel c = plane 2 - c of
    the RGB image), and a cv2 INTER_CUBIC resize of the prediction back to the crop.  The engine supplies _crops_network."""

    BOOST_MEAN = (0.485, 0.456, 0.406)
    BOOST_STD = (0.229, 0.224, 0.225)

    def _boost_consts(self):
        return (ctypes.c_float * 3)(*self.BOOST_MEAN), (ctypes.c_float * 3)(*self.BOOST_STD), (ctypes.c_int * 3)(*self.CHAN_MAP)

    def _forward_crop(self, planar, rect, msize):
        """estimatemidasBoost's network and resize on one crop -> [1, h, w] (not normalised)"""
        return self.forward_crops(planar, [rect], msize)[0].unsqueeze(0)

    def forward_crops(self, planar, rects, msize):
        """B crops (x0, y0, w, h) of one planar fp32 image [3, Hi, Wi] -> [fp32 CUDA [h, w]] in the order of `rects`: each crop at its
        upper-bound net size for msize, then cv2-cubic back to the crop.  Crops clipped at the image border are not square, so the
        crops are grouped by net shape, one batched forward per shape."""
        import torch
        hi, wi, groups = _midas_crop_groups(planar, rects, msize)
        out = [None] * len(rects)
        for (nh, nw), ks in groups.items():
            r = torch.tensor([[int(v) for v in rects[k]] for k in ks], dtype=torch.int32).to(self.device)
            d = self._crops_network(planar, hi, wi, r, len(ks), nh, nw)
            for i, k in enumerate(ks):
                w, h = int(rects[k][2]), int(rects[k][3])
                o = torch.empty(h, w, dtype=torch.float32, device=self.device)
                self.ops.call("dm_boost_resize_cubic", d[i], nw, 0, nh, nw, o, w, 0, h, w, 1)
                out[k] = o
        return out


class _MidasDptEngine(_MidasBoost, DepthAnythingV2Engine):
    """What the MiDaS DPT networks (DptBeitEngine, DptVitEngine) share on the Depth-Anything-V2 engine: the checkpoint layout
    (trunk under 'pretrained.model.', decoder under 'scratch.'), the readout projection of the reassemble stage, DPT /
    DPTDepthModel (dmidas/dpt_depth.py:31-166), estimatemidas' pre-processing and bicubic resize back (src/depthmap_generation.py:
    455-499), and BOOST (_MidasBoost)."""

    PATCH = 16
    MEAN = (0.5, 0.5, 0.5)
    STD = (0.5, 0.5, 0.5)
    SUPPORTS_SPLIT = False
    CHAN_MAP = (2, 1, 0)        # estimatemidas receives the BGR-swapped image of get_raw_prediction (:381) unchanged
    FINAL_RESIZE_MODE = 1       # bicubic, align_corners=False (:487-497)
    NEEDS_READOUT = True

    def net_size(self, W, H, net_w, net_h):
        return midas_net_size(W, H, net_w, net_h)

    def _block_keys(self, sd, blk):
        """hook: the full qkv bias and the LayerScale gammas of the block with checkpoint prefix `blk`, under Depth-Anything-V2's keys"""
        raise NotImplementedError

    def _pack(self, sd):
        """the MiDaS checkpoint mapped to the layout of DepthAnythingV2Engine._pack, plus the readout projections"""
        p = 'pretrained.model.'
        m = {'pretrained.' + k: sd[p + k] for k in ('patch_embed.proj.weight', 'patch_embed.proj.bias', 'cls_token')}
        if self.POS_EMBED:
            m['pretrained.pos_embed'] = sd[p + 'pos_embed']
        for i in range(self.cfg['depth']):
            b, d = p + f'blocks.{i}.', f'pretrained.blocks.{i}.'
            for k in ('norm1.weight', 'norm1.bias', 'attn.qkv.weight', 'attn.proj.weight', 'attn.proj.bias', 'norm2.weight', 'norm2.bias',
                      'mlp.fc1.weight', 'mlp.fc1.bias', 'mlp.fc2.weight', 'mlp.fc2.bias'):
                m[d + k] = sd[b + k]
            m.update({d + k: v for k, v in self._block_keys(sd, b).items()})
        for j in range(4):
            a = f'pretrained.act_postprocess{j + 1}.'
            m[f'depth_head.projects.{j}.weight'] = sd[a + '3.weight']
            m[f'depth_head.projects.{j}.bias'] = sd[a + '3.bias']
        for j in (0, 1, 3):
            a = f'pretrained.act_postprocess{j + 1}.4.'
            m[f'depth_head.resize_layers.{j}.weight'] = sd[a + 'weight']
            m[f'depth_head.resize_layers.{j}.bias'] = sd[a + 'bias']
        for k, v in sd.items():
            if k.startswith('scratch.layer') or k.startswith('scratch.refinenet'):
                m['depth_head.' + k] = v
        for d, k in (('output_conv1', 'output_conv.0'), ('output_conv2.0', 'output_conv.2'), ('output_conv2.2', 'output_conv.4')):
            m[f'depth_head.scratch.{d}.weight'] = sd[f'scratch.{k}.weight']
            m[f'depth_head.scratch.{d}.bias'] = sd[f'scratch.{k}.bias']
        super()._pack(m)
        key = lambda k: sd[f'pretrained.act_postprocess{k}'].detach().to(self.device)
        self.w['readout'] = [(_mat(key(f'{j + 1}.0.project.0.weight')), _vec(key(f'{j + 1}.0.project.0.bias'))) for j in range(4)]

    def emit_feature(self, b, fi, B, N, C):
        """forward hook on the raw block output + ProjectReadout: GELU(Linear(cat(tokens, cls)))."""
        rw, rb = self.w['readout'][fi]
        self.ops.call("dm_concat_readout_f16", b['x'], B, N, C, b['cat'])
        self.ops.gemm(b['cat'], 2 * C, rw, 2 * C, B * (N - 1), C, 2 * C, act=_lib.ACT_GELU, bias=rb, C=b['feat'][fi], ldc=C)

    # ---- BOOST: estimatemidasBoost on float crops ---------------------------------------------------------------------
    def forward_batch(self, rgb, net_w, net_h=None, out_hw=None, planar=None):
        """rgb: uint8 CUDA [B,H,W,3] -> float32 CUDA [B,H,W] (estimatemidas).  planar = (fp32 CUDA [3,Hi,Wi] image, (x0, y0, w, h))
        instead of `rgb`: _forward_crop with msize = net_w."""
        if planar is not None:
            return self._forward_crop(*planar, net_w)
        return super().forward_batch(rgb, net_w, net_h, out_hw)

    def _crops_network(self, planar, hi, wi, r, B, nh, nw):
        # eager: BOOST alternates crop net sizes, and a new shape drops the graphs (_buffers), so a capture would not replay
        b = self._buffers(B, nh, nw)
        self.ops.call("dm_preprocess_patchify_f32_crops", planar, hi, wi, r, B, nh, nw, self.PATCH, *self._boost_consts(), b['patches'],
                      self.kpad, launches=1 + (self.kpad > 3 * self.PATCH ** 2))
        return self._network(b, B, nh, nw)


class DptBeitEngine(_MidasDptEngine):
    """MiDaS 3.1 DPT-BEiT (dpt_beit_large_512 / _384) on the sm_90a kernels.

    Mirrors the reference's overriding forwards (dmidas/backbones/beit.py:18-129), the reassemble stage
    (dmidas/backbones/utils.py:28-39,83-124,144-249), DPT / DPTDepthModel (dmidas/dpt_depth.py:110-166) and estimatemidas
    (src/depthmap_generation.py:455-499).  No absolute position embedding (use_abs_pos_emb=False).  The relative-position bias,
    which the reference rebuilds (bilinear table resize + gather) in every block of every forward, is resized once per resolution
    into a per-head fp32 table per block; the fused attention kernel gathers from it (csrc/attention_wgmma.cu), so no
    [heads, N, N] tensor exists."""

    CONFIGS = BEIT_CONFIGS
    POS_EMBED = None

    def _block_keys(self, sd, blk):
        import torch
        qkv_b = torch.cat((sd[blk + 'attn.q_bias'].float(), torch.zeros(self.cfg['embed_dim']), sd[blk + 'attn.v_bias'].float()))  # no key bias
        return {'attn.qkv.bias': qkv_b, 'ls1.gamma': sd[blk + 'gamma_1'], 'ls2.gamma': sd[blk + 'gamma_2']}

    def _pack(self, sd):
        import torch
        super()._pack(sd)
        self._tables = [sd[f'pretrained.model.blocks.{i}.attn.relative_position_bias_table'].detach().to(self.device, torch.float32).contiguous()
                        for i in range(self.cfg['depth'])]
        self._bias_cache = {}

    TABLE_RESOLUTIONS = 4      # resized tables kept resident: BOOST alternates between its whole-image and patch windows

    def rel_tables(self, gh, gw):
        """Table half of _get_rel_pos_bias (dmidas/backbones/beit.py:29-50): per block, the [nrd, heads] table resized
        (bilinear) to the current window, laid out [heads, nrd] in fp32 and multiplied by log2(e).  Once per resolution.
        The gather half (:52-62, relative_position_index) happens inside the attention kernel."""
        import torch
        import torch.nn.functional as F
        key = (gh, gw)
        if key not in self._bias_cache:
            win = self.cfg['window']
            old_h = old_w = 2 * win - 1
            new_h, new_w = 2 * gh - 1, 2 * gw - 1
            out = []
            nrd_new = new_h * new_w + 3
            heads = self.cfg['heads']
            for t in self._tables:
                # host arithmetic in float32 and torch's operation order (csrc/pos_tables.cu)
                src = np.ascontiguousarray(t.cpu().numpy(), dtype=np.float32)
                dst = np.empty((heads, nrd_new), dtype=np.float32)
                _lib.check(self.ops.L.dm_beit_rel_table(src.ctypes.data, win, heads, gh, gw, dst.ctypes.data), "dm_beit_rel_table")
                out.append(torch.from_numpy(dst).to(self.device))
            while len(self._bias_cache) >= self.TABLE_RESOLUTIONS:
                self._bias_cache.pop(next(iter(self._bias_cache)))
            self._bias_cache[key] = (out, new_h * new_w + 3)
        return self._bias_cache[key]

    def attention(self, i, b, B, N, heads, C, gh, gw):
        tabs, nrd = self.rel_tables(gh, gw)
        self.ops.call("dm_attention_relpos_f16", b['qkv'], B, gh, gw, heads, (C // heads) ** -0.5, tabs[i], nrd, b['att'])


class DptVitEngine(_MidasDptEngine):
    """MiDaS 3.0 dpt_large_384 (model type 3) on the sm_90a kernels, op-level path: timm's vit_large_patch16_384 driven by
    the reference's forward_flex (dmidas/backbones/vit.py:12-79,107-118) — absolute position embedding resized bilinearly to
    the current grid, plain (un-biased) attention, no LayerScale — with the hooks, ProjectReadout, reassemble stage and DPT
    decoder it shares with the BEiT models (dmidas/dpt_depth.py:31-166)."""

    CONFIGS = {
        'vitl16_384': dict(embed_dim=1024, depth=24, heads=16, features=256, out_channels=[256, 512, 1024, 1024], layers=[5, 11, 17, 23], window=24),
        'vit_tiny': dict(embed_dim=128, depth=4, heads=2, features=64, out_channels=[64, 64, 128, 128], layers=[0, 1, 2, 3], window=4),
    }
    POS_EMBED = "dm_vit_pos_embed"      # _resize_pos_embed (vit.py:16-31)

    def _block_keys(self, sd, blk):
        import torch
        # no LayerScale: gammas of one, as the residual epilogue takes a gamma
        C = self.cfg['embed_dim']
        return {'attn.qkv.bias': sd[blk + 'attn.qkv.bias'], 'ls1.gamma': torch.ones(C), 'ls2.gamma': torch.ones(C)}


class _ResNeXtEngine:
    """The ResNeXt-101 32x8d encoder LeReS and MiDaS v2.1 share (torchvision's ResNet(Bottleneck, [3, 4, 23, 3], groups=32,
    width_per_group=8); lib/Resnext_torch.py:60-220), with the buffer pool and CUDA-graph cache of their op-level engines.
    NHWC fp16 activations, fp32 accumulation.  1x1 convolutions are GEMMs, 3x3 ones the implicit-GEMM conv; the 32-group 3x3
    convolutions use block-diagonal dense filters (exact: the extra products are zeros), the three stride-2 ones go through the
    strided im2col; BatchNorm (running statistics, eps 1e-5) is folded into filters and biases when the checkpoint is packed; the
    bottleneck's `relu(out + identity)` comes out of the GEMM epilogue's relu copy (C2).  circular=True: tiling mode, the stem and
    every 3x3 convolution pad circularly (the max-pool keeps its padding)."""

    LAYERS = (3, 4, 23, 3)
    GROUPS = 32
    MEAN = (0.485, 0.456, 0.406)
    STD = (0.229, 0.224, 0.225)
    GRAPH_ENV, NAME = None, None     # environment switch and name of the engine's CUDA-graph cache

    def __init__(self, state_dict, device, circular=False):
        self.device = device
        self.circular = circular
        self._cv = "_circular" if circular else ""      # entry-point suffix of the circular stem / im2col
        self.ops = _lib.Ops()
        self._bufs = {}
        # from the second call on at a given (B, net size) the ~500 launches of the network replay from a CUDA graph
        self._graphs = _lib.GraphCache(self.ops, self.GRAPH_ENV, self.NAME)
        self._pooled_bytes, self._pool_limit = 0, None
        self._pack(state_dict)

    # ---- weights -------------------------------------------------------------------------------------------------------
    def _fold(self, sd, conv, bn):
        """conv weight [Co, Ci/g, kh, kw] (+ optional bias) followed by BatchNorm (inference) -> (weight, bias) in fp32"""
        import torch
        w = sd[conv + '.weight'].detach().float()
        b = sd[conv + '.bias'].detach().float() if conv + '.bias' in sd else torch.zeros(w.shape[0])
        if bn is not None:
            scale = sd[bn + '.weight'].detach().float() / torch.sqrt(sd[bn + '.running_var'].detach().float() + 1e-5)
            w = w * scale.view(-1, 1, 1, 1)
            b = (b - sd[bn + '.running_mean'].detach().float()) * scale + sd[bn + '.bias'].detach().float()
        return w, b

    def _packed(self, sd, conv, bn, groups=1, npad=None):
        """_fold, then the kernels' layout on the device: a 1x1 conv as an fp16 [Co, Ci] matrix, a 3x3 one as an fp16 (ky, kx, ci)
        filter with its groups as diagonal blocks (exact: the extra products are zeros) and Co zero padded to npad; fp32 bias"""
        w, b = self._fold(sd, conv, bn)
        wt = _mat(w) if w.shape[-1] == 1 else _conv_w(w, cout_pad=npad, groups=groups)
        return wt.to(self.device), _vec(b, npad).to(self.device)

    def _pack_encoder(self, sd, stem_conv, stem_bn, block):
        """folded stem (fp16 [64, 192], K ordered (ky, kx, c)) and bottleneck weights; block(li, bi) is the checkpoint prefix of
        bottleneck bi of stage li"""
        sw, sb = self._fold(sd, stem_conv, stem_bn)               # [64, 3, 7, 7] -> [64, (ky, kx, c)] padded to 192
        stem = _mat(sw.permute(0, 2, 3, 1), cols=192).to(self.device), _vec(sb).to(self.device)
        blocks = []
        for li, nb in enumerate(self.LAYERS, start=1):
            for bi in range(nb):
                p = block(li, bi)
                blk = dict(stride=2 if (bi == 0 and li > 1) else 1)
                blk['c1'] = self._packed(sd, p + '.conv1', p + '.bn1')
                blk['c2'] = self._packed(sd, p + '.conv2', p + '.bn2', groups=self.GROUPS)
                blk['c3'] = self._packed(sd, p + '.conv3', p + '.bn3')
                blk['down'] = self._packed(sd, p + '.downsample.0', p + '.downsample.1') if bi == 0 else None
                blk['width'], blk['cout'] = blk['c1'][0].shape[0], blk['c3'][0].shape[0]
                blocks.append(blk)
        return stem, blocks

    # ---- buffers: a simple keyed pool (every tensor of a forward has its own name) ---------------------------------
    def _buf(self, name, shape, dtype=None):
        import torch
        dtype = dtype or torch.float16
        key = (name, tuple(shape), dtype)          # one set of buffers per net size: BOOST alternates 448 / 896 / whole-image nets, and the
        t = self._bufs.get(key)                    # captured graphs below need stable addresses
        if t is None:
            t = torch.empty(*shape, dtype=dtype, device=self.device)
            self._bufs[key] = t
            self._pooled_bytes += t.numel() * t.element_size()
        return t

    def _trim_pools(self):
        """Called at the start of a forward, never inside one: BOOST's whole-image net size depends on the image, so a long run would
        otherwise collect one buffer set (and one graph) per size.  Past half of the device memory everything pooled is dropped and
        rebuilt lazily."""
        import torch
        if self._pool_limit is None:
            self._pool_limit = torch.cuda.get_device_properties(self.device).total_memory // 2
        if self._pooled_bytes > self._pool_limit and not torch.cuda.is_current_stream_capturing():
            torch.cuda.synchronize(self.device)
            self._graphs.clear()
            self._bufs.clear()
            self._pooled_bytes = 0
            torch.cuda.empty_cache()

    def _network(self, B, net_h, net_w, cols):
        """stem GEMM .. decoder output [B, net_h, net_w] fp32 (a pooled buffer)"""
        return self._graphs.run((B, net_h, net_w), lambda: self._network_eager(B, net_h, net_w, cols))

    def _encoder(self, B, net_h, net_w, cols, halo):
        """stem GEMM (folded BN + ReLU) on the stem's im2col `cols`, max-pool, the 33 bottlenecks -> [(feature, h, w, channels)] after
        each stage (1/4 .. 1/32); `halo`: the circular-padding scratch, or None"""
        ops, w = self.ops, self.w
        h1, w1 = (net_h + 6 - 7) // 2 + 1, (net_w + 6 - 7) // 2 + 1
        x = self._buf('stem', (B, h1, w1, 64))
        ops.gemm(cols, 192, w['stem'][0], 192, B * h1 * w1, 64, 192, act=_lib.ACT_RELU, bias=w['stem'][1], C=x, ldc=64)
        h, wd = (h1 + 2 - 3) // 2 + 1, (w1 + 2 - 3) // 2 + 1
        xp = self._buf('pool', (B, h, wd, 64))
        ops.call("dm_maxpool3x3s2_nhwc_f16", x, B, h1, w1, 64, xp)
        x, cin = xp, 64
        feats = []
        bi_global = 0
        for li, nb in enumerate(self.LAYERS, start=1):
            for bi in range(nb):
                blk = w['blocks'][bi_global]
                tag = f"l{li}b{bi % 2}" if bi > 0 else f"l{li}first"
                width, cout, stride = blk['width'], blk['cout'], blk['stride']
                M = B * h * wd
                t1 = self._buf(tag + '_t1', (B, h, wd, width))
                ops.gemm(x, cin, blk['c1'][0], cin, M, width, cin, act=_lib.ACT_RELU, bias=blk['c1'][1], C=t1, ldc=width)
                if stride == 1:
                    ho, wo = h, wd
                    t2 = self._buf(tag + '_t2', (B, ho, wo, width))
                    ops.conv3x3(t1, B, h, wd, width, blk['c2'][0], width, act=_lib.ACT_RELU, bias=blk['c2'][1], C=t2, halo=halo)
                else:
                    ho, wo = (h + 2 - 3) // 2 + 1, (wd + 2 - 3) // 2 + 1
                    c2 = self._buf(tag + '_cols', (B * ho * wo, 9 * width))
                    ops.call("dm_im2col_s2_circular_f16" if self.circular else "dm_im2col_s2_f16", t1, B, h, wd, width, c2)
                    t2 = self._buf(tag + '_t2', (B, ho, wo, width))
                    ops.gemm(c2, 9 * width, blk['c2'][0], 9 * width, B * ho * wo, width, 9 * width, act=_lib.ACT_RELU, bias=blk['c2'][1], C=t2, ldc=width)
                Mo = B * ho * wo
                if blk['down'] is not None:
                    xs = x
                    if stride == 2:
                        xs = self._buf(tag + '_xs', (B, ho, wo, cin))
                        ops.call("dm_subsample2_nhwc_f16", x, B, h, wd, cin, xs)
                    idn = self._buf(tag + '_idn', (B, ho, wo, cout))
                    ops.gemm(xs, cin, blk['down'][0], cin, Mo, cout, cin, bias=blk['down'][1], C=idn, ldc=cout)
                else:
                    idn = x
                pre = self._buf(tag + '_pre', (B, ho, wo, cout))
                last = bi == nb - 1
                out = self._buf(f"feat{li}" if last else tag + '_out', (B, ho, wo, cout))
                ops.gemm(t2, width, blk['c3'][0], width, Mo, cout, width, bias=blk['c3'][1], C=pre, ldc=cout, C2=out, R=idn, ldr=cout)
                x, cin, h, wd = out, cout, ho, wo
                bi_global += 1
            feats.append((x, h, wd, cin))
        return feats

    def _stem_cols(self, B, net_h, net_w):
        """the im2col of the 7x7 / 2 stem conv, K = (ky, kx, c) padded to 192"""
        return self._buf('stem_cols', (B * ((net_h + 6 - 7) // 2 + 1) * ((net_w + 6 - 7) // 2 + 1), 192))

    # ---- decoder steps: each output is the pooled buffer `name` -------------------------------------------------------
    def _conv(self, B, halo, name, xin, hh, ww, ci, wb, co, act=_lib.ACT_NONE, R=None, R2=None, C2=False):
        """3x3 conv (+ bias, act, residuals R / R2) -> its output, or with C2 the epilogue's relu copy of it"""
        outp = self._buf(name, (B, hh, ww, co))
        out2 = self._buf(name + '_r', (B, hh, ww, co)) if C2 else None
        self.ops.conv3x3(xin, B, hh, ww, ci, wb[0], co, act=act, bias=wb[1], C=outp, C2=out2, R=R, R2=R2, halo=halo)
        return out2 if C2 else outp

    def _up2(self, B, name, xin, hh, ww, c):
        """x2 bilinear up-sample, align_corners=True"""
        outp = self._buf(name, (B, 2 * hh, 2 * ww, c))
        self.ops.call("dm_resize_bilinear_nhwc_f16", xin, B, hh, ww, c, outp, 2 * hh, 2 * ww)
        return outp

    def to(self, device):
        return self


class LeresEngine(_ResNeXtEngine):
    """LeReS / res101 (model type 0) on the sm_90a kernels: estimateleres (src/depthmap_generation.py:406-440) around
    RelDepthModel('resnext101') (lib/multi_depth_model_woauxi.py:6-32, lib/Resnext_torch.py:60-220, lib/network_auxi.py:15-215).
    The shared ResNeXt-101 encoder, then the FTB / FFM / AO decoder on the implicit-GEMM conv; FTB's `relu(x + branch)` comes out of
    the epilogue's relu copy (C2).  circular=True: tiling mode, the stem, every 3x3 convolution of the encoder and the decoder pad
    circularly."""

    ENC = "depth_model.encoder_modules.encoder."
    DEC = "depth_model.decoder_modules."
    GRAPH_ENV, NAME = "DEPTHMAP_B200_LERES_GRAPH", "LeReS"

    def _pack(self, sd):
        E, D = self.ENC, self.DEC
        w = {}
        w['stem'], w['blocks'] = self._pack_encoder(sd, E + 'conv1', E + 'bn1', lambda li, bi: f"{E}layer{li}.{bi}")

        def ftb(p):
            return dict(c1=self._packed(sd, p + '.conv1', None), b1=self._packed(sd, p + '.conv_branch.1', p + '.conv_branch.2'),
                        b4=self._packed(sd, p + '.conv_branch.4', None))
        w['conv'] = ftb(D + 'conv')
        w['conv1'] = self._packed(sd, D + 'conv1', None)
        for k in ('ffm2', 'ffm1', 'ffm0'):
            w[k] = (ftb(D + k + '.ftb1'), ftb(D + k + '.ftb2'))
        a = D + 'outconv.adapt_conv'
        w['ao0'] = self._packed(sd, a + '.0', a + '.1')
        w['ao3'] = self._packed(sd, a + '.3', None, npad=32)
        self.w = w

    # ---- forward ---------------------------------------------------------------------------------------------------
    def forward_batch(self, rgb, net_w, net_h=None, out_hw=None, planar=None):
        """rgb: uint8 CUDA [B,H,W,3] -> float32 CUDA [B,H,W] (what estimateleres returns; invert = True).
        planar = (fp32 CUDA [3,Hi,Wi] image in network channel order, (x0, y0, w, h)) instead of `rgb`: estimateleres on a float
        crop, as BOOST calls it (src/depthmap_generation.py:1053-1056) — one image, result [1, h, w]."""
        import torch
        if planar is None:
            B, H, W, _ = rgb.shape
        else:
            pl_img, rect = planar
            pl_hi, pl_wi = int(pl_img.shape[1]), int(pl_img.shape[2])
            B, H, W = 1, int(rect[3]), int(rect[2])
        net_h = net_h if net_h is not None else net_w
        if net_w % 32 or net_h % 32:
            raise ValueError("LeReS needs a net size that is a multiple of 32")
        self._trim_pools()
        # stem: pre-processing + im2col of the 7x7 / 2 conv, folded BN + ReLU in the GEMM, max-pool
        cols = self._stem_cols(B, net_h, net_w)
        m = (ctypes.c_float * 3)(*self.MEAN)
        s = (ctypes.c_float * 3)(*self.STD)
        if planar is None:
            self.ops.call("dm_leres_stem_im2col" + self._cv, rgb, B, H, W, net_h, net_w, m, s, cols)
        else:
            self.ops.call("dm_leres_stem_im2col_f32" + self._cv, pl_img, pl_hi, pl_wi, rect[0], rect[1], rect[2], rect[3], net_h, net_w, m, s, cols)
        dn = self._network(B, net_h, net_w, cols)
        hh, ww = net_h // 2, net_w // 2
        oh, ow = out_hw if out_hw is not None else (H, W)
        out = torch.empty(B, oh, ow, dtype=torch.float32, device=self.device)
        if (oh, ow) == (2 * hh, 2 * ww):
            out.copy_(dn)                                      # cv2.resize to the same size is a copy
        else:
            self.ops.call("dm_resize_f32", dn, B, 2 * hh, 2 * ww, out, oh, ow, 1)   # cv2.INTER_CUBIC (A = -0.75, replicated borders)
        return out

    def net_size(self, W, H, net_w, net_h):
        return net_w, net_h           # estimateleres resizes every image to the net size

    def forward_ragged(self, packed, desc, net_w, net_h=None):
        """Ragged batch (DepthAnythingV2Engine.forward_ragged): every image at (net_w, net_h), cv2.INTER_CUBIC back to its own size"""
        net_w, net_h = _ragged_net_size(self, desc, net_w, net_h)
        if net_w % 32 or net_h % 32:
            raise ValueError("LeReS needs a net size that is a multiple of 32")
        self._trim_pools()
        B = desc.B
        cols = self._stem_cols(B, net_h, net_w)
        self.ops.call("dm_leres_stem_im2col_ragged" + self._cv, *desc.args(packed), net_h, net_w, (ctypes.c_float * 3)(*self.MEAN),
                      (ctypes.c_float * 3)(*self.STD), cols)
        dn = self._network(B, net_h, net_w, cols)
        # the uniform path copies a prediction already at the image size; the bicubic resize at scale 1 reproduces it exactly
        return _resize_ragged(self, dn, B, net_h, net_w, desc, 1)

    def forward_crops(self, planar, rects, net):
        """BOOST's patch batch: estimateleres' network on B crops of one planar fp32 image ([3, Hi, Wi], rects = [(x0, y0, w, h)]), all at the
        same square net size -> fp32 [B, net, net] (a pooled buffer, valid until the next call at this (B, net)); the caller does the
        per-crop resize back (each crop has its own size)."""
        import torch
        if net % 32:
            raise ValueError("LeReS needs a net size that is a multiple of 32")
        B = len(rects)
        self._trim_pools()
        hi, wi = int(planar.shape[1]), int(planar.shape[2])
        _check_rects(rects, hi, wi)
        r = torch.tensor([list(map(int, q)) for q in rects], dtype=torch.int32).to(self.device)
        cols = self._stem_cols(B, net, net)
        m = (ctypes.c_float * 3)(*self.MEAN)
        sdev = (ctypes.c_float * 3)(*self.STD)
        self.ops.call("dm_leres_stem_im2col_f32_batch" + self._cv, planar, hi, wi, r, B, net, net, m, sdev, cols)
        return self._network(B, net, net, cols)

    def _network_eager(self, B, net_h, net_w, cols):
        import torch
        ops, w = self.ops, self.w
        # circular padding: the halo copy of a 3x3 convolution's input, sized for the largest one (adapt_conv.0's 256 channels at
        # half the net size)
        halo = self._buf('halo', (B * (net_h // 2 + 2) * (net_w // 2 + 2) * 256,)) if self.circular else None
        feats = self._encoder(B, net_h, net_w, cols, halo)
        conv, up2 = functools.partial(self._conv, B, halo), functools.partial(self._up2, B)

        def ftb(name, xin, hh, ww, ci, f, cm):
            x1 = conv(name + '_x1', xin, hh, ww, ci, f['c1'], cm, act=_lib.ACT_RELU)           # the in-place ReLU also rewrites the skip operand
            b1 = conv(name + '_b1', x1, hh, ww, cm, f['b1'], cm, act=_lib.ACT_RELU)
            return conv(name + '_o', b1, hh, ww, cm, f['b4'], cm, R=x1, C2=True)             # relu(x1 + branch)

        f3, h3, w3, c3 = feats[3]
        x = ftb('dconv', f3, h3, w3, c3, w['conv'], 512)
        x = conv('dconv1', x, h3, w3, 512, w['conv1'], 256)
        x = up2('up32', x, h3, w3, 256)
        hh, ww = 2 * h3, 2 * w3
        for k, fi in (('ffm2', 2), ('ffm1', 1), ('ffm0', 0)):
            low, hl, wl, cl = feats[fi]
            assert (hl, wl) == (hh, ww)
            a1 = ftb(k + 'a', low, hl, wl, cl, w[k][0], 256)
            sm = self._buf(k + '_sum', (B, hl, wl, 256))
            ops.call("dm_add_f16", a1, x, sm, sm.numel())
            x = ftb(k + 'b', sm, hl, wl, 256, w[k][1], 256)
            x = up2(k + '_up', x, hl, wl, 256)
            hh, ww = 2 * hl, 2 * wl
        x = conv('ao0', x, hh, ww, 256, w['ao0'], 128, act=_lib.ACT_RELU)
        d32 = self._buf('ao3', (B * hh * ww, 32), torch.float32)
        ops.conv3x3(x, B, hh, ww, 128, w['ao3'][0], 32, epi=_lib.EPI_STORE_F32, bias=w['ao3'][1], X=d32, ldx=32, halo=halo)
        dn = self._buf('dnet', (B, 2 * hh, 2 * ww), torch.float32)
        ops.call("dm_resize_f32_ld", d32, 32, B, hh, ww, dn, 2 * hh, 2 * ww, 0)
        assert (2 * hh, 2 * ww) == (net_h, net_w)
        return dn


class _RequiredKeys(dict):
    """a state dict whose missing keys raise ValueError naming the key"""

    def __init__(self, sd, what):
        super().__init__(sd)
        self.what = what

    def __missing__(self, key):
        raise ValueError(f"{self.what} checkpoint lacks {key!r}")


class MidasV21Engine(_MidasBoost, _ResNeXtEngine):
    """MiDaS v2.1 (midas_v21, model type 5) on the sm_90a kernels: estimatemidas (src/depthmap_generation.py:455-499) with the
    'upper_bound' resize and ImageNet statistics, around MidasNet (dmidas/midas_net.py:12-76, dmidas/blocks.py:136-320).

    The encoder is the ResNeXt-101 32x8d of LeReS (`pretrained.layer1` = conv1, bn1, relu, maxpool, layer1), its stem fed by a cv2
    INTER_CUBIC pre-processing + im2col.  The decoder: layer{1..4}_rn (3x3, no bias, 256 channels), the four FeatureFusionBlocks and
    the head, all on the implicit-GEMM conv.  ResidualConvUnit's ReLU is in place, so its skip operand is relu(x):
    RCU(x) = conv2(relu(conv1(relu(x)))) + relu(x), and only relu(layer_rn) is ever read.  FeatureFusionBlock: relu(path + RCU1(l))
    leaves conv2's epilogue as its relu copy (the sum itself is dead), RCU2, then a x2 bilinear up-sample with align_corners=True.
    refinenet4 has one input, and its resConfUnit1 is never used.  Head: conv3x3 256 -> 128, x2 bilinear with align_corners=False,
    then conv3x3 128 -> 32, ReLU, conv1x1 32 -> 1, ReLU fused into one epilogue.  The prediction goes back to the image size by
    bicubic interpolation (align_corners=False).

    BOOST (estimatemidasBoost, :1180-1220) calls forward_batch(None, msize, msize, planar=(img, rect)) and
    forward_crops(img, rects, msize) on float crops of a planar fp32 image, as for the DPT engines.  circular=True: tiling mode,
    every padded convolution (stem, encoder and decoder 3x3s, head) pads circularly."""

    FEATURES = 256
    CHAN_MAP = (2, 1, 0)     # the network sees the BGR-swapped image of get_raw_prediction (:381): channel c reads source channel 2-c
    GRAPH_ENV, NAME = "DEPTHMAP_B200_MIDAS_GRAPH", "MiDaS v2.1"

    @staticmethod
    def _block(li, bi):
        return f"pretrained.layer1.4.{bi}" if li == 1 else f"pretrained.layer{li}.{bi}"

    def _pack(self, sd):
        sd = _RequiredKeys(sd, "MiDaS v2.1")
        w = {}
        w['stem'], w['blocks'] = self._pack_encoder(sd, 'pretrained.layer1.0', 'pretrained.layer1.1', self._block)
        def conv(key, bias=True):
            if bias and key + '.bias' not in sd:       # _fold would take a missing bias for zeros
                raise ValueError(f"MiDaS v2.1 checkpoint lacks {key + '.bias'!r}")
            return self._packed(sd, key, None)
        w['rn'] = [conv(f'scratch.layer{i}_rn', bias=False) for i in range(1, 5)]
        for i in range(1, 5):
            for u in ((2,) if i == 4 else (1, 2)):
                for c in (1, 2):
                    w[f'rf{i}_u{u}c{c}'] = conv(f'scratch.refinenet{i}.resConfUnit{u}.conv{c}')
        w['oc0'] = conv('scratch.output_conv.0')
        w['oc2'] = conv('scratch.output_conv.2')
        w['oc4_w'] = _vec(sd['scratch.output_conv.4.weight'].detach().to(self.device))
        self.oc4_b = float(sd['scratch.output_conv.4.bias'].detach().float().reshape(-1)[0])
        self.w = w

    # ---- forward ---------------------------------------------------------------------------------------------------
    def net_size(self, W, H, net_w, net_h):
        nw, nh = midas_upper_bound_net_size(W, H, net_w, net_h)
        if nw <= 0 or nh <= 0:
            raise ValueError(f"a {W}x{H} image is too elongated for a net of at most {net_w}x{net_h} px")
        return nw, nh

    def forward_batch(self, rgb, net_w, net_h=None, out_hw=None, planar=None):
        """rgb: uint8 CUDA [B,H,W,3] -> float32 CUDA [B,H,W] (what estimatemidas returns; invert = False).  planar = (fp32 CUDA [3,Hi,Wi]
        image, (x0, y0, w, h)) instead of `rgb`: _forward_crop with msize = net_w."""
        import torch
        if planar is not None:
            return self._forward_crop(*planar, net_w)
        B, H, W, _ = rgb.shape
        nw, nh = self.net_size(W, H, net_w, net_h if net_h is not None else net_w)
        self._trim_pools()
        cols = self._stem_cols(B, nh, nw)
        m, s, c = (ctypes.c_float * 3)(*self.MEAN), (ctypes.c_float * 3)(*self.STD), (ctypes.c_int * 3)(*self.CHAN_MAP)
        self.ops.call("dm_midas_stem_im2col" + self._cv, rgb, B, H, W, nh, nw, m, s, c, cols)
        d = self._network(B, nh, nw, cols)
        oh, ow = out_hw if out_hw is not None else (H, W)
        out = torch.empty(B, oh, ow, dtype=torch.float32, device=self.device)
        self.ops.call("dm_resize_f32", d, B, nh, nw, out, oh, ow, 1)     # F.interpolate(bicubic, align_corners=False)
        return out

    def forward_ragged(self, packed, desc, net_w, net_h=None):
        """Ragged batch (DepthAnythingV2Engine.forward_ragged)"""
        nw, nh = _ragged_net_size(self, desc, net_w, net_h)
        self._trim_pools()
        B = desc.B
        cols = self._stem_cols(B, nh, nw)
        m, s, c = (ctypes.c_float * 3)(*self.MEAN), (ctypes.c_float * 3)(*self.STD), (ctypes.c_int * 3)(*self.CHAN_MAP)
        self.ops.call("dm_midas_stem_im2col_ragged" + self._cv, *desc.args(packed), nh, nw, m, s, c, cols)
        d = self._network(B, nh, nw, cols)
        return _resize_ragged(self, d, B, nh, nw, desc, 1)

    def _crops_network(self, planar, hi, wi, r, B, nh, nw):
        self._trim_pools()          # each crop group is a forward of its own
        cols = self._stem_cols(B, nh, nw)
        self.ops.call("dm_midas_stem_im2col_f32_crops" + self._cv, planar, hi, wi, r, B, nh, nw, *self._boost_consts(), cols)
        return self._network(B, nh, nw, cols)

    def _network_eager(self, B, net_h, net_w, cols):
        """stem GEMM .. head: the depth at the net size, fp32 [B, net_h, net_w] (a pooled buffer)"""
        import torch
        ops, w, F = self.ops, self.w, self.FEATURES
        # circular padding: the halo copy of a 3x3 convolution's input, sized for the largest one (the head's second conv: 128
        # channels at the net size, or its first: 256 at half of it)
        halo = self._buf('halo', (B * max((net_h + 2) * (net_w + 2) * 128, (net_h // 2 + 2) * (net_w // 2 + 2) * F),)) if self.circular else None
        feats = self._encoder(B, net_h, net_w, cols, halo)
        conv, up2 = functools.partial(self._conv, B, halo), functools.partial(self._up2, B)

        # layer{i}_rn, followed by the in-place ReLU of the first RCU that reads it
        lr = [conv(f'rn{i}', x, h, wd, c, w['rn'][i], F, act=_lib.ACT_RELU) for i, (x, h, wd, c) in enumerate(feats)]
        _, h, wd, _ = feats[3]
        t = conv('rf4_t', lr[3], h, wd, F, w['rf4_u2c1'], F, act=_lib.ACT_RELU)
        path = up2('rf4_up', conv('rf4_o', t, h, wd, F, w['rf4_u2c2'], F, R=lr[3]), h, wd, F)
        for i in (3, 2, 1):                                   # refinenet{i} reads layer{i}_rn = lr[i - 1]
            _, h, wd, _ = feats[i - 1]
            t = conv(f'rf{i}_t1', lr[i - 1], h, wd, F, w[f'rf{i}_u1c1'], F, act=_lib.ACT_RELU)
            s = conv(f'rf{i}_s', t, h, wd, F, w[f'rf{i}_u1c2'], F, R=lr[i - 1], R2=path, C2=True)     # relu(path + RCU1(l))
            t = conv(f'rf{i}_t2', s, h, wd, F, w[f'rf{i}_u2c1'], F, act=_lib.ACT_RELU)
            path = up2(f'rf{i}_up', conv(f'rf{i}_o', t, h, wd, F, w[f'rf{i}_u2c2'], F, R=s), h, wd, F)
        h, wd = 2 * h, 2 * wd
        a = conv('oc0', path, h, wd, F, w['oc0'], 128)
        au = self._buf('oc0_up', (B, net_h, net_w, 128))
        ops.call("dm_resize_bilinear_half_nhwc_f16", a, B, h, wd, 128, au, net_h, net_w)
        d = self._buf('dnet', (B, net_h, net_w), torch.float32)
        ops.conv3x3(au, B, net_h, net_w, 128, w['oc2'][0], 32, epi=_lib.EPI_HEAD, act=_lib.ACT_RELU, bias=w['oc2'][1], X=d,
                    gamma=w['oc4_w'], head_b2=self.oc4_b, halo=halo)
        assert (2 * h, 2 * wd) == (net_h, net_w)
        return d


ZOE_CONFIG = dict(n_bins=64, emb=128, min_temp=0.0212, max_temp=50.0, router_dim=128, router_heads=4, router_layers=4)


def _nbytes(obj):
    """device bytes of the tensors in a (nested) buffer dict"""
    if isinstance(obj, dict):
        return sum(_nbytes(v) for v in obj.values())
    if isinstance(obj, (list, tuple)):
        return sum(_nbytes(v) for v in obj)
    return obj.numel() * obj.element_size() if hasattr(obj, "element_size") else 0


def _zoe_pads(H, W):
    """DepthModel.infer_pil's reflect pad of an H x W image (depth_model.py:80-82, fh = fw = 3)"""
    return int(np.sqrt(H / 2) * 3.0), int(np.sqrt(W / 2) * 3.0)


def _zoe_lin(sd, dev, key, rows=None):
    """(weight, bias) of one 1x1 conv / linear layer: fp16 [rows, cin], fp32 [rows], output rows zero padded to `rows`"""
    return _mat(sd[key + '.weight'].detach().to(dev), rows), _vec(sd[key + '.bias'].detach().to(dev), rows)


def _zoe_mlp(sd, dev, key):
    """the two layers of a ZoeDepth MLP block (key._net.0, key._net.2)"""
    return _zoe_lin(sd, dev, key + '._net.0'), _zoe_lin(sd, dev, key + '._net.2')


class _ZoeDepthBase(DptBeitEngine):
    """What ZoeDepth-NK and ZoeDepth-N / -K share on the sm_90a kernels: DepthModel.infer_pil's pad + flip test-time augmentation
    (dzoedepth/models/depth_model.py:57-152; image b and its horizontal flip run as forwards 2b / 2b+1 of ONE batch), PrepForMidas
    (base_models/midas.py:175-186), the DPT-BEiT-L-384 core with MidasCore's hooks (midas.py:258-319), the seed projector, the
    attractor levels (projector -> resize-add of the previous bin embedding -> attractor MLP -> attractor kernel) and the
    log-binomial's bin-embedding GEMM.  Subclasses supply the seed bins, the attractor kernel, the log-binomial kernel and the
    layer widths below.  Checkpoint layout: MiDaS weights under "core.core.", head weights at the top level."""

    PROJ = ATT_HID = ATT_OUT = None     # hidden width of the projectors, of the attractor MLPs, and the attractor MLPs' output

    def __init__(self, state_dict, device, core_name='beitl16_384', circular=False):
        core_sd = {k[len("core.core."):]: v for k, v in state_dict.items() if k.startswith("core.core.")}
        self._sets, self._set_bytes, self._set_limit = {}, {}, None
        super().__init__(core_sd, core_name, device, circular)
        self._pack_head({k: v for k, v in state_dict.items() if not k.startswith("core.")})

    def _buffers(self, B, nh, nw):
        """One buffer set per forward shape, least recently used dropped first once the sets pass half of the device memory.
        BOOST alternates its crops between two net sizes (and the whole image between two others), so a single set would be
        rebuilt on every call.  The forward is eager (no CUDA graph reads a dropped set)."""
        import torch
        key = (B, nh, nw)
        b = self._sets.pop(key, None)
        if b is None:
            if self._set_limit is None:
                self._set_limit = torch.cuda.get_device_properties(self.device).total_memory // 2
            while self._sets and sum(self._set_bytes.values()) > self._set_limit:
                oldest = next(iter(self._sets))
                del self._sets[oldest], self._set_bytes[oldest]
            self._buf_key = None
            b = super()._buffers(B, nh, nw)
            self._set_bytes[key] = _nbytes(b)
        self._sets[key] = b                         # most recently used last
        self._bufs, self._buf_key = b, key
        return b

    @property
    def _zbufs(self):
        """the head's buffers at the current shape (ZoeDepth tests and tools read them)"""
        return self._bufs['z']

    def _head_buffers(self, b, F, nh, nw):
        """the head's buffers, b['z']"""
        import torch
        dev = self.device
        h16 = lambda *s: torch.empty(*s, dtype=torch.float16, device=dev)
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        s3 = b['sizes'][3]
        n0 = s3[0] * s3[1]
        levels = list(b['up_sizes'])                       # (h, w) of refinenet4..1 outputs
        zb = dict(x16=h16(F * n0, self.Fp), bprev=f32(F * n0, 64), p0=h16(F * n0, self.PROJ), pemb=h16(F * n0, 128), n0=n0, levels=levels)
        zb['t'] = [h16(F * h * w, self.PROJ) for h, w in levels]
        zb['bemb'] = [h16(F * h * w, 128) for h, w in levels]
        zb['xin'] = [h16(F * h * w, 128) for h, w in levels]
        zb['a0'] = [h16(F * h * w, self.ATT_HID) for h, w in levels]
        zb['A'] = [f32(F * h * w, self.ATT_OUT) for h, w in levels]
        zb['bnew'] = [f32(F * h * w, 64) for h, w in levels]
        zb['ze'] = f32(F * levels[3][0] * levels[3][1], 128)
        zb['o32'] = h16(F, nh, nw, 32)
        zb['d'] = f32(F, nh, nw)
        zb.update(self._seed_buffers(F, n0, h16, f32))
        b['z'] = zb

    def lin(self, a, lda, wb, M, N, K, out=None, act=_lib.ACT_NONE, f32out=None, resid=None):
        """a [M, K] (row pitch lda) times a (weight, bias) pair -> fp16 `out`, fp32 `f32out`, or added into the fp32 stream `resid`"""
        wt, bias = wb
        if resid is not None:
            self.ops.gemm(a, lda, wt, K, M, N, K, epi=_lib.EPI_RESID_F32, bias=bias, X=resid, ldx=N, gamma=self.z['ones128'])
        elif f32out is not None:
            self.ops.gemm(a, lda, wt, K, M, N, K, epi=_lib.EPI_STORE_F32, act=act, bias=bias, X=f32out, ldx=N)
        else:
            self.ops.gemm(a, lda, wt, K, M, N, K, act=act, bias=bias, C=out, ldc=N)

    def forward_batch(self, rgb, net_w, net_h=None, out_hw=None, planar=None):
        """rgb: uint8 CUDA [B,H,W,3] -> float32 CUDA [B,H,W] metric depth (what estimatezoedepth returns; invert = True).
        planar = (fp32 CUDA [3,Hi,Wi] image, (x0, y0, w, h)) instead of `rgb`: BOOST's estimate of one crop at msize = net_w,
        [1, h, w] (forward_crops)."""
        import torch
        if planar is not None:
            return self.forward_crops(planar[0], [planar[1]], net_w)[0].unsqueeze(0)
        ops = self.ops
        B, H, W, _ = rgb.shape
        net_h = net_h if net_h is not None else net_w
        pad_h, pad_w = _zoe_pads(H, W)
        nw, nh = self.net_size(W, H, net_w, net_h)
        F = 2 * B
        b = self._buffers(F, nh, nw)
        ops.call("dm_zoe_preprocess_patchify", rgb, B, H, W, pad_h, pad_w, nh, nw, self.PATCH, b['patches'], self.kpad)
        zb = self._zoe_network(b, F, nh, nw)
        out = torch.empty(B, H, W, dtype=torch.float32, device=self.device)
        ops.call("dm_zoe_tta_combine", zb['d'], B, nh, nw, pad_h, pad_w, H, W, out)
        return out

    def net_size(self, W, H, net_w, net_h):
        """PrepForMidas (keep aspect, x32, "minimal") of the reflect-padded image"""
        pad_h, pad_w = _zoe_pads(H, W)
        return midas_net_size(W + 2 * pad_w, H + 2 * pad_h, net_w, net_h)

    def forward_ragged(self, packed, desc, net_w, net_h=None):
        """Ragged batch (DepthAnythingV2Engine.forward_ragged): each image with its own reflect pad and flip, one forward of 2B"""
        import torch
        nw, nh = _ragged_net_size(self, desc, net_w, net_h)
        B = desc.B
        F = 2 * B
        b = self._buffers(F, nh, nw)
        self.ops.call("dm_zoe_preprocess_patchify_ragged", *desc.args(packed), nh, nw, self.PATCH, b['patches'], self.kpad)
        zb = self._zoe_network(b, F, nh, nw)
        out_desc = _lib.Ragged(desc.sizes, 1, self.device)
        out = torch.empty(out_desc.size, dtype=torch.float32, device=self.device)
        self.ops.call("dm_zoe_tta_combine_ragged", zb['d'], B, nh, nw, out, out_desc.size, out_desc.host.ctypes.data, out_desc.dev)
        return out

    def _zoe_network(self, b, F, nh, nw):
        """patch matrix of the F = 2B forwards in b['patches'] -> the head's buffers, the net-size metric depth in zb['d']"""
        ops, z, P, RELU = self.ops, self.z, self.PROJ, _lib.ACT_RELU
        self.run_network(b, F, nh, nw)
        zb, Fp = b['z'], self.Fp
        # out_conv activation (MidasCore hooks output_conv[3], the 32-channel ReLU)
        self.run_output_conv1(b, F, nh, nw)
        ops.conv3x3(b['oc1u'], F, nh, nw, self.F2p, self.w['oc2_w'], 32, act=RELU, bias=self.w['oc2_b'], C=zb['o32'], halo=b['halo'])
        n0 = zb['n0']
        # x = conv2(bottleneck); seed bins; seed embedding
        self.lin(b['l'][3], Fp, z['conv2'], F * n0, Fp, Fp, out=zb['x16'])
        self.seed_bins(zb, F)
        self.lin(zb['x16'], Fp, z['sproj'][0], F * n0, P, Fp, out=zb['p0'], act=RELU)
        self.lin(zb['p0'], P, z['sproj'][1], F * n0, 128, P, out=zb['pemb'])
        # attractor levels
        bprev, pemb, (hp, wp) = zb['bprev'], zb['pemb'], b['sizes'][3]
        for i, (h, w) in enumerate(zb['levels']):
            M = F * h * w
            self.lin(b['path'][i], Fp, z['proj'][i][0], M, P, Fp, out=zb['t'][i], act=RELU)
            self.lin(zb['t'][i], P, z['proj'][i][1], M, 128, P, out=zb['bemb'][i])
            ops.call("dm_resize_add_nhwc_f16", zb['bemb'][i], pemb, F, hp, wp, 128, zb['xin'][i], h, w)
            self.lin(zb['xin'][i], 128, z['att'][i][0], M, self.ATT_HID, 128, out=zb['a0'][i], act=RELU)
            self.lin(zb['a0'][i], self.ATT_HID, z['att'][i][1], M, self.ATT_OUT, self.ATT_HID, f32out=zb['A'][i])
            self.attractor(i, zb, bprev, F, hp, wp, h, w)
            bprev, pemb, (hp, wp) = zb['bnew'][i], zb['bemb'][i], (h, w)
        # conditional log-binomial + expectation, then un-pad / un-flip / average (depth_model.py:88-129)
        ops.gemm(zb['bemb'][3], 128, z['clb'][0], 128, F * hp * wp, 128, 128, epi=_lib.EPI_STORE_F32, X=zb['ze'], ldx=128)
        self.log_binomial(zb, bprev, F, nh, nw, hp, wp)
        return zb

    def forward_crops(self, planar, rects, msize):
        """BOOST's estimates: singleestimate's ZoeDepth branch (src/depthmap_generation.py:1062-1064, estimatezoedepth :443-452) on
        crops (x0, y0, w, h) of one planar fp32 image [3, Hi, Wi] -> [fp32 CUDA [h, w]] metric depth at each crop's size (no
        normalisation), in the order of `rects`.  Each crop is quantised as PIL receives it (np.uint8(crop * 255) of the R/B-swapped
        image, dm_boost_quantise_crops_u8), then runs infer_pil at msize x msize: the forward above.  Its reflect pad and keep-aspect
        net size depend on the crop's shape, so the crops are grouped by exact (h, w), one batched forward per shape."""
        import torch
        hi, wi = _check_planar(planar)
        _check_rects(rects, hi, wi)
        groups = {}
        for k, (_, _, w, h) in enumerate(rects):
            groups.setdefault((int(h), int(w)), []).append(k)
        out = [None] * len(rects)
        for (h, w), ks in groups.items():
            r = torch.tensor([[int(v) for v in rects[k]] for k in ks], dtype=torch.int32).to(self.device)
            u8 = torch.empty(len(ks), h, w, 3, dtype=torch.uint8, device=self.device)
            self.ops.call("dm_boost_quantise_crops_u8", planar, hi, wi, r, len(ks), h, w, u8)
            d = self.forward_batch(u8, msize, msize)
            for i, k in enumerate(ks):
                out[k] = d[i]
        return out


class ZoeDepthNKEngine(_ZoeDepthBase):
    """ZoeDepth-NK (model type 9, zoedepth_nk): the metric head of ZoeDepthNK.forward (zoedepth_nk/zoedepth_nk_v1.py:159-243) on
    the shared ZoeDepth skeleton.  The router picks nyu / kitti per forward on the device (argmax of two logits, no host sync, no
    cross-image vote); both heads' layers are packed side by side."""

    PROJ, ATT_HID, ATT_OUT = 64, 256, 64

    # ---- weights -------------------------------------------------------------------------------------------------------
    def _pack_head(self, sd):
        import torch
        dev = self.device
        lin = functools.partial(_zoe_lin, sd, dev)
        cat = lambda pairs: tuple(torch.cat(t) for t in zip(*pairs))       # layers of both heads stacked
        z = {'conv2': lin('conv2'), 'emb': lin('patch_transformer.embedding_convPxP')}
        layers = []
        for i in range(ZOE_CONFIG['router_layers']):
            q = f'patch_transformer.transformer_encoder.layers.{i}'
            f32 = lambda k: _vec(sd[k].detach().to(dev))
            layers.append(dict(
                in_w=_mat(sd[q + '.self_attn.in_proj_weight'].detach().to(dev)), in_b=f32(q + '.self_attn.in_proj_bias'),
                out=lin(q + '.self_attn.out_proj'), l1=lin(q + '.linear1'), l2=lin(q + '.linear2'),
                n1=(f32(q + '.norm1.weight'), f32(q + '.norm1.bias')), n2=(f32(q + '.norm2.weight'), f32(q + '.norm2.bias'))))
        z['layers'] = layers
        z['cls0'] = lin('mlp_classifier.0')
        z['cls2'] = lin('mlp_classifier.2', 32)
        z['ones128'] = torch.ones(128, dtype=torch.float32, device=dev)
        z['zeros128'] = torch.zeros(128, dtype=torch.float32, device=dev)
        names = ('nyu', 'kitti')
        # seed bin regressors of both heads side by side: net.0 stacked, net.2 block-diagonal (nyu -> columns 0..63, kitti 64..127)
        z['seed0'] = cat([lin(f'seed_bin_regressors.{n}._net.0') for n in names])
        w2 = torch.zeros(128, 128, dtype=torch.float16, device=dev)
        b2 = torch.zeros(128, dtype=torch.float32, device=dev)
        for k, n in enumerate(names):
            w2[64 * k:64 * k + 64, 64 * k:64 * k + 64], b2[64 * k:64 * k + 64] = lin(f'seed_bin_regressors.{n}._net.2')
        z['seed2'] = (w2, b2)
        z['sproj'] = _zoe_mlp(sd, dev, 'seed_projector')
        z['proj'] = [_zoe_mlp(sd, dev, f'projectors.{i}') for i in range(4)]
        att = []
        for i in range(4):
            a0 = cat([lin(f'attractors.{n}.{i}._net.0') for n in names])
            w2 = torch.zeros(64, 256, dtype=torch.float16, device=dev)
            b2 = torch.zeros(64, dtype=torch.float32, device=dev)
            for k, n in enumerate(names):
                t, bk = lin(f'attractors.{n}.{i}._net.2')
                if t.shape[0] != 16:
                    raise NotImplementedError("ZoeDepth-NK attractor layers with other than 16 attractors (the reference always builds 16)")
                w2[32 * k:32 * k + 16, 128 * k:128 * k + 128] = t
                b2[32 * k:32 * k + 16] = bk
            att.append((a0, (w2, b2)))
        z['att'] = att
        # conditional log-binomial: mlp.0 split into its out_conv part (32 inputs, evaluated per pixel in clb_final) and its bin
        # embedding part (128 inputs, a GEMM before the up-sampling: a 1x1 conv commutes with bilinear interpolation)
        we = torch.zeros(128, 128, dtype=torch.float16, device=dev)
        wo = torch.zeros(2, 32, 40, dtype=torch.float32, device=dev)
        b0 = torch.zeros(2, 40, dtype=torch.float32, device=dev)
        w2c = torch.zeros(2, 4, 40, dtype=torch.float32, device=dev)
        b2c = torch.zeros(2, 4, dtype=torch.float32, device=dev)
        for k, n in enumerate(names):
            m0 = sd[f'conditional_log_binomial.{n}.mlp.0.weight'].detach().to(dev).float().reshape(40, 160)
            wo[k] = m0[:, :32].t()
            we[64 * k:64 * k + 40] = m0[:, 32:].to(torch.float16)
            b0[k] = sd[f'conditional_log_binomial.{n}.mlp.0.bias'].detach().to(dev).float()
            w2c[k] = sd[f'conditional_log_binomial.{n}.mlp.2.weight'].detach().to(dev).float().reshape(4, 40)
            b2c[k] = sd[f'conditional_log_binomial.{n}.mlp.2.bias'].detach().to(dev).float()
        z['clb'] = (we, wo.contiguous(), b0.contiguous(), w2c.contiguous(), b2c.contiguous())
        self.z = z
        self._pe_cache = {}

    def _router_pe(self, S):
        """PositionalEncodingPermute1D replacement of patch_transformer.py:45-62: sin | cos of position * 10000^(-2i/E)."""
        import torch
        if S not in self._pe_cache:
            E = ZOE_CONFIG['router_dim']
            pos = torch.arange(0, S, dtype=torch.float32, device=self.device).unsqueeze(1)
            idx = torch.arange(0, E, 2, dtype=torch.float32, device=self.device).unsqueeze(0)
            div = torch.exp(idx * (-torch.log(torch.tensor(10000.0, device=self.device)) / E))
            pe = pos * div
            self._pe_cache = {S: torch.cat([torch.sin(pe), torch.cos(pe)], dim=1).contiguous()}
        return self._pe_cache[S]

    def _seed_buffers(self, F, n0, h16, f32):
        S = n0 + 1
        return dict(emb=h16(F * n0, 128), X=f32(F * S, 128), h=h16(F * S, 128), qkv=h16(F * S, 384), att=h16(F * S, 128), ff=h16(F * S, 1024),
                    c1=h16(F, 128), logits=f32(F, 32), s0=h16(F * n0, 128), seed=f32(F * n0, 128), S=S)

    # ---- the NK-specific steps of the forward --------------------------------------------------------------------------
    def seed_bins(self, zb, F):
        """router: PatchTransformerEncoder (patch size 1) + MLP classifier (zoedepth_nk_v1.py:186-195); the seed bins of both heads
        and the routed head's softplus (:197-206)"""
        ops, z, RELU = self.ops, self.z, _lib.ACT_RELU
        n0, S, Fp = zb['n0'], zb['S'], self.Fp
        self.lin(zb['x16'], Fp, z['emb'], F * n0, 128, Fp, out=zb['emb'])
        ops.call("dm_assemble_tokens", zb['emb'], z['zeros128'], self._router_pe(S), zb['X'], F, n0, 128)
        ops.call("dm_cast_f32_f16", zb['X'], F * S * 128, zb['h'])
        for lay in z['layers']:
            self.lin(zb['h'], 128, (lay['in_w'], lay['in_b']), F * S, 384, 128, out=zb['qkv'])
            ops.call("dm_attention_small_f16", zb['qkv'], F, S, ZOE_CONFIG['router_heads'], 1.0 / math.sqrt(32.0), zb['att'])
            self.lin(zb['att'], 128, lay['out'], F * S, 128, 128, resid=zb['X'])
            ops.call("dm_layernorm_post_f16", zb['X'], F * S, 128, lay['n1'][0], lay['n1'][1], 1e-5, zb['h'])
            self.lin(zb['h'], 128, lay['l1'], F * S, 1024, 128, out=zb['ff'], act=RELU)
            self.lin(zb['ff'], 1024, lay['l2'], F * S, 128, 1024, resid=zb['X'])
            ops.call("dm_layernorm_post_f16", zb['X'], F * S, 128, lay['n2'][0], lay['n2'][1], 1e-5, zb['h'])
        self.lin(zb['h'], S * 128, z['cls0'], F, 128, 128, out=zb['c1'], act=RELU)       # token 0 of every forward (row pitch S*128)
        self.lin(zb['c1'], 128, z['cls2'], F, 32, 128, f32out=zb['logits'])
        self.lin(zb['x16'], Fp, z['seed0'], F * n0, 128, Fp, out=zb['s0'], act=RELU)
        self.lin(zb['s0'], 128, z['seed2'], F * n0, 128, 128, f32out=zb['seed'])
        ops.call("dm_zoe_select_softplus", zb['seed'], 128, zb['logits'], 32, F, n0, zb['bprev'])

    def attractor(self, i, zb, bprev, F, hp, wp, h, w):
        """(:207-214)"""
        self.ops.call("dm_zoe_attractor", zb['A'][i], 64, zb['logits'], 32, bprev, F, hp, wp, h, w, zb['bnew'][i])

    def log_binomial(self, zb, bprev, F, nh, nw, hp, wp):
        """(:216-236)"""
        _, wo, b0, w2c, b2c = self.z['clb']
        self.ops.call("dm_zoe_clb_final", zb['o32'], 32, zb['ze'], 128, bprev, zb['logits'], 32, wo, b0, w2c, b2c, F, nh, nw, hp, wp,
                      ZOE_CONFIG['min_temp'], ZOE_CONFIG['max_temp'], zb['d'])


# ZoeDepth-N / -K: get_config("zoedepth", "infer") and its "kitti" version.  Neither sets min_depth / max_depth, so both keep
# ZoeDepth.__init__'s 1e-3 / 10 (dzoedepth/models/zoedepth/zoedepth_v1.py:39); K's centres are clipped at 10 like the reference's.
ZOE_SINGLE_CONFIG = dict(n_bins=64, bin_embedding_dim=128, n_attractors=[16, 8, 4, 1], min_temp=0.0212, max_temp=50.0, min_depth=1e-3, max_depth=10.0)
ZOE_SINGLE_VARIANTS = {'n': dict(model_type=7, bin_centers_type='softplus', checkpoint='ZoeD_M12_N.pt'),
                       'k': dict(model_type=8, bin_centers_type='normed', checkpoint='ZoeD_M12_K.pt')}


class ZoeDepthEngine(_ZoeDepthBase):
    """Single-head ZoeDepth: ZoeDepth-N (variant 'n', model type 7, softplus bin centres) and ZoeDepth-K ('k', model type 8, bin
    centres normed to [min_depth, max_depth]) on the shared ZoeDepth skeleton.  The head is ZoeDepth.forward
    (dzoedepth/models/zoedepth/zoedepth_v1.py:124-192): seed bins, four attractor levels with [16, 8, 4, 1] attractors, and a
    log-binomial whose 33rd input is the core's own relative depth.  Bin centres, attractor points and the log-binomial stay in
    fp32."""

    PROJ, ATT_HID, ATT_OUT = 128, 128, 32

    def __init__(self, state_dict, device, variant, core_name='beitl16_384', circular=False):
        if variant not in ZOE_SINGLE_VARIANTS:
            raise ValueError(f"ZoeDepthEngine: variant must be 'n' or 'k', not {variant!r}")
        self.variant = variant
        self.normed = ZOE_SINGLE_VARIANTS[variant]['bin_centers_type'] == 'normed'
        super().__init__(state_dict, device, core_name, circular)

    def _pack_head(self, sd):
        dev = self.device
        lin = functools.partial(_zoe_lin, sd, dev)
        z = {'conv2': lin('conv2'), 'seed': _zoe_mlp(sd, dev, 'seed_bin_regressor'), 'sproj': _zoe_mlp(sd, dev, 'seed_projector'),
             'proj': [_zoe_mlp(sd, dev, f'projectors.{i}') for i in range(4)]}
        if z['seed'][1][0].shape[0] != ZOE_SINGLE_CONFIG['n_bins']:
            raise ValueError(f"ZoeDepthEngine: the seed bin regressor has {z['seed'][1][0].shape[0]} outputs, not 64 bins")
        per = 2 if self.normed else 1
        att = []
        for i, n in enumerate(ZOE_SINGLE_CONFIG['n_attractors']):
            key = f'attractors.{i}._net.2'
            if sd[key + '.weight'].shape[0] != per * n:
                raise ValueError(f"ZoeDepthEngine({self.variant!r}): {key} has {sd[key + '.weight'].shape[0]} outputs, expected {per * n} "
                                 f"({n} attractors{' x 2 for the normed layer' if self.normed else ''})")
            att.append((lin(f'attractors.{i}._net.0'), lin(key, 32)))
        z['att'] = att
        # conditional log-binomial: mlp.0 over cat(out_conv (32), rel_depth (1), b_emb (128)), 80 outputs.  Its out_conv and
        # rel-depth part is evaluated per pixel in clb_single, its bin-embedding part is a GEMM before the up-sampling (a 1x1 conv
        # commutes with bilinear interpolation), as in ZoeDepth-NK
        m0 = sd['conditional_log_binomial.mlp.0.weight'].detach().to(dev).float()
        if tuple(m0.shape[:2]) != (80, 161):
            raise ValueError(f"ZoeDepthEngine: conditional_log_binomial.mlp.0 is {tuple(m0.shape)}, expected (80, 161, 1, 1)")
        m0 = m0.reshape(80, 161)
        z['clb'] = (_mat(m0[:, 33:], 128), m0[:, :33].t().contiguous(), _vec(sd['conditional_log_binomial.mlp.0.bias'].detach().to(dev)),
                    sd['conditional_log_binomial.mlp.2.weight'].detach().to(dev).float().reshape(4, 80).contiguous(),
                    _vec(sd['conditional_log_binomial.mlp.2.bias'].detach().to(dev)))
        self.z = z

    def _seed_buffers(self, F, n0, h16, f32):
        return dict(s0=h16(F * n0, 256), seed=f32(F * n0, 64))

    # ---- the N / K-specific steps of the forward -----------------------------------------------------------------------
    def seed_bins(self, zb, F):
        """seed bins (zoedepth_v1.py:151-159)"""
        cfg, z, n0, Fp = ZOE_SINGLE_CONFIG, self.z, zb['n0'], self.Fp
        self.lin(zb['x16'], Fp, z['seed'][0], F * n0, 256, Fp, out=zb['s0'], act=_lib.ACT_RELU)
        self.lin(zb['s0'], 256, z['seed'][1], F * n0, 64, 256, f32out=zb['seed'])
        self.ops.call("dm_zoe_seed_bins", zb['seed'], 64, F * n0, int(self.normed), cfg['min_depth'], cfg['max_depth'], zb['bprev'])

    def attractor(self, i, zb, bprev, F, hp, wp, h, w):
        """(:164-169); the normed head's last level hands on sorted, clipped centres"""
        cfg = ZOE_SINGLE_CONFIG
        sort_clip = int(self.normed and i == len(zb['levels']) - 1)
        self.ops.call("dm_zoe_attractor_single", zb['A'][i], 32, cfg['n_attractors'][i], int(self.normed), bprev, F, hp, wp, h, w, sort_clip,
                      cfg['min_depth'], cfg['max_depth'], zb['bnew'][i])

    def log_binomial(self, zb, bprev, F, nh, nw, hp, wp):
        """on cat(out_conv, rel_depth) + expectation (:171-192); the core's relative depth, the final 1x1 conv + ReLU on out_conv,
        is evaluated inside clb_single"""
        _, wo, b0, w2c, b2c = self.z['clb']
        self.ops.call("dm_zoe_clb_single", zb['o32'], 32, zb['ze'], 128, bprev, wo, b0, w2c, b2c, self.w['oc3_w'], self.oc3_b, F, nh, nw, hp, wp,
                      ZOE_SINGLE_CONFIG['min_temp'], ZOE_SINGLE_CONFIG['max_temp'], zb['d'])


def _unwrap_key(key, where):
    """training checkpoints wrap the weights in a dict; a flat state dict never has these top-level keys"""
    return lambda sd: sd[key] if where in sd else sd


def _unwrap_leres(sd):
    """src/depthmap_generation.py:113-116: strip_prefix_if_present(checkpoint['depth_model'], "module.")"""
    if "depth_model" not in sd:
        return sd
    return {(k[len("module."):] if k.startswith("module.") else k): v for k, v in sd["depth_model"].items()}


_flat = lambda sd: sd
_midas = _unwrap_key("model", "optimizer")      # dmidas/base_model.py:13
_zoe = _unwrap_key("model", "model")            # dzoedepth/models/model_io.py:52-53


def _vit(cls, name):
    return lambda sd, dev, tiling, split: cls(sd, name, dev, tiling, split)


# model type -> (default checkpoint path, unwrap, engine(state_dict, device, tiling, split)).  `split` (the no_half path) is only
# ever set for Depth-Anything-V2 (no_half_route).
CHECKPOINTS = {
    0: ("./models/leres/res101.pth", _unwrap_leres, lambda sd, dev, tiling, split: LeresEngine(sd, dev, tiling)),
    1: ("./models/midas/dpt_beit_large_512.pt", _midas, _vit(DptBeitEngine, 'beitl16_512')),
    2: ("./models/midas/dpt_beit_large_384.pt", _midas, _vit(DptBeitEngine, 'beitl16_384')),
    3: ("./models/midas/dpt_large-midas-2f21e586.pt", _midas, _vit(DptVitEngine, 'vitl16_384')),
    5: ("./models/midas/midas_v21-f6b98070.pt", _midas, lambda sd, dev, tiling, split: MidasV21Engine(sd, dev, tiling)),
    7: ("./models/zoedepth/" + ZOE_SINGLE_VARIANTS['n']['checkpoint'], _zoe,
        lambda sd, dev, tiling, split: ZoeDepthEngine(sd, dev, 'n', circular=tiling)),
    8: ("./models/zoedepth/" + ZOE_SINGLE_VARIANTS['k']['checkpoint'], _zoe,
        lambda sd, dev, tiling, split: ZoeDepthEngine(sd, dev, 'k', circular=tiling)),
    9: ("./models/zoedepth/ZoeD_M12_NK.pt", _zoe, lambda sd, dev, tiling, split: ZoeDepthNKEngine(sd, dev, circular=tiling)),
    12: ("./models/depth_anything_v2/depth_anything_v2_vits.pth", _flat, _vit(DepthAnythingV2Engine, 'vits')),
    13: ("./models/depth_anything_v2/depth_anything_v2_vitb.pth", _flat, _vit(DepthAnythingV2Engine, 'vitb')),
    14: ("./models/depth_anything_v2/depth_anything_v2_vitl.pth", _flat, _vit(DepthAnythingV2Engine, 'vitl')),
}
PIX2PIX_CHECKPOINT = "./models/pix2pix/latest_net_G.pth"
DAV2_ENCODERS = {12: 'vits', 13: 'vitb', 14: 'vitl'}


def no_half_route(model_type, boost, precision):
    """What the `no_half` setting does to a model load: "split" (Depth-Anything-V2: the reference then runs the whole network in
    fp32, src/depthmap_generation.py:548-559, so it gets the fp32-class split path), "unchanged" (the reference's arithmetic does
    not change either: 0 and 7 always run in fp32 here and there, BOOST never halves its base network, and MiDaS 1, 2, 3, 5 under
    precision "autocast" keep fp16 convolutions and matmuls through torch.autocast, :455-499), or NotImplementedError where the
    reference would run an fp32 network this build has no fp32-class path for."""
    if model_type in DAV2_ENCODERS:
        return "split"
    if model_type in (8, 9):
        raise NotImplementedError(f"no_half is not implemented in depthmap_b200 for model type {model_type} (ZoeDepth on the BEiT core); "
                                  f"it is implemented for Depth-Anything-V2 (12, 13, 14) and leaves 0, 7, BOOST and autocast MiDaS as they are")
    if model_type in (1, 2, 3, 5) and not boost and precision == "full":
        raise NotImplementedError(f"no_half with precision \"full\" is not implemented in depthmap_b200 for model type {model_type} (an fp32 "
                                  f"MiDaS network); with precision \"autocast\" the reference keeps fp16 arithmetic and so does this build")
    return "unchanged"


class ModelHolder:
    """Same public surface as the reference's ModelHolder (src/depthmap_generation.py:40-403)."""

    def __init__(self):
        self.depth_model = None
        self.pix2pix_model = None
        self.depth_model_type = None
        self.device = None
        self.offloaded = False
        self.resize_mode = None
        self.normalization = None
        self.tiling_mode = False
        # settings injected by update_settings(**ops) in the reference (src/backbone.py:36-49,132-137)
        self.no_half = False
        self.precision = "autocast"
        self.boost_rmax = 1600
        self.weights_provider = None  # callable(model_type) -> state_dict; default: torch.load of ./models/... like the reference

    def update_settings(self, **kvargs):
        for k, v in kvargs.items():
            setattr(self, k, v)

    def ensure_models(self, model_type, device, boost: bool, tiling_mode: bool = False):
        if model_type == -1 or model_type is None:
            self.unload_models()
            return
        if (model_type != self.depth_model_type or boost != (self.pix2pix_model is not None) or device != self.device or
                tiling_mode != self.tiling_mode):
            self.unload_models()
            self.load_models(model_type, device, boost, tiling_mode)
        self.reload()

    def load_models(self, model_type, device, boost: bool, tiling_mode: bool = False):
        """Ensure that the depth model is loaded (reference: src/depthmap_generation.py:76-301)."""
        import torch
        _lib.require_cuda()
        from .boost import BASE_NETWORKS
        if boost and model_type not in BASE_NETWORKS:
            raise NotImplementedError(f"BOOST is implemented in depthmap_b200 for the base networks LeReS res101 (model type 0), "
                                      f"DPT-BEiT-L 512 / 384 (1, 2), DPT-Large 384 (3), MiDaS v2.1 (5) and ZoeDepth-NK (9), not for "
                                      f"model type {model_type}")
        # `no_half` is read here, at load time; like the reference, ensure_models does not reload when only the setting changes
        route = no_half_route(model_type, boost, self.precision) if self.no_half else "unchanged"
        if model_type not in CHECKPOINTS:
            raise NotImplementedError(f"model_type {model_type} is not implemented in depthmap_b200 yet "
                                      f"(implemented: 0 = LeReS res101; 1, 2 = DPT-BEiT-L 512/384; 3 = DPT-Large 384; 5 = MiDaS v2.1; 7 = ZoeDepth-N; "
                                      f"8 = ZoeDepth-K; 9 = ZoeDepth-NK; 12, 13, 14 = Depth-Anything-V2 S/B/L)")
        dev = torch.device(device)
        path, unwrap, make = CHECKPOINTS[model_type]
        model = make(self._load_checkpoint(model_type, path, unwrap), dev, bool(tiling_mode), route == "split")
        if boost:      # reference :284-299: the pix2pix merge network ('latest_net_G.pth', netG = unet_1024, norm none)
            from .boost import BoostPipeline, UnetMergeEngine
            self.pix2pix_model = BoostPipeline(model, UnetMergeEngine(self._load_checkpoint("pix2pix", PIX2PIX_CHECKPOINT), dev), dev, model_type)
        self.depth_model = model
        self.depth_model_type = model_type
        self.resize_mode = "upper_bound" if model_type == 5 else "minimal"
        self.normalization = None
        self.tiling_mode = tiling_mode
        self.device = device

    def _load_checkpoint(self, key, path, unwrap=_flat):
        """weights_provider(key), or torch.load of the default path; unwrapped to the flat state dict"""
        import torch
        if self.weights_provider is not None:
            sd = self.weights_provider(key)
        else:
            if not os.path.exists(path):
                raise FileNotFoundError(f"{path} not found (depthmap_b200 does not download checkpoints)")
            sd = torch.load(path, map_location='cpu')
        return unwrap(sd)

    @staticmethod
    def get_default_net_size(model_type):
        sizes = {0: [448, 448], 1: [512, 512], 2: [384, 384], 3: [384, 384], 4: [384, 384], 5: [384, 384], 6: [256, 256],
                 7: [384, 512], 8: [384, 768], 9: [384, 512], 10: [768, 768], 11: [518, 518], 12: [518, 518], 13: [518, 518],
                 14: [518, 518]}
        if model_type in sizes:
            return sizes[model_type]
        return [512, 512]

    def offload(self):
        """The reference swaps the model to host RAM between calls to free VRAM for Stable Diffusion (:344-348).
        Packed weights stay resident on a 180 GB part; the flag is kept so callers observe the same state machine."""
        if self.device is not None and not self.offloaded:
            self.offloaded = True

    def reload(self):
        if self.offloaded:
            self.offloaded = False

    def move_models_to(self, device):
        pass

    def unload_models(self):
        if self.depth_model is not None or self.pix2pix_model is not None:
            self.depth_model = None
            self.pix2pix_model = None
            gc.collect()
            try:
                import torch
                torch.cuda.empty_cache()
            except Exception:
                pass
        self.depth_model_type = None
        self.device = None

    # ---- prediction ------------------------------------------------------------------------------------------------
    def get_raw_prediction_batch(self, rgb, net_width, net_height):
        """uint8 CUDA [B,H,W,3] -> (float32 CUDA [B,H,W], invert flag).  Batched form of get_raw_prediction."""
        import torch
        if self.depth_model is None:
            raise RuntimeError("no depth model loaded; call ensure_models first")
        if not torch.is_tensor(rgb) or rgb.dtype != torch.uint8 or rgb.dim() != 4 or rgb.shape[-1] != 3:
            raise ValueError("rgb must be a uint8 tensor [B,H,W,3]")      # the kernels read the tensor's memory as such
        rgb = rgb.contiguous()
        if self.pix2pix_model is not None:
            # boost: estimateboost works on one image at a time (its resolutions and patches depend on the image); the net size is ignored
            preds = [self.pix2pix_model.run(rgb[i].cpu().numpy(), self.boost_rmax, to_host=False) for i in range(rgb.shape[0])]
            return torch.stack(preds), self.depth_model_type in [0, 7, 8, 9, 10]
        if self.depth_model_type in (0, 1, 2, 3, 5, 7, 8, 9, 12, 13, 14):
            pred = self.depth_model.forward_batch(rgb, net_width, net_height)
        else:
            raise NotImplementedError(f"model_type {self.depth_model_type}")
        return pred, self.depth_model_type in [0, 7, 8, 9, 10]

    def net_size(self, w, h, net_w, net_h):
        """the network input size (width, height) the loaded depth model gives a w x h image for the requested net size: images
        that share it can run as one ragged batch (get_raw_prediction_ragged)"""
        if self.depth_model is None:
            raise RuntimeError("no depth model loaded; call ensure_models first")
        return tuple(self.depth_model.net_size(int(w), int(h), net_w, net_h))

    def get_raw_prediction_ragged(self, images, net_width, net_height):
        """list of uint8 CUDA [Hi, Wi, 3] images of any sizes -> (list of float32 CUDA [Hi, Wi] in input order, invert flag).  The images
        are grouped by network input size, one forward per group; each result equals get_raw_prediction_batch of that image alone.
        With BOOST loaded each image runs through the BOOST pipeline on its own, as in get_raw_prediction_batch."""
        import torch
        if self.depth_model is None:
            raise RuntimeError("no depth model loaded; call ensure_models first")
        for t in images:
            if not torch.is_tensor(t) or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[-1] != 3 or t.shape[0] < 1 or t.shape[1] < 1:
                raise ValueError("every image must be a uint8 tensor [H,W,3]")      # the kernels read the tensors' memory as such
        invert = self.depth_model_type in [0, 7, 8, 9, 10]
        if self.pix2pix_model is not None:
            return [self.pix2pix_model.run(t.cpu().numpy(), self.boost_rmax, to_host=False) for t in images], invert
        dev = self.depth_model.device
        groups = {}
        for i, t in enumerate(images):
            groups.setdefault(self.net_size(t.shape[1], t.shape[0], net_width, net_height), []).append(i)
        out = [None] * len(images)
        for idx in groups.values():
            desc = _lib.Ragged([tuple(images[i].shape[:2]) for i in idx], 3, dev)
            packed = torch.cat([images[i].to(dev).reshape(-1) for i in idx])
            pred = self.depth_model.forward_ragged(packed, desc, net_width, net_height)
            for i, p in zip(idx, _lib.Ragged(desc.sizes, 1, None).split(pred)):
                out[i] = p
        return out, invert

    def get_raw_prediction(self, input, net_width, net_height):
        """Get prediction from the model currently loaded by the ModelHolder object (reference :375-403)."""
        import torch
        dev = _lib.require_cuda()
        img = np.asarray(input)
        if img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.uint8:
            img = np.asarray(input.convert('RGB')) if hasattr(input, 'convert') else img
        if self.pix2pix_model is not None:       # boost: net_width / net_height are ignored (reference :376-377, :399-401)
            return self.pix2pix_model.run(img, self.boost_rmax), self.depth_model_type in [0, 7, 8, 9, 10]
        t = torch.from_numpy(np.ascontiguousarray(img)).to(dev).unsqueeze(0)
        pred, invert = self.get_raw_prediction_batch(t, net_width, net_height)
        return pred[0].cpu().numpy(), invert
