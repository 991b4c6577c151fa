"""ORACLE (test infrastructure only — the product never imports this): plain-torch fp32 functional restatement of the
single-head ZoeDepth metric head, ZoeDepth-N (model type 7, softplus bins) and ZoeDepth-K (model type 8, "normed" bins), on
top of the same DPT-BEiT-L-384 core as ZoeDepth-NK, with seeded synthetic weights in the reference's checkpoint layout.

Follows the reference tree:
  dzoedepth/models/zoedepth/zoedepth_v1.py:124-192          ZoeDepth.forward (seed bins, attractors, log-binomial on
                                                            cat(out_conv, rel_depth))
  dzoedepth/models/layers/localbins_layers.py:29-68         SeedBinRegressor (normed) / SeedBinRegressorUnnormed
  dzoedepth/models/layers/attractor.py:60-136               AttractorLayer (normed; A_normed override) / AttractorLayerUnnormed
  dzoedepth/models/layers/dist_layers.py:72-121             ConditionalLogBinomial(33, 128, 64): 80 hidden
The layers, the log-binomial, PrepForMidas and the pad + flip TTA wrapper it shares with ZoeDepth-NK are oracle/zoedepth.py's.
The core's relative depth, the 33rd log-binomial input, is oracle/beit_dpt.forward's own prediction, returned next to the
hooked features.  Pinned against the reference module around a stub core by tests/test_zoedepth_n_k_cpu.py."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.zoedepth import _conditional_log_binomial, _conv1x1, _inv_attractor, _mlp2, infer, prep_for_midas

# ---------------------------------------------------------------------------------------------------------------------
# single-head ZoeDepth: ZoeDepth-N (model type 7) and ZoeDepth-K (model type 8), dzoedepth/models/zoedepth/zoedepth_v1.py:124-192
# with get_config("zoedepth", "infer") / config_version="kitti" (config_zoedepth.json, config_zoedepth_kitti.json).  Neither
# config sets min_depth / max_depth, so ZoeDepth.__init__'s defaults 1e-3 / 10 apply to both (K's output is clipped at 10 m).
# Pinned against the reference module around a stub core by tests/test_zoedepth_n_k_cpu.py.
# ---------------------------------------------------------------------------------------------------------------------
SINGLE_CONFIG = dict(n_bins=64, bin_embedding_dim=128, n_attractors=[16, 8, 4, 1], min_temp=0.0212, max_temp=50.0, min_depth=1e-3, max_depth=10.0)
SINGLE_VARIANTS = {"n": dict(bin_centers_type="softplus"), "k": dict(bin_centers_type="normed")}


def _attractor_single(x, b_prev, prev_emb, sd, prefix, n_attractors, normed, dmin, dmax):
    """AttractorLayerUnnormed / AttractorLayer (attractor.py:60-136) with interpolate=True, kind 'mean', attractor_type 'inv'.
    Returns (b_new, B_centers): the next level's unsorted b_prev and the centres this level hands on (sorted and clipped for
    the normed layer)."""
    x = x + F.interpolate(prev_emb, x.shape[-2:], mode="bilinear", align_corners=True)
    if normed:
        A = F.relu(_mlp2(x, sd, prefix, F.relu)) + 1e-3
        A = A[:, 0::2]                             # the A_normed override (attractor.py:104-106): attractor i is channel 2i
    else:
        A = F.softplus(_mlp2(x, sd, prefix, F.relu))
    assert A.shape[1] == n_attractors
    h, w = A.shape[-2:]
    b_centers = F.interpolate(b_prev, (h, w), mode="bilinear", align_corners=True)
    delta = torch.mean(_inv_attractor(A.unsqueeze(2) - b_centers.unsqueeze(1)), dim=1)
    b_new = b_centers + delta
    if not normed:
        return b_new, b_new
    B_centers, _ = torch.sort((dmax - dmin) * b_new + dmin, dim=1)
    return b_new, torch.clip(B_centers, dmin, dmax)


def _seed_normed(x, sd, dmin, dmax):
    """SeedBinRegressor (localbins_layers.py:52-68), then b_prev = (centres - min) / (max - min) (zoedepth_v1.py:155-157)."""
    B = F.relu(_mlp2(x, sd, "seed_bin_regressor", F.relu)) + 1e-3
    widths = (dmax - dmin) * (B / B.sum(dim=1, keepdim=True))
    edges = torch.cumsum(F.pad(widths, (0, 0, 0, 0, 1, 0), mode="constant", value=dmin), dim=1)
    centres = 0.5 * (edges[:, :-1] + edges[:, 1:])
    return (centres - dmin) / (dmax - dmin)


def metric_head_single(features, rel_depth, sd, variant):
    """features = [out_conv, btlnck, x_block4, x_block3, x_block2, x_block1] (fp32 NCHW), rel_depth [N, h, w] = the core's own
    prediction (MidasCore return_rel_depth=True), variant 'n' or 'k'.  Returns metric depth [N, 1, H, W]."""
    normed = SINGLE_VARIANTS[variant]["bin_centers_type"] == "normed"
    cfg = SINGLE_CONFIG
    dmin, dmax = cfg["min_depth"], cfg["max_depth"]
    outconv, btlnck, x_blocks = features[0], features[1], features[2:]
    x = _conv1x1(btlnck, sd, "conv2")
    if normed:
        b_prev = _seed_normed(x, sd, dmin, dmax)
    else:
        b_prev = F.softplus(_mlp2(x, sd, "seed_bin_regressor", F.relu))                # SeedBinRegressorUnnormed
    prev_emb = _mlp2(x, sd, "seed_projector", F.relu)
    b_centers = b_emb = None
    for i, xb in enumerate(x_blocks):
        b_emb = _mlp2(xb, sd, f"projectors.{i}", F.relu)
        b_prev, b_centers = _attractor_single(b_emb, b_prev, prev_emb, sd, f"attractors.{i}", cfg["n_attractors"][i], normed, dmin, dmax)
        prev_emb = b_emb
    rel = F.interpolate(rel_depth.unsqueeze(1), size=outconv.shape[2:], mode="bilinear", align_corners=True)
    last = torch.cat([outconv, rel], dim=1)
    b_emb = F.interpolate(b_emb, last.shape[-2:], mode="bilinear", align_corners=True)
    probs = _conditional_log_binomial(last, b_emb, sd, "conditional_log_binomial", cfg["n_bins"])
    b_centers = F.interpolate(b_centers, probs.shape[-2:], mode="bilinear", align_corners=True)
    return torch.sum(probs * b_centers, dim=1, keepdim=True)


def split_state_dict(sd):
    """ZoeDepth checkpoint -> (MiDaS core weights without "core.core.", head weights at the top level)."""
    core_sd = {k[len("core.core."):]: v for k, v in sd.items() if k.startswith("core.core.")}
    head_sd = {k: v for k, v in sd.items() if not k.startswith("core.")}
    return core_sd, head_sd


@torch.no_grad()
def get_raw_prediction_single(rgb_uint8, sd, variant, net_w=512, net_h=384, core_name="beitl16_384"):
    """ModelHolder.get_raw_prediction for model types 7 ('n') and 8 ('k'): (float32 metric depth [H,W], invert=True).  The core's
    relative depth (beit_dpt.forward's prediction) is the 33rd input of the log-binomial."""
    import numpy as np
    from oracle import beit_dpt
    core_sd, head_sd = split_state_dict(sd)

    def model_fn(x):
        xin = prep_for_midas(x, net_w, net_h)
        rel, feats = beit_dpt.forward(core_sd, xin, core_name, return_features=True)
        return metric_head_single(feats, rel, head_sd, variant)

    img = np.asarray(rgb_uint8)
    x = torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1).float().div(255.0).unsqueeze(0)
    out = infer(model_fn, x, pad_input=True, with_flip_aug=True)
    return out.squeeze().cpu().numpy(), True


def make_zoedepth_single_head_state_dict(variant, feat_ch=256, out_conv_ch=32, seed=0, dtype=torch.float32, gain=1.0):
    """Seeded single-head ZoeDepth metric-head weights (ZoeDepth-N: variant 'n', softplus bins; ZoeDepth-K: 'k', normed bins) in
    the checkpoint layout of dzoedepth/models/zoedepth/zoedepth_v1.py (keys as `ZoeDepth.state_dict()` minus "core."): 64 bins,
    128-d bin embedding, a 256-wide seed MLP, 128-wide projector and attractor MLPs, attractors [16, 8, 4, 1] (twice the channels
    for the normed layers), log-binomial on 32 + 1 + 128 inputs with 80 hidden.  tests/test_zoedepth_n_k_cpu.py checks the layout
    against the reference module.  `gain` as in make_zoedepth_head_state_dict."""
    if variant not in ("n", "k"):
        raise ValueError(f"variant must be 'n' or 'k', not {variant!r}")
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def conv(key, cout, cin):
        sd[key + ".weight"] = (torch.randn(cout, cin, 1, 1, generator=g) * (0.05 if gain == 1.0 else gain * cin ** -0.5)).to(dtype)
        sd[key + ".bias"] = (torch.randn(cout, generator=g) * (0.02 if gain == 1.0 else 0.3)).to(dtype)

    emb, nb = 128, 64
    conv("conv2", feat_ch, feat_ch)
    conv("seed_bin_regressor._net.0", 256, feat_ch)
    conv("seed_bin_regressor._net.2", nb, 256)
    conv("seed_projector._net.0", 128, feat_ch)
    conv("seed_projector._net.2", emb, 128)
    for i in range(4):
        conv(f"projectors.{i}._net.0", 128, feat_ch)
        conv(f"projectors.{i}._net.2", emb, 128)
    for i, n in enumerate((16, 8, 4, 1)):
        conv(f"attractors.{i}._net.0", 128, emb)
        conv(f"attractors.{i}._net.2", 2 * n if variant == "k" else n, 128)
    cin = out_conv_ch + 1 + emb
    conv("conditional_log_binomial.mlp.0", cin // 2, cin)
    conv("conditional_log_binomial.mlp.2", 4, cin // 2)
    return sd
