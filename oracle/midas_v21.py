"""ORACLE (test infrastructure only — the product never imports this): plain-torch fp32 functional restatement of MiDaS v2.1
inference (midas_v21, model type 5).

Follows /root/reference:
  src/depthmap_generation.py:375-403,455-499  get_raw_prediction + estimatemidas: Resize(keep_aspect_ratio, multiple of 32,
                                              "upper_bound", INTER_CUBIC) of the BGR-swapped float64 image, ImageNet mean / std,
                                              the network, bicubic align_corners=False back to the image size
  dmidas/transforms.py:48-231                 Resize.get_size / NormalizeImage / PrepareForNet
  dmidas/midas_net.py:12-76                   MidasNet: encoder, layer{1..4}_rn, refinenet4..1, output_conv
  dmidas/blocks.py:60-66,136-320              _make_resnet_backbone (pretrained.layer1 = conv1, bn1, relu, maxpool, layer1),
                                              _make_scratch (3x3, no bias), Interpolate (align_corners=False),
                                              ResidualConvUnit (in-place ReLU: the skip operand is relu(x)), FeatureFusionBlock
The encoder is torchvision's resnext101_32x8d (the WSL hub entry); its bottleneck is oracle.leres's, under MidasNet's key names.
BatchNorm is evaluated in inference mode (eps 1e-5).  state_dict keys are the reference module's (`MidasNet.state_dict()`).
Pinned by a strict load of a seeded state_dict (make_state_dict below) into the reference module (tests/test_midas_v21_cpu.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import leres

LAYERS = (3, 4, 23, 3)
MEAN = np.array([0.485, 0.456, 0.406])
STD = np.array([0.229, 0.224, 0.225])


def block_prefix(li, bi):
    """bottleneck bi of stage li: pretrained.layer1 is Sequential(conv1, bn1, relu, maxpool, layer1), so its blocks sit under .4"""
    return f"pretrained.layer1.4.{bi}" if li == 1 else f"pretrained.layer{li}.{bi}"


def encoder(sd, x):
    """pretrained.layer1..layer4 -> features at 1/4 .. 1/32"""
    x = F.relu(leres._bn(F.conv2d(x, sd["pretrained.layer1.0.weight"], stride=2, padding=3), sd, "pretrained.layer1.1"))
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    feats = []
    for li, nblocks in enumerate(LAYERS, start=1):
        for bi in range(nblocks):
            x = leres._bottleneck(x, sd, block_prefix(li, bi), 2 if (bi == 0 and li > 1) else 1, bi == 0)
        feats.append(x)
    return feats


def _conv(sd, key, x, padding=1):
    return F.conv2d(x, sd[key + ".weight"], sd.get(key + ".bias"), padding=padding)


def _rcu(sd, key, x):
    """ResidualConvUnit: nn.ReLU(inplace=True) rewrites x, so the skip operand is relu(x)"""
    x = F.relu(x)
    return _conv(sd, key + ".conv2", F.relu(_conv(sd, key + ".conv1", x))) + x


def _fusion(sd, key, x0, x1=None):
    out = x0 if x1 is None else x0 + _rcu(sd, key + ".resConfUnit1", x1)
    out = _rcu(sd, key + ".resConfUnit2", out)
    return F.interpolate(out, scale_factor=2, mode="bilinear", align_corners=True)


def forward(sd, x):
    """MidasNet.forward: x [B, 3, H, W] (H, W multiples of 32) -> [B, H, W].  The weights are read as `sd[k].float()`, so a
    precision.HalfView runs the whole network in fp16."""
    sd = {k: v.float() for k, v in sd.items()}
    l1, l2, l3, l4 = encoder(sd, x)
    rn = [_conv(sd, f"scratch.layer{i + 1}_rn", f) for i, f in enumerate((l1, l2, l3, l4))]
    path = _fusion(sd, "scratch.refinenet4", rn[3])
    path = _fusion(sd, "scratch.refinenet3", path, rn[2])
    path = _fusion(sd, "scratch.refinenet2", path, rn[1])
    path = _fusion(sd, "scratch.refinenet1", path, rn[0])
    o = _conv(sd, "scratch.output_conv.0", path)
    o = F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=False)
    o = F.relu(_conv(sd, "scratch.output_conv.2", o))
    o = F.relu(_conv(sd, "scratch.output_conv.4", o, padding=0))
    return o.squeeze(1)


def _constrain(x, multiple_of, max_val):
    y = int(np.round(x / multiple_of) * multiple_of)
    if y > max_val:
        y = int(np.floor(x / multiple_of) * multiple_of)
    if y < 0:
        y = int(np.ceil(x / multiple_of) * multiple_of)
    return y


def net_size(width, height, net_w, net_h, multiple_of=32):
    """Resize.get_size, 'upper_bound' with keep_aspect_ratio (transforms.py:106-160) -> (width, height); a side may be 0"""
    scale_h, scale_w = net_h / height, net_w / width
    if scale_w < scale_h:
        scale_h = scale_w
    else:
        scale_w = scale_h
    return _constrain(scale_w * width, multiple_of, net_w), _constrain(scale_h * height, multiple_of, net_h)


def preprocess(img, net_w, net_h):
    """estimatemidas' transform of the float image it is handed -> float32 tensor [1, 3, nh, nw]"""
    import cv2
    w, h = net_size(img.shape[1], img.shape[0], net_w, net_h)
    x = cv2.resize(img, (w, h), interpolation=cv2.INTER_CUBIC)
    x = (x - MEAN) / STD
    return torch.from_numpy(np.ascontiguousarray(np.transpose(x, (2, 0, 1))).astype(np.float32)).unsqueeze(0)


@torch.no_grad()
def estimatemidas(img, sd, net_w, net_h):
    """the reference function (:455-499) in fp32 for whatever float image it is handed -> float32 [H, W]"""
    pred = forward(sd, preprocess(np.asarray(img), net_w, net_h))
    return F.interpolate(pred.unsqueeze(1), size=np.asarray(img).shape[:2], mode="bicubic", align_corners=False).squeeze().cpu().numpy()


@torch.no_grad()
def get_raw_prediction(rgb_uint8, sd, net_w=384, net_h=384):
    """ModelHolder.get_raw_prediction for model type 5 -> (float32 [H, W], invert=False).  The holder hands estimatemidas
    `cv2.cvtColor(image, COLOR_BGR2RGB) / 255.0` (:381)."""
    import cv2
    img = cv2.cvtColor(np.asarray(rgb_uint8), cv2.COLOR_BGR2RGB) / 255.0
    return estimatemidas(img, sd, net_w, net_h), False


def make_state_dict(seed=0, dtype=torch.float32):
    """Seeded synthetic state_dict with the keys and shapes of the reference's MidasNet(None).state_dict() (dmidas/midas_net.py,
    dmidas/blocks.py; torchvision's resnext101_32x8d as the encoder; `num_batches_tracked` buffers left out).  The encoder follows
    synth_weights.make_leres_state_dict's recipe (bn3 scaled down so 33 residual blocks keep activations O(1)); the final 1x1 conv has
    non-negative weights and a positive bias, so the depth after its ReLU is positive everywhere and varies."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def conv(key, co, ci, k, bias=False):
        sd[key + '.weight'] = (torch.randn(co, ci, k, k, generator=g) * (1.0 / (ci * k * k) ** 0.5)).to(dtype)
        if bias:
            sd[key + '.bias'] = (0.05 * torch.randn(co, generator=g)).to(dtype)

    def bn(key, c, gain=1.0):
        sd[key + '.weight'] = (gain + 0.05 * torch.randn(c, generator=g)).to(dtype)
        sd[key + '.bias'] = (0.05 * torch.randn(c, generator=g)).to(dtype)
        sd[key + '.running_mean'] = (0.1 * torch.randn(c, generator=g)).to(dtype)
        sd[key + '.running_var'] = (0.5 + torch.rand(c, generator=g)).to(dtype)

    conv('pretrained.layer1.0', 64, 3, 7)
    bn('pretrained.layer1.1', 64)
    inplanes = 64
    for li, (planes, nb) in enumerate(zip((64, 128, 256, 512), (3, 4, 23, 3)), start=1):
        width = planes * 8 // 64 * 32
        for bi in range(nb):
            p = f'pretrained.layer1.4.{bi}' if li == 1 else f'pretrained.layer{li}.{bi}'
            conv(p + '.conv1', width, inplanes, 1)
            bn(p + '.bn1', width)
            conv(p + '.conv2', width, width // 32, 3)
            bn(p + '.bn2', width)
            conv(p + '.conv3', planes * 4, width, 1)
            bn(p + '.bn3', planes * 4, gain=0.3)
            if bi == 0:
                conv(p + '.downsample.0', planes * 4, inplanes, 1)
                bn(p + '.downsample.1', planes * 4)
            inplanes = planes * 4
    for i, ci in enumerate((256, 512, 1024, 2048), start=1):
        conv(f'scratch.layer{i}_rn', 256, ci, 3)
    for i in range(1, 5):
        for u in (1, 2):
            for c in (1, 2):
                conv(f'scratch.refinenet{i}.resConfUnit{u}.conv{c}', 256, 256, 3, bias=True)
    conv('scratch.output_conv.0', 128, 256, 3, bias=True)
    conv('scratch.output_conv.2', 32, 128, 3, bias=True)
    conv('scratch.output_conv.4', 1, 32, 1, bias=True)
    # the last two convolutions see non-negative inputs: non-negative weights and a positive bias keep the depth positive
    sd['scratch.output_conv.4.weight'] = sd['scratch.output_conv.4.weight'].abs()
    sd['scratch.output_conv.4.bias'] = torch.full((1,), 0.1, dtype=dtype)
    return sd
