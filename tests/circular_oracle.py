"""Tiling mode in the fp32 oracles: circular padding for every padded conv2d of chosen oracle modules.

The reference's tiling mode sets padding_mode = 'circular' on every nn.Conv2d of the depth network (src/depthmap_generation.py:251-260).
PyTorch evaluates such a layer as conv2d(F.pad(x, (p, p, p, p), mode='circular'), w, stride=s, padding=0).  The functional oracles
call `F.conv2d` through their module's `F`; `circular_convs(module, ...)` swaps that name for a view of torch.nn.functional whose
conv2d does exactly this when the padding is non-zero, and counts those calls.  Only the modules named are affected, so the
pix2pix merge network, ConvTranspose, pooling, F.pad and interpolation keep their zero padding / behaviour, as in the reference."""
from __future__ import annotations

import contextlib

import torch.nn.functional as _F


class CircularFunctional:
    """torch.nn.functional with a circular-padding conv2d; `padded` counts the padded convolutions evaluated"""

    def __init__(self):
        self.padded = 0

    def __getattr__(self, name):
        return getattr(_F, name)

    def conv2d(self, input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
        ph, pw = (padding, padding) if isinstance(padding, int) else tuple(padding)
        if ph or pw:
            self.padded += 1
            input = _F.pad(input, (pw, pw, ph, ph), mode="circular")
            padding = 0
        return _F.conv2d(input, weight, bias, stride, padding, dilation, groups)


@contextlib.contextmanager
def circular_convs(*modules):
    """Within the block, the padded conv2d calls of `modules` (oracle modules that `import torch.nn.functional as F`) pad circularly.
    Yields the CircularFunctional, whose `padded` counts them."""
    view = CircularFunctional()
    saved = [(m, m.F) for m in modules]
    for m in modules:
        m.F = view
    try:
        yield view
    finally:
        for m, f in saved:
            m.F = f


def padded_conv2d_modules(model):
    """the nn.Conv2d / nn.Conv1d modules of `model` the reference's hijack sets circular (exact type, as it checks), with non-zero padding"""
    import torch
    return [m for m in model.modules() if type(m) in (torch.nn.Conv2d, torch.nn.Conv1d) and any(p != 0 for p in m.padding)]


def set_circular(model):
    """the reference's tiling hijack (src/depthmap_generation.py:251-260) on a module"""
    import torch
    for m in model.modules():
        if type(m) in (torch.nn.Conv2d, torch.nn.Conv1d):
            m.padding_mode = "circular"
    return model
