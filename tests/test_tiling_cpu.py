"""CPU: tiling mode (circular padding in every padded convolution of the depth networks), the parts that need no GPU.

- The circular oracle (tests/circular_oracle.py around the fp32 functional oracles) equals the reference's own modules with their
  nn.Conv2d set circular the way its tiling hijack does (src/depthmap_generation.py:251-260): DepthAnythingV2 S / B and RelDepthModel.
  The reference's results and the number of padded Conv2d modules a forward reaches are stored in tests/golden/tiling_pin.npz;
      DEPTHMAP_MINT_GOLDEN=1 python -m pytest tests/test_tiling_cpu.py
  recomputes them where the reference tree is present.
- The op-level engines with circular=True, recorded against the fake library of test_engine_trace_cpu.py: the call sequence is the
  zero-padded one with the circular entry point at every padded-convolution call site and nothing else changed, there is one such
  call per padded convolution of the oracle, and the launch counter equals the kernels issued.
"""
from __future__ import annotations

import os
import re

import numpy as np
import pytest

from circular_oracle import circular_convs, padded_conv2d_modules, set_circular
from oracle import ref_loader
from synth import synth_rgb
from test_engine_trace_cpu import _cpu, _planar, _rgb, _zoe_core, fake  # noqa: F401  (fake: the recording-library fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiling_pin.npz")
MINT = os.environ.get("DEPTHMAP_MINT_GOLDEN") == "1"
_stored = dict(np.load(GOLDEN)) if os.path.exists(GOLDEN) else {}
_minted = {}


def pinned(key, compute):
    """the reference's result for `key`: the stored one, or, when minting, compute()"""
    if MINT:
        _minted[key] = np.asarray(compute())
        return _minted[key]
    if key not in _stored:
        pytest.fail(f"no stored reference result for {key}: mint {GOLDEN} with the reference tree present")
    return _stored[key]


@pytest.fixture(scope="module", autouse=True)
def _write_minted():
    yield
    if MINT and _minted:
        np.savez_compressed(GOLDEN, **dict(_stored, **_minted))


def _count_forward(model, run):
    """run() with forward hooks on the padded convolutions of `model` -> (result, number of padded convolutions evaluated)"""
    n = [0]
    hooks = [m.register_forward_hook(lambda *a: n.__setitem__(0, n[0] + 1)) for m in padded_conv2d_modules(model)]
    try:
        out = run()
    finally:
        for h in hooks:
            h.remove()
    return out, n[0]


# ---- the circular oracle against the reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("encoder,hw,net", [("vits", (70, 98), 70), ("vitb", (70, 70), 70)])
def test_dav2_circular_oracle_equals_reference(encoder, hw, net):
    """get_raw_prediction (:375-403, :548-559) of the reference's DepthAnythingV2 with circular Conv2d layers"""
    import cv2
    import torch
    import torch.nn.functional as F
    from oracle import dav2 as odav2
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict(encoder, seed=1)
    cfg = odav2.CONFIGS[encoder]
    rgb = synth_rgb(hw[0], hw[1], 3)
    ref_count = []

    def reference():
        model = ref_loader.dav2_class()(encoder=encoder, features=cfg['features'], out_channels=cfg['out_channels']).eval()
        res = model.load_state_dict(sd, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        set_circular(model)
        img = cv2.cvtColor(np.asarray(rgb), cv2.COLOR_BGR2RGB) / 255.0
        with torch.no_grad():
            image = cv2.cvtColor((img * 255.1).astype('uint8'), cv2.COLOR_BGR2RGB)
            image, (h, w) = model.image2tensor(image, net)
            depth, n = _count_forward(model, lambda: model.forward(image.to('cpu')))
            depth = F.interpolate(depth[:, None], (h, w), mode="bilinear", align_corners=True)[0, 0]
        ref_count.append(n)
        return depth.cpu().numpy()
    want = pinned(f"dav2/{encoder}/{hw[0]}x{hw[1]}/{net}", reference)
    with circular_convs(odav2) as c:
        got, _ = odav2.get_raw_prediction(rgb, sd, encoder, net)
    with torch.no_grad():
        zero, _ = odav2.get_raw_prediction(rgb, sd, encoder, net)
    assert got.shape == want.shape == tuple(hw)
    assert float(np.abs(got - want).max()) <= 1e-5 * float(np.abs(want).max())
    assert float(np.abs(zero - want).max()) > 1e-3 * float(np.abs(want).max())      # circular padding is visible in the output
    assert c.padded == int(pinned(f"count/dav2/{encoder}", lambda: ref_count[0])) == 21


def test_leres_circular_oracle_equals_reference():
    """RelDepthModel.depth_model with circular Conv2d layers: the 7x7 stem (pad 3), the bottlenecks' grouped 3x3 convs (stride 1 and 2)
    and the decoder's FTB / FFM / AO convs"""
    import torch
    from oracle import leres, synth_weights
    sd = synth_weights.make_leres_state_dict(seed=2)
    x = torch.randn(1, 3, 64, 96, generator=torch.Generator().manual_seed(4))
    ref_count = []

    def reference():
        ref_loader.bootstrap()
        from lib.multi_depth_model_woauxi import RelDepthModel
        model = RelDepthModel(backbone="resnext101").eval()
        res = model.load_state_dict(sd, strict=False)
        assert not res.unexpected_keys and all(k.endswith("num_batches_tracked") for k in res.missing_keys)
        set_circular(model)
        with torch.no_grad():
            out, n = _count_forward(model, lambda: model.depth_model(x))
        ref_count.append(n)
        return out.numpy()
    want = torch.from_numpy(pinned("leres/network", reference))
    with torch.no_grad(), circular_convs(leres) as c:
        got = leres.forward(sd, x)
    with torch.no_grad():
        zero = leres.forward(sd, x)
    scale = want.abs().max().item()
    assert got.shape == want.shape == (1, 1, 64, 96) and scale > 0
    assert (got - want).abs().max().item() <= 1e-5 * scale
    assert (zero - want).abs().max().item() > 1e-3 * scale
    assert c.padded == int(pinned("count/leres", lambda: ref_count[0])) == 58


def test_circular_oracle_leaves_other_modules_alone():
    """only the modules named pad circularly; outside the block the oracle is zero padded again"""
    import torch
    import torch.nn.functional as F
    from oracle import dav2 as odav2
    from oracle import pix2pix
    x = torch.randn(1, 4, 5, 6, generator=torch.Generator().manual_seed(0))
    w = torch.randn(3, 4, 3, 3, generator=torch.Generator().manual_seed(1))
    with circular_convs(odav2) as c:
        assert pix2pix.F is F
        got = odav2.F.conv2d(x, w, padding=1)
        assert torch.equal(odav2.F.conv2d(x, w), F.conv2d(x, w))                # unpadded: unchanged, not counted
    assert odav2.F is F and c.padded == 1
    torch.testing.assert_close(got, F.conv2d(F.pad(x, (1, 1, 1, 1), mode="circular"), w), rtol=0, atol=0)


# ---- the engines' call sequences with tiling on ---------------------------------------------------------------------------------
CIRCULAR = {"dm_conv3x3_circular_ex": "dm_conv3x3_ex", "dm_im2col_s2_circular_f16": "dm_im2col_s2_f16",
            "dm_leres_stem_im2col_circular": "dm_leres_stem_im2col", "dm_leres_stem_im2col_f32_circular": "dm_leres_stem_im2col_f32",
            "dm_leres_stem_im2col_f32_batch_circular": "dm_leres_stem_im2col_f32_batch"}
ZERO_PADDED = set(CIRCULAR.values())


def kernels(name, k):
    """kernels a recorded call issues: the circular conv is the halo copy plus the implicit GEMM; the rest as recorded"""
    return 2 if name == "dm_conv3x3_circular_ex" else k


def _relabel(calls):
    """pointer and stream labels renumbered by first appearance: dropping the halo argument shifts the recorder's numbering, and
    every BoostPipeline makes its own side streams"""
    labels = {}

    def v(x):
        if isinstance(x, str) and re.fullmatch(r"(p|stream)\d+", x):
            return labels.setdefault(x, f"{x.rstrip('0123456789')}{len(labels)}")
        if isinstance(x, dict):
            return {k: v(y) for k, y in x.items()}
        return x
    return [[n, [v(a) for a in args]] for n, args in calls]


def _record(fake, run):
    """run() -> launch counter; returns (the calls recorded meanwhile, the counter)"""
    start = len(fake.calls)
    launches = run()
    return fake.calls[start:], launches


def _compare(fake, make_and_run, per_forward, forwards):
    """make_and_run(circular) builds the engine(s), runs them and returns their launch counter.  The circular trace, with each
    circular entry point renamed to its zero-padded one and the halo argument dropped, equals the zero-padded trace; there are
    per_forward circular calls per network forward; the counter equals the kernels issued."""
    zero_calls, _ = _record(fake, lambda: make_and_run(False))
    circ_calls, launches = _record(fake, lambda: make_and_run(True))
    if forwards is None:            # one stem call per network forward
        forwards = sum(n.startswith("dm_leres_stem_im2col") for n, _, _ in circ_calls)
    assert not any(n in ZERO_PADDED for n, _, _ in circ_calls), "a zero-padded convolution ran in tiling mode"
    halos = {args[1] for n, args, _ in circ_calls if n == "dm_conv3x3_circular_ex"}
    assert 1 <= len(halos) <= forwards, "a pooled halo scratch per engine and shape"
    mapped = [[CIRCULAR.get(n, n), args[:1] + args[2:] if n == "dm_conv3x3_circular_ex" else args] for n, args, _ in circ_calls]
    assert _relabel(mapped) == _relabel([[n, a] for n, a, _ in zero_calls])
    n_circ = sum(n in CIRCULAR for n, _, _ in circ_calls)
    assert n_circ == per_forward * forwards, (n_circ, per_forward, forwards)
    assert launches == sum(kernels(n, k) for n, _, k in circ_calls)
    return circ_calls


def _oracle_count(module, run):
    import torch
    with torch.no_grad(), circular_convs(module) as c:
        run()
    return c.padded


def test_tiling_trace_dav2(fake):
    import torch
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import dav2 as odav2
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=0)
    per = _oracle_count(odav2, lambda: odav2.forward(sd, torch.zeros(1, 3, 70, 98), 'vits'))

    def run(circular):
        eng = DepthAnythingV2Engine(sd, 'vits', _cpu(), circular=circular)
        eng.forward_batch(_rgb(2, 60, 80, 1), 70)
        return eng.ops.launches
    _compare(fake, run, per, 1)


@pytest.mark.parametrize("name", ["beit_tiny", "vit_tiny"])
def test_tiling_trace_dpt(fake, name):
    import torch
    from depthmap_b200.depthmap_generation import DptBeitEngine, DptVitEngine
    from oracle import beit_dpt, synth_weights
    sd = synth_weights.make_beit_dpt_state_dict(name, seed=0)
    per = _oracle_count(beit_dpt, lambda: beit_dpt.forward(sd, torch.zeros(1, 3, 64, 96), name))
    cls = DptBeitEngine if name == "beit_tiny" else DptVitEngine

    def run(circular):
        eng = cls(sd, name, _cpu(), circular=circular)
        eng.forward_batch(_rgb(2, 60, 80, 1), 96)
        eng.forward_crops(_planar(100, 120, 2), [(0, 0, 64, 64), (10, 20, 48, 80), (30, 5, 64, 64)], 64)
        return eng.ops.launches
    _compare(fake, run, per, 3)       # one batched forward, then two crop groups (64 x 64 and 32 x 64 nets)


@pytest.mark.parametrize("variant", ["nk", "n", "k"])
def test_tiling_trace_zoedepth(fake, variant):
    import torch
    from depthmap_b200.depthmap_generation import ZoeDepthEngine, ZoeDepthNKEngine
    from oracle import beit_dpt, synth_weights
    from oracle import zoedepth_single as ozs
    sd = _zoe_core('beit_tiny', 0)
    feat = beit_dpt.CONFIGS['beit_tiny']['features']
    sd.update(synth_weights.make_zoedepth_head_state_dict(feat_ch=feat, seed=100) if variant == "nk" else
              ozs.make_zoedepth_single_head_state_dict(variant, feat_ch=feat, seed=100))
    core = {k[len("core.core."):]: v for k, v in sd.items() if k.startswith("core.core.")}
    per = _oracle_count(beit_dpt, lambda: beit_dpt.forward(core, torch.zeros(1, 3, 64, 96), 'beit_tiny', return_features=True))

    def run(circular):
        if variant == "nk":
            eng = ZoeDepthNKEngine(sd, _cpu(), core_name='beit_tiny', circular=circular)
        else:
            eng = ZoeDepthEngine(sd, _cpu(), variant, core_name='beit_tiny', circular=circular)
        eng.forward_batch(_rgb(2, 60, 80, 1), 96)
        return eng.ops.launches
    _compare(fake, run, per, 1)       # the 2B test-time-augmentation forwards run as one batch


@pytest.fixture(scope="module")
def leres_sd():
    from oracle import synth_weights
    return synth_weights.make_leres_state_dict(seed=0)


def _leres_per_forward(sd):
    import torch
    from oracle import leres
    return _oracle_count(leres, lambda: leres.forward(sd, torch.zeros(1, 3, 64, 64)))


def test_tiling_trace_leres(fake, leres_sd):
    from depthmap_b200.depthmap_generation import LeresEngine

    def run(circular):
        eng = LeresEngine(leres_sd, _cpu(), circular=circular)
        eng.forward_batch(_rgb(1, 60, 80, 1), 64)
        eng.forward_batch(_rgb(1, 64, 64, 2), 64)
        eng.forward_batch(None, 64, planar=(_planar(100, 120, 2), (10, 20, 64, 64)))
        eng.forward_crops(_planar(100, 120, 2), [(0, 0, 64, 64), (10, 20, 64, 64)], 64)
        return eng.ops.launches
    _compare(fake, run, _leres_per_forward(leres_sd), 4)


def test_tiling_trace_boost_leres(fake, leres_sd):
    """BOOST with tiling: a circular base network and the usual merge network, whose calls do not change"""
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import LeresEngine
    from oracle import synth_weights
    p2p = synth_weights.make_pix2pix_state_dict(seed=0)

    def run(circular):
        depth = LeresEngine(leres_sd, _cpu(), circular=circular)
        pipe = BoostPipeline(depth, UnetMergeEngine(p2p, _cpu()), _cpu(), 0)
        pipe.run(synth_rgb(300, 420, 12), 1600)
        return pipe.ops.launches + depth.ops.launches + pipe.merge.ops.launches
    calls = _compare(fake, run, _leres_per_forward(leres_sd), None)
    assert sum(n.startswith("dm_leres_stem_im2col") for n, _, _ in calls) >= 2
