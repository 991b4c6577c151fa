"""CPU: pins the oracle to the REAL reference.

What the reference computed on each test's seeded inputs is stored in tests/golden/oracle_pin.npz, so the comparisons run
anywhere.  Where a test fills a reference module with seeded weights, the order and shapes of that module's parameters and
buffers are stored too, and `_seeded_state` draws the identical tensors from them without the module.  With the reference
tree present (oracle/ref_loader.py: DEPTHMAP_REFERENCE_ROOT),

    DEPTHMAP_MINT_GOLDEN=1 python -m pytest tests/test_oracle_pin.py

runs the reference again and replaces the keys it computed (keys of tests that did not run are kept); outputs larger than
the 1 MB file limit allows are stored strided, and the network pins have a file of their own (oracle_pin_nets.npz)."""
import json
import os
import warnings

import numpy as np
import pytest

from oracle import normalmap as onm
from oracle import ref_loader
from oracle import stereo as ost
from synth import noise_depth_u16, noise_rgb, synth_depth_u16, synth_rgb

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MINT = os.environ.get("DEPTHMAP_MINT_GOLDEN") == "1"
_stored, _minted = {}, {}


def _store(name):
    if name not in _stored:
        path = os.path.join(GOLDEN_DIR, name + ".npz")
        _stored[name] = dict(np.load(path)) if os.path.exists(path) else {}
        _minted[name] = {}
    return _stored[name], _minted[name]


def pinned(key, compute, store="oracle_pin"):
    """The reference's result for `key` (an array, or a list of arrays): the stored one, or, when minting, compute()."""
    stored, minted = _store(store)
    if MINT:
        val = compute()
        vals = val if isinstance(val, (list, tuple)) else [val]
        for i, v in enumerate(vals):
            minted[f"{key}#{i}"] = np.asarray(v)
        minted[f"{key}#n"] = np.asarray(len(vals) if isinstance(val, (list, tuple)) else -1)
    src = minted if MINT else stored
    if f"{key}#n" not in src:
        pytest.fail(f"no stored reference result for {key}: mint tests/golden/oracle_pin.npz with the reference tree present")
    n = int(src[f"{key}#n"])
    return src[f"{key}#0"] if n < 0 else [src[f"{key}#{i}"] for i in range(n)]


def pinned_json(key, compute, store="oracle_pin"):
    return json.loads(str(pinned(key, lambda: np.asarray(json.dumps(compute())), store)))


@pytest.fixture(scope="module", autouse=True)
def _write_minted():
    yield
    if MINT:
        for name, minted in _minted.items():
            if minted:                             # a partial run replaces its own keys and keeps the others
                np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **dict(_stored[name], **minted))


NETS = "oracle_pin_nets"


def _layout(module):
    """[[name, shape, dtype] ...] of a module's parameters and of its buffers, each in the module's own order."""
    def rows(it):
        return [[n, list(t.shape), str(t.dtype).replace("torch.", "")] for n, t in it]
    kept = set(module.state_dict())                # buffers registered as non-persistent are not part of a state dict
    return {"parameters": rows(module.named_parameters()), "buffers": rows((n, b) for n, b in module.named_buffers() if n in kept)}


def _seeded_state(layout, g, param_fn, buffer_fn=None):
    """The state dict a test gets by filling a module of this layout in place: param_fn(name, shape, g) per parameter in order,
    then buffer_fn per buffer (None = the buffer keeps its stored value, layout["buffer_values"]); drawing from `g` in the
    same order as the in-place fill gives the identical tensors."""
    import torch
    sd = {}
    for name, shape, _ in layout["parameters"]:
        sd[name] = param_fn(name, tuple(shape), g)
    for name, shape, dtype in layout["buffers"]:
        t = buffer_fn(name, tuple(shape), g) if buffer_fn else None
        if t is None:
            t = torch.tensor(layout.get("buffer_values", {}).get(name, 0), dtype=getattr(torch, dtype)).reshape(shape) if name in layout.get("buffer_values", {}) \
                else torch.zeros(shape, dtype=getattr(torch, dtype))
        sd[name] = t
    return sd


def _assert_same_state(sd, model_sd):
    import torch
    assert set(sd) == set(model_sd)
    for k in sd:
        assert sd[k].dtype == model_sd[k].dtype and torch.equal(sd[k], model_sd[k]), k


def ref():
    warnings.filterwarnings("ignore")
    return ref_loader.stereo_module(), ref_loader.normalmap_module()



@pytest.mark.parametrize("fill", ['none', 'naive', 'naive_interpolating', 'polylines_soft', 'polylines_sharp'])
def test_stereo_oracle_equals_reference(fill):
    rng = np.random.default_rng(11)
    for (h, w, seed, kind) in [(21, 67, 10, 'smooth'), (16, 50, 11, 'noise')]:
        img = synth_rgb(h, w, seed) if kind == 'smooth' else noise_rgb(h, w, seed)
        dep = synth_depth_u16(h, w, seed) if kind == 'smooth' else noise_depth_u16(h, w, seed)
        for rep in range(3):
            div, sep = float(rng.uniform(0.05, 15)), float(rng.uniform(-5, 5))
            bal, ex = float(rng.uniform(-1, 1)), float(rng.choice([1.0, 2.0]))
            a = pinned(f"stereo/{fill}/{kind}/{rep}", lambda: [np.asarray(x) for x in ref()[0].create_stereoimages(
                img, dep, div, sep, ['left-right', 'red-cyan-anaglyph'], bal, ex, fill)])
            b = ost.create_stereoimages(img, dep, div, sep, ['left-right', 'red-cyan-anaglyph'], bal, ex, fill)
            for x, y in zip(a, b):
                assert np.array_equal(np.asarray(x), np.asarray(y)), (fill, div, sep, bal, ex)


def test_stereo_oracle_float_depth_equals_reference():
    img = noise_rgb(12, 40, 5)
    dep = np.random.default_rng(5).random((12, 40)).astype(np.float32)
    for fill in ['naive', 'polylines_sharp']:
        a = pinned(f"stereo_float/{fill}", lambda: np.asarray(ref()[0].create_stereoimages(img, dep, 3.0, fill_technique=fill)[0]))
        b = ost.create_stereoimages(img, dep, 3.0, fill_technique=fill)[0]
        assert np.array_equal(np.asarray(a), np.asarray(b))


def test_normalmap_oracle_equals_reference():
    for seed in range(3):
        dep = synth_depth_u16(30, 41, seed) if seed else noise_depth_u16(30, 41, seed)
        for (pb, sb, qb, inv) in [(None, 3, None, False), (None, 5, None, True), (None, None, None, False),
                                  (3, 3, 3, False), (None, 11, None, False), (9, 3, None, True), (None, 3, 11, False),
                                  (None, 31, None, False), (31, 3, 31, False)]:
            a = pinned(f"normalmap/{seed}/{pb}/{sb}/{qb}/{inv}", lambda: np.asarray(ref()[1].create_normalmap(dep, pb, sb, qb, inv)))
            b = onm.create_normalmap(dep, pb, sb, qb, inv, return_array=True)
            assert np.array_equal(a, b), (seed, pb, sb, qb, inv)


# ---------------------------------------------------------------------------------------------------------------------
# D7 (round-2 row): the ZoeDepth-NK metric head oracle against the reference module built around a stub core
# ---------------------------------------------------------------------------------------------------------------------
def _zoedepth_feats(g, base_hw):
    import torch
    h, w = base_hw
    shapes = [(32, 16 * h, 16 * w), (256, h, w), (256, 2 * h, 2 * w), (256, 4 * h, 4 * w), (256, 8 * h, 8 * w), (256, 16 * h, 16 * w)]
    feats = [torch.randn(2, c, hh, ww, generator=g) * 0.7 for c, hh, ww in shapes]
    feats[0] = feats[0].abs()                      # out_conv is a post-ReLU activation in the core
    return feats


def _zoedepth_param(name, shape, g):               # seeded weights with enough spread to exercise every branch
    import torch
    t = torch.randn(shape, generator=g) * (0.05 if len(shape) > 1 else 0.02)
    return t + 1.0 if name.endswith("norm1.weight") or name.endswith("norm2.weight") else t


def _zoedepth_inputs(seed, base_hw):
    """feats and head state dict of _zoedepth_reference_head(seed, base_hw), without the reference."""
    import torch
    g = torch.Generator().manual_seed(seed)
    feats = _zoedepth_feats(g, base_hw)

    def reference():
        model, _, sd = _zoedepth_reference_head(seed, base_hw)
        lay = _layout(model)
        lay["buffer_values"] = {n: b.tolist() for n, b in model.named_buffers()}
        return lay
    layout = pinned_json("zoedepth_head/layout", reference, NETS)
    sd = _seeded_state(layout, g, _zoedepth_param)
    if MINT:
        _assert_same_state(sd, _zoedepth_reference_head(seed, base_hw)[2])
    return feats, sd


def _zoedepth_reference_head(seed, base_hw):
    import torch
    import torch.nn as nn
    ref_loader.bootstrap()
    from dzoedepth.models.zoedepth_nk.zoedepth_nk_v1 import ZoeDepthNK
    from oracle import zoedepth as ozd
    g = torch.Generator().manual_seed(seed)
    feats = _zoedepth_feats(g, base_hw)

    class StubCore(nn.Module):                     # hands the head fixed activations (MidasCore.forward, midas.py:258-276)
        output_channels = (256, 256, 256, 256, 256)

        def forward(self, x, denorm=False, return_rel_depth=False):
            return torch.zeros(x.shape[0], x.shape[2], x.shape[3]), [f.clone() for f in feats]

    cfg = {k: ozd.CONFIG[k] for k in ("bin_embedding_dim", "n_attractors", "attractor_alpha", "attractor_gamma", "min_temp", "max_temp")}

    class AttrDict(dict):                          # the reference reads its config entries as attributes (EasyDict)
        __getattr__ = dict.__getitem__

    model = ZoeDepthNK(StubCore(), bin_conf=[AttrDict(c) for c in ozd.CONFIG["bin_conf"]], bin_centers_type="softplus", attractor_kind="mean",
                       attractor_type="inv", memory_efficient=True, **cfg).eval()
    with torch.no_grad():
        for name, p in model.named_parameters():
            p.copy_(_zoedepth_param(name, tuple(p.shape), g))
    sd = {k: v.detach().clone() for k, v in model.state_dict().items() if not k.startswith("core.")}
    return model, feats, sd


@pytest.mark.parametrize("seed,base_hw", [(0, (3, 4)), (1, (4, 3)), (2, (2, 2))])
def test_zoedepth_head_oracle_equals_reference(seed, base_hw):
    import torch
    from oracle import zoedepth as ozd
    feats, sd = _zoedepth_inputs(seed, base_hw)

    def reference():
        model = _zoedepth_reference_head(seed, base_hw)[0]
        with torch.no_grad():
            out = model(torch.zeros(2, 3, feats[0].shape[2], feats[0].shape[3]))
        return [out["domain_logits"].numpy(), out["metric_depth"].numpy()]
    want_logits, want_depth = [torch.from_numpy(a) for a in pinned(f"zoedepth_head/{seed}", reference, NETS)]
    with torch.no_grad():
        got_depth, got_logits, name = ozd.metric_head(feats, sd)
    assert torch.equal(got_logits, want_logits) or (got_logits - want_logits).abs().max() < 1e-5
    err = (got_depth - want_depth).abs().max().item()
    assert err <= 1e-5 * want_depth.abs().max().item(), (name, err)


@pytest.mark.parametrize("pad,flip", [(True, True), (True, False), (False, True)])
def test_zoedepth_tta_wrapper_equals_reference(pad, flip):
    """DepthModel.infer (pad + flip augmentation) around the same head: the stub core ignores its input, so this pins the
    padding arithmetic, the bicubic resize back to the padded size, the crop and the flip average."""
    import torch
    from oracle import zoedepth as ozd
    feats, sd = _zoedepth_inputs(3, (2, 3))
    x = torch.rand(2, 3, 40, 56, generator=torch.Generator().manual_seed(5))

    def reference():
        with torch.no_grad():
            return _zoedepth_reference_head(3, (2, 3))[0].infer(x, pad_input=pad, with_flip_aug=flip).numpy()
    want = torch.from_numpy(pinned(f"zoedepth_tta/{pad}/{flip}", reference, NETS))
    with torch.no_grad():
        got = ozd.infer(lambda t: ozd.metric_head(feats, sd)[0], x, pad_input=pad, with_flip_aug=flip)
    assert got.shape == want.shape == (2, 1, 40, 56)
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()


@pytest.mark.parametrize("smoothening", ["none", "experimental", "something-else"])
def test_video_normalisation_equals_reference(smoothening):
    """§8(f) rank 1 groundwork: cross-frame normalisation of video mode (src/video_mode.py:103-128)."""
    from oracle import video as ovid
    rng = np.random.default_rng(11)
    frames = [(rng.standard_normal((24, 32)) * (1 + 0.3 * i) + 0.1 * i).astype(np.float32) for i in range(7)]

    def reference():
        ref_loader.bootstrap()
        from src import video_mode
        return video_mode.process_predicitons([f.copy() for f in frames], smoothening)
    want = pinned(f"video/{smoothening}", reference)
    got = ovid.process_predictions([f.copy() for f in frames], smoothening)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w)


# ---------------------------------------------------------------------------------------------------------------------
# D8 (round-2 row): LeReS ResNeXt-101 32x8d + decoder oracle against the reference module with the same state_dict
# ---------------------------------------------------------------------------------------------------------------------
def _leres_param(name, shape, g):              # seeded weights / running statistics that keep activations O(1) through 100+ layers
    import torch
    if len(shape) == 4:
        return torch.randn(shape, generator=g) * (1.0 / (shape[1] * shape[2] * shape[3]) ** 0.5)
    if name.endswith(".weight"):
        return (0.3 if "bn3" in name else 1.0) + 0.05 * torch.randn(shape, generator=g)
    return 0.05 * torch.randn(shape, generator=g)


def _leres_buffer(name, shape, g):
    import torch
    if name.endswith("running_mean"):
        return 0.1 * torch.randn(shape, generator=g)
    if name.endswith("running_var"):
        return 0.5 + torch.rand(shape, generator=g)
    return None


_leres_model = []


def _leres_reference_model():
    """The reference's RelDepthModel filled with the seeded weights (built once per session, minting only)."""
    import torch
    if not _leres_model:
        ref_loader.bootstrap()
        from lib.multi_depth_model_woauxi import RelDepthModel
        model = RelDepthModel(backbone="resnext101").eval()
        g = torch.Generator().manual_seed(21)
        with torch.no_grad():
            for name, p in model.named_parameters():
                p.copy_(_leres_param(name, tuple(p.shape), g))
            for name, b in model.named_buffers():
                t = _leres_buffer(name, tuple(b.shape), g)
                if t is not None:
                    b.copy_(t)
        _leres_model.append(model)
    return _leres_model[0]


@pytest.fixture(scope="module")
def leres_sd():
    """The state dict of _leres_reference_model(), drawn from the stored layout of the reference module."""
    import torch
    layout = pinned_json("leres/layout", lambda: _layout(_leres_reference_model()), NETS)
    sd = _seeded_state(layout, torch.Generator().manual_seed(21), _leres_param, _leres_buffer)
    if MINT:
        model_sd = _leres_reference_model().state_dict()
        _assert_same_state(sd, model_sd)
    return sd


def test_leres_synthetic_state_dict_matches_reference_module():
    """oracle.synth_weights.make_leres_state_dict has exactly the reference module's keys and shapes (strict load, only the
    BatchNorm step counters are left out) and the oracle reproduces the reference module with it."""
    import torch
    from oracle import leres, synth_weights
    sd = synth_weights.make_leres_state_dict(seed=2)
    x = torch.randn(1, 3, 64, 96, generator=torch.Generator().manual_seed(4))

    def reference():
        ref_loader.bootstrap()
        from lib.multi_depth_model_woauxi import RelDepthModel
        model = RelDepthModel(backbone="resnext101").eval()
        res = model.load_state_dict(sd, strict=False)
        assert not res.unexpected_keys and all(k.endswith("num_batches_tracked") for k in res.missing_keys)
        with torch.no_grad():
            return model.depth_model(x).numpy()
    want = torch.from_numpy(pinned("leres_synth", reference))
    with torch.no_grad():
        got = leres.forward(sd, x)
    assert torch.isfinite(want).all() and want.abs().max().item() > 1e-3
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()


def test_leres_network_oracle_equals_reference(leres_sd):
    import torch
    from oracle import leres
    sd = leres_sd
    x = torch.randn(1, 3, 96, 128, generator=torch.Generator().manual_seed(4))

    def reference():
        with torch.no_grad():
            return _leres_reference_model().depth_model(x).numpy()
    want = torch.from_numpy(pinned("leres/network", reference, NETS))
    with torch.no_grad():
        got = leres.forward(sd, x)
    assert got.shape == want.shape == (1, 1, 96, 128)
    scale = want.abs().max().item()
    assert scale > 0 and torch.isfinite(want).all()
    assert (got - want).abs().max().item() <= 1e-5 * scale


def test_leres_estimate_equals_reference(leres_sd):
    """estimateleres (BGR flip, cv2 resize, scale_torch, cubic resize back) around the same network."""
    import torch
    from oracle import leres
    sd = leres_sd
    import cv2
    rgb = synth_rgb(70, 90, 3)
    img = cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0       # what ModelHolder.get_raw_prediction hands over (:381)

    def reference(image, w, h):
        ref_loader.bootstrap()
        from src import depthmap_generation as dg
        dg.depthmap_device = torch.device("cpu")
        return dg.estimateleres(image, _leres_reference_model(), w, h)
    want = pinned("leres/estimate_float", lambda: reference(img, 64, 96), NETS)
    got, invert = leres.get_raw_prediction(rgb, sd, 64, 96)
    assert invert is True and got.shape == want.shape == (70, 90)
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()
    want = pinned("leres/estimate_uint8", lambda: reference(rgb, 96, 64), NETS)   # and the function itself on a uint8 array
    got = leres.estimateleres(rgb, sd, 96, 64)
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


def _pix2pix_param(name, shape, g):
    import torch
    if len(shape) == 4:
        return torch.randn(shape, generator=g) * (1.6 / (shape[1] * 16) ** 0.5)
    return 0.05 * torch.randn(shape, generator=g)


def _pix2pix_reference_net(seeded=True):
    import torch
    ref_loader.bootstrap()
    from pix2pix.models import networks
    net = networks.define_G(2, 1, 64, 'unet_1024', 'none', False, 'normal', 0.02, []).eval()
    if seeded:
        g = torch.Generator().manual_seed(31)
        with torch.no_grad():
            for name, p in net.named_parameters():
                p.copy_(_pix2pix_param(name, tuple(p.shape), g))
    return net


def test_pix2pix_unet_oracle_equals_reference():
    """D9 groundwork: the BOOST merge network (10-level U-Net, norm 'none') and its input preparation."""
    import torch
    from oracle import pix2pix as op2p
    layout = pinned_json("pix2pix/layout", lambda: _layout(_pix2pix_reference_net(False)), NETS)
    sd = _seeded_state(layout, torch.Generator().manual_seed(31), _pix2pix_param)
    rng = np.random.default_rng(5)
    outer = rng.standard_normal((1024, 1024)).astype(np.float32)
    inner = (outer * 0.5 + rng.standard_normal((1024, 1024)).astype(np.float32)).astype(np.float32)
    x = op2p.merge_input(outer, inner)
    assert x.shape == (1, 2, 1024, 1024) and float(x.min()) == -1.0 and float(x.max()) == 1.0

    def reference():                               # the 1024 x 1024 result is stored as every fourth row and column (file size)
        net = _pix2pix_reference_net()
        _assert_same_state(sd, net.state_dict())
        with torch.no_grad():
            return net(x.clone())[:, :, ::4, ::4].numpy()
    want = torch.from_numpy(pinned("pix2pix/unet", reference, NETS))
    with torch.no_grad():
        got = op2p.unet(sd, x.clone())
    assert got.shape == (1, 1, 1024, 1024) and want.shape == (1, 1, 256, 256)
    assert float(want.abs().max()) > 1e-3          # the seeded weights keep a signal through the 20 layers
    assert (got[:, :, ::4, ::4] - want).abs().max().item() <= 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# Depth-Anything-V2 (D5 / D6): the oracle restatement against the reference's own DepthAnythingV2 module
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("encoder,hw,net", [("vits", (70, 98), 70), ("vits", (84, 56), 56), ("vitb", (70, 70), 70)])
def test_dav2_oracle_equals_reference(encoder, hw, net):
    """ddepth_anything_v2/depth_anything_v2/dpt.py:176-221 + src/depthmap_generation.py:375-403,548-559: strict
    state_dict load of the synthetic weights into the reference module, then the reference's own pre-processing /
    forward / final resize against oracle.dav2.get_raw_prediction on the same uint8 image -> identical floats."""
    import cv2
    import torch
    import torch.nn.functional as F
    from oracle import dav2 as odav2
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict(encoder, seed=1)
    cfg = odav2.CONFIGS[encoder]
    rgb = synth_rgb(hw[0], hw[1], 3)

    def reference():
        model = ref_loader.dav2_class()(encoder=encoder, features=cfg['features'], out_channels=cfg['out_channels']).eval()
        missing = model.load_state_dict(sd, strict=True)
        assert not missing.missing_keys and not missing.unexpected_keys
        # the reference's call chain, verbatim: get_raw_prediction (:381) -> estimatedepthanything_v2 (:548-559)
        img = cv2.cvtColor(np.asarray(rgb), cv2.COLOR_BGR2RGB) / 255.0
        with torch.no_grad():
            image = cv2.cvtColor((img * 255.1).astype('uint8'), cv2.COLOR_BGR2RGB)
            image, (h, w) = model.image2tensor(image, net)
            image = image.to('cpu')
            depth = model.forward(image)
            depth = F.interpolate(depth[:, None], (h, w), mode="bilinear", align_corners=True)[0, 0]
        return depth.cpu().numpy()
    want = pinned(f"dav2/{encoder}/{hw[0]}x{hw[1]}/{net}", reference)
    got, invert = odav2.get_raw_prediction(rgb, sd, encoder, net)
    assert invert is False
    assert want.max() - want.min() > 0.1          # a non-degenerate map (default init would be identically zero)
    assert got.shape == want.shape == tuple(hw)
    # identical floats when both sides run on one machine (minting).  The stored result may come from another CPU, whose
    # fp32 GEMM kernels sum in another order through the 12 blocks: between two x86 hosts the three cases differed by
    # 5.4e-7, 7.3e-7 and 1.2e-6 of the map's maximum, so the stored comparison allows 1e-5
    tol = 1e-6 if MINT else 1e-5
    assert float(np.abs(got - want).max()) <= tol * float(np.abs(want).max()), float(np.abs(got - want).max())


# ---------------------------------------------------------------------------------------------------------------------
# D9: the BOOST driver (resolution search, patch selection, double estimation, merge + blend) against the reference's own
# functions.  The two networks are stand-ins (cheap, deterministic, the same on both sides): the real ones are pinned above.
# ---------------------------------------------------------------------------------------------------------------------
class _FakeLeres:
    """stands for RelDepthModel: estimateleres calls model.depth_model(normalised [1,3,h,w])"""

    @staticmethod
    def depth_model(x):
        import torch
        import torch.nn.functional as F
        g = x.mean(dim=1, keepdim=True)
        return F.avg_pool2d(g, 9, 1, 4) + 0.25 * torch.sin(3.0 * x[:, :1]) + 0.1 * x[:, 2:3]


class _FakePix2Pix:
    """stands for Pix2Pix4DepthModel: set_input / test / get_current_visuals (pix2pix/models/pix2pix4depth_model.py:96-116)"""

    def set_input(self, outer, inner):
        from oracle import pix2pix as op2p
        self.real_A = op2p.merge_input(outer, inner)

    def test(self):
        import torch
        o, i = self.real_A[:, :1], self.real_A[:, 1:]
        self.fake_B = torch.tanh(0.7 * o + 0.5 * i + 0.1 * o * i)

    def get_current_visuals(self):
        return {"fake_B": self.fake_B}


def _boost_reference_module():
    import torch
    ref_loader.bootstrap()
    from src import depthmap_generation as dg
    dg.depthmap_device = torch.device("cpu")
    import skimage.measure as sm
    from oracle import boost
    sm.block_reduce = lambda img, block, func: boost.block_reduce_max(img, block[0])   # skimage is absent here (SURVEY A.5); zero-padded max pool
    dg.skimage = __import__("skimage")
    return dg


def _fake_estimate(img, msize):
    import cv2
    from oracle import leres
    with __import__("torch").no_grad():
        pred = _FakeLeres.depth_model(leres.preprocess(img, msize, msize)).squeeze().numpy()
    return cv2.resize(pred, (img.shape[1], img.shape[0]), interpolation=cv2.INTER_CUBIC)


def _fake_merge(outer, inner):
    p = _FakePix2Pix()
    p.set_input(outer, inner)
    p.test()
    return p.fake_B.squeeze().numpy()


@pytest.mark.parametrize("hw,rmax", [((300, 420), 1600), ((520, 360), 1200)])
def test_boost_selection_equals_reference(hw, rmax):
    """calculateprocessingres + generatepatchs + generatemask: integer / index results, compared exactly."""
    import cv2
    from oracle import boost
    rgb = synth_rgb(hw[0], hw[1], 11)
    img = cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0
    key = f"boost_select/{hw[0]}x{hw[1]}/{rmax}"
    want = pinned_json(key + "/res", lambda: [float(v) for v in _boost_reference_module().calculateprocessingres(img, 448, 0.2, 3, rmax)[:2]])
    got = boost.calculateprocessingres(img, 448, 0.2, 3, rmax)
    assert got[0] == want[0] and got[1] == want[1]
    factor = max(min(1, 4 * got[1] * got[0] / rmax), 0.2)
    a, b = boost.target_size(img.shape, got[0], factor)
    big = cv2.resize(img, (b, a), interpolation=cv2.INTER_CUBIC)
    wantp = pinned_json(key + "/rects", lambda: [[int(v) for v in kv[1]["rect"]] for kv in _boost_reference_module().generatepatchs(big, 896, factor)])
    gotp = boost.generatepatchs(big, 896, factor)
    assert len(gotp) == len(wantp) and len(gotp) > 0
    assert [[int(v) for v in kv[1]["rect"]] for kv in gotp] == wantp
    # stored as every third row and column: the mask is a separable Gaussian ramp, far larger in full than a golden file may be
    assert np.array_equal(boost.generatemask((300, 300))[::3, ::3], pinned("boost_mask300", lambda: _boost_reference_module().generatemask((300, 300))[::3, ::3]))


def test_boost_estimate_equals_reference():
    """estimateboost end to end (model type 0: receptive field 448, patches at 896) with the stand-in networks."""
    import cv2
    from oracle import boost
    rgb = synth_rgb(300, 420, 12)
    img = cv2.cvtColor(rgb, cv2.COLOR_BGR2RGB) / 255.0
    # the reference's 300 x 420 result is stored as every second row and column (file size)
    want = pinned("boost_estimate", lambda: _boost_reference_module().estimateboost(img.copy(), _FakeLeres(), 0, _FakePix2Pix(), 1600)[::2, ::2])
    info = {}
    got = boost.estimateboost(img.copy(), 0, _fake_estimate, _fake_merge, 1600, info=info)
    assert got.shape == (300, 420) and want.shape == (150, 210) and len(info["patches"]) >= 2
    assert np.abs(got[::2, ::2] - want).max() <= 1e-6 * np.abs(want).max()


def test_pix2pix_synthetic_state_dict_matches_reference_module():
    """oracle.synth_weights.make_pix2pix_state_dict loads strictly into the reference generator: the same keys with the same
    shapes and types as the generator's own state dict (stored), which is what a strict load checks"""
    from oracle import synth_weights
    sd = synth_weights.make_pix2pix_state_dict(seed=1)

    def reference():
        net = _pix2pix_reference_net(False)
        res = net.load_state_dict(sd, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        return sorted([k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in net.state_dict().items())
    want = pinned_json("pix2pix/state_dict", reference, NETS)
    assert sorted([k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()) == want
