"""CPU: pins the single-head ZoeDepth oracle (oracle/zoedepth_single.py: metric_head_single, model types 7 = ZoeDepth-N and
8 = ZoeDepth-K) to the reference's ZoeDepth module (dzoedepth/models/zoedepth/zoedepth_v1.py), built around a stub core
from the reference's own get_config("zoedepth", "infer") (config_version "kitti" for K).

What the reference computed on each test's seeded inputs, the parameter layout of its module and its resolved configuration
are stored in tests/golden/zoedepth_n_k_pin.npz, so the comparisons run anywhere.  With the reference tree present,

    DEPTHMAP_MINT_GOLDEN=1 python -m pytest tests/test_zoedepth_n_k_cpu.py

runs the reference again and replaces the keys it computed (keys of tests that did not run are kept)."""
import json
import os
import warnings

import numpy as np
import pytest

from oracle import ref_loader

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zoedepth_n_k_pin.npz")
MINT = os.environ.get("DEPTHMAP_MINT_GOLDEN") == "1"
_stored = dict(np.load(GOLDEN)) if os.path.exists(GOLDEN) else {}
_minted = {}


def pinned(key, compute):
    """The reference's result for `key` (an array): the stored one, or, when minting, compute()."""
    if MINT:
        _minted[key] = np.asarray(compute())
    src = _minted if MINT else _stored
    if key not in src:
        pytest.fail(f"no stored reference result for {key}: mint {GOLDEN} with the reference tree present")
    return src[key]


def pinned_json(key, compute):
    return json.loads(str(pinned(key, lambda: np.asarray(json.dumps(compute())))))


@pytest.fixture(scope="module", autouse=True)
def _write_minted():
    yield
    if MINT and _minted:
        np.savez_compressed(GOLDEN, **dict(_stored, **_minted))


VARIANTS = {"n": None, "k": "kitti"}
BUILD_ARGS = ("midas_model_type", "pretrained_resource", "use_pretrained_midas", "train_midas", "freeze_midas_bn")


def _reference_config(variant):
    warnings.filterwarnings("ignore")
    ref_loader.bootstrap()
    from dzoedepth.utils.config import get_config
    v = VARIANTS[variant]
    conf = get_config("zoedepth", "infer", config_version=v) if v else get_config("zoedepth", "infer")
    return {k: val for k, val in dict(conf).items() if k not in BUILD_ARGS}


def _feats(g, base_hw):
    import torch
    h, w = base_hw
    shapes = [(32, 16 * h, 16 * w), (256, h, w), (256, 2 * h, 2 * w), (256, 4 * h, 4 * w), (256, 8 * h, 8 * w), (256, 16 * h, 16 * w)]
    feats = [torch.randn(2, c, hh, ww, generator=g) * 0.7 for c, hh, ww in shapes]
    feats[0] = feats[0].abs()                      # out_conv is a post-ReLU activation in the core
    rel = torch.rand(2, 16 * h, 16 * w, generator=g) * 3.0          # the core's (non-negative) relative depth
    return feats, rel


def _param(name, shape, g):
    import torch
    return torch.randn(shape, generator=g) * (0.05 if len(shape) > 1 else 0.02)


def _reference_head(variant, seed, base_hw):
    import torch
    import torch.nn as nn
    conf = _reference_config(variant)
    from dzoedepth.models.zoedepth.zoedepth_v1 import ZoeDepth
    g = torch.Generator().manual_seed(seed)
    feats, rel = _feats(g, base_hw)

    class StubCore(nn.Module):                     # hands the head fixed activations (MidasCore.forward, midas.py:258-276)
        output_channels = (256, 256, 256, 256, 256)

        def forward(self, x, denorm=False, return_rel_depth=False):
            out = [f.clone() for f in feats]
            return (rel.clone(), out) if return_rel_depth else out

    model = ZoeDepth(StubCore(), **conf).eval()
    with torch.no_grad():
        for name, p in model.named_parameters():
            p.copy_(_param(name, tuple(p.shape), g))
    # parameters only: the module's buffers (the log-binomial's k_idx / K_minus_1) are constants the oracle builds itself
    sd = {k: v.detach().clone() for k, v in model.named_parameters() if not k.startswith("core.")}
    return model, sd


def _layout(variant):
    model = _reference_head(variant, 0, (2, 2))[0]
    return [[n, list(p.shape)] for n, p in model.named_parameters() if not n.startswith("core.")]


def _inputs(variant, seed, base_hw):
    """feats, rel and head state dict of _reference_head(variant, seed, base_hw), without the reference."""
    import torch
    g = torch.Generator().manual_seed(seed)
    feats, rel = _feats(g, base_hw)
    layout = pinned_json(f"{variant}/layout", lambda: _layout(variant))
    sd = {name: _param(name, tuple(shape), g) for name, shape in layout}
    if MINT:
        want = _reference_head(variant, seed, base_hw)[1]
        assert set(sd) == set(want) and all(torch.equal(sd[k], want[k]) for k in sd)
    return feats, rel, sd


@pytest.mark.parametrize("variant", ["n", "k"])
def test_resolved_config_matches_reference(variant):
    """get_config + ZoeDepth.__init__ defaults: both models bound their bins to [1e-3, 10] (no dataset sets min / max depth)."""
    from depthmap_b200.depthmap_generation import ZOE_SINGLE_CONFIG, ZOE_SINGLE_VARIANTS, ModelHolder
    from oracle import zoedepth_single as ozs

    def reference():
        conf = _reference_config(variant)
        model = _reference_head(variant, 0, (2, 2))[0]
        return dict(bin_centers_type=model.bin_centers_type, min_depth=model.min_depth, max_depth=model.max_depth,
                    min_temp=model.min_temp, n_bins=conf["n_bins"], n_attractors=[a.n_attractors for a in model.attractors],
                    kinds=sorted({a.kind for a in model.attractors}), types=sorted({a.attractor_type for a in model.attractors}),
                    max_temp=model.conditional_log_binomial.max_temp, bin_embedding_dim=conf["bin_embedding_dim"], img_size=conf["img_size"],
                    clb_hidden=model.conditional_log_binomial.mlp[0].out_channels, clb_in=model.conditional_log_binomial.mlp[0].in_channels)
    want = pinned_json(f"{variant}/config", reference)
    assert want["min_depth"] == 1e-3 and want["max_depth"] == 10
    assert want["kinds"] == ["mean"] and want["types"] == ["inv"] and want["clb_in"] == 32 + 1 + 128 and want["clb_hidden"] == 80
    for cfg in (ozs.SINGLE_CONFIG, ZOE_SINGLE_CONFIG):
        for k in ("min_depth", "max_depth", "min_temp", "max_temp", "n_bins", "n_attractors", "bin_embedding_dim"):
            assert cfg[k] == pytest.approx(want[k]), k
    assert ozs.SINGLE_VARIANTS[variant]["bin_centers_type"] == ZOE_SINGLE_VARIANTS[variant]["bin_centers_type"] == want["bin_centers_type"]
    # ModelHolder's default net size for the type (src/depthmap_generation.py:331-332) is the config's img_size
    assert ModelHolder.get_default_net_size(ZOE_SINGLE_VARIANTS[variant]["model_type"]) == [want["img_size"][0], want["img_size"][1]]


@pytest.mark.parametrize("variant", ["n", "k"])
def test_synthetic_state_dict_matches_reference_layout(variant):
    from oracle import zoedepth_single as ozs
    layout = pinned_json(f"{variant}/layout", lambda: _layout(variant))
    sd = ozs.make_zoedepth_single_head_state_dict(variant, seed=1)
    assert {k: list(v.shape) for k, v in sd.items()} == {n: s for n, s in layout}


@pytest.mark.parametrize("variant", ["n", "k"])
@pytest.mark.parametrize("seed,base_hw", [(0, (3, 4)), (1, (4, 3)), (2, (2, 2)), (3, (1, 5))])
def test_single_head_oracle_equals_reference(variant, seed, base_hw):
    import torch
    from oracle import zoedepth_single as ozs
    feats, rel, sd = _inputs(variant, seed, base_hw)

    def reference():
        model = _reference_head(variant, seed, base_hw)[0]
        with torch.no_grad():
            return model(torch.zeros(2, 3, feats[0].shape[2], feats[0].shape[3]))["metric_depth"].numpy()
    want = torch.from_numpy(pinned(f"{variant}/head/{seed}", reference))
    with torch.no_grad():
        got = ozs.metric_head_single(feats, rel, sd, variant)
    assert got.shape == want.shape == (2, 1, 16 * base_hw[0], 16 * base_hw[1])
    assert float(want.max() - want.min()) > 1e-3             # the seeded weights give a depth map that varies
    if variant == "k":
        assert float(want.max()) <= 10.0 and float(want.min()) >= 1e-3
    err = (got - want).abs().max().item()
    assert err <= 1e-5 * want.abs().max().item(), err


@pytest.mark.parametrize("variant", ["n", "k"])
def test_single_head_tta_wrapper_equals_reference(variant):
    """DepthModel.infer (pad + flip augmentation) around the single head: the stub core ignores its input."""
    import torch
    from oracle import zoedepth as ozd
    from oracle import zoedepth_single as ozs
    feats, rel, sd = _inputs(variant, 3, (2, 3))
    x = torch.rand(2, 3, 40, 56, generator=torch.Generator().manual_seed(5))

    def reference():
        with torch.no_grad():
            return _reference_head(variant, 3, (2, 3))[0].infer(x, pad_input=True, with_flip_aug=True).numpy()
    want = torch.from_numpy(pinned(f"{variant}/tta", reference))
    with torch.no_grad():
        got = ozd.infer(lambda t: ozs.metric_head_single(feats, rel, sd, variant), x, pad_input=True, with_flip_aug=True)
    assert got.shape == want.shape == (2, 1, 40, 56)
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()
