"""The op-level engines' native call sequences, recorded on the CPU against a fake library.

Every engine forward is a sequence of C-ABI calls.  Here `_lib.load()` returns a recorder in which every `dm_*` returns DM_OK;
the engines run on CPU tensors with seeded synthetic weights, so nothing is computed, but each call is recorded with its entry
point, its scalar arguments, the scalar fields of a GemmDesc and every pointer as a label numbered by first appearance (so the
trace also pins which buffer is wired where).  The trace must equal tests/golden/engine_trace.json.gz, and each engine's launch
counter must equal the kernels the recorded calls issue (kernels() below, read from csrc/).

    DEPTHMAP_MINT_GOLDEN=1 python -m pytest tests/test_engine_trace_cpu.py      # rewrite the stored trace
"""
from __future__ import annotations

import contextlib
import ctypes
import gzip
import json
import os
import types

import numpy as np
import pytest

from synth import synth_rgb

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "engine_trace.json.gz")
MINT = os.environ.get("DEPTHMAP_MINT_GOLDEN") == "1"
PARTIALS = 16                     # what the fake dm_boost_partials returns

# host-side table helpers: no stream, no kernel
HOST_ONLY = {"dm_dinov2_pos_embed", "dm_vit_pos_embed", "dm_beit_rel_table", "dm_boost_partials"}


def kernels(name, args):
    """kernels one call issues (csrc/*.cu): one, except the patchify pre-processing, which first zero-fills the K padding of the
    patch matrix when kpad exceeds 3 * patch * patch (vit_kernels.cu: patchify_setup), and a circularly padded 3x3 convolution,
    which first copies its input into the halo buffer"""
    if name in HOST_ONLY:
        return 0
    if name in ("dm_preprocess_patchify", "dm_preprocess_patchify_split"):
        return 1 + (args[11] > 3 * args[6] ** 2)
    if name == "dm_preprocess_patchify_f32_crops":
        return 1 + (args[12] > 3 * args[7] ** 2)
    if name == "dm_conv3x3_circular_ex":
        return 2
    if name == "dm_conv3x3_split_ex":
        return 1 + bool(args[1])
    return 1


class _Stream:
    def __init__(self, ident):
        self.cuda_stream = ident

    def wait_stream(self, other):
        pass


class _Recorder:
    """Stands in for the ctypes library: dm_* attributes are recording functions that return DM_OK."""

    def __init__(self):
        self.calls = []
        self.alive = []
        self._labels = {}

    def __getattr__(self, name):
        if not name.startswith("dm_"):
            raise AttributeError(name)
        rec = self

        def fn(*args):
            assert len(args) == len(fn.argtypes), name
            rec.calls.append([name, [rec._value(a, t) for a, t in zip(args, fn.argtypes)], kernels(name, args)])
            return PARTIALS if name == "dm_boost_partials" else 0

        fn.argtypes = None
        setattr(self, name, fn)
        return fn

    def _label(self, ptr):
        if not ptr:
            return "NULL"
        return self._labels.setdefault(ptr, f"p{len(self._labels)}")

    def _value(self, a, argtype):
        if isinstance(a, ctypes.c_void_p):                                  # the stream
            return f"stream{a.value}"
        if argtype is ctypes.c_void_p:                                      # a tensor or numpy address
            return self._label(a)
        if type(a).__name__ == "CArgObject":                                # byref(GemmDesc)
            d = a._obj
            out = {}
            for f, t in d._fields_:
                v = getattr(d, f)
                out[f] = self._label(v) if t is ctypes.c_void_p else v
            return out
        if isinstance(a, ctypes.Array):                                     # mean / std / channel map
            return list(a)
        if isinstance(a, float):
            return float(np.float32(a))                                     # every float parameter is a C float
        return a


@pytest.fixture
def fake(monkeypatch):
    """Fake library, stream and the few torch.cuda calls the eager paths make; CUDA-graph capture off."""
    import torch
    from depthmap_b200 import _lib
    rec = _Recorder()
    _lib._bind_optional(rec)                 # argtypes tell pointers from scalars
    for name in HOST_ONLY - {"dm_boost_partials"}:
        getattr(rec, name).argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    rec.dm_boost_partials.argtypes = []
    cur = [_Stream(1)]
    made = [0]

    def new_stream(device=None):
        made[0] += 1
        return _Stream(1 + made[0])

    @contextlib.contextmanager
    def use(s):
        prev, cur[0] = cur[0], s
        try:
            yield
        finally:
            cur[0] = prev

    # a tensor whose address entered the trace stays alive, so no later tensor can take its address (and its label)
    data_ptr = torch.Tensor.data_ptr
    monkeypatch.setattr(torch.Tensor, "data_ptr", lambda t: rec.alive.append(t) or data_ptr(t))
    monkeypatch.setattr(_lib, "load", lambda: rec)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: ctypes.c_void_p(cur[0].cuda_stream))
    monkeypatch.setattr(torch.cuda, "get_device_properties", lambda *a: types.SimpleNamespace(total_memory=1 << 40, multi_processor_count=132))
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    monkeypatch.setattr(torch.cuda, "Stream", new_stream)
    monkeypatch.setattr(torch.cuda, "stream", use)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: cur[0])
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.cuda, "empty_cache", lambda: None)
    monkeypatch.setenv("DEPTHMAP_B200_MODEL_GRAPH", "0")
    monkeypatch.setenv("DEPTHMAP_B200_LERES_GRAPH", "0")
    monkeypatch.setenv("DEPTHMAP_B200_UNET_GRAPH", "0")
    return rec


_STORED = None
_MINTED = {}


def check_trace(key, rec, launches):
    """the recorded calls equal the stored trace; the launch counter equals the kernels those calls issue"""
    global _STORED
    calls = json.loads(json.dumps(rec.calls))            # tuples -> lists, as stored
    if MINT:
        _MINTED[key] = calls                              # minting runs the whole module: every key is rewritten
        with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
            f.write(json.dumps(_MINTED, separators=(",", ":"), sort_keys=True).encode())
    else:
        if _STORED is None:
            with gzip.open(GOLDEN, "rt") as f:
                _STORED = json.load(f)
        want = _STORED[key]
        for i, (g, w) in enumerate(zip(calls, want)):
            assert g == w, f"{key}: call {i} differs\n got  {g}\n want {w}"
        assert len(calls) == len(want), f"{key}: {len(calls)} calls, stored {len(want)}"
    issued = sum(k for _, _, k in calls)
    assert launches == issued, f"{key}: launch counter {launches}, kernels issued {issued}"


def _cpu():
    import torch
    return torch.device("cpu")


def _rgb(B, h, w, seed):
    import torch
    return torch.from_numpy(np.stack([synth_rgb(h, w, seed + i) for i in range(B)]))


def _planar(h, w, seed):
    import torch
    return torch.from_numpy(synth_rgb(h, w, seed).transpose(2, 0, 1).astype(np.float32) / 255.0).contiguous()


def _trace_dav2(fake, split=False, circular=False):
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import synth_weights
    eng = DepthAnythingV2Engine(synth_weights.make_dav2_state_dict('vits', seed=0), 'vits', _cpu(), circular=circular, split=split)
    eng.forward_batch(_rgb(2, 60, 80, 1), 70)
    check_trace("dav2_vits" + "_split" * split + "_circular" * circular, fake, eng.ops.launches)


def test_trace_dav2(fake):
    _trace_dav2(fake)


@pytest.mark.parametrize("split, circular", [(True, False), (False, True), (True, True)])
def test_trace_dav2_modes(fake, split, circular):
    """the split (no_half) path and tiling mode"""
    _trace_dav2(fake, split, circular)


@pytest.mark.parametrize("name, circular", [pytest.param(n, c, id=n + "-circular" * c)
                                            for c in (False, True) for n in ("beit_tiny", "vit_tiny")])
def test_trace_dpt(fake, name, circular):
    from depthmap_b200.depthmap_generation import DptBeitEngine, DptVitEngine
    from oracle import synth_weights
    cls = DptBeitEngine if name == "beit_tiny" else DptVitEngine
    eng = cls(synth_weights.make_beit_dpt_state_dict(name, seed=0), name, _cpu(), circular=circular)
    eng.forward_batch(_rgb(2, 60, 80, 1), 96)
    eng.forward_crops(_planar(100, 120, 2), [(0, 0, 64, 64), (10, 20, 48, 80), (30, 5, 64, 64)], 64)
    check_trace(f"dpt_{name}" + "_circular" * circular, fake, eng.ops.launches)


def _zoe_core(core, seed):
    from oracle import synth_weights
    return {"core.core." + k: v for k, v in synth_weights.make_beit_dpt_state_dict(core, seed=seed).items()}


def test_trace_zoedepth_nk(fake):
    _trace_zoedepth_nk(fake)


def test_trace_zoedepth_nk_circular(fake):
    _trace_zoedepth_nk(fake, circular=True)


def _trace_zoedepth_nk(fake, circular=False):
    from depthmap_b200.depthmap_generation import ZoeDepthNKEngine
    from oracle import beit_dpt, synth_weights
    sd = _zoe_core('beit_tiny', 0)
    sd.update(synth_weights.make_zoedepth_head_state_dict(feat_ch=beit_dpt.CONFIGS['beit_tiny']['features'], seed=100))
    eng = ZoeDepthNKEngine(sd, _cpu(), core_name='beit_tiny', circular=circular)
    eng.forward_batch(_rgb(2, 60, 80, 1), 96)
    check_trace("zoedepth_nk" + "_circular" * circular, fake, eng.ops.launches)


@pytest.mark.parametrize("variant, circular", [pytest.param(v, c, id=v + "-circular" * c) for c in (False, True) for v in ("n", "k")])
def test_trace_zoedepth_single(fake, variant, circular):
    from depthmap_b200.depthmap_generation import ZoeDepthEngine
    from oracle import beit_dpt
    from oracle import zoedepth_single as ozs
    sd = _zoe_core('beit_tiny', 0)
    sd.update(ozs.make_zoedepth_single_head_state_dict(variant, feat_ch=beit_dpt.CONFIGS['beit_tiny']['features'], seed=100))
    eng = ZoeDepthEngine(sd, _cpu(), variant, core_name='beit_tiny', circular=circular)
    eng.forward_batch(_rgb(2, 60, 80, 1), 96)
    check_trace(f"zoedepth_{variant}" + "_circular" * circular, fake, eng.ops.launches)


@pytest.fixture(scope="module")
def leres_sd():
    from oracle import synth_weights
    return synth_weights.make_leres_state_dict(seed=0)


@pytest.fixture(scope="module")
def pix2pix_sd():
    from oracle import synth_weights
    return synth_weights.make_pix2pix_state_dict(seed=0)


@pytest.fixture(scope="module")
def midas_v21_sd():
    from oracle import midas_v21
    return midas_v21.make_state_dict(seed=1)


def test_trace_leres(fake, leres_sd):
    _trace_leres(fake, leres_sd)


def test_trace_leres_circular(fake, leres_sd):
    _trace_leres(fake, leres_sd, circular=True)


def _trace_leres(fake, leres_sd, circular=False):
    from depthmap_b200.depthmap_generation import LeresEngine
    eng = LeresEngine(leres_sd, _cpu(), circular=circular)
    eng.forward_batch(_rgb(1, 60, 80, 1), 64)
    eng.forward_batch(_rgb(1, 64, 64, 2), 64)                  # output at net size: a copy, no resize kernel
    eng.forward_crops(_planar(100, 120, 2), [(0, 0, 64, 64), (10, 20, 64, 64)], 64)
    check_trace("leres" + "_circular" * circular, fake, eng.ops.launches)


@pytest.mark.parametrize("circular", [False, True])
def test_trace_midas_v21(fake, midas_v21_sd, circular):
    from depthmap_b200.depthmap_generation import MidasV21Engine
    eng = MidasV21Engine(midas_v21_sd, _cpu(), circular=circular)
    eng.forward_batch(_rgb(2, 100, 150, 1), 384, 384)
    # 200 x 200 crops at a 384 x 384 net, the 100 x 300 one at 128 x 384: two net shapes
    eng.forward_crops(_planar(300, 400, 3), [(0, 0, 200, 200), (100, 50, 200, 200), (300, 0, 100, 300)], 384)
    check_trace("midas_v21" + "_circular" * circular, fake, eng.ops.launches)


def test_trace_unet_merge(fake, pix2pix_sd):
    import torch
    from depthmap_b200.boost import UnetMergeEngine
    eng = UnetMergeEngine(pix2pix_sd, _cpu())
    eng.forward(torch.zeros(1024, 1024, 2))
    check_trace("unet_split", fake, eng.ops.launches)


@pytest.mark.parametrize("model_type", [0, 1, 5])
def test_trace_boost(fake, leres_sd, pix2pix_sd, midas_v21_sd, model_type):
    from depthmap_b200.boost import BoostPipeline, UnetMergeEngine
    from depthmap_b200.depthmap_generation import DptBeitEngine, LeresEngine, MidasV21Engine
    from oracle import synth_weights
    if model_type == 0:
        depth = LeresEngine(leres_sd, _cpu())
    elif model_type == 5:
        depth = MidasV21Engine(midas_v21_sd, _cpu())
    else:
        depth = DptBeitEngine(synth_weights.make_beit_dpt_state_dict('beit_tiny', seed=0), 'beit_tiny', _cpu())
    pipe = BoostPipeline(depth, UnetMergeEngine(pix2pix_sd, _cpu()), _cpu(), model_type)
    info = {}
    pipe.run(synth_rgb(300, 420, 12), 1600, info=info)
    assert len(info["rects"]) >= 1
    check_trace(f"boost_{model_type}", fake, pipe.ops.launches + depth.ops.launches + pipe.merge.ops.launches)
