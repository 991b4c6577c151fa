"""CPU: ragged batches without a GPU.
  * the funnel's grouping: consecutive images by network input size (custom depth maps and BOOST by pixel size), each group bounded
    by max_batch_for of its largest image, against a fake holder;
  * an engine's ragged call sequence, recorded against the fake library of test_engine_trace_cpu.py: the ragged pre-processing,
    then exactly the network calls of a uniform batch of the same size, then the ragged final resize;
  * the host-side descriptor layout (_lib.Ragged)."""
import numpy as np
import pytest
from PIL import Image

from test_engine_trace_cpu import HOST_ONLY, _cpu, _rgb, fake  # noqa: F401  (fake is a fixture)


class _Holder:
    """net size = the image's aspect ratio class, as a keep-aspect model would give; records the calls"""

    def __init__(self):
        self.calls = []

    def net_size(self, w, h, nw, nh):
        return (round(w / h, 2), nw, nh)


def _groups(sizes, custom=(), boost=False, env=None, monkeypatch=None):
    from depthmap_b200 import core
    if env is not None:
        monkeypatch.setenv("DEPTHMAP_B200_MAX_BATCH", env)
    imgs = [Image.new('RGB', (w, h)) for h, w in sizes]
    inp = core.CoreGenerationFunnelInp(dict(net_width=70, net_height=70, boost=boost))
    holder = _Holder()
    key = lambda i: core._group_key(holder, inp, imgs[i], i in custom, boost)
    out, i = [], 0
    while i < len(imgs):
        g, largest = [i], imgs[i].width * imgs[i].height
        while g[-1] + 1 < len(imgs):
            nxt = imgs[g[-1] + 1]
            grown = max(largest, nxt.width * nxt.height)
            if len(g) + 1 > core.max_batch_for(grown, 1) or key(g[-1] + 1) != key(i):
                break
            g.append(g[-1] + 1)
            largest = grown
        out.append(g)
        i = g[-1] + 1
    return out


def test_grouping_by_net_size(monkeypatch):
    from depthmap_b200 import core
    sizes = [(60, 80), (90, 120), (30, 40), (40, 40), (80, 80), (60, 80)]
    assert _groups(sizes) == [[0, 1, 2], [3, 4], [5]]
    assert _groups(sizes, custom={1}) == [[0], [1], [2], [3, 4], [5]]      # a custom depth map keeps the pixel size
    assert _groups(sizes, boost=True) == [[0], [1], [2], [3], [4], [5]]
    assert _groups(sizes, env="2", monkeypatch=monkeypatch) == [[0, 1], [2], [3, 4], [5]]
    monkeypatch.delenv("DEPTHMAP_B200_MAX_BATCH")
    # the bound is that of the group's largest image: 2048 x 2048 allows 4 images, so a small first image does not set it
    big = [(64, 64)] + [(2048, 2048)] * 6
    assert core.max_batch_for(64, 64) == 64 and core.max_batch_for(2048, 2048) == 4
    assert _groups(big) == [[0, 1, 2, 3], [4, 5, 6]]


def test_funnel_uses_the_same_grouping(monkeypatch):
    """core_generation_funnel forms the groups _groups models: one ragged call per mixed group, the uniform call otherwise"""
    import torch
    from depthmap_b200 import core
    calls = []

    class H(_Holder):
        def update_settings(self, **kw):
            pass

        def ensure_models(self, *a):
            pass

        def offload(self):
            pass

        def get_raw_prediction_batch(self, rgb, nw, nh):
            calls.append(("batch", tuple(rgb.shape)))
            return torch.zeros(rgb.shape[:3]), False

        def get_raw_prediction_ragged(self, images, nw, nh):
            calls.append(("ragged", [tuple(t.shape) for t in images]))
            return [torch.zeros(t.shape[:2]) for t in images], False

    monkeypatch.setattr(core, "_model_holder", H())
    monkeypatch.setattr(core._lib, "require_cuda", lambda: torch.device("cpu"))
    monkeypatch.setattr(core, "normalize_prediction_batch", lambda p, *a, **k: (torch.zeros(p.shape, dtype=torch.int32), torch.zeros(p.shape[0])))
    sizes = [(60, 80), (90, 120), (90, 120), (40, 40)]
    imgs = [Image.fromarray(np.zeros((h, w, 3), np.uint8)) for h, w in sizes]
    out = list(core.core_generation_funnel(None, imgs, None, None, dict(net_width=70, net_height=70), ops={}))
    assert [i for i, _, _ in out] == [0, 1, 2, 3]
    assert calls == [("ragged", [(60, 80, 3), (90, 120, 3), (90, 120, 3)]), ("batch", (1, 40, 40, 3))]


def test_ragged_layout():
    from depthmap_b200 import _lib
    r = _lib.Ragged([(2, 3), (4, 5)], 3, None)
    assert r.size == 2 * 3 * 3 + 4 * 5 * 3 and r.host.itemsize == 16
    assert [tuple(x) for x in r.host.tolist()] == [(0, 2, 3), (18, 4, 5)]
    import torch
    a, b = r.split(torch.arange(r.size))
    assert a.shape == (2, 3, 3) and b.shape == (4, 5, 3) and int(b[0, 0, 0]) == 18


def _names(rec, start):
    """the kernel calls from `start` on (host-side tables are computed once per resolution, by whichever call comes first)"""
    return [c[0] for c in rec.calls[start:] if c[0] not in HOST_ONLY]


def test_ragged_trace_dav2(fake):  # noqa: F811
    """forward_ragged: the ragged patchify, the network calls of forward_batch at the same B and net size, the ragged resize"""
    import torch
    from depthmap_b200 import _lib
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import synth_weights
    eng = DepthAnythingV2Engine(synth_weights.make_dav2_state_dict('vits', seed=0), 'vits', _cpu())
    eng.forward_batch(_rgb(3, 60, 80, 1), 70)
    uniform = _names(fake, 0)
    n0 = len(fake.calls)
    imgs = [_rgb(1, h, w, 2)[0] for h, w in ((60, 80), (37, 53), (90, 120))]
    desc = _lib.Ragged([tuple(t.shape[:2]) for t in imgs], 3, _cpu())
    out = eng.forward_ragged(torch.cat([t.reshape(-1) for t in imgs]), desc, 70)
    ragged = _names(fake, n0)
    assert out.numel() == 60 * 80 + 37 * 53 + 90 * 120
    assert ragged[0] == "dm_preprocess_patchify_ragged" and uniform[0] == "dm_preprocess_patchify"
    assert ragged[-1] == "dm_resize_f32_ragged" and uniform[-1] == "dm_resize_f32"
    assert ragged[1:-1] == uniform[1:-1]


@pytest.mark.parametrize("engine", ["leres", "zoe"])
def test_ragged_trace_stems(fake, engine):  # noqa: F811
    import torch
    from depthmap_b200 import _lib
    from depthmap_b200.depthmap_generation import LeresEngine, ZoeDepthNKEngine
    from oracle import beit_dpt, synth_weights
    if engine == "leres":
        eng, sizes, net = LeresEngine(synth_weights.make_leres_state_dict(seed=0), _cpu()), ((60, 80), (37, 53)), 64
        first, last = "dm_leres_stem_im2col", "dm_resize_f32"
    else:
        sd = {"core.core." + k: v for k, v in synth_weights.make_beit_dpt_state_dict('beit_tiny', seed=0).items()}
        sd.update(synth_weights.make_zoedepth_head_state_dict(feat_ch=beit_dpt.CONFIGS['beit_tiny']['features'], seed=100))
        eng, sizes, net = ZoeDepthNKEngine(sd, _cpu(), core_name='beit_tiny'), ((60, 80), (75, 100)), 96
        first, last = "dm_zoe_preprocess_patchify", "dm_zoe_tta_combine"
    eng.forward_batch(_rgb(2, *sizes[0], 1), net)
    uniform = _names(fake, 0)
    n0 = len(fake.calls)
    imgs = [_rgb(1, h, w, 2)[0] for h, w in sizes]
    eng.forward_ragged(torch.cat([t.reshape(-1) for t in imgs]), _lib.Ragged(sizes, 3, _cpu()), net)
    ragged = _names(fake, n0)
    assert uniform[0] == first and ragged[0] == first + "_ragged"
    assert uniform[-1] == last and ragged[-1] == last + "_ragged"
    assert ragged[1:-1] == uniform[1:-1]
