"""GPU: the ViT / DPT engines' CUDA-graph path (DepthAnythingV2Engine, DptBeitEngine, DptVitEngine through _lib.GraphCache)
against the same engine kept eager (DEPTHMAP_B200_MODEL_GRAPH=0).  Call 1 of a shape runs eagerly, call 2 captures, later calls
replay; every one must equal the eager engine BIT FOR BIT (the same kernels on the same packed weights), also after a shape change
(the buffers are rebuilt, the graphs dropped) and when recorded into a caller's CUDA graph.  The resolution tables the graphs
read come from the host routines dm_dinov2_pos_embed, dm_vit_pos_embed and dm_beit_rel_table, at native and resized grids."""
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _imgs(B, h, w, seed=0):
    from synth import synth_rgb
    return np.stack([synth_rgb(h, w, seed + s) for s in range(B)])


def _engines(monkeypatch, cls, sd, *args, **kw):
    """(graphed, eager) engines of one checkpoint"""
    monkeypatch.delenv("DEPTHMAP_B200_MODEL_GRAPH", raising=False)
    graphed = cls(sd, *args, **kw)
    monkeypatch.setenv("DEPTHMAP_B200_MODEL_GRAPH", "0")
    eager = cls(sd, *args, **kw)
    assert graphed._graphs.enabled and not eager._graphs.enabled
    return graphed, eager


def _calls_equal_eager(graphed, eager, rgb, net_w, net_h, calls):
    """`calls` forwards of the graphed engine at one shape, each equal to the eager engine's; the first is eager, the second
    captures, and a replay adds as many launches as an eager forward"""
    import torch
    n0 = eager.ops.launches
    want = eager.forward_batch(rgb, net_w, net_h)
    per_forward = eager.ops.launches - n0
    for call in range(calls):
        n0 = graphed.ops.launches
        got = graphed.forward_batch(rgb, net_w, net_h)
        assert torch.equal(got, want), (call, float((got - want).abs().max()))
        assert graphed.ops.launches - n0 == per_forward, (call, graphed.ops.launches - n0, per_forward)
        assert bool(graphed._graphs._graphs) == (call >= 1), call
    return want


@pytest.mark.parametrize("encoder,hw,net,circular,split", [
    ('vits', (70, 98), 70, False, False), ('vits', (64, 64), 56, False, False), ('vitb', (84, 84), 84, False, False),
    ('vits', (120, 90), 140, False, False), ('vits', (70, 98), 70, True, False), ('vits', (70, 98), 70, False, True)])
def test_graph_dav2_equals_eager(cuda_device, monkeypatch, encoder, hw, net, circular, split):
    """Depth-Anything-V2, zero padding, tiling mode (circular) and no_half (split); DINOv2 position embedding resized from the
    37 x 37 grid (dm_dinov2_pos_embed)"""
    import torch
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict(encoder, seed=1)
    graphed, eager = _engines(monkeypatch, DepthAnythingV2Engine, sd, encoder, cuda_device, circular=circular, split=split)
    rgb = torch.from_numpy(_imgs(2, *hw)).to(cuda_device)
    _calls_equal_eager(graphed, eager, rgb, net, net, 4)


@pytest.mark.parametrize("hw,net", [((64, 96), (64, 64)), ((96, 96), (96, 96)), ((80, 50), (64, 64))])
def test_graph_beit_equals_eager(cuda_device, monkeypatch, hw, net):
    """DPT-BEiT (structural configuration) with resized relative-position tables (dm_beit_rel_table).  A different batch size and
    resolution rebuilds the buffers and drops the graphs; back at the first shape the engine runs eagerly, captures again and
    still equals the eager engine."""
    import torch
    from depthmap_b200.depthmap_generation import DptBeitEngine
    from oracle import synth_weights
    sd = synth_weights.make_beit_dpt_state_dict('beit_tiny', seed=3)
    graphed, eager = _engines(monkeypatch, DptBeitEngine, sd, 'beit_tiny', cuda_device)
    rgb = torch.from_numpy(_imgs(3, *hw, seed=7)).to(cuda_device)
    _calls_equal_eager(graphed, eager, rgb, net[0], net[1], 3)
    rgb2 = torch.from_numpy(_imgs(1, 96, 64, seed=9)).to(cuda_device)
    _calls_equal_eager(graphed, eager, rgb2, 64, 96, 3)
    _calls_equal_eager(graphed, eager, rgb, net[0], net[1], 3)
    assert len(graphed._graphs._graphs) == 1


@pytest.mark.parametrize("hw,net", [((64, 64), (64, 64)), ((96, 128), (96, 96))])
def test_graph_vit_equals_eager(cuda_device, monkeypatch, hw, net):
    """the dpt_large_384 family (structural configuration), absolute position embedding resized bilinearly (dm_vit_pos_embed)"""
    import torch
    from depthmap_b200.depthmap_generation import DptVitEngine
    from oracle import synth_weights
    sd = synth_weights.make_beit_dpt_state_dict('vit_tiny', seed=5)
    graphed, eager = _engines(monkeypatch, DptVitEngine, sd, 'vit_tiny', cuda_device)
    rgb = torch.from_numpy(_imgs(2, *hw, seed=11)).to(cuda_device)
    _calls_equal_eager(graphed, eager, rgb, net[0], net[1], 3)


def test_graph_beit512_outer_capture_and_latency(cuda_device, monkeypatch):
    """dpt_beit_large_512 at its native window: replays equal the eager engine, recording forward_batch into a caller's CUDA
    graph gives the eager result, and at B = 1 (the reference's call shape, ModelHolder.get_raw_prediction) the graphed engine
    is faster than the eager one"""
    import torch
    from depthmap_b200.depthmap_generation import DptBeitEngine
    from oracle import synth_weights
    sd = synth_weights.make_beit_dpt_state_dict('beitl16_512', seed=3)
    graphed, eager = _engines(monkeypatch, DptBeitEngine, sd, 'beitl16_512', cuda_device)
    rgb = torch.from_numpy(_imgs(2, 512, 512, seed=70)).to(cuda_device)
    want = _calls_equal_eager(graphed, eager, rgb, 512, 512, 4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graphed.forward_batch(rgb, 512, 512)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = graphed.forward_batch(rgb, 512, 512)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    one = rgb[:1].contiguous()

    def lat(fn, n=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n * 1e3
    t_eager = lat(lambda: eager.forward_batch(one, 512, 512))
    t_graph = lat(lambda: graphed.forward_batch(one, 512, 512))
    print(f"[latency] dpt_beit_large_512 B=1: eager {t_eager:.2f} ms/forward, graph replay {t_graph:.2f} ms/forward")
    assert t_graph < t_eager


def test_get_raw_prediction_batch_rejects_bad_input(cuda_device):
    """the kernels read the batch's memory as uint8 [B,H,W,3]: anything else is refused before a kernel runs"""
    import torch
    from depthmap_b200.depthmap_generation import ModelHolder
    from oracle import synth_weights
    sd = synth_weights.make_dav2_state_dict('vits', seed=1)
    mh = ModelHolder()
    mh.weights_provider = lambda t: sd
    mh.ensure_models(12, cuda_device, False)
    with pytest.raises(ValueError):
        mh.get_raw_prediction_batch(torch.zeros(1, 56, 56, 3, dtype=torch.float32, device=cuda_device), 56, 56)
    with pytest.raises(ValueError):
        mh.get_raw_prediction_batch(torch.zeros(1, 56, 56, 4, dtype=torch.uint8, device=cuda_device), 56, 56)
    pred, invert = mh.get_raw_prediction_batch(torch.zeros(1, 56, 56, 3, dtype=torch.uint8, device=cuda_device), 56, 56)
    assert pred.shape == (1, 56, 56) and invert is False
    mh.unload_models()
