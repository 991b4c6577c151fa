"""CPU: the `no_half` setting without a device — its routing table, the split weight packing, and the split engine's call sequence.

The split (fp32-class) path of Depth-Anything-V2 is the fp16 path layer for layer on split operands (gemm_wgmma.cu): its trace,
recorded against the fake library of test_engine_trace_cpu.py, must be the fp16 trace with every entry point replaced by its split
counterpart, the depths and pitches of the split operands tripled, and a launch counter equal to the kernels the calls issue."""
from __future__ import annotations

import json

import pytest

from test_engine_trace_cpu import _cpu, _rgb, fake  # noqa: F401  (fake: the recording library fixture)

# fp16 entry point -> its split counterpart (the split path's only entry points)
SPLIT_OF = {
    "dm_preprocess_patchify": "dm_preprocess_patchify_split",
    "dm_assemble_tokens": "dm_assemble_tokens_f32",
    "dm_layernorm_f16": "dm_layernorm_split",
    "dm_gemm_ex": "dm_gemm_split_ex",
    "dm_attention_f16": "dm_attention_split",
    "dm_conv3x3_ex": "dm_conv3x3_split_ex",
    "dm_conv3x3_circular_ex": "dm_conv3x3_split_ex",
    "dm_resize_bilinear_nhwc_f16": "dm_resize_bilinear_nhwc_split",
    "dm_im2col_s2_f16": "dm_im2col_s2_f16",
    "dm_im2col_s2_circular_f16": "dm_im2col_s2_circular_f16",
    "dm_resize_f32": "dm_resize_f32",
}


# ---- routing table ------------------------------------------------------------------------------------------------------------
def _expected_route(t, boost, precision):
    """the table of the no_half design (DESIGN.md, "no_half")"""
    if t in (12, 13, 14):
        return "split"
    if t in (8, 9):
        return "raise"
    if t in (1, 2, 3, 5) and not boost and precision == "full":
        return "raise"
    return "unchanged"


@pytest.mark.parametrize("t", range(15))
@pytest.mark.parametrize("boost", [False, True])
@pytest.mark.parametrize("precision", ["autocast", "full"])
def test_no_half_route(t, boost, precision):
    from depthmap_b200.depthmap_generation import no_half_route
    want = _expected_route(t, boost, precision)
    if want == "raise":
        with pytest.raises(NotImplementedError, match=rf"model type {t}\b.*"):
            no_half_route(t, boost, precision)
    else:
        assert no_half_route(t, boost, precision) == want


def test_ensure_models_does_not_reload_on_no_half():
    """like the reference (src/depthmap_generation.py:60-74), only type, boost, device or tiling reload; no_half is read at load"""
    from depthmap_b200.depthmap_generation import ModelHolder
    mh = ModelHolder()
    loads = []
    mh.load_models = lambda *a: (loads.append(a), setattr(mh, "depth_model_type", a[0]), setattr(mh, "device", a[1]),
                                 setattr(mh, "tiling_mode", a[3]))
    mh.ensure_models(12, "cuda:0", False)
    mh.update_settings(no_half=True)
    mh.ensure_models(12, "cuda:0", False)
    mh.update_settings(no_half=False)
    mh.ensure_models(12, "cuda:0", False)
    assert len(loads) == 1


# ---- split weight packing -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [1, 9])
def test_split_weight_reconstructs_fp32(groups):
    import torch
    from depthmap_b200.depthmap_generation import split_weight
    g = torch.Generator().manual_seed(0)
    N, Kg = 48, 64
    w = torch.randn(N, groups * Kg, generator=g) * torch.logspace(-4, 1, N)[:, None]      # rows of very different magnitudes
    w[5] = 0                                                                                 # an all-zero (padding) row
    w[7, :3] = torch.tensor([1e-9, -3e-7, 2.5e-12])                                           # tiny entries next to large ones
    sw = split_weight(w, groups)
    assert sw.t.dtype == torch.float16 and sw.t.shape == (N, 3 * groups * Kg) and sw.scale.shape == (N,)
    s = torch.log2(sw.scale)
    assert torch.equal(s, s.round()), "the pre-scale is a power of two"
    parts = sw.t.float().reshape(N, groups, 3, Kg)
    assert torch.equal(parts[:, :, 0], parts[:, :, 1]), "each tap packs [w_hi | w_hi | w_lo]"
    rec = ((parts[:, :, 0].double() + parts[:, :, 2].double()) * sw.scale.double()[:, None, None]).reshape(N, -1)
    err = (rec - w.double()).abs()
    rowmax = w.double().abs().amax(dim=1, keepdim=True)
    # 2^-22 relative wherever the low half is a normal fp16 number; an entry 2^-24 below its row's largest lands among the fp16
    # subnormals of the pre-scaled row, whose spacing is 2^-24, i.e. 2^-35 of the row maximum at most
    assert bool((err <= 2.0 ** -22 * w.double().abs() + 2.0 ** -35 * rowmax).all()), float((err / rowmax.clamp_min(1e-300)).max())
    hi = parts[:, :, 0][w.reshape(N, groups, Kg).abs() > 0]
    assert bool((hi.abs().max() < 2048) & (sw.scale[5] == 1))


@pytest.mark.parametrize("cls", ["DptBeitEngine", "DptVitEngine"])
def test_split_refused_by_dpt_engines(cls):
    from depthmap_b200 import depthmap_generation as dg
    with pytest.raises(NotImplementedError, match="no split"):
        getattr(dg, cls)({}, 'beit_tiny', None, split=True)


# ---- split engine trace -------------------------------------------------------------------------------------------------------
def _kernels(name, args):
    """kernels one recorded call issues (csrc/*.cu): the patchify pre-processing zero-fills the K padding first when there is any
    (vit_kernels.cu: patchify_setup); a circular convolution is the halo copy plus the implicit GEMM (gemm_wgmma.cu)"""
    if name in ("dm_preprocess_patchify", "dm_preprocess_patchify_split"):
        return 1 + (args[11] > 3 * args[6] ** 2)
    if name == "dm_conv3x3_circular_ex" or (name == "dm_conv3x3_split_ex" and args[1] != "NULL"):
        return 2
    if name == "dm_dinov2_pos_embed":
        return 0
    return 1


def _run(fake, split, circular, encoder='vits'):
    from depthmap_b200.depthmap_generation import DepthAnythingV2Engine
    from oracle import synth_weights
    fake.calls.clear()
    eng = DepthAnythingV2Engine(synth_weights.make_dav2_state_dict(encoder, seed=0), encoder, _cpu(), circular=circular, split=split)
    eng.forward_batch(_rgb(2, 60, 80, 1), 70)
    calls = json.loads(json.dumps(fake.calls))
    assert eng.ops.launches == sum(_kernels(n, a) for n, a, _ in calls)
    return [(n, a) for n, a, _ in calls if n != "dm_dinov2_pos_embed"], eng


@pytest.mark.parametrize("circular", [False, True])
def test_split_trace_mirrors_fp16(fake, circular):
    f16, _ = _run(fake, False, circular)
    spl, eng = _run(fake, True, circular)
    assert len(spl) == len(f16)
    used = set()
    first_gemm = True
    for i, ((n16, a16), (ns, a)) in enumerate(zip(f16, spl)):
        assert ns == SPLIT_OF[n16], (i, n16, ns)
        used.add(ns)
        if ns == "dm_gemm_split_ex":
            d16, d = a16[4], a[5]
            assert a[1] == 3 * a16[1] and a[3] == 3 * a16[3], i                 # split operand pitches
            assert a[4] != "NULL" and d["K"] == 3 * d16["K"], i                   # wscale; the tripled depth
            if first_gemm:                                                       # the patch embedding: fp32 into the token assembly
                assert d16["epi"] == 0 and d["epi"] == 4 and d["X"] != "NULL" and d["ldx"] == d16["ldc"], i
                first_gemm = False
                continue
            assert (d["M"], d["N"], d["epi"], d["act"]) == (d16["M"], d16["N"], d16["epi"], d16["act"]), i
            assert d["ldc"] == 3 * d16["ldc"] and d["ldx"] == d16["ldx"], i
        elif ns == "dm_conv3x3_split_ex":
            d16 = a16[-2]
            d = a[-2]
            assert (a[1] != "NULL") == circular, i                                # halo scratch = circular padding
            assert a[2:6] == (a16[2:6] if circular else a16[1:5]), i               # B, H, W, Cin (logical)
            assert (d["N"], d["epi"], d["act"], d["ldc"]) == (d16["N"], d16["epi"], d16["act"], 3 * d16["ldc"]), i
            assert d["ldr"] == 3 * d16["ldr"] and d["ldr2"] == 3 * d16["ldr2"], i
            assert (d["R"] == "NULL") == (d16["R"] == "NULL") and (d["C2"] == "NULL") == (d16["C2"] == "NULL"), i
        elif ns.startswith("dm_im2col"):
            assert a[4] == 3 * a16[4] and a[1:4] == a16[1:4], i                    # the gather runs on the 3C-wide split tensor
        elif ns == "dm_attention_split":
            assert a[1:5] == a16[1:5], i                                         # B, N, heads, scale
        elif ns in ("dm_layernorm_split", "dm_resize_bilinear_nhwc_split", "dm_preprocess_patchify_split", "dm_assemble_tokens_f32"):
            scal = lambda args: [v for v in args if not (isinstance(v, str) and v.startswith("p"))]
            assert scal(a) == scal(a16), i                                       # the same logical shapes
    assert used >= {"dm_preprocess_patchify_split", "dm_assemble_tokens_f32", "dm_layernorm_split", "dm_gemm_split_ex",
                    "dm_attention_split", "dm_conv3x3_split_ex", "dm_resize_bilinear_nhwc_split"}
    assert eng.w['blocks'][0]['qkv_w'].t.shape == (3 * 384, 3 * 384)


def test_split_buffers_are_three_wide(fake):
    _, eng = _run(fake, True, False)
    b = eng._bufs
    C = eng.cfg['embed_dim']
    assert b['h'].shape[-1] == 3 * C and b['qkv'].shape[-1] == 9 * C and b['mlp'].shape[-1] == 12 * C
    assert b['x'].dtype.is_floating_point and b['x'].element_size() == 4 and b['pe'].element_size() == 4
    assert b['path'][3].shape[-1] == 3 * eng.Fp and b['patches'].shape[-1] == 3 * eng.kpad


def test_split_weights_cover_every_gemm(fake):
    from depthmap_b200.depthmap_generation import SplitWeight
    _, eng = _run(fake, True, False)
    w = eng.w
    names = [k for k in w if k.endswith('_w') and k not in ('norm_w', 'oc3_w')]
    assert names and all(isinstance(w[k], SplitWeight) for k in names), [k for k in names if not isinstance(w[k], SplitWeight)]
    for blk in w['blocks']:
        for k in ('qkv_w', 'proj_w', 'fc1_w', 'fc2_w'):
            assert isinstance(blk[k], SplitWeight)
    assert w['oc3_w'].element_size() == 4                                        # the fused 1x1 head's weights stay fp32
