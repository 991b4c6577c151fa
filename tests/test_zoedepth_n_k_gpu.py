"""GPU: ZoeDepth-N and ZoeDepth-K (model types 7 and 8) — the single-head kernels against torch fp32 restatements, and the
whole model (uint8 image in, metric depth out) against the fp32 oracle (oracle/zoedepth_single.py: metric_head_single + pad / flip
TTA, pinned to the reference module by tests/test_zoedepth_n_k_cpu.py; core = oracle/beit_dpt.py).

Bars.  Type 8 is `.half()`-ed by the reference on CUDA: tests/precision.py's rule against an fp16-policy run of the same oracle.
Type 7 is never halved by the reference (fp16 gives black images there): the LeReS bar, max < 3e-3 and mean < 6e-4 of the
range, with the fp16-policy figure printed for information.  The tiny test networks get precision.py's 1.5 slack on the max."""
import numpy as np
import pytest

import precision

pytestmark = pytest.mark.gpu

TYPE = {'n': 7, 'k': 8}


def make_state_dict(core, variant, seed, gain=1.5):
    """Seeded synthetic checkpoint.  For N the seed bins get an increasing bias ramp, ordered centres like a trained model's:
    with random order the expectation over 64 unordered softplus centres is a nearly flat map (range ~20 % of the mean), on
    which an error normalised by the range measures the flatness rather than the arithmetic."""
    import torch
    from oracle import beit_dpt, synth_weights
    from oracle import zoedepth_single as ozs
    csd = synth_weights.make_beit_dpt_state_dict(core, seed=seed)
    hsd = ozs.make_zoedepth_single_head_state_dict(variant, feat_ch=beit_dpt.CONFIGS[core]['features'], seed=seed + 100, gain=gain)
    if variant == 'n':
        hsd['seed_bin_regressor._net.2.bias'] = hsd['seed_bin_regressor._net.2.bias'] + torch.linspace(-3.0, 3.0, 64)
    sd = {"core.core." + k: v for k, v in csd.items()}
    sd.update(hsd)
    return sd


def reference_fp16_error_single(img, sd, variant, net_w, net_h, core_name, want, dev):
    """The single-head model under the reference's GPU policy for type 8 (`.half()`): core, head, TTA and the resize back all
    in fp16 on the GPU, through the oracle's own functions."""
    import torch
    from oracle import beit_dpt
    from oracle import zoedepth as ozd
    from oracle import zoedepth_single as ozs
    core_sd, head_sd = ozs.split_state_dict(sd)
    core_sd = precision.HalfView(core_sd, dev)
    head_sd = {k: v.to(dev, torch.float16) for k, v in head_sd.items()}

    def model_fn(x):
        xin = ozd.prep_for_midas(x, net_w, net_h)
        rel, feats = beit_dpt.forward(core_sd, xin, core_name, return_features=True)
        return ozs.metric_head_single(feats, rel, head_sd, variant)

    x = torch.from_numpy(np.ascontiguousarray(np.asarray(img))).permute(2, 0, 1).float().div(255.0).unsqueeze(0).to(dev, torch.float16)
    with torch.no_grad():
        out = ozd.infer(model_fn, x, pad_input=True, with_flip_aug=True)
    return precision.norm_err(out.squeeze().float().cpu().numpy(), want)


def check_bar(label, variant, got, want, ref16, tiny=False):
    """tiny: the beit_tiny test networks, whose near-argmax bin selection turns rounding noise into isolated outlier pixels, get
    tests/precision.py's slack of 1.5 on the max (type 7: 4.5e-3); the real core gets the bars above."""
    if variant == 'k':
        return precision.check(label, got, want, ref16, slack=1.5 if tiny else 1.25)
    mx, mean = precision.norm_err(got, want)
    print(f"[precision] {label}: ours max {mx:.3e} mean {mean:.3e} | fp16 policy (information) max {ref16[0]:.3e} mean {ref16[1]:.3e}")
    assert mx < (1.5 if tiny else 1.0) * 3e-3 and mean < 6e-4, (label, mx, mean)
    return mx, mean


# ---- kernels ---------------------------------------------------------------------------------------------------------------
def _lib():
    from depthmap_b200 import _lib as L
    return L, L.load()


@pytest.mark.parametrize("normed", [0, 1])
def test_seed_bins_kernel(cuda_device, normed):
    import torch
    L, lib = _lib()
    g = torch.Generator().manual_seed(3 + normed)
    rows = 1000
    seed = (torch.randn(rows, 64, generator=g) * 2.0).to(cuda_device)
    seed[:7] = -1.0                                    # whole rows at the ReLU floor: uniform widths
    out = torch.empty(rows, 64, device=cuda_device)
    L.check(lib.dm_zoe_seed_bins(seed.data_ptr(), 64, rows, normed, 1e-3, 10.0, out.data_ptr(), L.stream_ptr()), "dm_zoe_seed_bins")
    if normed:
        Bv = torch.relu(seed) + 1e-3
        w = (10.0 - 1e-3) * Bv / Bv.sum(dim=1, keepdim=True)
        e = torch.cumsum(torch.nn.functional.pad(w, (1, 0), value=1e-3), dim=1)
        want = (0.5 * (e[:, :-1] + e[:, 1:]) - 1e-3) / (10.0 - 1e-3)
    else:
        want = torch.nn.functional.softplus(seed)
    torch.cuda.synchronize()
    assert (out - want).abs().max().item() < 2e-6 * max(1.0, want.abs().max().item())


def _attractor_restated(A, n, normed, b_prev, H, W, sort_clip, dmin=1e-3, dmax=10.0):
    import torch
    import torch.nn.functional as F
    Fn, Hp, Wp, _ = b_prev.shape
    a = A.view(Fn, H, W, -1).permute(0, 3, 1, 2)
    a = torch.relu(a[:, 0:2 * n:2]) + 1e-3 if normed else F.softplus(a[:, :n])
    b = F.interpolate(b_prev.permute(0, 3, 1, 2), (H, W), mode="bilinear", align_corners=True)
    dx = a.unsqueeze(2) - b.unsqueeze(1)
    bn = b + torch.mean(dx / (1 + 300.0 * dx * dx), dim=1)
    if sort_clip:
        bn = torch.clip(torch.sort((dmax - dmin) * bn + dmin, dim=1)[0], dmin, dmax)
    return bn.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("n", [16, 8, 4, 1])
@pytest.mark.parametrize("normed,sort_clip", [(0, 0), (1, 0), (1, 1)])
def test_attractor_single_kernel(cuda_device, n, normed, sort_clip):
    import torch
    L, lib = _lib()
    g = torch.Generator().manual_seed(10 * n + 2 * normed + sort_clip)
    Fn, Hp, Wp, H, W = 3, 5, 7, 9, 13
    A = (torch.randn(Fn * H * W, 32, generator=g) * 0.6).to(cuda_device)
    # normed: b in [-0.3, 1.3] so that (max - min) b + min leaves [min, max] on both sides; pairs of equal bins make ties
    bp = torch.rand(Fn, Hp, Wp, 64, generator=g) * (1.6 if normed else 2.0) - (0.3 if normed else 0.0)
    bp[..., 1::2] = bp[..., 0::2]
    bp = bp.to(cuda_device)
    out = torch.empty(Fn, H, W, 64, device=cuda_device)
    L.check(lib.dm_zoe_attractor_single(A.data_ptr(), 32, n, normed, bp.data_ptr(), Fn, Hp, Wp, H, W, sort_clip, 1e-3, 10.0, out.data_ptr(),
                                        L.stream_ptr()), "dm_zoe_attractor_single")
    want = _attractor_restated(A, n, normed, bp, H, W, sort_clip)
    torch.cuda.synchronize()
    err = (out - want).abs().max().item()
    assert err < 2e-5 * max(1.0, want.abs().max().item()), err
    if sort_clip:
        assert bool((out[..., 1:] >= out[..., :-1]).all()) and out.min().item() >= 1e-3 and out.max().item() <= 10.0
        assert out.min().item() == pytest.approx(1e-3) and out.max().item() == 10.0     # the clip is exercised at both ends


def test_single_head_kernels_reject_bad_arguments(cuda_device):
    import torch
    L, lib = _lib()
    t = torch.zeros(64 * 64, device=cuda_device)
    p = t.data_ptr()
    assert lib.dm_zoe_attractor_single(p, 32, 3, 0, p, 1, 1, 1, 1, 1, 0, 1e-3, 10.0, p, L.stream_ptr()) == -4
    assert b"3 attractors" in lib.dm_last_error()
    assert lib.dm_zoe_attractor_single(p, 32, 16, 0, p, 1, 1, 1, 1, 1, 1, 1e-3, 10.0, p, L.stream_ptr()) == -1        # sort_clip, softplus
    assert lib.dm_zoe_attractor_single(p, 16, 16, 1, p, 1, 1, 1, 1, 1, 0, 1e-3, 10.0, p, L.stream_ptr()) == -1        # lda < 2n
    assert lib.dm_zoe_seed_bins(p, 63, 4, 0, 1e-3, 10.0, p, L.stream_ptr()) == -1
    assert lib.dm_zoe_seed_bins(p, 64, 4, 1, 10.0, 1e-3, p, L.stream_ptr()) == -1
    assert lib.dm_zoe_clb_single(p, 32, p, 64, p, p, p, p, p, p, 0.0, 1, 1, 1, 1, 1, 0.0212, 50.0, p, L.stream_ptr()) == -1  # ldz < 80
    assert b"ldz" in lib.dm_last_error()


def test_clb_single_kernel(cuda_device):
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    g = torch.Generator().manual_seed(21)
    Fn, nh, nw, h3, w3 = 2, 37, 150, 19, 75
    o32 = (torch.randn(Fn, nh, nw, 32, generator=g).abs() * 0.8).half()
    ze = torch.randn(Fn, h3, w3, 128, generator=g) * 0.7
    bc = torch.sort(torch.rand(Fn, h3, w3, 64, generator=g) * 10.0, dim=-1)[0]
    wo = torch.randn(33, 80, generator=g) * 0.25
    b0 = torch.randn(80, generator=g) * 0.3
    w2 = torch.randn(4, 80, generator=g) * 0.3
    b2 = torch.randn(4, generator=g) * 0.3
    wr = torch.randn(32, generator=g) * 0.3
    br = 0.1
    dev = [x.to(cuda_device).contiguous() for x in (o32, ze, bc, wo, b0, w2, b2, wr)]
    out = torch.empty(Fn, nh, nw, device=cuda_device)
    L.check(lib.dm_zoe_clb_single(dev[0].data_ptr(), 32, dev[1].data_ptr(), 128, dev[2].data_ptr(), dev[3].data_ptr(), dev[4].data_ptr(),
                                  dev[5].data_ptr(), dev[6].data_ptr(), dev[7].data_ptr(), br, Fn, nh, nw, h3, w3, 0.0212, 50.0, out.data_ptr(),
                                  L.stream_ptr()), "dm_zoe_clb_single")
    # restatement: rel = relu(wr . o + br); pre = [o, rel] . wo + b0 + up(ze); log-binomial over 64 bins; expectation of up(bc)
    from oracle import zoedepth as ozd
    from oracle import zoedepth_single as ozs
    o = o32.float()
    rel = torch.relu(o @ wr + br)
    up = lambda t: F.interpolate(t.permute(0, 3, 1, 2), (nh, nw), mode="bilinear", align_corners=True)
    pre = (torch.cat([o, rel.unsqueeze(-1)], dim=-1) @ wo + b0).permute(0, 3, 1, 2) + up(ze[..., :80])
    pt = F.softplus(torch.einsum('jk,nkyx->njyx', w2, F.gelu(pre)) + b2.view(1, 4, 1, 1))
    p = (pt[:, 0] + 1e-4) / (pt[:, 0] + pt[:, 1] + 2e-4)
    t = (50.0 - 0.0212) * ((pt[:, 2] + 1e-4) / (pt[:, 2] + pt[:, 3] + 2e-4)) + 0.0212
    k = torch.arange(64.0).view(1, -1, 1, 1)
    xx = p.unsqueeze(1)
    y = ozd._log_binom(torch.tensor(63.0), k) + k * torch.log(xx.clamp(1e-4, 1)) + (63 - k) * torch.log((1 - xx).clamp(1e-4, 1))
    probs = torch.softmax(y / t.unsqueeze(1), dim=1)
    want = (probs * up(bc)).sum(dim=1)
    torch.cuda.synchronize()
    err = (out.cpu() - want).abs().max().item()
    assert float(want.max() - want.min()) > 1.0 and err < 1e-4 * float(want.abs().max()), err


# ---- the model -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["n", "k"])
@pytest.mark.parametrize("seed,hw,net", [(1, (96, 128), (64, 64)), (3, (70, 50), (64, 96)), (2, (64, 64), (96, 64))])
def test_tiny_core_vs_oracle(cuda_device, variant, seed, hw, net):
    import torch
    from depthmap_b200.depthmap_generation import ZoeDepthEngine
    from oracle import zoedepth as ozd
    from oracle import zoedepth_single as ozs
    from synth import synth_rgb
    sd = make_state_dict('beit_tiny', variant, seed)
    eng = ZoeDepthEngine(sd, cuda_device, variant, core_name='beit_tiny')
    imgs = [synth_rgb(hw[0], hw[1], 5 + s) for s in range(2)]
    got = eng.forward_batch(torch.from_numpy(np.stack(imgs)).to(cuda_device), net[0], net[1]).cpu().numpy()
    assert got.shape == (2, hw[0], hw[1]) and got.dtype == np.float32
    for i, img in enumerate(imgs):
        want, invert = ozs.get_raw_prediction_single(img, sd, variant, net[0], net[1], core_name='beit_tiny')
        assert invert is True and want.max() - want.min() > 0.02
        ref16 = reference_fp16_error_single(img, sd, variant, net[0], net[1], 'beit_tiny', want, cuda_device)
        check_bar(f"zoedepth_{variant} tiny seed{seed} {hw} net {net} img{i}", variant, got[i], want, ref16, tiny=True)
        if variant == 'k':
            assert got[i].max() <= 10.0


@pytest.mark.parametrize("variant", ["n", "k"])
def test_batch_of_three_equals_three_single_calls(cuda_device, variant):
    import torch
    from depthmap_b200.depthmap_generation import ZoeDepthEngine
    from synth import synth_rgb
    eng = ZoeDepthEngine(make_state_dict('beit_tiny', variant, 4), cuda_device, variant, core_name='beit_tiny')
    imgs = torch.from_numpy(np.stack([synth_rgb(80, 112, 30 + s) for s in range(3)])).to(cuda_device)
    whole = eng.forward_batch(imgs, 96, 64).clone()
    for i in range(3):
        assert torch.equal(eng.forward_batch(imgs[i:i + 1], 96, 64)[0], whole[i]), i


def test_k_output_is_clipped_at_max_depth(cuda_device):
    """K's bins are bounded by ZoeDepth's default max_depth = 10 (no dataset config overrides it).  Head weights that put all
    but the first seed bin at the top of the range and every attractor just above it (normalised 1.02) push the centres past
    10; the last level clips them, so the log-binomial's expectation reaches 10 and never exceeds it.  The tiny-core model tests
    check the same bound on ordinary outputs."""
    import torch
    from depthmap_b200.depthmap_generation import ZoeDepthEngine
    from synth import synth_rgb
    sd = make_state_dict('beit_tiny', 'k', 5)
    w = sd['seed_bin_regressor._net.2.weight']
    sd['seed_bin_regressor._net.2.weight'] = torch.zeros_like(w)
    sd['seed_bin_regressor._net.2.bias'] = torch.cat([torch.tensor([1000.0]), torch.zeros(63)])     # width of bin 0 ~ 10
    for i in range(4):
        k = f'attractors.{i}._net.2'
        sd[k + '.weight'] = torch.zeros_like(sd[k + '.weight'])
        sd[k + '.bias'] = torch.full_like(sd[k + '.bias'], 1.02 - 1e-3)
    eng = ZoeDepthEngine(sd, cuda_device, 'k', core_name='beit_tiny')
    got = eng.forward_batch(torch.from_numpy(synth_rgb(64, 96, 2)).unsqueeze(0).to(cuda_device), 64, 64)
    net = eng._zbufs['d']                                          # the expectation at net size, before the bicubic resize back
    torch.cuda.synchronize()
    assert net.max().item() <= 10.0 and net.max().item() > 9.9, (net.min().item(), net.max().item())
    # the bicubic resize back to the image (the reference's as well) may ring a little above the largest net value
    assert got.max().item() <= 10.0 + 0.1 * (net.max() - net.min()).item()


@pytest.mark.parametrize("variant", ["n", "k"])
def test_beit384_core_through_model_holder(cuda_device, variant):
    """The real configuration: DPT-BEiT-L-384 core at the type's default net size (7: 384 x 512, 8: 384 x 768)."""
    from PIL import Image
    from depthmap_b200.depthmap_generation import ModelHolder
    from oracle import zoedepth as ozd
    from oracle import zoedepth_single as ozs
    from synth import synth_rgb
    t = TYPE[variant]
    sd = make_state_dict('beitl16_384', variant, 3)
    mh = ModelHolder()
    mh.weights_provider = lambda mt: {"model": sd}                 # the checkpoint wrapper of ZoeD_M12_{N,K}.pt
    mh.ensure_models(t, cuda_device, False)
    net = ModelHolder.get_default_net_size(t)
    assert net == {7: [384, 512], 8: [384, 768]}[t]
    img = synth_rgb(384, 320, 21)
    pred, invert = mh.get_raw_prediction(Image.fromarray(img), net[0], net[1])
    assert invert is True and pred.shape == (384, 320) and pred.dtype == np.float32
    want, _ = ozs.get_raw_prediction_single(img, sd, variant, net[0], net[1], core_name='beitl16_384')
    ref16 = reference_fp16_error_single(img, sd, variant, net[0], net[1], 'beitl16_384', want, cuda_device)
    check_bar(f"zoedepth_{variant} beitl16_384 (384x320 image, net {net})", variant, pred, want, ref16)
    with pytest.raises(NotImplementedError):
        mh.ensure_models(t, cuda_device, True)                     # BOOST on 7 / 8 is not implemented
    mh.unload_models()


@pytest.mark.parametrize("model_type", [7, 8])
def test_funnel_yields_depth(cuda_device, model_type):
    """core_generation_funnel (the drop-in entry point) with model type 7 / 8 loads ZoeDepthEngine through ModelHolder and yields
    the prediction and the depth image."""
    from PIL import Image
    from depthmap_b200 import core
    from synth import synth_rgb
    sd = make_state_dict('beitl16_384', {7: 'n', 8: 'k'}[model_type], 1)
    holder = core.get_model_holder()
    holder.unload_models()
    holder.weights_provider = lambda t: sd
    try:
        inp = dict(compute_device='GPU', model_type=model_type, net_width=128, net_height=96, net_size_match=False, boost=False,
                   do_output_depth=True, gen_stereo=False, gen_normalmap=False, do_output_depth_prediction=True)
        out = list(core.core_generation_funnel(None, [Image.fromarray(synth_rgb(96, 144, 3))], None, None, inp, ops={}))
        assert [k for _, k, _ in out][:2] == ['depth_prediction', 'depth']
        pred = out[0][2]
        assert pred.shape == (96, 144) and pred.dtype == np.float32 and np.isfinite(pred).all() and pred.max() > pred.min()
        assert type(holder.depth_model).__name__ == 'ZoeDepthEngine' and holder.depth_model.variant == {7: 'n', 8: 'k'}[model_type]
    finally:
        holder.unload_models()
        holder.weights_provider = None
