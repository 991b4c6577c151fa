"""GPU: the BOOST glue kernels (csrc/boost_kernels.cu) one by one, each against a float64 (or bit-exact) restatement of what the
reference's estimateboost does with numpy and cv2 at that step: the min-max normalisations, the fp64 fit sums, the blend (the
rank-truncated np.polyfit line, cv2's cubic resize, generatemask resized bilinearly), cv2.resize(INTER_CUBIC) of pitched crops,
the uint8 -> float conversion and the fixed-order chunk sum of the merge network.  Bars and the wrong-variant checks:
tests/op_bars.py."""
import functools
import math
import warnings

import numpy as np
import pytest

from op_bars import check_exact, check_f32, teeth

pytestmark = pytest.mark.gpu

N_CASES = [1, 255, 257, 528 * 256 + 3, 1024 * 1024]      # 528 partial blocks of 256 threads: below, at and past one grid stride


def _lib():
    import depthmap_b200._lib as L
    return L, L.load()


def _minmax(L, lib, x):
    import torch
    P = int(lib.dm_boost_partials())
    p = torch.full((2 * P,), float("nan"), device=x.device)
    L.check(lib.dm_boost_minmax(x.data_ptr(), x.numel(), p.data_ptr(), L.stream_ptr()), "dm_boost_minmax")
    return p


@pytest.mark.parametrize("n", N_CASES)
def test_boost_minmax_merge_post_normalise(cuda_device, n):
    """minmax partials fold to the exact extremes; merge_input (each estimate to [-1, 1]), post with normalise 0 and 1 and
    minmax_normalise against float64 of the reference's numpy expressions"""
    import torch
    L, lib = _lib()
    g = torch.Generator().manual_seed(n)
    outer = torch.randn(n, generator=g) * 3 + 1
    inner = torch.rand(n, generator=g) * 5 - 2
    t = 0.6 * torch.tanh(torch.randn(n, generator=g) * 2) + 0.2
    outer[-1], inner[-1] = 40.0, -9.0                      # the extremes sit in the grid's tail
    od, idd, td = (v.to(cuda_device) for v in (outer, inner, t))
    po, pi, pt = _minmax(L, lib, od), _minmax(L, lib, idd), _minmax(L, lib, td)
    torch.cuda.synchronize()
    for name, p, v in (("outer", po, outer), ("inner", pi, inner), ("t", pt, t)):
        p = p.cpu()
        check_exact(f"boost_minmax {name} n={n}", torch.stack([p[0::2].min(), p[1::2].max()]), torch.stack([v.min(), v.max()]))

    # post, normalise = 0: (t + 1) / 2
    out = torch.full((n,), float("nan"), device=cuda_device)
    L.check(lib.dm_boost_post(td.data_ptr(), n, None, 0, out.data_ptr(), L.stream_ptr()), "dm_boost_post")
    torch.cuda.synchronize()
    check_f32(f"boost_post normalise=0 n={n}", out.cpu(), (t.double() + 1) / 2, (t + 1) / 2, 1e-7)

    # minmax_normalise: (x - min) / (max - min); one element is a constant map (the degenerate flag, zeros)
    flag = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    L.check(lib.dm_boost_minmax_normalise(od.data_ptr(), n, po.data_ptr(), out.data_ptr(), flag.data_ptr(), L.stream_ptr()),
            "dm_boost_minmax_normalise")
    torch.cuda.synchronize()
    if n == 1:
        assert int(flag) == 1 and float(out.cpu().abs().max()) == 0.0
        return
    assert int(flag) == 0

    def mm(x):
        return (x - x.min()) / (x.max() - x.min())
    want = mm(outer.double())
    bar = check_f32(f"boost_minmax_normalise n={n}", out.cpu(), want, mm(outer), 1e-7)
    teeth("minmax_normalise without the shift by the minimum", outer.double() / (outer.max() - outer.min()).double(), want, bar)

    # merge_input: cat(2 mm(outer) - 1, 2 mm(inner) - 1) per pixel
    x2 = torch.full((n, 2), float("nan"), device=cuda_device)
    L.check(lib.dm_boost_merge_input(od.data_ptr(), idd.data_ptr(), n, po.data_ptr(), pi.data_ptr(), x2.data_ptr(), L.stream_ptr()),
            "dm_boost_merge_input")
    torch.cuda.synchronize()
    want = torch.stack([mm(outer.double()) * 2 - 1, mm(inner.double()) * 2 - 1], dim=1)
    bar = check_f32(f"boost_merge_input n={n}", x2.cpu(), want, torch.stack([mm(outer) * 2 - 1, mm(inner) * 2 - 1], dim=1), 1e-7)
    teeth("merge_input with the estimates swapped", want.flip(1), want, bar)

    # post, normalise = 1: m = (t + 1) / 2, then min-max of m
    L.check(lib.dm_boost_post(td.data_ptr(), n, pt.data_ptr(), 1, out.data_ptr(), L.stream_ptr()), "dm_boost_post")
    torch.cuda.synchronize()
    want = mm((t.double() + 1) / 2)
    bar = check_f32(f"boost_post normalise=1 n={n}", out.cpu(), want, mm((t + 1) / 2), 1e-7)
    teeth("boost_post without the min-max step", (t.double() + 1) / 2, want, bar)


@pytest.mark.parametrize("span,flat", [(0.0, True), (2e-16, True), (3e-16, False)])
def test_boost_minmax_normalise_float64_eps(cuda_device, span, flat):
    """estimatemidasBoost stops when max - min <= float64 eps (2.2e-16): a span just below is flagged and written as zeros, one
    just above normalises (a float32-eps threshold would flag both)"""
    import torch
    L, lib = _lib()
    n = 1000
    x = torch.full((n,), 0.75 if span == 0.0 else 0.0)
    x[::3] += span
    xd = x.to(cuda_device)
    p = _minmax(L, lib, xd)
    out = torch.full((n,), float("nan"), device=cuda_device)
    flag = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    L.check(lib.dm_boost_minmax_normalise(xd.data_ptr(), n, p.data_ptr(), out.data_ptr(), flag.data_ptr(), L.stream_ptr()),
            "dm_boost_minmax_normalise")
    torch.cuda.synchronize()
    want = torch.zeros(n) if flat else (x - x.min()) / (x.max() - x.min())
    assert int(flag) == int(flat) and (float(x.max() - x.min()) > 2.220446049250313e-16) != flat
    check_exact(f"boost_minmax_normalise span {span:g}", out.cpu(), want)
    if not flat:
        assert float(want.max()) == 1.0            # a degenerate answer (all zeros) would miss this


@pytest.mark.parametrize("n", N_CASES)
def test_boost_fit_sums(cuda_device, n):
    """the four fp64 sums of np.polyfit's normal equations: within 1e-10 relative of math.fsum of the same (exact) products"""
    import torch
    L, lib = _lib()
    g = torch.Generator().manual_seed(n + 1)
    x = 0.5 + 0.2 * torch.randn(n, generator=g)
    y = 0.3 * x + 0.1 + 0.01 * torch.randn(n, generator=g)
    P = int(lib.dm_boost_partials())
    sums = torch.full((4 * P,), float("nan"), dtype=torch.float64, device=cuda_device)
    xd_, yd_ = x.to(cuda_device), y.to(cuda_device)
    L.check(lib.dm_boost_fit_sums(xd_.data_ptr(), yd_.data_ptr(), n, sums.data_ptr(), L.stream_ptr()),
            "dm_boost_fit_sums")
    torch.cuda.synchronize()
    part = sums.cpu().numpy().reshape(P, 4)
    got = [math.fsum(part[:, k]) for k in range(4)]
    xd, yd = x.double().numpy(), y.double().numpy()
    terms = [xd, yd, xd * xd, xd * yd]                       # products of two floats are exact in float64
    want = [math.fsum(t) for t in terms]
    rel = max(abs(a - b) / abs(b) for a, b in zip(got, want))
    print(f"[kernel] boost_fit_sums n={n}: max relative error {rel:.3e} (bar 1e-10)")
    assert rel <= 1e-10, (got, want)
    if n >= 528 * 256:
        f32 = [float(np.cumsum(t.astype(np.float32), dtype=np.float32)[-1]) for t in terms]
        rel32 = max(abs(a - b) / abs(b) for a, b in zip(f32, want))
        print(f"[kernel] boost_fit_sums with float32 accumulation: off by {rel32:.3e} relative")
        assert rel32 >= 1e-9


@functools.lru_cache(maxsize=None)
def _generatemask(n):
    from oracle.boost import generatemask
    return generatemask((n, n))


def _blend_ref(mapped, upd, slope, icpt, rect, dtype):
    """estimateboost's merge step (:911-924): the fitted patch cv2-cubic-resized to the rect, generatemask(3000^2) resized
    bilinearly, updated = updated (1 - mask) + merged mask inside the rect"""
    import cv2
    x, y, w, h = rect
    mask = cv2.resize(_generatemask(3000).astype(dtype), (w, h), interpolation=cv2.INTER_LINEAR)
    if dtype == np.float64:
        merged = cv2.resize(mapped.astype(np.float64), (w, h), interpolation=cv2.INTER_CUBIC) * slope + icpt
    else:
        merged = cv2.resize((slope * mapped.astype(np.float64) + icpt).astype(np.float32), (w, h), interpolation=cv2.INTER_CUBIC)
    region = upd[y:y + h, x:x + w].astype(dtype)
    return (region * (1 - mask) + merged * mask).astype(dtype)


@pytest.mark.parametrize("spread", [0.5, 0.05])
@pytest.mark.parametrize("Hu,Wu,rect", [(900, 1200, (500, 400, 700, 500)), (1200, 1500, (200, 100, 1300, 1100))])
def test_boost_blend(cuda_device, spread, Hu, Wu, rect):
    """the fit (both np.polyfit regimes: spread 0.5 is the regression line, 0.05 the rank-truncated solution), the cubic resize
    of the fitted 1024^2 patch and the Gaussian mask, for rects smaller and larger than 1024 that touch the right and bottom
    border of an `updated` whose pitch exceeds the rect's width; pixels outside the rect stay untouched"""
    import torch
    from depthmap_b200.boost import MASK_SIZE, PIX2PIX_SIZE, mask_profile
    from test_polyfit_model import closed_form
    L, lib = _lib()
    S = PIX2PIX_SIZE
    x, y, w, h = rect
    assert x + w == Wu and y + h == Hu and w != h
    rng = np.random.default_rng(int(spread * 100) + w)
    mapped = (0.5 + spread * rng.standard_normal((S, S))).astype(np.float32)
    base = (0.3 * mapped + 0.1 + 0.01 * rng.standard_normal((S, S))).astype(np.float32)
    upd = (2.0 + rng.standard_normal((Hu, Wu))).astype(np.float32)
    md = torch.from_numpy(mapped).to(cuda_device)
    P = int(lib.dm_boost_partials())
    sums = torch.empty(4 * P, dtype=torch.float64, device=cuda_device)
    bd = torch.from_numpy(base).to(cuda_device)
    L.check(lib.dm_boost_fit_sums(md.data_ptr(), bd.data_ptr(), S * S, sums.data_ptr(), L.stream_ptr()),
            "dm_boost_fit_sums")
    ud = torch.from_numpy(upd).to(cuda_device)
    prof = torch.from_numpy(mask_profile()).to(cuda_device)
    L.check(lib.dm_boost_blend(md.data_ptr(), S, sums.data_ptr(), prof.data_ptr(), MASK_SIZE, ud.data_ptr(), Wu, x, y, w, h, L.stream_ptr()),
            "dm_boost_blend")
    torch.cuda.synchronize()
    got = ud.cpu().numpy()

    slope, icpt, full = closed_form(mapped.ravel(), base.ravel())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pf = np.polyfit(mapped.ravel(), base.ravel(), deg=1)
    assert abs(pf[0] - slope) < 1e-3 and abs(pf[1] - icpt) < 1e-3 and full == (spread == 0.5)
    want = _blend_ref(mapped, upd, slope, icpt, rect, np.float64)
    inside = np.zeros((Hu, Wu), bool)
    inside[y:y + h, x:x + w] = True
    check_exact("boost_blend outside the rect", got[~inside], upd[~inside])
    bar = check_f32(f"boost_blend spread {spread} rect {rect} in {Hu}x{Wu} (slope {slope:.4f})", got[y:y + h, x:x + w], want,
                    _blend_ref(mapped, upd, slope, icpt, rect, np.float32), 1e-6 * float(np.abs(want).max()))
    if not full:
        ols = np.polyfit(mapped.ravel().astype(np.float64), base.ravel().astype(np.float64), deg=1)
        assert abs(ols[0] - slope) > 0.02, (ols, slope)         # the truncated fit is far from the regression line here
        teeth("boost_blend with the least-squares line", _blend_ref(mapped, upd, ols[0], ols[1], rect, np.float64), want, bar)
    flipped = _blend_ref(mapped.T.copy(), upd, slope, icpt, rect, np.float64)
    teeth("boost_blend with the patch transposed (w and h swapped)", flipped, want, bar)


@pytest.mark.parametrize("planes,Hin,Win,Hout,Wout", [(1, 300, 200, 1024, 1024), (3, 257, 301, 129, 97), (1, 1024, 1024, 700, 500),
                                                      (3, 120, 160, 120, 333), (1, 77, 55, 77, 55)])
def test_boost_resize_cubic(cuda_device, planes, Hin, Win, Hout, Wout):
    """cv2.resize(INTER_CUBIC) of a crop given as a pointer offset into a pitched parent (touching its right and bottom border):
    3 planes, up and down, one dimension unchanged, and the same-size copy"""
    import cv2
    import torch
    L, lib = _lib()
    Hpar, Wpar = Hin + 9, Win + 13
    y0, x0 = Hpar - Hin, Wpar - Win
    rng = np.random.default_rng(Hin * Win + planes)
    parent = (rng.standard_normal((planes, Hpar, Wpar)) * 2 + 1).astype(np.float32)
    pd = torch.from_numpy(parent).to(cuda_device)
    out = torch.full((planes, Hout, Wout), float("nan"), device=cuda_device)
    L.check(lib.dm_boost_resize_cubic(pd.data_ptr() + 4 * (y0 * Wpar + x0), Wpar, Hpar * Wpar, Hin, Win, out.data_ptr(), Wout,
                                      Hout * Wout, Hout, Wout, planes, L.stream_ptr()), "dm_boost_resize_cubic")
    torch.cuda.synchronize()

    def cv(src, dtype):
        return np.stack([cv2.resize(src[p].astype(dtype), (Wout, Hout), interpolation=cv2.INTER_CUBIC) for p in range(planes)])
    crop = parent[:, y0:, x0:]
    want = cv(crop, np.float64)
    bar = check_f32(f"boost_resize_cubic {planes} x {Hin}x{Win} -> {Hout}x{Wout}", out.cpu(), want, cv(crop, np.float32),
                    1e-6 * float(np.abs(want).max()))
    teeth("boost_resize_cubic ignoring the crop offset", cv(parent[:, :Hin, :Win], np.float64), want, bar)


@pytest.mark.parametrize("H,W", [(1, 1), (16, 16), (37, 53), (480, 641)])
def test_boost_u8_to_planar(cuda_device, H, W):
    """uint8 HWC -> planar fp32 x / 255, bit-exact against numpy's (x / 255.0).astype(float32); every byte value occurs"""
    import torch
    L, lib = _lib()
    rgb = np.random.default_rng(H * W).integers(0, 256, (H, W, 3), dtype=np.uint8)
    flat = rgb.reshape(-1)
    flat[:min(256, flat.size)] = np.arange(min(256, flat.size), dtype=np.uint8)
    out = torch.full((3, H, W), float("nan"), device=cuda_device)
    rgb_d = torch.from_numpy(rgb).to(cuda_device)
    L.check(lib.dm_boost_u8_to_planar(rgb_d.data_ptr(), H, W, out.data_ptr(), L.stream_ptr()),
            "dm_boost_u8_to_planar")
    torch.cuda.synchronize()
    want = (rgb.transpose(2, 0, 1) / 255.0).astype(np.float32)
    check_exact(f"boost_u8_to_planar {H}x{W}", out.cpu().numpy(), want)
    if H * W > 1:
        teeth("u8_to_planar in BGR order", want[::-1], want, 0.0)


@pytest.mark.parametrize("nchunks", [1, 2, 3, 5])
def test_sum_chunks_f32(cuda_device, nchunks):
    """out = gamma[i % N] * (ws[0] + ws[1] + ...): a sequential fp32 sum in chunk order, bit-exact; M * N / 4 = 592 threads"""
    import torch
    L, lib = _lib()
    M, N = 37, 64
    mn = M * N
    rng = np.random.default_rng(nchunks)
    ws = (rng.standard_normal((nchunks, mn)) * (10.0 ** rng.integers(-3, 4, (nchunks, 1)))).astype(np.float32)
    gamma = (0.5 + rng.random(N)).astype(np.float32)
    out = torch.full((mn,), float("nan"), device=cuda_device)
    wsd, gd = torch.from_numpy(ws).to(cuda_device), torch.from_numpy(gamma).to(cuda_device)
    L.check(lib.dm_sum_chunks_f32(wsd.data_ptr(), nchunks, mn, N, gd.data_ptr(),
                                  out.data_ptr(), L.stream_ptr()), "dm_sum_chunks_f32")
    torch.cuda.synchronize()

    def seq(order, g):
        acc = ws[order[0]].copy()
        for c in order[1:]:
            acc = (acc + ws[c]).astype(np.float32)
        return (acc * np.tile(g, M)).astype(np.float32)
    want = seq(list(range(nchunks)), gamma)
    check_exact(f"sum_chunks_f32 {nchunks} chunks", out.cpu().numpy(), want)
    if nchunks >= 3:
        teeth("sum_chunks in reverse chunk order", seq(list(range(nchunks))[::-1], gamma), want, 0.0)
    teeth("sum_chunks with gamma indexed by the row", seq(list(range(nchunks)), np.roll(gamma, 4)), want, 0.0)
