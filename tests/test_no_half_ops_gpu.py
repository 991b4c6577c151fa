"""GPU: every split (no_half, fp32-class) entry point against a float64 restatement of its operation, on inputs that only the
low halves can get right.

A split tensor stores an fp32 value v as fp16 hi = rn(v), lo = rn(v - hi), each row [hi | lo | hi].  The network test
(test_no_half_gpu.py) averages over a whole Depth-Anything-V2 forward, so one op that drops lo, reads it from the wrong third or
rounds it away would hide there.  Here each kernel gets
- one case where hi is the same constant everywhere (1.5 + u, |u| < 2^-11) and all the information is in lo: a kernel that
  ignores lo returns a near-constant and misses the bar by orders of magnitude;
- values across fp16's range: hi subnormal (|v| < 6e-5), lo subnormal (|v| < 0.125), up to 3e4 (the format holds |v| < 65504);
- the shapes the engine sends and the kernels' own edges (tile tails, 1-wide maps, B > 1, the two split GEMM tiles).
Operands are made exactly representable in the split format first (`_rep`), so the bars measure the kernel's arithmetic, not
the split of its inputs.  Bars (tests/op_bars.py): split outputs `check_split` (format, then 8 x the fp32 evaluation's error
plus the format's own), fp32 outputs `check_fp32_class`, data movement `check_exact`; every check has a `teeth` line, the main
wrong variant being the hi-only evaluation (the same operation with lo = 0)."""
import ctypes

import numpy as np
import pytest

from op_bars import check_exact, check_fp32_class, check_split, split_parts, teeth

pytestmark = pytest.mark.gpu

LO_U = 0.999 * 2.0 ** -11          # |u| < half an fp16 ulp at 1.5: rn(1.5 + u) = 1.5


# ---- split helpers --------------------------------------------------------------------------------------------------------------
def _lib():
    import depthmap_b200._lib as L
    return L, L.load()


def _no_tf32():
    import contextlib

    import torch

    @contextlib.contextmanager
    def cm():
        saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        try:
            yield
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
    return cm()


def _parts(x):
    hi = x.half()
    return hi, (x - hi.float()).half()


def _split(x):
    """fp32 [..., n] -> split fp16 [..., 3n] = [hi | lo | hi]"""
    import torch
    hi, lo = _parts(x)
    return torch.cat([hi, lo, hi], dim=-1).contiguous()


def _rep(x):
    """x as the split format holds it: hi + lo (exact in fp32)"""
    hi, lo = _parts(x)
    return hi.float() + lo.float()


def _hi(x):
    return x.half().float()


def _unsplit64(t):
    hi, lo, _ = split_parts(t)
    return hi.double() + lo.double()


def _gen(seed, dev):
    import torch
    return torch.Generator(device=dev).manual_seed(seed)


def _lo_signal(shape, g, dev, scale=1.0, sign=False):
    """scale * (1.5 + u), |u| < 2^-11: hi = 1.5 * scale everywhere (scale a power of two), all the information in lo; sign: a
    random sign per element"""
    import torch
    x = scale * (1.5 + (torch.rand(*shape, generator=g, device=dev) * 2 - 1) * LO_U)
    if sign:
        x = x * (torch.randint(0, 2, shape, generator=g, device=dev) * 2 - 1)
    return _rep(x)


def _magnitudes(shape, g, dev, dim=-1, top=1e4):
    """normal values in four bands along `dim`: hi subnormal (sd 2e-5), lo subnormal (sd 0.04), O(1), and large (sd `top`,
    clamped to 3e4)"""
    import torch
    x = torch.randn(*shape, generator=g, device=dev)
    n = shape[dim]
    s = torch.tensor([2e-5, 0.04, 1.0, top], device=dev)[torch.arange(n, device=dev) % 4]
    view = [1] * len(shape)
    view[dim] = n
    return _rep((x * s.view(view)).clamp(-3e4, 3e4))


BANDS = ("hi-subnormal", "lo-subnormal", "O(1)", "large")


def _band(n):
    """the `_magnitudes` band of index i along its dim, as a CPU array"""
    return np.arange(n) % 4


def _ftz(x):
    """x with its subnormal fp16 halves flushed to zero, as a kernel that flushes denormals would read it"""
    import torch
    hi, lo = _parts(x)
    flush = lambda t: torch.where(t.abs() < 2.0 ** -14, torch.zeros_like(t), t).float()
    return flush(hi) + flush(lo)


def _band_wrong(x, band_in):
    """the wrong-variant input of a `_magnitudes` operand: subnormals flushed in the hi-subnormal band (hi only would change
    nothing there: lo is zero), hi only in the other three; band_in: the band of each element, broadcastable to x"""
    import torch
    return torch.where(torch.as_tensor(band_in, device=x.device) == 0, _ftz(x), _hi(x))


def _band_teeth(label, wrong, ref, bar, band_out):
    """one teeth line per band: the outputs of that band only (band_out: the band of each output, broadcastable to ref)"""
    wrong, ref = wrong.double().cpu().numpy(), ref.double().cpu().numpy()
    band_out = np.broadcast_to(band_out, ref.shape)
    for k, name in enumerate(BANDS):
        m = band_out == k
        teeth(f"{label}, {name} band, {'subnormals flushed' if k == 0 else 'hi only'}", wrong[m], ref[m], np.broadcast_to(bar, ref.shape)[m])


def _wrep(sw, groups=1):
    """the fp32 weights a SplitWeight carries: (w_hi + w_lo) * scale (exact in fp32)"""
    N, K3 = sw.t.shape
    t = sw.t.view(N, groups, 3, K3 // (3 * groups))
    return ((t[:, :, 0].float() + t[:, :, 2].float()) * sw.scale[:, None, None]).reshape(N, K3 // 3)


def _sparse(w, nnz, g):
    """w [N, ...] with all but `nnz` entries of each row (at random places) zeroed: in the lo-carrying cases a dense row's fp32
    accumulation error, 8 x of which is the bar, grows with the depth until it comes within 100x of the lo signal (2^-12 of the
    value); a few products per output keep the two apart"""
    import torch
    flat = w.reshape(w.shape[0], -1)
    keep = torch.zeros_like(flat)
    keep.scatter_(1, torch.rand(flat.shape, generator=g, device=w.device).argsort(1)[:, :nnz], 1.0)
    return (flat * keep).view(w.shape)


def _same(a, b):
    import torch
    v = lambda t: t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)
    return a.shape == b.shape and torch.equal(v(a), v(b))


def _split_logical(t):
    """split [..., 3n] -> (hi, lo) [..., n] each, for bit comparisons across different row widths"""
    hi, lo, _ = split_parts(t)
    return hi, lo


# ---- 1. dm_preprocess_patchify_split ----------------------------------------------------------------------------------------------
def _cubic_matrix(n_in, n_out, dtype):
    """cv2.resize INTER_CUBIC along one axis as an [n_out, n_in] matrix: A = -0.75, replicated border, the coefficients of
    cv_cubic.cuh evaluated in `dtype` (np.float64 for the reference, np.float32 for the fp32 evaluation)"""
    f = np.dtype(dtype).type
    A = f(-0.75)
    m = np.zeros((n_out, n_in), dtype)
    s = f(n_in) / f(n_out)
    for o in range(n_out):
        x = (f(o) + f(0.5)) * s - f(0.5)
        i = int(np.floor(x))
        x = f(x - f(i))
        c0 = ((A * (x + f(1)) - f(5) * A) * (x + f(1)) + f(8) * A) * (x + f(1)) - f(4) * A
        c1 = ((A + f(2)) * x - (A + f(3))) * x * x + f(1)
        c2 = ((A + f(2)) * (f(1) - x) - (A + f(3))) * (f(1) - x) * (f(1) - x) + f(1)
        c3 = f(1) - c0 - c1 - c2
        for k, c in enumerate((c0, c1, c2, c3)):
            m[o, min(max(i - 1 + k, 0), n_in - 1)] += c
    return m


def _patchify_ref(img, nh, nw, dtype, patch=14):
    """uint8 [B, H, W, 3] -> normalised patch rows [B*gh*gw, 588], network channel c from source channel 2 - c, in `dtype`"""
    B, H, W, _ = img.shape
    mean = np.array([0.485, 0.456, 0.406], dtype)
    std = np.array([0.229, 0.224, 0.225], dtype)
    x = img.astype(dtype)[..., ::-1]
    if (H, W) != (nh, nw):
        my, mx = _cubic_matrix(H, nh, dtype), _cubic_matrix(W, nw, dtype)
        x = np.einsum("yh,bhwc,xw->byxc", my, x, mx)
    x = (x / dtype(255) - mean) / std
    gh, gw = nh // patch, nw // patch
    return np.ascontiguousarray(x.reshape(B, gh, patch, gw, patch, 3).transpose(0, 1, 3, 5, 2, 4).reshape(B * gh * gw, 3 * patch * patch))


@pytest.mark.parametrize("H,W,nh,nw", [(70, 98, 70, 98), (42, 168, 56, 84)])
def test_preprocess_patchify_split(cuda_device, H, W, nh, nw):
    """identity size and a real cubic resize, CHAN_MAP (2, 1, 0), K padded 588 -> 640 in each third; the hi third equals the
    fp16 patchify bit for bit (the same fp32 arithmetic, one rounding).  The buffer is NaN before the call, so padding the
    kernel leaves unwritten fails the bit-exact check on it.  The resize scales by 3/4 and 2, which keep every sample
    position exact in fp32: at a scale like 97/70 the fp32 position alone moves a sample of a noise image by 3e-3 of a grey
    level, which would set the bar far above the split's precision."""
    import cv2
    import torch
    L, lib = _lib()
    B, patch, kpad = 2, 14, 640
    img = np.random.default_rng(H).integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    if (H, W) != (nh, nw):    # the float64 formula is cv2's INTER_CUBIC (cv2 rounds its coefficients to fp32)
        want = np.stack([cv2.resize(i.astype(np.float64), (nw, nh), interpolation=cv2.INTER_CUBIC) for i in img])
        got = np.einsum("yh,bhwc,xw->byxc", _cubic_matrix(H, nh, np.float64), img.astype(np.float64), _cubic_matrix(W, nw, np.float64))
        assert np.abs(got - want).max() < 1e-4
    rgb = torch.from_numpy(img).to(cuda_device)
    rows = B * (nh // patch) * (nw // patch)
    args = (B, H, W, nh, nw, patch, (ctypes.c_float * 3)(0.485, 0.456, 0.406), (ctypes.c_float * 3)(0.229, 0.224, 0.225),
            (ctypes.c_int * 3)(2, 1, 0))
    out = torch.full((rows, 3 * kpad), float("nan"), dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_preprocess_patchify_split(rgb.data_ptr(), *args, out.data_ptr(), kpad, L.stream_ptr()), "dm_preprocess_patchify_split")
    o16 = torch.full((rows, kpad), float("nan"), dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_preprocess_patchify(rgb.data_ptr(), *args, o16.data_ptr(), kpad, L.stream_ptr()), "dm_preprocess_patchify")
    torch.cuda.synchronize()
    out = out.cpu().numpy().reshape(rows, 3, kpad)
    label = f"patchify_split {H}x{W} -> {nh}x{nw}"
    pad = out[:, :, 588:]
    check_exact(f"{label} K padding (3 x 52 columns)", pad, np.zeros_like(pad))
    check_exact(f"{label} hi third vs dm_preprocess_patchify", out[:, 0], o16.cpu().numpy())
    ref = _patchify_ref(img, nh, nw, np.float64)
    bar = check_split(label, out[:, :, :588].reshape(rows, 3 * 588), ref, _patchify_ref(img, nh, nw, np.float32))
    teeth(f"{label} hi only", out[:, 0, :588].astype(np.float64), ref, bar)


# ---- 2. dm_assemble_tokens_f32 ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [384, 768, 1024])
@pytest.mark.parametrize("with_pos", [True, False])
def test_assemble_tokens_f32(cuda_device, C, with_pos):
    """X[b, 0] = cls + pos[0], X[b, 1 + p] = pe[b, p] + pos[1 + p]: one fp32 add, bit-exact against torch's"""
    import torch
    L, lib = _lib()
    B, Np = 3, 37
    g = _gen(C + with_pos, cuda_device)
    pe = _magnitudes((B * Np, C), g, cuda_device)
    cls = torch.randn(C, generator=g, device=cuda_device)
    pos = torch.randn(Np + 1, C, generator=g, device=cuda_device) if with_pos else None
    X = torch.full((B, Np + 1, C), float("nan"), device=cuda_device)
    L.check(lib.dm_assemble_tokens_f32(pe.data_ptr(), cls.data_ptr(), pos.data_ptr() if with_pos else None, X.data_ptr(), B, Np, C,
                                       L.stream_ptr()), "dm_assemble_tokens_f32")
    tok = lambda first: torch.cat([cls.expand(B, 1, C), pe.view(B, Np, C)], 1) if first else torch.cat([pe.view(B, Np, C), cls.expand(B, 1, C)], 1)
    want = tok(True) + pos if with_pos else tok(True)
    torch.cuda.synchronize()
    label = f"assemble_tokens_f32 C={C} pos={'yes' if with_pos else 'NULL'}"
    check_exact(label, X, want)
    teeth(f"{label} with the class token last", tok(False) + (pos if with_pos else 0), want, 0.0)
    if with_pos:
        teeth(f"{label} with pos shifted by one token", tok(True) + torch.roll(pos, 1, 0), want, 0.0)


# ---- 3. dm_layernorm_split ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [384, 768, 1024])
@pytest.mark.parametrize("drop", [0, 1])
def test_layernorm_split(cuda_device, C, drop):
    """rows of mean 1000 next to centred ones, gamma up to 300; the hi third equals dm_layernorm_f16's output bit for bit.  The
    two kinds of row are checked apart: fp32 loses 6e-5 of a mean-1000 row's values to cancellation, so there it loses more
    than lo holds, and only the centred rows can tell a kernel that drops lo."""
    import torch
    L, lib = _lib()
    B, T = 3, 50
    g = _gen(C * 2 + drop, cuda_device)
    x = torch.randn(B * T, C, generator=g, device=cuda_device) * 3 + 1
    x[::3] += 1000.0                                      # large mean: the two-pass variance must not cancel
    gamma = 1 + 0.1 * torch.randn(C, generator=g, device=cuda_device)
    gamma[::7] *= 300.0
    beta = 0.1 * torch.randn(C, generator=g, device=cuda_device)
    rows_out = B * (T - 1) if drop else B * T
    out = torch.full((rows_out + 8, 3 * C), float("nan"), dtype=torch.float16, device=cuda_device)
    o16 = torch.full((rows_out, C), float("nan"), dtype=torch.float16, device=cuda_device)
    args = (B * T, C, gamma.data_ptr(), beta.data_ptr(), 1e-6)
    L.check(lib.dm_layernorm_split(x.data_ptr(), *args, out.data_ptr(), T, drop, L.stream_ptr()), "dm_layernorm_split")
    L.check(lib.dm_layernorm_f16(x.data_ptr(), *args, o16.data_ptr(), T, drop, L.stream_ptr()), "dm_layernorm_f16")

    def ln(xx):
        mu = xx.mean(-1, keepdim=True)
        return (xx - mu) / torch.sqrt(((xx - mu) ** 2).mean(-1, keepdim=True) + 1e-6) * gamma.to(xx.dtype) + beta.to(xx.dtype)

    sel = (lambda y: y.view(B, T, C)[:, 1:].reshape(-1, C)) if drop else (lambda y: y)
    ref = sel(ln(x.double()))
    with _no_tf32():
        e32 = sel(ln(x))
    torch.cuda.synchronize()
    label = f"layernorm_split C={C} drop_first={drop}"
    assert torch.isnan(out[rows_out:].float()).all(), "rows past the output were written"
    check_exact(f"{label} hi third vs dm_layernorm_f16", out[:rows_out, :C], o16)
    flag = torch.zeros(B * T, C)
    flag[::3] = 1.0
    big = sel(flag)[:, 0] > 0
    o, bar = out[:rows_out].cpu(), torch.empty(rows_out, C, dtype=torch.float64)
    for name, m in (("centred rows", ~big), ("rows of mean 1000", big)):
        bar[m] = torch.from_numpy(check_split(f"{label}, {name}", o[m], ref.cpu()[m], e32.cpu()[m]))
    teeth(f"{label}, centred rows, hi only", _hi(o[~big, :C].float()), ref.cpu()[~big], bar[~big])
    if drop:
        teeth(f"{label} dropping the last token instead of the first", ln(x.double()).view(B, T, C)[:, :-1].reshape(-1, C), ref, bar)
    with pytest.raises(NotImplementedError):
        L.check(lib.dm_layernorm_split(x.data_ptr(), B * T, 128, gamma.data_ptr(), beta.data_ptr(), 1e-6, out.data_ptr(), T, drop,
                                       L.stream_ptr()), "dm_layernorm_split")


# ---- 4. dm_resize_bilinear_nhwc_split -------------------------------------------------------------------------------------------------
# the decoder's up-samples at a 70 x 98 net (5 x 7 patches): refinenet4..1 (3x4 -> 5x7, 5x7 -> 10x14, 10x14 -> 20x28,
# 20x28 -> 40x56) at Fp, and output_conv1's 40x56 -> 70x98 at F2p; Fp = 64 / 128 / 256 and F2p = 64 / 64 / 128 for ViT-S / B / L
RESIZE_CASES = ([(c, 3, 4, 5, 7) for c in (64, 128, 256)] + [(c, 20, 28, 40, 56) for c in (64, 256)] + [(c, 40, 56, 70, 98) for c in (64, 128)]
                + [(64, 9, 13, 17, 1), (64, 9, 13, 1, 17), (128, 10, 14, 10, 14), (64, 1, 1, 3, 5)])


def _bilinear(x, Hout, Wout):
    """bilinear align_corners=True resize of NHWC x, arithmetic in x's dtype, at the sample positions and weights the kernel's
    (and torch's fp32 upsample's) fp32 index math gives: on a noise map the rounding of an fp32 position alone moves a sample
    by 7e-6 of the value, 30 x the split's precision, so the float64 reference interpolates at those positions"""
    import torch
    B, Hin, Win, C = x.shape

    def axis(n_in, n_out):
        f32 = lambda v: torch.tensor(float(v), dtype=torch.float32, device=x.device)
        s = f32(n_in - 1) / f32(n_out - 1) if n_out > 1 else f32(0.0)
        f = s * torch.arange(n_out, device=x.device, dtype=torch.float32)
        i0 = f.long().clamp_max(n_in - 1)
        lam = f - i0.float()
        return i0, (i0 + 1).clamp_max(n_in - 1), lam.to(x.dtype), (1 - lam).to(x.dtype)

    y0, y1, ly, hy = axis(Hin, Hout)
    x0, x1, lx, hx = axis(Win, Wout)
    hx, lx = hx[:, None], lx[:, None]
    row = lambda yy: hx * x[:, yy][:, :, x0] + lx * x[:, yy][:, :, x1]
    return hy[:, None, None] * row(y0) + ly[:, None, None] * row(y1)


@pytest.mark.parametrize("C,Hin,Win,Hout,Wout", RESIZE_CASES)
@pytest.mark.parametrize("kind", ["lo", "range"])
def test_resize_bilinear_nhwc_split(cuda_device, C, Hin, Win, Hout, Wout, kind):
    import torch
    import torch.nn.functional as F
    L, lib = _lib()
    B = 2
    g = _gen(C + Hin * Win + Hout * Wout, cuda_device)
    x = _lo_signal((B, Hin, Win, C), g, cuda_device, sign=True) if kind == "lo" else _magnitudes((B, Hin, Win, C), g, cuda_device)
    out = torch.full((B, Hout, Wout, 3 * C), float("nan"), dtype=torch.float16, device=cuda_device)
    L.check(lib.dm_resize_bilinear_nhwc_split(_split(x).data_ptr(), B, Hin, Win, C, out.data_ptr(), Hout, Wout, L.stream_ptr()),
            "dm_resize_bilinear_nhwc_split")

    def rs(t, ac=True):
        return F.interpolate(t.permute(0, 3, 1, 2), (Hout, Wout), mode="bilinear", align_corners=ac).permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    label = f"resize_split {kind} C={C} {Hin}x{Win} -> {Hout}x{Wout}"
    if (Hin, Win) == (Hout, Wout):
        # value-exact: hi + lo unchanged (re-splitting may move a half-ulp tie from lo into hi, and 1 * -0 + 0 * y is +0, so
        # not the bits)
        v, want = _unsplit64(out).cpu().numpy(), x.double().cpu().numpy()
        diff = int(np.count_nonzero(v != want))
        print(f"[kernel] {label} (identity): {diff} values of hi + lo changed (bar: value-exact)")
        assert diff == 0, label
        return
    ref = _bilinear(x.double(), Hout, Wout)
    assert (ref - rs(x.double())).abs().max() <= 3e-5 * x.abs().max()      # the torch operation, at fp32 sample positions
    chans = _band(C) if kind == "range" else None                         # "range": channels in the four bands, a bar each
    bar = check_split(label, out, ref, _bilinear(x, Hout, Wout), groups=chans)
    if kind == "range":
        _band_teeth(label, _bilinear(_band_wrong(x, _band(C)).double(), Hout, Wout), ref, bar, chans)
    else:
        teeth(f"{label} hi only", _bilinear(_hi(x).double(), Hout, Wout), ref, bar, at_least=100)
    if Hin * Win > 1:
        teeth(f"{label} with align_corners flipped", rs(x.double(), ac=False), ref, bar)


# ---- 5. dm_im2col_s2_f16 / _circular_f16 on split tensors, through the split GEMM -----------------------------------------------
@pytest.mark.parametrize("circular", [False, True])
@pytest.mark.parametrize("ocp,H,W", [(384, 5, 7), (64, 9, 4), (128, 1, 3)])
def test_im2col_s2_split_then_gemm(cuda_device, circular, ocp, H, W):
    """the reassemble stage's stride-2 conv on a split map as the engine runs it: the channel-agnostic im2col over 3 * ocp
    channels (bit-exact against torch unfold of the split tensor), then the split GEMM against down3's per-tap split weights"""
    import torch
    import torch.nn.functional as F
    from depthmap_b200 import _lib as Lm
    from depthmap_b200.depthmap_generation import _conv_w, split_weight
    L, lib = _lib()
    B = 2
    g = _gen(ocp + H * W + circular, cuda_device)
    x = _lo_signal((B, H, W, ocp), g, cuda_device, sign=True)
    w = _sparse(torch.randn(ocp, ocp, 3, 3, generator=g, device=cuda_device) * 0.3, 16, g)
    bias = torch.randn(ocp, generator=g, device=cuda_device) * 0.1
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xs = _split(x)
    cols = torch.full((B * Ho * Wo, 9 * 3 * ocp), float("nan"), dtype=torch.float16, device=cuda_device)
    name = "dm_im2col_s2_circular_f16" if circular else "dm_im2col_s2_f16"
    L.check(getattr(lib, name)(xs.data_ptr(), B, H, W, 3 * ocp, cols.data_ptr(), L.stream_ptr()), name)
    pad = (lambda t: F.pad(t, (1, 1, 1, 1), mode="circular")) if circular else (lambda t: F.pad(t, (1, 1, 1, 1)))
    unf = F.unfold(pad(xs.permute(0, 3, 1, 2).float()), 3, stride=2).view(B, 3 * ocp, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, -1)
    torch.cuda.synchronize()
    label = f"im2col_s2 split {'circular' if circular else 'zero'} {H}x{W}x3*{ocp}"
    check_exact(label, cols, unf.half())
    sw = split_weight(_conv_w(w, ocp, ocp, torch.float32), 9)
    out = torch.empty(B * Ho * Wo, 3 * ocp, dtype=torch.float16, device=cuda_device)
    Lm.Ops().gemm_split(cols, 27 * ocp, sw.t, 27 * ocp, sw.scale, B * Ho * Wo, ocp, 27 * ocp, bias=bias, C=out, ldc=3 * ocp)
    wr = _wrep(sw, 9).view(ocp, 3, 3, ocp).permute(0, 3, 1, 2)
    conv = lambda t, p=pad: F.conv2d(p(t.permute(0, 3, 1, 2)), wr.to(t.dtype), bias.to(t.dtype), stride=2).permute(0, 2, 3, 1).reshape(-1, ocp)
    ref = conv(x.double())
    with _no_tf32():
        e32 = conv(x)
    torch.cuda.synchronize()
    bar = check_split(f"{label} -> gemm_split (down3)", out, ref, e32)
    teeth(f"{label} -> gemm_split hi only", conv(_hi(x).double()), ref, bar, at_least=100)
    if circular:
        teeth(f"{label} -> gemm_split with zero padding", conv(x.double(), lambda t: F.pad(t, (1, 1, 1, 1))), ref, bar)


# ---- 6. dm_gemm_split_ex -------------------------------------------------------------------------------------------------------------
def _gemm_split(ops, As, K, sw, M, N, **kw):
    """split GEMM of logical depth K"""
    ops.gemm_split(As, 3 * K, sw.t, 3 * K, sw.scale, M, N, 3 * K, **kw)


def _acc(A, Wr, bias):
    """A Wr^T + bias in float64 and in fp32 (TF32 off)"""
    with _no_tf32():
        return A.double() @ Wr.double().t() + bias.double(), A @ Wr.t() + bias


# the trunk's GEMMs at C = 384 / 768 / 1024 (qkv N = 3C, fc1 N = 4C with GELU, proj / fc2 into the fp32 stream), the reassemble
# projections' ocp widths, N % 64 != 0 (128 x 32 tiles), M tails of 1, 63 and 127 rows, and the shortest depth (K = 64: three
# k-blocks of the tripled depth)
GEMM_CASES = ([(301, c, 3 * c, "qkv") for c in (384, 768, 1024)] + [(301, c, 4 * c, "fc1") for c in (384, 768, 1024)]
              + [(301, c, c, "proj") for c in (384, 768, 1024)] + [(301, 4 * c, c, "fc2") for c in (384, 768, 1024)]
              + [(301, 384, n, "qkv") for n in (64, 128, 192, 256, 512)] + [(130, 768, n, "qkv") for n in (96, 160, 32)]
              + [(m, 384, 192, "qkv") for m in (1, 63, 127)] + [(1, 64, 64, "fc1"), (200, 64, 96, "proj")])


@pytest.mark.parametrize("M,K,N,kind", GEMM_CASES)
def test_gemm_split_shapes(cuda_device, M, K, N, kind):
    import torch
    from depthmap_b200 import _lib as Lm
    from depthmap_b200.depthmap_generation import split_weight
    g = _gen(M * 7 + K * 3 + N, cuda_device)
    banded = M > 4                      # A's rows in the four bands of _magnitudes, each checked against its own bar
    A = _magnitudes((M, K), g, cuda_device, dim=0, top=3e3) if banded else _rep(torch.randn(M, K, generator=g, device=cuda_device))
    rows = _band(M)[:, None] if banded else None
    Wf = torch.randn(N, K, generator=g, device=cuda_device) * (0.5 / K ** 0.5)
    bias = torch.randn(N, generator=g, device=cuda_device) * 0.1
    sw = split_weight(Wf)
    Wr = _wrep(sw)
    ops = Lm.Ops()
    acc64, acc32 = _acc(A, Wr, bias)
    label = f"gemm_split {kind} M={M} K={K} N={N}"
    if kind in ("proj", "fc2"):
        gamma = torch.rand(N, generator=g, device=cuda_device) + 0.5
        X0 = _magnitudes((M, N), g, cuda_device, dim=0, top=3e3) if banded else torch.randn(M, N, generator=g, device=cuda_device)
        X = X0.clone()
        _gemm_split(ops, _split(A), K, sw, M, N, epi=Lm.EPI_RESID_F32, bias=bias, X=X, ldx=N, gamma=gamma)
        ref, e32 = X0.double() + gamma.double() * acc64, X0 + gamma * acc32
        torch.cuda.synchronize()
        bar = check_fp32_class(label, X, ref, e32, groups=rows)
        wrong = lambda A_: X0.double() + gamma.double() * _acc(A_, Wr, bias)[0]
    else:
        act = Lm.ACT_GELU if kind == "fc1" else Lm.ACT_NONE
        C = torch.full((M, 3 * N), float("nan"), dtype=torch.float16, device=cuda_device)
        _gemm_split(ops, _split(A), K, sw, M, N, act=act, bias=bias, C=C, ldc=3 * N)
        f = (lambda t: 0.5 * t * (1 + torch.erf(t / np.sqrt(2.0)))) if kind == "fc1" else (lambda t: t)
        ref, e32 = f(acc64), (torch.nn.functional.gelu(acc32) if kind == "fc1" else acc32)
        torch.cuda.synchronize()
        bar = check_split(label, C, ref, e32, groups=rows)
        wrong = lambda A_: f(_acc(A_, Wr, bias)[0])
    if banded:
        _band_teeth(label, wrong(_band_wrong(A, _band(M)[:, None])), ref, bar, rows)
    else:
        teeth(f"{label} hi only", wrong(_hi(A)), ref, bar)


@pytest.mark.parametrize("N", [64, 96, 256])
def test_gemm_split_lo_operands(cuda_device, N):
    """A with all its information in lo (sparse weights, see _sparse), then the relu-copy epilogue with residuals R, R2 whose
    information is in lo"""
    import torch
    from depthmap_b200 import _lib as Lm
    from depthmap_b200.depthmap_generation import split_weight
    M, K = 200, 768
    g = _gen(N, cuda_device)
    A = _lo_signal((M, K), g, cuda_device, sign=True)
    Wf = _sparse(torch.randn(N, K, generator=g, device=cuda_device) * 0.3, 8, g)
    bias = torch.randn(N, generator=g, device=cuda_device) * 0.1
    sw, ops = split_weight(Wf), Lm.Ops()
    Wr = _wrep(sw)
    acc64, acc32 = _acc(A, Wr, bias)
    C = torch.empty(M, 3 * N, dtype=torch.float16, device=cuda_device)
    _gemm_split(ops, _split(A), K, sw, M, N, bias=bias, C=C, ldc=3 * N)
    torch.cuda.synchronize()
    label = f"gemm_split lo-carrying A N={N}"
    bar = check_split(label, C, acc64, acc32)
    teeth(f"{label} hi only", _acc(_hi(A), Wr, bias)[0], acc64, bar, at_least=100)
    # C = acc + bias + R + R2, C2 = relu(C): R and R2 near +-1.5 each, their sum and the accumulator of comparable size
    R = _lo_signal((M, N), g, cuda_device)
    R2 = -_lo_signal((M, N), g, cuda_device)
    Wsmall = split_weight(Wf * 1e-3)
    acc64, acc32 = _acc(A, _wrep(Wsmall), bias * 1e-3)
    C1, C2 = torch.empty_like(C), torch.empty_like(C)
    _gemm_split(ops, _split(A), K, Wsmall, M, N, bias=bias * 1e-3, C=C1, ldc=3 * N, C2=C2, R=_split(R), ldr=3 * N, R2=_split(R2), ldr2=3 * N)
    torch.cuda.synchronize()
    s64, s32 = acc64 + R.double() + R2.double(), acc32 + R + R2
    label = f"gemm_split residuals R + R2 in lo N={N}"
    bar = check_split(label, C1, s64, s32)
    teeth(f"{label} hi-only residuals", acc64 + _hi(R).double() + _hi(R2).double(), s64, bar, at_least=100)
    bar = check_split(f"{label} relu copy", C2, s64.clamp_min(0), s32.clamp_min(0))
    teeth(f"{label} relu copy, hi-only residuals", (acc64 + _hi(R).double() + _hi(R2).double()).clamp_min(0), s64.clamp_min(0), bar, at_least=100)
    teeth(f"{label} relu copy without the relu", s64, s64.clamp_min(0), bar)


def test_gemm_split_row_scales(cuda_device):
    """weight rows whose magnitudes span 2^-20 to 2^10 (the per-row power of two differs from column to column) and all-zero
    rows (e = 0, as ocp padding gives): a wscale read for the neighbouring column is off by the ratio of the two scales"""
    import torch
    from depthmap_b200 import _lib as Lm
    from depthmap_b200.depthmap_generation import split_weight
    M, K, N = 257, 512, 192
    g = _gen(11, cuda_device)
    A = _rep(torch.randn(M, K, generator=g, device=cuda_device))
    e = torch.randint(-20, 11, (N,), generator=g, device=cuda_device).float()
    Wf = torch.randn(N, K, generator=g, device=cuda_device) * torch.exp2(e)[:, None] / K ** 0.5
    Wf[N - 40:] = 0.0
    Wf[5] = 0.0
    sw = split_weight(Wf)
    assert (sw.scale[N - 40:] == 1).all() and sw.scale[:N - 40].unique().numel() > 20
    Wr = _wrep(sw)
    bias = torch.randn(N, generator=g, device=cuda_device) * torch.exp2(e) * 0.1
    acc64, acc32 = _acc(A, Wr, bias)
    ops = Lm.Ops()
    C = torch.empty(M, 3 * N, dtype=torch.float16, device=cuda_device)
    _gemm_split(ops, _split(A), K, sw, M, N, bias=bias, C=C, ldc=3 * N)
    X = torch.empty(M, N, device=cuda_device)
    _gemm_split(ops, _split(A), K, sw, M, N, epi=Lm.EPI_STORE_F32, bias=bias, X=X, ldx=N)
    torch.cuda.synchronize()
    label = "gemm_split per-row weight scales 2^-20 .. 2^10"
    # columns of 2^-20-sized values next to 2^10-sized ones: the fp32 evaluation's error is taken per column
    cols = np.arange(N)[None, :]
    bar = check_split(label, C, acc64, acc32, groups=cols)
    bar32 = check_fp32_class(f"{label} (fp32 store)", X, acc64, acc32, groups=cols)
    assert _same(X[:, N - 40:], bias[N - 40:].expand(M, 40)) and _same(X[:, 5], bias[5].expand(M))
    nb = torch.arange(N, device=cuda_device) ^ 1                     # the other column of the epilogue's float2 pair
    wrong = (acc64 - bias.double()) * (sw.scale[nb] / sw.scale).double() + bias.double()
    teeth(f"{label}: wscale of the neighbouring column", wrong, acc64, bar32)
    teeth(f"{label}: hi only", _acc(_hi(A), Wr, bias)[0], acc64, bar)


@pytest.mark.parametrize("cout", [64, 256])
def test_gemm_split_pixel_shuffle_s4(cuda_device, cout):
    """ConvTranspose2d(k = s = 4) as up0 runs it: N = 16 cout, each output pixel [hi | lo | hi] of cout channels"""
    import torch
    from depthmap_b200 import _lib as Lm
    from depthmap_b200.depthmap_generation import split_weight
    B, gh, gw, s = 2, 5, 7, 4
    M, K, N = B * gh * gw, cout, s * s * cout
    g = _gen(cout, cuda_device)
    A = _lo_signal((M, K), g, cuda_device, sign=True)
    Wf = _sparse(torch.randn(N, K, generator=g, device=cuda_device) * 0.3, 8, g)
    bias = torch.randn(N, generator=g, device=cuda_device) * 0.1
    sw = split_weight(Wf)
    Wr = _wrep(sw)
    P = torch.full((B, gh * s, gw * s, 3 * cout), float("nan"), dtype=torch.float16, device=cuda_device)
    _gemm_split(Lm.Ops(), _split(A), K, sw, M, N, epi=Lm.EPI_PIXSHUF, bias=bias, C=P, ps=(s, cout, gh, gw))
    acc64, acc32 = _acc(A, Wr, bias)
    shuf = lambda t, p=(0, 1, 3, 2, 4, 5): t.reshape(B, gh, gw, s, s, cout).permute(*p).reshape(B, gh * s, gw * s, cout)
    torch.cuda.synchronize()
    ref = shuf(acc64)
    label = f"gemm_split pixel shuffle s=4 cout={cout}"
    bar = check_split(label, P, ref, shuf(acc32))
    teeth(f"{label} hi only", shuf(_acc(_hi(A), Wr, bias)[0]), ref, bar, at_least=100)
    teeth(f"{label} with i and j swapped", shuf(acc64, (0, 1, 4, 2, 3, 5)), ref, bar)


class _SplitCase:
    """the operands of one split epilogue; run(r0, r1, n0, n1) computes rows [r0, r1) x columns [n0, n1) as one call into fresh
    outputs and returns them in logical form (split outputs as (hi, lo) pairs)"""

    def __init__(self, epi, M, N, K, dev):
        import torch
        from depthmap_b200.depthmap_generation import split_weight
        self.L, self.lib = _lib()
        self.epi, self.M, self.N, self.K, self.dev = epi, M, N, K, dev
        g = _gen({"gelu_r": 1, "relu_r2_c2": 2, "resid": 3, "f32": 4, "head": 5}[epi] * 1000 + N, dev)
        self.As = _split(torch.randn(M, K, generator=g, device=dev) * 0.5)
        self.sw = split_weight(torch.randn(N, K, generator=g, device=dev) * 0.05)
        self.bias = torch.randn(N, generator=g, device=dev)
        self.gamma = torch.randn(N, generator=g, device=dev) * 0.5
        self.R = torch.randn(M, N, generator=g, device=dev)
        self.R2 = torch.randn(M, N, generator=g, device=dev)
        self.X0 = torch.randn(M, N, generator=g, device=dev)

    def run(self, r0, r1, n0, n1, stream=None):
        import torch
        L = self.L
        m, n = r1 - r0, n1 - n0
        d = L.GemmDesc()
        d.M, d.N, d.K = m, n, 3 * self.K
        d.bias = self.bias.data_ptr() + 4 * n0
        keep = []                   # the split residuals, alive until the kernel has run
        if self.epi in ("gelu_r", "relu_r2_c2"):
            C = torch.zeros(m, 3 * n, dtype=torch.float16, device=self.dev)
            R = _split(self.R[r0:r1, n0:n1])
            d.epi, d.C, d.ldc, d.R, d.ldr = L.EPI_STORE_F16, C.data_ptr(), 3 * n, R.data_ptr(), 3 * n
            outs, keep = [C], [R]
            if self.epi == "gelu_r":
                d.act = L.ACT_GELU
            else:
                C2 = torch.zeros_like(C)
                R2 = _split(self.R2[r0:r1, n0:n1])
                d.act, d.C2, d.R2, d.ldr2 = L.ACT_RELU, C2.data_ptr(), R2.data_ptr(), 3 * n
                outs, keep = [C, C2], [R, R2]
        elif self.epi in ("resid", "f32"):
            X = self.X0[r0:r1, n0:n1].clone() if self.epi == "resid" else torch.zeros(m, n, device=self.dev)
            d.epi, d.X, d.ldx = (L.EPI_RESID_F32 if self.epi == "resid" else L.EPI_STORE_F32), X.data_ptr(), n
            d.gamma = self.gamma.data_ptr() + 4 * n0
            outs = [X]
        else:                                                            # head: N = 32, whole rows
            X = torch.zeros(m, device=self.dev)
            d.epi, d.act, d.X, d.gamma, d.head_b2 = L.EPI_HEAD, L.ACT_RELU, X.data_ptr(), self.gamma.data_ptr(), 0.25
            outs = [X]
        s = L.stream_ptr() if stream is None else ctypes.c_void_p(stream.cuda_stream)
        L.check(self.lib.dm_gemm_split_ex(self.As[r0:].data_ptr(), 3 * self.K, self.sw.t[n0:].data_ptr(), 3 * self.K,
                                          self.sw.scale.data_ptr() + 4 * n0, ctypes.byref(d), s), "dm_gemm_split_ex")
        torch.cuda.synchronize()
        keep.clear()
        return [p for o in outs for p in (_split_logical(o) if o.dtype == torch.float16 else (o,))]


M_POS = 8300                   # 65 m-tiles, a 108-row tail; N = 1024: 16 n-tiles of 64, about 8 tiles per CTA


# N = 1024 runs 128 x 64 tiles; the column slices (64 at an odd 64-offset: 128 x 64; 96 and 160: 128 x 32) switch between the two
@pytest.mark.parametrize("epi,N", [("gelu_r", 1024), ("relu_r2_c2", 1024), ("resid", 1024), ("f32", 1024), ("head", 32)])
def test_gemm_split_position_independent(cuda_device, epi, N):
    case = _SplitCase(epi, M_POS, N, 1024 if epi != "head" else 256, cuda_device)
    full = case.run(0, M_POS, 0, N)
    rows = [(0, 128), (64, 64 + 1000), (4321, 4321 + 2100), (M_POS - 700, M_POS), (1, 1 + 128 * 30 + 77)]
    cols = [] if N == 32 else [(320, 384), (N - 96, N), (64, 224), (0, 512)]
    for r0, r1 in rows:
        for f, p in zip(full, case.run(r0, r1, 0, N)):
            assert _same(f[r0:r1], p), (epi, "rows", r0, r1)
    for n0, n1 in cols:
        for f, p in zip(full, case.run(0, M_POS, n0, n1)):
            assert _same(f[:, n0:n1], p), (epi, "cols", n0, n1)
    print(f"[kernel] gemm_split {epi}: {len(rows)} row slices and {len(cols)} column slices bit-identical to the whole call")


def test_gemm_split_pixel_shuffle_position_independent(cuda_device):
    """s = 4, cout = 64 (N = 1024): a batch of 40 images equals calls on image subsets"""
    import torch
    from depthmap_b200 import _lib as Lm
    from depthmap_b200.depthmap_generation import split_weight
    nimg, h, w, s, cout, K = 40, 5, 7, 4, 64, 64
    N, M = s * s * cout, nimg * h * w
    g = _gen(5, cuda_device)
    As = _split(torch.randn(M, K, generator=g, device=cuda_device))
    sw = split_weight(torch.randn(N, K, generator=g, device=cuda_device) * 0.1)
    bias = torch.randn(N, generator=g, device=cuda_device)
    ops = Lm.Ops()

    def run(b0, b1):
        out = torch.zeros(b1 - b0, s * h, s * w, 3 * cout, dtype=torch.float16, device=cuda_device)
        _gemm_split(ops, As[b0 * h * w:], K, sw, (b1 - b0) * h * w, N, epi=Lm.EPI_PIXSHUF, bias=bias, C=out, ps=(s, cout, h, w))
        torch.cuda.synchronize()
        return out

    full = run(0, nimg)
    for b0, b1 in [(0, 1), (3, 17), (39, 40)]:
        assert _same(full[b0:b1], run(b0, b1)), (b0, b1)


def test_gemm_split_graph_replay_equals_eager(cuda_device):
    import torch
    case = _SplitCase("relu_r2_c2", 4100, 1024, 1024, cuda_device)
    eager = case.run(0, case.M, 0, case.N)
    L, lib = case.L, case.lib
    C = torch.zeros(case.M, 3 * case.N, dtype=torch.float16, device=cuda_device)
    C2 = torch.zeros_like(C)
    R, R2 = _split(case.R), _split(case.R2)
    d = L.GemmDesc()
    d.M, d.N, d.K, d.epi, d.act, d.bias = case.M, case.N, 3 * case.K, L.EPI_STORE_F16, L.ACT_RELU, case.bias.data_ptr()
    d.C, d.ldc, d.C2, d.R, d.ldr, d.R2, d.ldr2 = C.data_ptr(), 3 * case.N, C2.data_ptr(), R.data_ptr(), 3 * case.N, R2.data_ptr(), 3 * case.N
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            L.check(lib.dm_gemm_split_ex(case.As.data_ptr(), 3 * case.K, case.sw.t.data_ptr(), 3 * case.K, case.sw.scale.data_ptr(),
                                         ctypes.byref(d), ctypes.c_void_p(s.cuda_stream)), "dm_gemm_split_ex")
    torch.cuda.synchronize()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, _split_logical(C) + _split_logical(C2)):
        assert _same(a, b)


def test_gemm_split_promotion_bias(cuda_device):
    """All-positive operands at logical K = 4096: every partial sum grows, so the tensor core's truncating accumulator biases
    the result low in proportion to the k-steps it accumulates before the fp32 promotion.  gemm_wgmma.cu measured the mean
    signed relative error at -1.4e-7 with SPLIT_PROMOTE = 1, -3.8e-7 with 2 and -1.0e-6 with 4 (H100 SXM, one run).  The bar
    5e-7 lies between P = 1 and P = 4, so it catches P >= 4 only: P = 2 would pass.  It rests on that one measurement (one run of
    this test gave -1.8e-7) and has not been re-derived from repeated H100 runs."""
    import torch
    from depthmap_b200 import _lib as Lm
    from depthmap_b200.depthmap_generation import split_weight
    M, N, K = 512, 512, 4096
    g = _gen(4096, cuda_device)
    A = _rep(torch.rand(M, K, generator=g, device=cuda_device) + 0.01)
    sw = split_weight(torch.rand(N, K, generator=g, device=cuda_device) + 0.01)
    Wr = _wrep(sw)
    bias = torch.zeros(N, device=cuda_device)
    X = torch.empty(M, N, device=cuda_device)
    _gemm_split(Lm.Ops(), _split(A), K, sw, M, N, epi=Lm.EPI_STORE_F32, bias=bias, X=X, ldx=N)
    ref, e32 = _acc(A, Wr, bias)
    torch.cuda.synchronize()
    rel = float(((X.double() - ref) / ref).mean())
    rel32 = float(((e32.double() - ref) / ref).mean())
    print(f"[kernel] gemm_split promotion: mean signed relative error {rel:.3e} (bar: |.| <= 5e-7; fp32 torch {rel32:.3e})")
    assert abs(rel) <= 5e-7, rel
    check_fp32_class("gemm_split all-positive K=4096", X, ref, e32)


# ---- 7. dm_conv3x3_split_ex -----------------------------------------------------------------------------------------------------------
def _conv_split(lib, L, xs, B, H, W, cin, sw, cout, halo=None, **kw):
    """dm_conv3x3_split_ex with a desc built from keyword operands (as Ops.conv3x3_split)"""
    d = L._gemm_desc(0, cout, 0, kw.get("epi", L.EPI_STORE_F16), kw.get("act", L.ACT_NONE), kw.get("bias"), kw.get("C"), 3 * cout,
                     kw.get("C2"), kw.get("R"), 3 * cout, kw.get("R2"), 3 * cout, kw.get("X"), kw.get("ldx", 1), kw.get("gamma"),
                     kw.get("head_b2", 0.0))
    L.check(lib.dm_conv3x3_split_ex(xs.data_ptr(), halo.data_ptr() if halo is not None else None, B, H, W, cin, sw.t.data_ptr(),
                                    sw.scale.data_ptr(), ctypes.byref(d), L.stream_ptr()), "dm_conv3x3_split_ex")


def _conv64(x, wr, bias, circular):
    """3x3 pad-1 conv of NHWC x in x's dtype -> NHWC"""
    import torch.nn.functional as F
    xc = x.permute(0, 3, 1, 2)
    xc = F.pad(xc, (1, 1, 1, 1), mode="circular") if circular else F.pad(xc, (1, 1, 1, 1))
    return F.conv2d(xc, wr.to(x.dtype), bias.to(x.dtype)).permute(0, 2, 3, 1)


@pytest.mark.parametrize("circular", [False, True])
@pytest.mark.parametrize("cin,cout,B,H,W,kind", [(64, 32, 2, 7, 9, "lo"), (64, 192, 4, 5, 13, "range"), (128, 64, 2, 11, 3, "lo"),
                                                 (256, 192, 4, 9, 7, "range"), (256, 64, 2, 1, 5, "lo")])
def test_conv3x3_split(cuda_device, circular, cin, cout, B, H, W, kind):
    import torch
    from depthmap_b200.depthmap_generation import _conv_w, split_weight
    L, lib = _lib()
    g = _gen(cin + cout + H * W + circular, cuda_device)
    x = _lo_signal((B, H, W, cin), g, cuda_device, sign=True) if kind == "lo" else _magnitudes((B, H, W, cin), g, cuda_device, dim=0, top=1e3)
    w = torch.randn(cout, cin, 3, 3, generator=g, device=cuda_device) / (3 * cin ** 0.5)
    if kind == "lo":
        w = _sparse(w * (3 * cin ** 0.5) * 0.3, 16, g)
    bias = torch.randn(cout, generator=g, device=cuda_device) * 0.1
    sw = split_weight(_conv_w(w, cin, cout, torch.float32), 9)
    wr = _wrep(sw, 9).view(cout, 3, 3, cin).permute(0, 3, 1, 2)
    xs = _split(x)
    halo = (lambda b: torch.empty(b * (H + 2) * (W + 2) * 3 * cin, dtype=torch.float16, device=cuda_device)) if circular else (lambda b: None)
    out = torch.full((B, H, W, 3 * cout), float("nan"), dtype=torch.float16, device=cuda_device)
    _conv_split(lib, L, xs, B, H, W, cin, sw, cout, halo(B), bias=bias, C=out)
    ref = _conv64(x.double(), wr, bias, circular)
    with _no_tf32():
        e32 = _conv64(x, wr, bias, circular)
    torch.cuda.synchronize()
    label = f"conv3x3_split {kind} {'circular' if circular else 'zero'} B={B} {H}x{W} {cin}->{cout}"
    # "range": the images of the batch in the four bands of _magnitudes (a conv sums its input channels, so bands along them
    # would all land in every output), each image checked against its own bar
    imgs = _band(B)[:, None, None, None] if kind == "range" else None
    bar = check_split(label, out, ref, e32, groups=imgs)
    if kind == "range":
        _band_teeth(label, _conv64(_band_wrong(x, _band(B)[:, None, None, None]).double(), wr, bias, circular), ref, bar, imgs)
    else:
        teeth(f"{label} hi-only activations", _conv64(_hi(x).double(), wr, bias, circular), ref, bar, at_least=100)
    if circular:
        teeth(f"{label} with zero padding", _conv64(x.double(), wr, bias, False), ref, bar)
    for b in range(B):                                     # the batch equals per-image calls bit for bit
        one = torch.full((1, H, W, 3 * cout), float("nan"), dtype=torch.float16, device=cuda_device)
        _conv_split(lib, L, xs[b:b + 1], 1, H, W, cin, sw, cout, halo(1), bias=bias, C=one)
        torch.cuda.synchronize()
        assert _same(out[b:b + 1], one), (label, b)


@pytest.mark.parametrize("circular", [False, True])
def test_conv3x3_split_head(cuda_device, circular):
    """output_conv2 as oc2 runs it: 3x3 conv 64 -> 32, ReLU, 1x1 conv 32 -> 1, ReLU in the EPI_HEAD epilogue, fp32 out"""
    import torch
    from depthmap_b200 import _lib as Lm
    from depthmap_b200.depthmap_generation import _conv_w, split_weight
    L, lib = _lib()
    B, H, W, cin = 2, 13, 17, 64
    g = _gen(64 + circular, cuda_device)
    x = _lo_signal((B, H, W, cin), g, cuda_device, sign=True)
    w = _sparse(torch.randn(32, cin, 3, 3, generator=g, device=cuda_device) * 0.3, 16, g)
    bias = torch.randn(32, generator=g, device=cuda_device) * 0.1
    w2 = torch.rand(32, generator=g, device=cuda_device) - 0.3
    sw = split_weight(_conv_w(w, cin, 32, torch.float32), 9)
    wr = _wrep(sw, 9).view(32, 3, 3, cin).permute(0, 3, 1, 2)
    halo = torch.empty(B * (H + 2) * (W + 2) * 3 * cin, dtype=torch.float16, device=cuda_device) if circular else None
    D = torch.full((B * H * W,), float("nan"), device=cuda_device)
    _conv_split(lib, L, _split(x), B, H, W, cin, sw, 32, halo, epi=Lm.EPI_HEAD, act=Lm.ACT_RELU, bias=bias, X=D, gamma=w2, head_b2=0.05)
    head = lambda t: (_conv64(t, wr, bias, circular).clamp_min(0).reshape(-1, 32) @ w2.to(t.dtype) + 0.05).clamp_min(0)
    ref = head(x.double())
    with _no_tf32():
        e32 = head(x)
    torch.cuda.synchronize()
    label = f"conv3x3_split head 64->32->1 {'circular' if circular else 'zero'}"
    assert (ref > 0).float().mean() > 0.2
    bar = check_fp32_class(label, D, ref, e32)
    teeth(f"{label} hi-only activations", head(_hi(x).double()), ref, bar, at_least=100)


def test_conv3x3_split_refinenet_sum(cuda_device):
    """resConfUnit1's second conv of a refinenet: C = conv + bias + R + R2 (l_i and the up-sampled path, both carrying their
    information in lo) and the relu copy C2, at Fp = 128"""
    import torch
    from depthmap_b200.depthmap_generation import _conv_w, split_weight
    L, lib = _lib()
    B, H, W, F_ = 2, 9, 11, 128
    g = _gen(128, cuda_device)
    x = _rep(torch.randn(B, H, W, F_, generator=g, device=cuda_device).clamp_min(0))
    w = torch.randn(F_, F_, 3, 3, generator=g, device=cuda_device) * 1e-3 / (3 * F_ ** 0.5)
    bias = torch.randn(F_, generator=g, device=cuda_device) * 1e-3
    R = _lo_signal((B, H, W, F_), g, cuda_device, sign=True)
    R2 = _lo_signal((B, H, W, F_), g, cuda_device, sign=True)
    sw = split_weight(_conv_w(w, F_, F_, torch.float32), 9)
    wr = _wrep(sw, 9).view(F_, 3, 3, F_).permute(0, 3, 1, 2)
    C = torch.empty(B, H, W, 3 * F_, dtype=torch.float16, device=cuda_device)
    C2 = torch.empty_like(C)
    _conv_split(lib, L, _split(x), B, H, W, F_, sw, F_, bias=bias, C=C, C2=C2, R=_split(R), R2=_split(R2))
    s64 = _conv64(x.double(), wr, bias, False) + R.double() + R2.double()
    with _no_tf32():
        s32 = _conv64(x, wr, bias, False) + R + R2
    torch.cuda.synchronize()
    label = "conv3x3_split refinenet C = conv + R + R2"
    bar = check_split(label, C, s64, s32)
    wrong = _conv64(x.double(), wr, bias, False) + _hi(R).double() + _hi(R2).double()
    teeth(f"{label} hi-only residuals", wrong, s64, bar, at_least=100)
    bar = check_split(f"{label}, relu copy", C2, s64.clamp_min(0), s32.clamp_min(0))
    teeth(f"{label}, relu copy of hi-only residuals", wrong.clamp_min(0), s64.clamp_min(0), bar, at_least=100)


# ---- 8. dm_attention_split -----------------------------------------------------------------------------------------------------------
def _attn(qkv, B, N, heads, scale):
    """softmax(scale q k^T) v per image and head in qkv's dtype: qkv [B*N, 3C] -> [B*N, C]"""
    import torch
    q, k, v = qkv.view(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    o = torch.softmax((q @ k.transpose(-1, -2)) * scale, dim=-1) @ v
    return o.transpose(1, 2).reshape(B * N, heads * 64)


def _attn_unmasked(qkv, B, N, heads, scale):
    """the wrong variant: image b's last key tile read to its 128-row end without the mask, i.e. with image b + 1's first keys
    (zeros past the last image, as the tensor map fills them)"""
    import torch
    T = (N + 127) // 128 * 128
    flat = torch.cat([qkv, torch.zeros(T, qkv.shape[1], dtype=qkv.dtype, device=qkv.device)]).view(-1, 3, heads, 64)
    outs = []
    for b in range(B):
        q = flat[b * N:(b + 1) * N, 0].transpose(0, 1)
        k, v = flat[b * N:b * N + T, 1].transpose(0, 1), flat[b * N:b * N + T, 2].transpose(0, 1)
        outs.append((torch.softmax((q @ k.transpose(-1, -2)) * scale, -1) @ v).transpose(0, 1).reshape(N, heads * 64))
    return torch.cat(outs)


def _run_attention(qkv, B, N, heads, scale, dev):
    import torch
    L, lib = _lib()
    out = torch.full((B * N, 3 * heads * 64), float("nan"), dtype=torch.float16, device=dev)
    L.check(lib.dm_attention_split(_split(qkv).data_ptr(), B, N, heads, ctypes.c_float(scale), out.data_ptr(), L.stream_ptr()),
            "dm_attention_split")
    with _no_tf32():
        ref, e32 = _attn(qkv.double(), B, N, heads, scale), _attn(qkv, B, N, heads, scale)
    torch.cuda.synchronize()
    return out, ref, e32


@pytest.mark.parametrize("N", [63, 64, 65, 127, 128, 129])
@pytest.mark.parametrize("heads", [6, 12, 16])
def test_attention_split_tile_edges(cuda_device, N, heads):
    """B = 3: every image but the last has a key tile whose rows past N are the next image's, which the mask must drop"""
    import torch
    B, scale = 3, 0.125
    qkv = _rep(torch.randn(B * N, 3 * heads * 64, generator=_gen(N * 100 + heads, cuda_device), device=cuda_device))
    out, ref, e32 = _run_attention(qkv, B, N, heads, scale, cuda_device)
    label = f"attention_split N={N} heads={heads} B={B}"
    bar = check_split(label, out, ref, e32)
    teeth(f"{label} hi only", _attn(_hi(qkv).double(), B, N, heads, scale), ref, bar)
    if N % 128:
        teeth(f"{label} with the tail keys unmasked", _attn_unmasked(qkv.double(), B, N, heads, scale), ref, bar)


@pytest.mark.parametrize("N", [64, 65])
def test_attention_split_lo_operands(cuda_device, N):
    """q and k near +-3 and v near +-1.5, all their information in lo"""
    B, heads, scale = 3, 6, 0.125
    g = _gen(N, cuda_device)
    C = heads * 64
    import torch
    qkv = torch.cat([_lo_signal((B * N, 2 * C), g, cuda_device, scale=2.0, sign=True), _lo_signal((B * N, C), g, cuda_device, sign=True)], 1)
    out, ref, e32 = _run_attention(qkv, B, N, heads, scale, cuda_device)
    label = f"attention_split lo-carrying q, k, v N={N}"
    bar = check_split(label, out, ref, e32)
    teeth(f"{label} hi only", _attn(_hi(qkv).double(), B, N, heads, scale), ref, bar, at_least=100)


def test_attention_split_rising_scores(cuda_device):
    """keys grow along the sequence, so the running max rises from tile to tile: the O * alpha + PV rescale by FFMA"""
    import torch
    B, N, heads, scale = 2, 1025, 2, 0.125
    g = _gen(1025, cuda_device)
    x = torch.randn(B * N, 3, heads, 64, generator=g, device=cuda_device)
    ramp = torch.linspace(0.0, 6.0, N, device=cuda_device).repeat(B).view(B * N, 1, 1)
    x[:, 0] = x[:, 0].abs()
    x[:, 1] = x[:, 1].abs() * 0.2 + ramp
    qkv = _rep(x.reshape(B * N, 3 * heads * 64))
    q, k, _ = qkv.view(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * scale
    rise = float((s.max(-1).values - s[..., :128].max(-1).values).max())
    print(f"[kernel] attention_split rising scores: the row max rises by up to {rise:.1f} past the first key tile")
    assert rise > 16
    out, ref, e32 = _run_attention(qkv, B, N, heads, scale, cuda_device)
    label = "attention_split rising scores N=1025"
    bar = check_split(label, out, ref, e32)
    teeth(f"{label} hi only", _attn(_hi(qkv).double(), B, N, heads, scale), ref, bar)


@pytest.mark.parametrize("N", [129, 257])
def test_attention_split_peaked(cuda_device, N):
    """large scores: most probabilities lie below 2^-15 of their row's max, where p * 2^12 splits into a subnormal lo; v carries
    its information in lo, so the few keys that count must be read to their last bit"""
    import torch
    B, heads, scale = 2, 6, 0.125
    C = heads * 64
    g = _gen(N + 7, cuda_device)
    qk = torch.randn(B * N, 2 * C, generator=g, device=cuda_device) * 2.5
    qkv = torch.cat([_rep(qk), _lo_signal((B * N, C), g, cuda_device, sign=True)], 1)
    q, k, _ = qkv.view(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = (q.double() @ k.double().transpose(-1, -2)) * scale
    small = float(((s - s.max(-1, keepdim=True).values) * np.log2(np.e) < -15).double().mean())
    print(f"[kernel] attention_split peaked N={N}: {small:.2f} of the probabilities below 2^-15 of their row max")
    assert small > 0.5
    out, ref, e32 = _run_attention(qkv, B, N, heads, scale, cuda_device)
    label = f"attention_split peaked N={N}"
    bar = check_split(label, out, ref, e32)
    teeth(f"{label} hi only", _attn(_hi(qkv).double(), B, N, heads, scale), ref, bar, at_least=100)
