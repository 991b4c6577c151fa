"""Shared by the kernel-level GPU tests (test_zoe_nk_ops_gpu.py, test_boost_ops_gpu.py, test_leres_dpt_ops_gpu.py): the bar an
output earns from its type when a kernel is compared with a float64 restatement of its operation, and the "teeth" check that a
plausible wrong variant of the operation would miss that bar by a wide margin on the same input.

- data movement, max, casts: bit-exact (`check_exact`);
- fp16 outputs computed in fp32: within one fp16 ulp of the float64 value (`check_f16`); magnitudes below `floor` get the
  spacing at `floor`, where fp32 cancellation, not the final rounding, sets the error;
- fp32 outputs: 4 x the max error of the same formula evaluated in fp32 torch on the same inputs, with a stated floor
  (`check_f32`), in the spirit of tests/precision.py: a fixed number is either toothless or flaky where the formula amplifies
  fp32 rounding (the log-binomial softmax at min_temp, the cubic resize of a large map);
- split (fp32-class, no_half) outputs, rows [hi | lo | hi] of fp16 with hi = rn(v), lo = rn(v - hi): the format first (third 0
  equals third 2 bit for bit, |lo| <= ulp16(hi) / 2), then the value hi + lo within 8 x the max error of the same formula in fp32
  torch (TF32 off) plus the format's own error, 2^-22 |ref| + 2^-25 (the last for a subnormal lo) (`check_split`); fp32 outputs
  of the split kernels get the same 8 x with fp32's own rounding, 2^-24 |ref|, in place of the format's (`check_fp32_class`).
Every check prints its measured error next to its bar."""
import numpy as np


def _f64(x):
    if hasattr(x, "detach"):
        x = x.detach().cpu().double().numpy()
    return np.asarray(x, dtype=np.float64)


def ulp16(ref, floor=2.0 ** -6):
    """spacing of fp16 at |ref|, at least the spacing at `floor`"""
    a = np.maximum(np.abs(_f64(ref)), floor)
    return np.spacing(a.astype(np.float16)).astype(np.float64)


def check_exact(label, got, want):
    got, want = (x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x) for x in (got, want))
    assert got.shape == want.shape and got.dtype == want.dtype, (label, got.shape, want.shape, got.dtype, want.dtype)
    diff = int(np.count_nonzero(np.ascontiguousarray(got).view(np.uint8) != np.ascontiguousarray(want).view(np.uint8)))
    print(f"[kernel] {label}: {diff} differing bytes (bar: bit-exact)")
    assert diff == 0, label


def check_f16(label, got, ref, floor=2.0 ** -6):
    """|got - ref| <= 1 fp16 ulp of ref; returns the per-element bar (for `teeth`)"""
    got, ref = _f64(got), _f64(ref)
    assert got.shape == ref.shape, (label, got.shape, ref.shape)
    u = ulp16(ref, floor)
    worst = float((np.abs(got - ref) / u).max()) if got.size else 0.0
    print(f"[kernel] {label}: max error {worst:.3f} fp16 ulp, max abs {float(np.abs(got - ref).max()):.3e} (bar: 1 ulp, floor |x| {floor:.1e})")
    assert np.isfinite(got).all() and worst <= 1.0, (label, worst)
    return u


def check_f32(label, got, ref, eval32, floor):
    """|got - ref| <= max(4 x |eval32 - ref|_max, floor); returns the bar"""
    got, ref, eval32 = _f64(got), _f64(ref), _f64(eval32)
    assert got.shape == ref.shape == eval32.shape, (label, got.shape, ref.shape, eval32.shape)
    e32 = float(np.abs(eval32 - ref).max())
    bar = max(4.0 * e32, floor)
    err = float(np.abs(got - ref).max())
    print(f"[kernel] {label}: max error {err:.3e}, bar {bar:.3e} (4 x fp32 evaluation {e32:.3e}, floor {floor:.1e})")
    assert np.isfinite(got).all() and err <= bar, (label, err, bar)
    return bar


def split_parts(t):
    """split [..., 3n] -> (hi, lo, third 2) as tensors / arrays of the same kind"""
    n = t.shape[-1] // 3
    return t[..., :n], t[..., n:2 * n], t[..., 2 * n:]


def _fp32_class(label, kind, v, ref, eval32, own, groups):
    dev32 = np.abs(eval32 - ref)
    if groups is None:
        e32 = float(dev32.max()) if ref.size else 0.0
        bar = 8.0 * e32 + own
    else:
        groups = np.broadcast_to(np.asarray(groups), ref.shape)
        e32g = np.zeros_like(ref)
        for k in np.unique(groups):
            e32g[groups == k] = dev32[groups == k].max()
        bar, e32 = 8.0 * e32g + own, float(dev32.max())
    err = np.abs(v - ref)
    worst = float((err / bar).max()) if ref.size else 0.0
    print(f"[kernel] {label}: max error {float(err.max()):.3e}, {worst:.3f} of the bar (8 x fp32 evaluation {e32:.3e} + {kind} "
          f"{float(own.max()):.1e} at most)")
    assert np.isfinite(v).all() and worst <= 1.0, (label, worst)
    return bar


def check_split(label, got_split, ref64, eval32, groups=None):
    """a split output [..., 3n]: format, then |hi + lo - ref64| <= 8 max|eval32 - ref64| + 2^-22 |ref64| + 2^-25 per element;
    returns the per-element bar (for `teeth`).  groups: an integer label per element (broadcast to ref64's shape), the max
    taken within each label only, where parts of the output differ in magnitude by orders: one bar for all would be set by the
    largest part and say nothing about the others."""
    if hasattr(got_split, "detach"):
        got_split = got_split.detach().cpu().numpy()
    got_split = np.asarray(got_split)
    assert got_split.dtype == np.float16, (label, got_split.dtype)
    hi, lo, hi2 = split_parts(got_split)
    ref, eval32 = _f64(ref64), _f64(eval32)
    assert hi.shape == ref.shape == eval32.shape, (label, hi.shape, ref.shape, eval32.shape)
    third = int(np.count_nonzero(np.ascontiguousarray(hi).view(np.uint16) != np.ascontiguousarray(hi2).view(np.uint16)))
    lo_over = int(np.count_nonzero(np.abs(lo.astype(np.float64)) > np.spacing(np.abs(hi)).astype(np.float64) / 2))
    print(f"[kernel] {label}: split format: {third} third-2 halves differ from third 0, {lo_over} |lo| > ulp(hi)/2 (bar: 0, 0)")
    assert third == 0 and lo_over == 0, (label, third, lo_over)
    v = hi.astype(np.float64) + lo.astype(np.float64)
    return _fp32_class(label, "split format", v, ref, eval32, 2.0 ** -22 * np.abs(ref) + 2.0 ** -25, groups)


def check_fp32_class(label, got, ref64, eval32, groups=None):
    """an fp32 output of a split kernel: |got - ref64| <= 8 max|eval32 - ref64| + 2^-24 |ref64| per element (groups: as in
    `check_split`); returns the bar"""
    got, ref, eval32 = _f64(got), _f64(ref64), _f64(eval32)
    assert got.shape == ref.shape == eval32.shape, (label, got.shape, ref.shape, eval32.shape)
    return _fp32_class(label, "fp32 rounding", got, ref, eval32, 2.0 ** -24 * np.abs(ref), groups)


def teeth(label, wrong, ref, bar, at_least=10):
    """the wrong variant differs from the right reference by at least `at_least` x the bar somewhere (and at all, for bit-exact
    bars, bar = 0); `bar` is a scalar or a per-element array (`check_f16`, `check_split`).  A NaN in the wrong variant (an
    output never written) counts as off without bound."""
    dev = np.abs(_f64(wrong) - _f64(ref))
    dev[np.isnan(dev)] = np.inf
    d = float(dev.max())
    bar = np.asarray(bar, np.float64)
    ratio = float((dev / bar).max()) if bar.any() else (float("inf") if d > 0 else 0.0)
    print(f"[kernel] {label}: wrong variant off by up to {d:.3e} ({ratio:.0f} x the bar)")
    assert d > 0 and ratio >= at_least, (label, d, ratio, at_least)
