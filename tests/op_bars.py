"""Shared by the kernel-level GPU tests (test_zoe_nk_ops_gpu.py, test_boost_ops_gpu.py, test_leres_dpt_ops_gpu.py): the bar an
output earns from its type when a kernel is compared with a float64 restatement of its operation, and the "teeth" check that a
plausible wrong variant of the operation would miss that bar by a wide margin on the same input.

- data movement, max, casts: bit-exact (`check_exact`);
- fp16 outputs computed in fp32: within one fp16 ulp of the float64 value (`check_f16`); magnitudes below `floor` get the
  spacing at `floor`, where fp32 cancellation, not the final rounding, sets the error;
- fp32 outputs: 4 x the max error of the same formula evaluated in fp32 torch on the same inputs, with a stated floor
  (`check_f32`), in the spirit of tests/precision.py: a fixed number is either toothless or flaky where the formula amplifies
  fp32 rounding (the log-binomial softmax at min_temp, the cubic resize of a large map).
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


def teeth(label, wrong, ref, bar):
    """the wrong variant differs from the right reference by at least 10 x the bar somewhere (and at all, for bit-exact bars,
    bar = 0); `bar` is a scalar or, for fp16 outputs, the per-element ulp array `check_f16` returns"""
    dev = np.abs(_f64(wrong) - _f64(ref))
    d = float(dev.max())
    bar = np.asarray(bar, np.float64)
    ratio = float((dev / bar).max()) if bar.any() else (float("inf") if d > 0 else 0.0)
    print(f"[kernel] {label}: wrong variant off by up to {d:.3e} ({ratio:.0f} x the bar)")
    assert d > 0 and ratio >= 10, (label, d, ratio)
