"""Host check of the single-MUFU GELU used by the GEMM epilogue (csrc/gemm_wgmma.cu: gelu_erf): the same fp32
arithmetic, step by step in numpy, against x * Phi(x) in float64 (torch.nn.GELU() of the reference networks is the erf form:
dmidas/backbones/beit.py Mlp, ddepth_anything_v2/dinov2_layers/mlp.py)."""
import numpy as np
from scipy.special import erf

COEF = [1.1511471271514893, 0.45891568064689636, 0.05323820561170578, -0.007977476343512535, 0.0007398786256089807,
        -2.992472582263872e-05]
CLAMP = 5.75


def gelu_kernel_formula(x):
    x = x.astype(np.float32)
    u = np.minimum(np.abs(x), np.float32(CLAMP))
    q = np.full_like(u, np.float32(COEF[-1]))
    for c in COEF[-2::-1]:
        q = (q.astype(np.float64) * u + np.float32(c)).astype(np.float32)       # one fused multiply-add, rounded once
    t = (-(u.astype(np.float64)) * q - 1.0).astype(np.float32)
    e = np.exp2(t.astype(np.float64)).astype(np.float32)
    return (np.maximum(x, 0).astype(np.float64) - u.astype(np.float64) * e).astype(np.float32)


def test_gelu_formula_matches_erf_gelu():
    x = np.concatenate([np.linspace(-12, 12, 600001), np.array([0.0, -0.0, 1e-8, -1e-8, 100.0, -100.0, 6e4, -6e4])])
    ref = 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))
    got = gelu_kernel_formula(x)
    err = np.abs(got - ref)
    assert (err < 3.5e-7 + 1.2e-7 * np.abs(x)).all(), err.max()      # formula error + one fp32 rounding of the result
    # far below the fp16 rounding of the stored activation everywhere it is representable
    big = np.abs(ref) > 1e-3
    assert (err[big] / np.abs(ref[big])).max() < 2 ** -11 / 8
