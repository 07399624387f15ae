"""Float64 replay of one torch.optim.Adam step on float32 tensors (test infrastructure).

torch.optim.Adam (the foreach path, which torch picks on CUDA for `torch.optim.Adam(params, lr=0.0, eps=1e-15)`, and the
single-tensor path) keeps beta1, beta2, lr and eps as Python doubles and rounds a constant to float32 only where its
kernel takes it:

    exp_avg.lerp_(grad, w1)                      w1 = (float)(1 - beta1)
    exp_avg_sq.mul_(b2).addcmul_(grad, grad, w2) b2 = (float)beta2, w2 = (float)(1 - beta2)
    denom = exp_avg_sq.sqrt() / bc2s + e         bc2s = (float)sqrt(1 - beta2^step), e = (float)eps
    param.addcdiv_(exp_avg, denom, -ss)          ss = (float)(lr / (1 - beta1^step))

with both powers taken in double and `step` the count after this step.  `adam_step` carries out exactly that with those
float32 constants and everything else exact in float64, from a float32 state (p, g, m, v).  A float32 result that
overflows (|x| >= 2^128 - 2^103) is infinite in every implementation, so the replay stores m' and v' as +-inf there.

The error scales are what a float32 implementation may add to the exact value per rounding it performs:
    p':  0.5 ulp(p') + 2^-24 (|u| + ss (b1 |m| + w1 |g|) / d),   u = ss m' / d, d = sqrt(v') / bc2s + e, b1 = 1 - w1
         (the rounding of the update itself, and the rounding of m' carried into it);
    m':  0.5 ulp(m') + 2^-24 w1 |g - m|;
    v':  0.5 ulp(v') + 2^-24 (b2 v + w2 g^2).
torch's own float32 step stays within 2 of these units on both paths (tests/test_adam64_cpu.py).  The p' scale leaves out
the rounding of v' carried into d: relative to d it is at most 2^-25 while v' is normal, and while v' is subnormal
sqrt(v') / bc2s < 2^-63 / bc2s is far below any eps this project uses (1e-15, 1e-8), so d is eps to float32 precision.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

ULP_UNIT = 2.0 ** -24
_F32_INF_AT = 2.0 ** 128 - 2.0 ** 103        # the smallest magnitude that rounds to inf in float32


def f32(x: float) -> float:
    """The float32 rounding of a double, as a double."""
    return float(np.float32(x))


@dataclass(frozen=True)
class AdamConstants:
    w1: float          # (float)(1 - beta1)
    b2: float          # (float)beta2
    w2: float          # (float)(1 - beta2)
    ss: float          # (float)(lr / (1 - beta1^step))
    bc2s: float        # (float)sqrt(1 - beta2^step)
    eps: float         # (float)eps


def torch_constants(lr: float, betas=(0.9, 0.999), eps: float = 1e-15, step: int = 1) -> AdamConstants:
    """torch.optim.Adam's float32 constants for step `step` (>= 1, the count after the step)."""
    b1, b2 = float(betas[0]), float(betas[1])
    return AdamConstants(w1=f32(1.0 - b1), b2=f32(b2), w2=f32(1.0 - b2), ss=f32(lr / (1.0 - b1 ** step)),
                         bc2s=f32((1.0 - b2 ** step) ** 0.5), eps=f32(eps))


def _store(x: np.ndarray) -> np.ndarray:
    """x with the values that overflow float32 replaced by +-inf (exact otherwise)."""
    return np.where(np.abs(x) >= _F32_INF_AT, np.copysign(np.inf, x), x)


def half_ulp(x: np.ndarray) -> np.ndarray:
    """Half the float32 spacing at |x| (subnormal spacing near 0), as float64."""
    with np.errstate(invalid="ignore"):
        return 0.5 * np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


@dataclass
class AdamStep:
    p: np.ndarray          # exact p', m', v' (float64; +-inf where float32 overflows, NaN where torch's is NaN)
    m: np.ndarray
    v: np.ndarray
    scale_p: np.ndarray    # the per-element error units above
    scale_m: np.ndarray
    scale_v: np.ndarray


def adam_step(p, g, m, v, step: int, lr: float, betas=(0.9, 0.999), eps: float = 1e-15,
              consts: AdamConstants | None = None) -> AdamStep:
    """One torch.optim.Adam step from the float32 state (p, g, m, v), `step` = the count after it.  `consts` replaces
    torch's constants (to show what other constants would do)."""
    c = consts or torch_constants(lr, betas, eps, step)
    p, g, m, v = (np.asarray(a, dtype=np.float32).astype(np.float64) for a in (p, g, m, v))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        m1 = _store(m + c.w1 * (g - m))
        v1 = _store(c.b2 * v + c.w2 * g * g)
        d = np.sqrt(v1) / c.bc2s + c.eps
        u = c.ss * m1 / d
        p1 = p - u
        scale_p = half_ulp(p1) + ULP_UNIT * (np.abs(u) + c.ss * ((1.0 - c.w1) * np.abs(m) + c.w1 * np.abs(g)) / d)
        scale_m = half_ulp(m1) + ULP_UNIT * c.w1 * np.abs(g - m)
        scale_v = half_ulp(v1) + ULP_UNIT * (c.b2 * v + c.w2 * g * g)
    return AdamStep(p1, m1, v1, scale_p, scale_m, scale_v)


def units(actual, want: np.ndarray, scale: np.ndarray, what: str = "") -> float:
    """The largest |actual - want| / scale over the finite elements of `want`; the non-finite ones (NaN, +-inf) must be
    matched exactly by `actual`."""
    a = np.asarray(actual, dtype=np.float32).astype(np.float64).reshape(-1)
    w, s = np.asarray(want, dtype=np.float64).reshape(-1), np.asarray(scale, dtype=np.float64).reshape(-1)
    fin = np.isfinite(w)
    bad_nan = np.flatnonzero(np.isnan(a) != np.isnan(w))
    assert bad_nan.size == 0, f"{what}: NaN where the replay has none or vice versa at {bad_nan[:8]}"
    inf = np.isinf(w)
    assert np.array_equal(a[inf], w[inf]), f"{what}: an infinite replay value is not matched"
    assert np.all(np.isfinite(a[fin])), f"{what}: non-finite where the replay is finite"
    if not fin.any():
        return 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        e = np.abs(a[fin] - w[fin]) / s[fin]
    return float(e.max())
