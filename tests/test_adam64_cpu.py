"""CPU tests of the float64 Adam replay (tests/_adam64.py) that the GPU tests check gh_adam_step, gh_adam_step_capturable
and gh_camera_adam_step against:

  * which float32 constants torch.optim.Adam uses: (float)(1 - beta2) = 1.0000000e-3, not 1.0f - 0.999f = 9.999871e-4;
  * torch.optim.Adam in float32, foreach=False and foreach=True, stays within 2 of the replay's error units for p', m'
    and v' over 1200 steps whose gradient scale jumps between 1e-3 and 1e3 (p is reset to 0 before each step, so the
    update is never hidden under the rounding of p), and at the edges: zero, subnormal-v and overflowing gradients,
    +-inf and NaN gradients, lr = 0, eps 1e-8, betas (0.8, 0.99), and states injected at step 1000 and 30000;
  * the bound separates: a float32 step with constants derived in float32 from float betas (what the kernels did
    before they took torch's constants) lands tens of units away from the replay.
"""
import numpy as np
import pytest
import torch

import _adam64 as A

STEPS = 1200
N = 4096


def _torch_step(opt, p, g):
    """One torch.optim.Adam step on the single parameter `p`: -> the float32 pre-step state (p, m, v) and the step count
    after it."""
    st = opt.state.get(p, {})
    m0 = st["exp_avg"].clone() if st else torch.zeros_like(p)
    v0 = st["exp_avg_sq"].clone() if st else torch.zeros_like(p)
    step = int(st["step"]) + 1 if st else 1
    p0 = p.detach().clone()
    p.grad = g.clone()
    opt.step()
    return p0, m0, v0, step


def _check(opt, p, g, pre, lr, betas, eps, bound=2.0, what=""):
    p0, m0, v0, step = pre
    r = A.adam_step(p0.numpy(), g.numpy(), m0.numpy(), v0.numpy(), step, lr, betas, eps)
    st = opt.state[p]
    e = (A.units(p.detach().numpy(), r.p, r.scale_p, f"{what} p"), A.units(st["exp_avg"].numpy(), r.m, r.scale_m, f"{what} m"),
         A.units(st["exp_avg_sq"].numpy(), r.v, r.scale_v, f"{what} v"))
    assert max(e) <= bound, f"{what} step {step}: p / m / v off by {e} units"
    return e


def test_torch_float_constants():
    """torch rounds 1 - beta1 and 1 - beta2 formed in double: one step from zero moments with g = 1 leaves exactly
    those constants in exp_avg and exp_avg_sq, and they differ from the constants formed in float32."""
    c = A.torch_constants(1e-3)
    assert np.float32(c.w2) == np.float32(1.0000000e-3) and np.float32(c.w2) != np.float32(1) - np.float32(0.999)
    assert abs((float(np.float32(1) - np.float32(0.999)) - c.w2) / c.w2 + 1.29e-5) < 0.01e-5
    assert np.float32(c.w1) != np.float32(1) - np.float32(0.9)
    for foreach in (False, True):
        p = torch.zeros(4, requires_grad=True)
        opt = torch.optim.Adam([p], lr=1e-3, eps=1e-15, foreach=foreach)
        p.grad = torch.ones(4)
        opt.step()
        assert torch.all(opt.state[p]["exp_avg"] == np.float32(c.w1))
        assert torch.all(opt.state[p]["exp_avg_sq"] == np.float32(c.w2))


@pytest.mark.parametrize("foreach", [False, True], ids=["single_tensor", "foreach"])
def test_replay_matches_torch_sweep(foreach):
    rng = np.random.default_rng(7)
    lr, betas, eps = 1e-3, (0.9, 0.999), 1e-15
    p = torch.zeros(N, requires_grad=True)
    opt = torch.optim.Adam([p], lr=lr, eps=eps, foreach=foreach)
    worst = np.zeros(3)
    for _ in range(STEPS):
        g = torch.from_numpy((rng.standard_normal(N) * 10.0 ** rng.uniform(-3, 3)).astype(np.float32))
        with torch.no_grad():
            p.zero_()
        pre = _torch_step(opt, p, g)
        worst = np.maximum(worst, _check(opt, p, g, pre, lr, betas, eps, what=f"foreach={foreach}"))
    assert int(opt.state[p]["step"]) == STEPS
    assert worst[0] > 0.05, "the sweep never resolved the update's rounding: the check would not see an error"


def _edge_gradients(rng, n):
    """N(0,1) gradients with runs of edge values: 0, subnormal v (w2 g^2 below 2^-126), values whose g^2 overflows
    float32 while w2 g^2 does not (1e20) and whose w2 g^2 overflows too (3e21), +-inf and NaN."""
    g = rng.standard_normal(n).astype(np.float32)
    edges = [0.0, -0.0, 1e-21, -3e-22, 1e-24, 1e-19, 1e20, -1e20, 3e21, np.inf, -np.inf, np.nan]
    for k, x in enumerate(edges):
        g[k * 16:(k + 1) * 16] = x
    return g


@pytest.mark.parametrize("foreach", [False, True], ids=["single_tensor", "foreach"])
@pytest.mark.parametrize("lr,betas,eps,late", [
    (1e-3, (0.9, 0.999), 1e-15, 0),
    (0.0, (0.9, 0.999), 1e-15, 0),
    (5e-2, (0.9, 0.999), 1e-8, 0),
    (1e-3, (0.8, 0.99), 1e-15, 0),
    (1e-3, (0.9, 0.999), 1e-15, 1000),
    (2.5e-3, (0.9, 0.999), 1e-15, 30000),
], ids=["default", "lr0", "eps1e-8", "betas_0.8_0.99", "late1000", "late30000"])
def test_replay_matches_torch_edges(foreach, lr, betas, eps, late):
    rng = np.random.default_rng(11)
    n = 1024
    p = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).requires_grad_(True)
    opt = torch.optim.Adam([p], lr=lr, betas=betas, eps=eps, foreach=foreach)
    if late:
        # a state as a long run leaves it: m ~ g, v ~ g^2 over a spread of scales, one zero-moment run
        scale = (10.0 ** rng.uniform(-4, 2, n)).astype(np.float32)
        m = (rng.standard_normal(n) * scale * 0.3).astype(np.float32)
        v = (scale * scale * rng.uniform(0.5, 2.0, n)).astype(np.float32)
        m[-32:] = 0
        v[-32:] = 0
        opt.state[p] = {"step": torch.tensor(float(late)), "exp_avg": torch.from_numpy(m), "exp_avg_sq": torch.from_numpy(v)}
    for k in range(4):
        g = torch.from_numpy(_edge_gradients(rng, n))
        if k == 0:
            g[-32:] = 0.0          # zero moments and a zero gradient: the update is exactly 0
        pre = _torch_step(opt, p, g)
        _check(opt, p, g, pre, lr, betas, eps, what=f"foreach={foreach} lr={lr} betas={betas} eps={eps} late={late}")
        if k == 0:
            assert torch.equal(p.detach()[-32:], pre[0][-32:]), "m = 0, g = 0 must leave p bit-identical"
        if lr == 0.0:
            fin = torch.isfinite(p.detach())
            assert torch.equal(p.detach()[fin], pre[0][fin]), "lr = 0 must leave every finite p bit-identical"


def _float32_step(p, g, m, v, w1, b2, w2, ss, bc2s, eps):
    """A float32 step with exact sqrt and division (numpy), the constants given as float32."""
    f = np.float32
    m1 = (f(w1) * (g - m) + m).astype(f)
    v1 = (v * f(b2) + (f(w2) * g) * g).astype(f)
    p1 = (p - (f(ss) * m1) / (np.sqrt(v1) / f(bc2s) + f(eps))).astype(f)
    return p1, m1, v1


def test_float_derived_constants_are_outside_the_bound():
    """What the bound catches: float32 steps with torch's constants stay within 2 units of the replay, steps whose
    constants were formed in float32 from float betas (1.0f - beta2 and powf(beta, step)) do not."""
    rng = np.random.default_rng(3)
    f = np.float32
    n, lr = 4096, 1e-3
    b1f, b2f = f(0.9), f(0.999)
    state = {"torch": [np.zeros(n, f), np.zeros(n, f)], "float": [np.zeros(n, f), np.zeros(n, f)]}
    worst = {"torch": 0.0, "float": 0.0}
    for s in range(1, 301):
        g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3)).astype(f)
        p = np.zeros(n, f)
        c = A.torch_constants(lr, step=s)
        consts = {"torch": (c.w1, c.b2, c.w2, c.ss, c.bc2s, c.eps),
                  "float": (f(1) - b1f, b2f, f(1) - b2f, f(lr) / (f(1) - np.power(b1f, f(s))),
                            np.sqrt(f(1) - np.power(b2f, f(s))), f(1e-15))}
        for k in ("torch", "float"):
            m, v = state[k]
            r = A.adam_step(p, g, m, v, s, lr)
            p1, m1, v1 = _float32_step(p, g, m, v, *consts[k])
            worst[k] = max(worst[k], A.units(p1, r.p, r.scale_p), A.units(v1, r.v, r.scale_v))
            state[k] = [m1, v1]
    assert worst["torch"] <= 2.0, worst
    assert worst["float"] > 10.0, worst
