"""Float64 replay of the projection kernels (gaussianhaircut_b200/csrc/gh_project_math.h, gh_project.cu's camera
reduction, gh_strands.cu) that carries, with every value, a bound on the error of the kernels' float32 evaluation.

`E` is a pair (value, bound) of float64 arrays.  Each operation rounds once in float32 (u = 2^-24) and propagates the
bounds of its operands:

    a +- b   e_a + e_b + u|v|              a * b    |a| e_b + |b| e_a + e_a e_b + u|v|
    a / b    (e_a + |v| e_b) / (|b| - e_b) + u|v|    sqrt(x)  e / (sqrt(x) + sqrt(x - e)) + u|v|
    expf     |v| expm1(e) + 4u|v|  (CUDA's expf is within 2 ulp)    fminf / fmaxf / select: exact

plus one float32 denormal step, and with u|v| taken on |v| + the propagated bound.  An operation on exact operands
whose result is a float32 is exact (correct rounding of a representable value).  A fused multiply-add rounds once
where this model rounds twice, so nvcc's contraction stays inside the bound; division and sqrtf are correctly
rounded because the library is built without --use_fast_math or -prec-div=false
(tests/test_project64_cpu.py checks the flags).

The replay restates the header line for line, in its operation order.  Each branch is decided in float64 with the
bounds of its operands; a decision whose interval straddles its threshold is *ambiguous* and recorded per row
(`Replay.amb`).  A division or square root whose operand's bound exceeds 2^-10 of its value marks its row
*unresolved* (`Replay.unres`): the bound there is still a bound, but a loose one.  In `f32=False` mode the constants
are the reference's float64 ones and the replay is the float64 evaluation of the same formulas (checked against
float64 autograd of oracle/synth.py `project_reference`)."""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -149                 # one float32 denormal step: the absolute floor of any rounding
REL_UNRESOLVED = 2.0 ** -10        # beyond this relative bound on an operand, first-order analysis no longer applies
EXP_ULP = 2                        # CUDA expf: maximum error 2 ulp

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def _is_f32(v):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.isfinite(v) & (v.astype(np.float32).astype(np.float64) == v)


def _round(v, p, ulps=1):
    """bound of a float32 result whose exact-operand value is v, with the operands' bounds propagated to p"""
    b = p + ulps * U * (np.abs(v) + p) + TINY
    exact = p == 0
    if not exact.any():
        return b
    return np.where(exact & _is_f32(v), 0.0, b)


class E:
    """(value, bound): a float64 value and a bound on |float32 evaluation - value|."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.asarray(e, dtype=np.float64)

    def __add__(self, o):
        o = _e(o)
        v = self.v + o.v
        return E(v, _round(v, self.e + o.e))

    __radd__ = __add__

    def __sub__(self, o):
        o = _e(o)
        v = self.v - o.v
        return E(v, _round(v, self.e + o.e))

    def __rsub__(self, o):
        return _e(o) - self

    def __mul__(self, o):
        o = _e(o)
        v = self.v * o.v
        return E(v, _round(v, np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e))

    __rmul__ = __mul__

    def __neg__(self):
        return E(-self.v, self.e)


def _e(x):
    return x if isinstance(x, E) else E(x)


def _pick(a, b, first):
    """fminf / fmaxf: the selected operand's bound where the choice is decided, the larger bound where it is not"""
    a, b = _e(a), _e(b)
    decided = np.abs(a.v - b.v) > a.e + b.e
    e = np.where(decided, np.where(first, a.e, b.e), np.maximum(a.e, b.e))
    return E(np.where(first, a.v, b.v), e)


def fmin(a, b):
    return _pick(a, b, _e(a).v <= _e(b).v)


def fmax(a, b):
    return _pick(a, b, _e(a).v >= _e(b).v)


def select(cond, a, b):
    a, b = _e(a), _e(b)
    return E(np.where(cond, a.v, b.v), np.where(cond, a.e, b.e))


def zero(n):
    return E(np.zeros(n))


class Replay:
    """Ambiguous decisions and unresolved rows of one replay over n rows."""

    def __init__(self, n, f32=True):
        self.n, self.f32 = n, f32
        self.amb = {}                                   # key -> bool (n,)
        self.unres = np.zeros(n, dtype=bool)

    def k(self, x):
        """a constant of the header: its float32 value (or the reference's float64 one)"""
        return E(float(np.float32(x)) if self.f32 else float(x))

    def kk(self, a, b):
        """a constant product the compiler folds, `a.f * b.f`"""
        return E(float(np.float32(np.float32(a) * np.float32(b))) if self.f32 else float(a) * float(b))

    def _flag(self, key, m):
        m = np.broadcast_to(m, (self.n,))
        self.amb[key] = self.amb.get(key, np.zeros(self.n, dtype=bool)) | m

    def gt(self, a, b, key, tie=None):
        """a > b, decided in float64 with the operands' bounds; `tie`: rows where the two are equal by construction"""
        a, b = _e(a), _e(b)
        d, e = a.v - b.v, a.e + b.e
        amb = (np.abs(d) <= e) & (e > 0)
        if tie is not None:
            amb = amb & ~tie
            d = np.where(tie, 0.0, d)
        self._flag(key, amb)
        return d > 0

    def ge(self, a, b, key):
        a, b = _e(a), _e(b)
        d, e = a.v - b.v, a.e + b.e
        self._flag(key, (np.abs(d) <= e) & (e > 0))
        return d >= 0

    def div(self, a, b):
        a, b = _e(a), _e(b)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = a.v / b.v
            den = np.abs(b.v) - b.e
            p = np.where(den > 0, (a.e + np.abs(v) * b.e) / np.where(den > 0, den, 1.0), np.inf)
        p = np.where((a.e == 0) & (b.e == 0), 0.0, p)
        self.unres |= np.broadcast_to(b.e > REL_UNRESOLVED * np.abs(b.v), (self.n,))
        return E(v, _round(v, p))

    def sqrt(self, x, track=True):
        """`track=False`: a value that only feeds an interval decision (the splat radius), not an output"""
        x = _e(x)
        v = np.sqrt(np.maximum(x.v, 0.0))
        with np.errstate(divide="ignore", invalid="ignore"):
            p = x.e / (v + np.sqrt(np.maximum(x.v - x.e, 0.0)))
        p = np.where(x.e == 0, 0.0, p)
        if track:
            self.unres |= np.broadcast_to(x.e > REL_UNRESOLVED * np.abs(x.v), (self.n,))
        return E(v, _round(v, p))

    def exp(self, x):
        x = _e(x)
        with np.errstate(over="ignore"):
            v = np.exp(x.v)
            p = np.abs(v) * np.expm1(x.e)
        return E(v, _round(v, p, EXP_ULP * 2))

    def sigmoid(self, x):
        return self.div(self.k(1.0), self.k(1.0) + self.exp(-x))

    def rows(self, key):
        return self.amb.get(key, np.zeros(self.n, dtype=bool))


# ------------------------------------------------------------------------------------------------ inputs
class Inputs:
    """One projection call as float64 arrays of the float32 values the kernels read."""

    def __init__(self, P, W, H, xyz, scaling, rotation, dirs, f_dc, f_rest, opacity, label, conf, V, Pm, campos,
                 tanx, tany, mod, sh_degree, cfg):
        d = lambda a, *shape: None if a is None else np.asarray(a, dtype=np.float32).astype(np.float64).reshape(*shape)  # noqa: E731
        f = lambda x: float(np.float32(x))  # noqa: E731
        self.P, self.W, self.H = int(P), int(W), int(H)
        self.strand = bool(cfg.get("strands", 0))
        self.xyz = d(xyz, P, 3)
        self.scaling = d(scaling, -1) if self.strand else d(scaling, P, 3)
        self.rotation = None if self.strand else d(rotation, P, 4)
        self.dirs = d(dirs, P, 3)
        self.f_dc = d(f_dc, P, 3)
        self.f_rest = d(f_rest, P, 45) if f_rest is not None else np.zeros((P, 45))
        self.opacity, self.label, self.conf = d(opacity, P), d(label, P), d(conf, P)
        self.V, self.Pm, self.campos = d(V, 16), d(Pm, 16), d(campos, 3)
        self.tanx, self.tany, self.mod = f(tanx), f(tany), f(mod)
        self.sh_degree = int(sh_degree)
        self.scale_act, self.opacity_act, self.label_act = int(cfg["scale_act"]), int(cfg["opacity_act"]), int(cfg["label_act"])
        self.conf_act, self.dir_mode = int(cfg["conf_act"]), int(cfg["dir_mode"])
        self.det_eps = f(cfg["det_eps"])


def _sel3(a0, a1, a2, j):
    return select(j == 0, a0, select(j == 1, a1, a2))


def sh_basis(rp, deg, x, y, z):
    k, kk = rp.k, rp.kk
    n = rp.n
    B = [zero(n) for _ in range(16)]
    B[0] = k(SH_C0)
    if deg > 0:
        B[1] = k(-SH_C1) * y; B[2] = k(SH_C1) * z; B[3] = k(-SH_C1) * x
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            B[4] = k(SH_C2[0]) * xy; B[5] = k(SH_C2[1]) * yz; B[6] = k(SH_C2[2]) * (k(2) * zz - xx - yy)
            B[7] = k(SH_C2[3]) * xz; B[8] = k(SH_C2[4]) * (xx - yy)
            if deg > 2:
                B[9] = k(SH_C3[0]) * y * (k(3) * xx - yy); B[10] = k(SH_C3[1]) * xy * z
                B[11] = k(SH_C3[2]) * y * (k(4) * zz - xx - yy); B[12] = k(SH_C3[3]) * z * (k(2) * zz - k(3) * xx - k(3) * yy)
                B[13] = k(SH_C3[4]) * x * (k(4) * zz - xx - yy); B[14] = k(SH_C3[5]) * z * (xx - yy)
                B[15] = k(SH_C3[6]) * x * (xx - k(3) * yy)
    del kk
    return B


def sh_basis_grad(rp, deg, x, y, z):
    k, kk, n = rp.k, rp.kk, rp.n
    Bx = [zero(n) for _ in range(16)]; By = [zero(n) for _ in range(16)]; Bz = [zero(n) for _ in range(16)]
    if deg > 0:
        By[1] = k(-SH_C1); Bz[2] = k(SH_C1); Bx[3] = k(-SH_C1)
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            C2, C3 = SH_C2, SH_C3
            Bx[4] = k(C2[0]) * y; By[4] = k(C2[0]) * x
            By[5] = k(C2[1]) * z; Bz[5] = k(C2[1]) * y
            Bx[6] = kk(-2, C2[2]) * x; By[6] = kk(-2, C2[2]) * y; Bz[6] = kk(4, C2[2]) * z
            Bx[7] = k(C2[3]) * z; Bz[7] = k(C2[3]) * x
            Bx[8] = kk(2, C2[4]) * x; By[8] = kk(-2, C2[4]) * y
            if deg > 2:
                Bx[9] = kk(6, C3[0]) * xy; By[9] = k(C3[0]) * (k(3) * xx - k(3) * yy)
                Bx[10] = k(C3[1]) * yz; By[10] = k(C3[1]) * xz; Bz[10] = k(C3[1]) * xy
                Bx[11] = kk(-2, C3[2]) * xy; By[11] = k(C3[2]) * (k(4) * zz - xx - k(3) * yy); Bz[11] = kk(8, C3[2]) * yz
                Bx[12] = kk(-6, C3[3]) * xz; By[12] = kk(-6, C3[3]) * yz; Bz[12] = k(C3[3]) * (k(6) * zz - k(3) * xx - k(3) * yy)
                Bx[13] = k(C3[4]) * (k(4) * zz - k(3) * xx - yy); By[13] = kk(-2, C3[4]) * xy; Bz[13] = kk(8, C3[4]) * xz
                Bx[14] = kk(2, C3[5]) * xz; By[14] = kk(-2, C3[5]) * yz; Bz[14] = k(C3[5]) * (xx - yy)
                Bx[15] = k(C3[6]) * (k(3) * xx - k(3) * yy); By[15] = kk(-6, C3[6]) * xy
    return Bx, By, Bz


def argmax3(rp, s, raw_tie):
    """gh_argmax3: first index on ties; `raw_tie[(a, b)]` marks rows whose scales a, b are equal by construction"""
    j = np.zeros(rp.n, dtype=int)
    g1 = rp.gt(s[1], s[0], "argmax", tie=raw_tie[(0, 1)])
    j = np.where(g1, 1, j)
    m = select(g1, s[1], s[0])
    tie2 = np.where(g1, raw_tie[(1, 2)], raw_tie[(0, 2)])
    g2 = rp.gt(s[2], m, "argmax", tie=tie2)
    return np.where(g2, 2, j)


# ------------------------------------------------------------------------------------------------ gh_proj_geometry
class Geo:
    pass


def geometry(rp, A: Inputs):
    k = rp.k
    n = A.P
    g = Geo()
    g.x = [E(A.xyz[:, c]) for c in range(3)]
    if A.strand:
        dx, dy, dz = (E(A.dirs[:, c]) for c in range(3))
        dn = rp.sqrt(dx * dx + dy * dy + dz * dz)
        th = E(A.scaling[0]) * k(A.mod)
        g.s = [(dn * k(0.5)) * k(A.mod), th, th]
        ib = rp.div(k(1.0), fmax(dn, k(1e-12)))
        q = [k(1.0) + dx * ib, zero(n), -(dz * ib), dy * ib]
        g.raw_tie = None
    else:
        raw = A.scaling
        if A.scale_act == 1:
            g.s = [rp.exp(E(raw[:, c])) * k(A.mod) for c in range(3)]
        else:
            # an exact float32 product, used only as a multiplicand and in comparisons: never contracted
            s32 = [np.float32(raw[:, c]) * np.float32(A.mod) for c in range(3)] if rp.f32 else [raw[:, c] * A.mod for c in range(3)]
            g.s = [E(np.asarray(v, dtype=np.float64)) if rp.f32 else E(v) for v in s32]
        g.raw_tie = {(a, b): raw[:, a] == raw[:, b] for a, b in ((0, 1), (0, 2), (1, 2))}
        q = [E(A.rotation[:, c]) for c in range(4)]
    g.qlen = rp.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    il = rp.div(k(1.0), g.qlen)
    r, x, y, z = q[0] * il, q[1] * il, q[2] * il, q[3] * il
    g.qn = [r, x, y, z]
    R = [[None] * 3 for _ in range(3)]
    R[0][0] = k(1) - k(2) * (y * y + z * z); R[1][0] = k(2) * (x * y - r * z); R[2][0] = k(2) * (x * z + r * y)
    R[0][1] = k(2) * (x * y + r * z); R[1][1] = k(1) - k(2) * (x * x + z * z); R[2][1] = k(2) * (y * z - r * x)
    R[0][2] = k(2) * (x * z - r * y); R[1][2] = k(2) * (y * z + r * x); R[2][2] = k(1) - k(2) * (x * x + y * y)
    g.R = R
    V = [E(v) for v in A.V]
    g.V = V
    g.t = [g.x[0] * V[j] + g.x[1] * V[4 + j] + g.x[2] * V[8 + j] + V[12 + j] for j in range(3)]
    tz = g.t[2]
    tanx, tany = k(A.tanx), k(A.tany)
    limx, limy = k(1.3) * tanx, k(1.3) * tany
    txtz, tytz = rp.div(g.t[0], tz), rp.div(g.t[1], tz)
    g.clx = rp.gt(-limx, txtz, "clamp") | rp.gt(txtz, limx, "clamp")
    g.cly = rp.gt(-limy, tytz, "clamp") | rp.gt(tytz, limy, "clamp")
    g.sgx = np.where(txtz.v < 0, -1.0, 1.0)
    g.sgy = np.where(tytz.v < 0, -1.0, 1.0)
    g.txc = fmin(limx, fmax(-limx, txtz)) * tz
    g.tyc = fmin(limy, fmax(-limy, tytz)) * tz
    g.fx = rp.div(k(A.W), k(2.0) * tanx)
    g.fy = rp.div(k(A.H), k(2.0) * tany)
    itz = rp.div(k(1.0), tz)
    itz2 = itz * itz
    g.j00 = g.fx * itz; g.j20 = -(g.fx * g.txc) * itz2
    g.j11 = g.fy * itz; g.j21 = -(g.fy * g.tyc) * itz2
    g.u0 = [V[4 * c + 0] * g.j00 + V[4 * c + 2] * g.j20 for c in range(3)]
    g.u1 = [V[4 * c + 1] * g.j11 + V[4 * c + 2] * g.j21 for c in range(3)]
    a = b = c_ = zero(n)
    g.w0, g.w1 = [], []
    for c in range(3):
        w0 = R[c][0] * g.u0[0] + R[c][1] * g.u0[1] + R[c][2] * g.u0[2]
        w1 = R[c][0] * g.u1[0] + R[c][1] * g.u1[1] + R[c][2] * g.u1[2]
        g.w0.append(w0); g.w1.append(w1)
        s2 = g.s[c] * g.s[c]
        a = a + s2 * w0 * w0; b = b + s2 * w0 * w1; c_ = c_ + s2 * w1 * w1
    g.a, g.b, g.c = a + k(0.3), b, c_ + k(0.3)
    return g


def visible(rp, A, g, m2x, m2y):
    """gh_proj_visible; ambiguous rows are flagged under "vis" (their value is then the one of the float64 values)"""
    k = rp.k
    det = g.a * g.c - g.b * g.b
    near = rp.gt(g.t[2], k(0.2), "vis")
    nz = ~((np.abs(det.v) <= det.e) & (det.e > 0)) & (det.v != 0)
    rp._flag("vis", (np.abs(det.v) <= det.e) & (det.e > 0))
    mid = k(0.5) * (g.a + g.c)
    sq = rp.sqrt(fmax(mid * mid - det, k(0.1)), track=False)
    r3 = k(3.0) * rp.sqrt(fmax(mid + sq, mid - sq), track=False)
    rad_lo, rad_hi = np.ceil(r3.v - r3.e), np.ceil(r3.v + r3.e)
    px = ((m2x + k(1.0)) * k(A.W) - k(1.0)) * k(0.5)
    py = ((m2y + k(1.0)) * k(A.H) - k(1.0)) * k(0.5)
    gx, gy = (A.W + 15) // 16, (A.H + 15) // 16

    def edge(p, sign, gmax):
        # (int)((p - rad) / 16) or (int)((p + rad + 15) / 16) over the intervals of p and rad, clamped to [0, gmax]:
        # (lowest, highest, float64 value)
        q = lambda rad: rp.div(p - E(rad), k(16.0)) if sign < 0 else rp.div(p + E(rad) + k(15.0), k(16.0))  # noqa: E731
        qa, qb, qm = q(rad_lo), q(rad_hi), q(np.ceil(r3.v))
        lo = np.minimum(np.trunc(qa.v - qa.e), np.trunc(qb.v - qb.e))
        hi = np.maximum(np.trunc(qa.v + qa.e), np.trunc(qb.v + qb.e))
        return np.clip(lo, 0, gmax), np.clip(hi, 0, gmax), np.clip(np.trunc(qm.v), 0, gmax)

    x0, y0 = edge(px, -1, gx), edge(py, -1, gy)
    x1, y1 = edge(px, 1, gx), edge(py, 1, gy)
    surely = (x1[0] > x0[1]) & (y1[0] > y0[1])
    never = (x1[1] <= x0[0]) | (y1[1] <= y0[0])
    rect = (x1[2] - x0[2]) * (y1[2] - y0[2]) != 0
    live = near & nz
    rp._flag("vis", live & ~surely & ~never)
    return live & rect


# ------------------------------------------------------------------------------------------------ forward
CHANNELS = 10


def forward(rp, A: Inputs, g=None):
    """gh_project_forward_one for every row -> dict of E: means2D [3], conic [3], opacity, color [10], cov3D [6],
    and `visible` (bool, the float64 decision)."""
    k = rp.k
    n = A.P
    if g is None:
        g = geometry(rp, A)
    Pm = [E(v) for v in A.Pm]
    h = [g.x[0] * Pm[j] + g.x[1] * Pm[4 + j] + g.x[2] * Pm[8 + j] + Pm[12 + j] for j in range(4)]
    p_w = rp.div(k(1.0), h[3] + k(0.0000001))
    o = {"means2D": [h[0] * p_w, h[1] * p_w, h[2] * p_w]}
    vis = visible(rp, A, g, o["means2D"][0], o["means2D"][1])
    o["visible"] = vis
    det = g.a * g.c - g.b * g.b
    inv = rp.div(k(1.0), det + k(A.det_eps))
    o["conic"] = [g.c * inv, -g.b * inv, g.a * inv]        # zero where culled (the caller compares those exactly)
    cov = [zero(n) for _ in range(6)]
    for c in range(3):
        s2 = g.s[c] * g.s[c]
        Rr = g.R[c]
        cov[0] = cov[0] + s2 * Rr[0] * Rr[0]; cov[1] = cov[1] + s2 * Rr[0] * Rr[1]; cov[2] = cov[2] + s2 * Rr[0] * Rr[2]
        cov[3] = cov[3] + s2 * Rr[1] * Rr[1]; cov[4] = cov[4] + s2 * Rr[1] * Rr[2]; cov[5] = cov[5] + s2 * Rr[2] * Rr[2]
    o["cov3D"] = cov
    op = k(1.0) if A.opacity_act == 2 else E(A.opacity)
    o["opacity"] = rp.sigmoid(op) if A.opacity_act == 1 else op * E(np.ones(n))
    d3 = _d3(rp, A, g, forward=True)
    dir2x = d3[0] * g.u0[0] + d3[1] * g.u0[1] + d3[2] * g.u0[2]
    dir2y = d3[0] * g.u1[0] + d3[1] * g.u1[1] + d3[2] * g.u1[2]
    v, ivl = _view_dir(rp, A, g)
    B = sh_basis(rp, A.sh_degree, *v)
    ncoef = (A.sh_degree + 1) ** 2
    col = []
    for ch in range(3):
        acc = _sh_acc(A, B, ncoef, ch)
        col.append(fmax(acc + k(0.5), k(0.0)))
    lab = _act(rp, A.label_act, A.label, n, rp.sigmoid)
    cf = zero(n) if A.conf_act == 3 else (rp.exp(E(A.conf)) if A.conf_act == 1 else E(A.conf))
    o["color"] = col + [lab, E(np.ones(n)), dir2x, dir2y, zero(n), cf, g.t[2]]
    return o, g


def _act(rp, mode, x, n, f):
    if mode == 2:
        return E(np.ones(n))
    if mode == 3:
        return zero(n)
    return f(E(x)) if mode == 1 else E(x)


def _sh_acc(A, B, ncoef, ch):
    acc = B[0] * E(A.f_dc[:, ch])
    for kk in range(1, ncoef):
        acc = acc + B[kk] * E(A.f_rest[:, 3 * (kk - 1) + ch])
    return acc


def _view_dir(rp, A, g):
    v = [g.x[c] - E(A.campos[c]) for c in range(3)]
    vl = rp.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    ivl = rp.div(rp.k(1.0), vl)
    return [v[0] * ivl, v[1] * ivl, v[2] * ivl], ivl


def _d3(rp, A, g, forward):
    k, n = rp.k, A.P
    g.jm, g.sjm, g.dl = None, None, None
    if A.dir_mode == 0:
        jm = argmax3(rp, g.s, g.raw_tie)
        sj = _sel3(*g.s, jm)
        g.jm, g.sjm = jm, sj
        return [_sel3(g.R[0][c], g.R[1][c], g.R[2][c], jm) * sj for c in range(3)]
    if A.dir_mode == 1:
        d = [E(A.dirs[:, c]) for c in range(3)]
        if forward:
            il = rp.div(k(1.0), fmax(rp.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), k(1e-12)))
            return [d[0] * il, d[1] * il, d[2] * il]
        dl = fmax(rp.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), k(1e-12))
        g.dl = dl
        return [rp.div(d[c], dl) for c in range(3)]
    return [zero(n) for _ in range(3)]


# ------------------------------------------------------------------------------------------------ backward
NCAM = 29


def backward(rp, A: Inputs, gi, live, g=None):
    """gh_project_backward_one for the rows with `live` (others are zero).  gi: dict of float64 arrays (float32
    values) m2x, m2y (n,), con (n,3) = [g00, 2 g01, g11], color (n,10), opacity (n,).  -> (dict of lists of E: xyz [3],
    scaling [3], rotation [4], dirs [3], f_dc [3], rest [45], opacity, label, conf; cam: list of 29 E per row)."""
    k = rp.k
    n = A.P
    if g is None:
        g = geometry(rp, A)
    V = g.V
    Pm = [E(v) for v in A.Pm]
    G = lambda a: E(np.asarray(a, dtype=np.float32).astype(np.float64))  # noqa: E731
    gcol = [G(gi["color"][:, c]) for c in range(CHANNELS)]
    gcon = [G(gi["con"][:, c]) for c in range(3)]
    cam = [zero(n) for _ in range(NCAM)]
    dx = [zero(n) for _ in range(3)]
    ds = [zero(n) for _ in range(3)]
    gt = [zero(n), zero(n), gcol[9]]
    go = {}
    go["opacity"] = zero(n)
    if A.opacity_act == 1:
        s = rp.sigmoid(E(A.opacity))
        go["opacity"] = G(gi["opacity"]) * s * (k(1.0) - s)
    elif A.opacity_act == 0:
        go["opacity"] = G(gi["opacity"])
    go["label"] = zero(n)
    if A.label_act == 1:
        s = rp.sigmoid(E(A.label))
        go["label"] = gcol[3] * s * (k(1.0) - s)
    elif A.label_act == 0:
        go["label"] = gcol[3]
    go["conf"] = zero(n)
    if A.conf_act == 1:
        go["conf"] = gcol[8] * rp.exp(E(A.conf))
    elif A.conf_act == 0:
        go["conf"] = gcol[8]
    go["dirs"] = [zero(n) for _ in range(3)]

    # ---- SH colour
    v, ivl = _view_dir(rp, A, g)
    B = sh_basis(rp, A.sh_degree, *v)
    ncoef = (A.sh_degree + 1) ** 2
    grgb, go["f_dc"] = [], []
    for ch in range(3):
        acc = _sh_acc(A, B, ncoef, ch)
        keep = rp.ge(acc + k(0.5), k(0.0), f"color{ch}")
        grgb.append(select(keep, gcol[ch], k(0.0)))
        go["f_dc"].append(B[0] * grgb[ch])
    gv = [zero(n) for _ in range(3)]
    if A.sh_degree > 0:
        Bx, By, Bz = sh_basis_grad(rp, A.sh_degree, *v)
        for kk in range(1, ncoef):
            r = [E(A.f_rest[:, 3 * (kk - 1) + ch]) for ch in range(3)]
            c = r[0] * grgb[0] + r[1] * grgb[1] + r[2] * grgb[2]
            gv[0] = gv[0] + Bx[kk] * c; gv[1] = gv[1] + By[kk] * c; gv[2] = gv[2] + Bz[kk] * c
    go["rest"] = [(B[kk] * grgb[ch]) if kk < ncoef else zero(n) for kk in range(1, 16) for ch in range(3)]
    dot = v[0] * gv[0] + v[1] * gv[1] + v[2] * gv[2]
    gd = [(gv[c] - v[c] * dot) * ivl for c in range(3)]
    for c in range(3):
        dx[c] = dx[c] + gd[c]
        cam[24 + c] = cam[24 + c] - gd[c]

    # ---- dir2D
    gu0 = [zero(n) for _ in range(3)]
    gu1 = [zero(n) for _ in range(3)]
    gR = [[zero(n) for _ in range(3)] for _ in range(3)]
    d3 = _d3(rp, A, g, forward=False)
    g5, g6 = gcol[5], gcol[6]
    gd3 = []
    for c in range(3):
        gd3.append(g5 * g.u0[c] + g6 * g.u1[c])
        gu0[c] = gu0[c] + g5 * d3[c]; gu1[c] = gu1[c] + g6 * d3[c]
    if A.dir_mode == 0:
        dsj = zero(n)
        for c in range(3):
            dsj = dsj + _sel3(g.R[0][c], g.R[1][c], g.R[2][c], g.jm) * gd3[c]
            for r in range(3):
                gR[r][c] = gR[r][c] + select(g.jm == r, g.sjm * gd3[c], k(0.0))
        for r in range(3):
            ds[r] = ds[r] + select(g.jm == r, dsj, k(0.0))
    elif A.dir_mode == 1:
        dot = d3[0] * gd3[0] + d3[1] * gd3[1] + d3[2] * gd3[2]
        go["dirs"] = [rp.div(gd3[c] - d3[c] * dot, g.dl) for c in range(3)]

    # ---- conic -> cov2D
    det = g.a * g.c - g.b * g.b
    inv = rp.div(k(1.0), det + k(A.det_eps))
    ga = gcon[2] * inv; gc = gcon[0] * inv; gb = -gcon[1] * inv
    ginv = gcon[0] * g.c - gcon[1] * g.b + gcon[2] * g.a
    gdet = -inv * inv * ginv
    ga = ga + gdet * g.c; gc = gc + gdet * g.a; gb = gb + k(-2.0) * g.b * gdet
    # ---- cov2D -> scales, rotation rows, u0 / u1
    for c in range(3):
        s2 = g.s[c] * g.s[c]
        w0, w1 = g.w0[c], g.w1[c]
        gw0 = s2 * (k(2.0) * ga * w0 + gb * w1)
        gw1 = s2 * (k(2.0) * gc * w1 + gb * w0)
        ds[c] = ds[c] + k(2.0) * g.s[c] * (ga * w0 * w0 + gb * w0 * w1 + gc * w1 * w1)
        for m in range(3):
            gR[c][m] = gR[c][m] + (gw0 * g.u0[m] + gw1 * g.u1[m])
            gu0[m] = gu0[m] + gw0 * g.R[c][m]; gu1[m] = gu1[m] + gw1 * g.R[c][m]
    # ---- u0 / u1 -> J entries and the view matrix
    gj00 = gj20 = gj11 = gj21 = zero(n)
    for c in range(3):
        gj00 = gj00 + gu0[c] * V[4 * c + 0]; gj20 = gj20 + gu0[c] * V[4 * c + 2]
        gj11 = gj11 + gu1[c] * V[4 * c + 1]; gj21 = gj21 + gu1[c] * V[4 * c + 2]
        cam[3 * c + 0] = cam[3 * c + 0] + gu0[c] * g.j00
        cam[3 * c + 1] = cam[3 * c + 1] + gu1[c] * g.j11
        cam[3 * c + 2] = cam[3 * c + 2] + (gu0[c] * g.j20 + gu1[c] * g.j21)
    tz = g.t[2]
    itz = rp.div(k(1.0), tz)
    itz2 = itz * itz
    itz3 = itz2 * itz
    gfx = gj00 * itz - g.txc * itz2 * gj20
    gfy = gj11 * itz - g.tyc * itz2 * gj21
    gt[2] = gt[2] + (-g.fx * itz2 * gj00 + k(2.0) * g.fx * g.txc * itz3 * gj20 - g.fy * itz2 * gj11
                     + k(2.0) * g.fy * g.tyc * itz3 * gj21)
    gtxc = -g.fx * itz2 * gj20
    gtyc = -g.fy * itz2 * gj21
    tanx, tany = k(A.tanx), k(A.tany)
    gt[2] = select(g.clx, gt[2] + E(g.sgx) * k(1.3) * tanx * gtxc, gt[2])
    glimx = select(g.clx, E(g.sgx) * tz * gtxc, k(0.0))
    gt[0] = select(g.clx, gt[0], gt[0] + gtxc)
    gt[2] = select(g.cly, gt[2] + E(g.sgy) * k(1.3) * tany * gtyc, gt[2])
    glimy = select(g.cly, E(g.sgy) * tz * gtyc, k(0.0))
    gt[1] = select(g.cly, gt[1], gt[1] + gtyc)
    cam[27] = cam[27] + (rp.div(-g.fx, tanx) * gfx + k(1.3) * glimx)
    cam[28] = cam[28] + (rp.div(-g.fy, tany) * gfy + k(1.3) * glimy)
    # ---- view transform
    for c in range(3):
        for j in range(3):
            dx[c] = dx[c] + gt[j] * V[4 * c + j]
            cam[3 * c + j] = cam[3 * c + j] + g.x[c] * gt[j]
    for j in range(3):
        cam[9 + j] = cam[9 + j] + gt[j]
    # ---- NDC mean
    h = [g.x[0] * Pm[j] + g.x[1] * Pm[4 + j] + g.x[2] * Pm[8 + j] + Pm[12 + j] for j in range(4)]
    p_w = rp.div(k(1.0), h[3] + k(0.0000001))
    m2x, m2y = G(gi["m2x"]), G(gi["m2y"])
    gh0, gh1 = m2x * p_w, m2y * p_w
    gh3 = -p_w * p_w * (m2x * h[0] + m2y * h[1])
    for c in range(3):
        dx[c] = dx[c] + (gh0 * Pm[4 * c + 0] + gh1 * Pm[4 * c + 1] + gh3 * Pm[4 * c + 3])
        cam[12 + 3 * c + 0] = cam[12 + 3 * c + 0] + g.x[c] * gh0
        cam[12 + 3 * c + 1] = cam[12 + 3 * c + 1] + g.x[c] * gh1
        cam[12 + 3 * c + 2] = cam[12 + 3 * c + 2] + g.x[c] * gh3
    cam[21] = cam[21] + gh0; cam[22] = cam[22] + gh1; cam[23] = cam[23] + gh3
    # ---- rotation matrix -> normalised quaternion -> raw quaternion
    r, x, y, z = g.qn
    two, four = k(2.0), k(4.0)
    gq = [two * (-z * gR[1][0] + y * gR[2][0] + z * gR[0][1] - x * gR[2][1] - y * gR[0][2] + x * gR[1][2]),
          two * (y * gR[1][0] + z * gR[2][0] + y * gR[0][1] - r * gR[2][1] + z * gR[0][2] + r * gR[1][2]) - four * x * (gR[1][1] + gR[2][2]),
          two * (x * gR[1][0] + r * gR[2][0] + x * gR[0][1] + z * gR[2][1] - r * gR[0][2] + z * gR[1][2]) - four * y * (gR[0][0] + gR[2][2]),
          two * (-r * gR[1][0] + x * gR[2][0] + r * gR[0][1] + y * gR[2][1] + x * gR[0][2] + y * gR[1][2]) - four * z * (gR[0][0] + gR[1][1])]
    dot = r * gq[0] + x * gq[1] + y * gq[2] + z * gq[3]
    il = rp.div(k(1.0), g.qlen)
    go["rotation"] = [(gq[0] - r * dot) * il, (gq[1] - x * dot) * il, (gq[2] - y * dot) * il, (gq[3] - z * dot) * il]
    go["scaling"] = [ds[c] * g.s[c] if A.scale_act == 1 else ds[c] * k(A.mod) for c in range(3)]
    go["xyz"] = dx
    if A.strand:
        nn = [E(A.dirs[:, c]) for c in range(3)]
        dl = fmax(rp.sqrt(nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2]), k(1e-12))
        b = [rp.div(nn[c], dl) for c in range(3)]
        gbv = [go["rotation"][0], go["rotation"][3], -go["rotation"][2]]
        dot = b[0] * gbv[0] + b[1] * gbv[1] + b[2] * gbv[2]
        hs = k(0.5) * go["scaling"][0]
        go["dirs"] = [go["dirs"][c] + (rp.div(gbv[c] - b[c] * dot, dl) + hs * b[c]) for c in range(3)]
        go["scaling"] = [zero(n) for _ in range(3)]
        go["rotation"] = [zero(n) for _ in range(4)]
    # rows the kernel does not run are exactly zero
    off = ~np.asarray(live, dtype=bool)
    kill = lambda e: E(np.where(off, 0.0, e.v), np.where(off, 0.0, e.e))  # noqa: E731
    for key, val in go.items():
        go[key] = [kill(e) for e in val] if isinstance(val, list) else kill(val)
    cam = [kill(e) for e in cam]
    return go, cam


# ------------------------------------------------------------------------------------------------ reductions
DEPTH_F32 = 5 + 3          # float32 additions on any path of gh_project.cu's camera reduction: 5 shuffle levels + 3 warp adds
U64 = 2.0 ** -53


def camera_sum(cam_rows, f32_depth=DEPTH_F32):
    """The 29 camera gradients: per-row E summed over the rows in any order (warp shuffle and CTA sums in float32,
    then float64 across CTAs, then one rounding to float32).  -> (value (29,), bound (29,)), each bound the sum of
    the rows' bounds plus the rounding of every partial sum, bounded by the sum of the absolute terms."""
    vals, bnds = [], []
    for e in cam_rows:
        n = e.v.size
        v = float(np.sum(e.v))
        sabs = float(np.sum(np.abs(e.v)) + np.sum(e.e))
        b = float(np.sum(e.e)) + f32_depth * U * sabs + n * U64 * sabs + U * (abs(v) + float(np.sum(e.e)) + f32_depth * U * sabs) + TINY
        vals.append(v); bnds.append(b)
    return np.array(vals), np.array(bnds)


def cam37(vals):
    """the 29 accumulators in the layout of d_camera (16 V + 16 Pm + 3 campos + 2 tan)"""
    out = np.zeros(37)
    for kk in range(12):
        out[4 * (kk // 3) + kk % 3] = vals[kk]
    for q in range(12):
        col = q % 3
        out[16 + 4 * (q // 3) + (3 if col == 2 else col)] = vals[12 + q]
    out[32:35] = vals[24:27]
    out[35:37] = vals[27:29]
    return out


def strand_midpoints(origins, dirs):
    """gh_strand_midpoints_kernel: origins (S,3), dirs (S,L,3) float32 values -> E list over segments of (S,3)"""
    o = E(np.asarray(origins, np.float32).astype(np.float64))
    d = np.asarray(dirs, np.float32).astype(np.float64)
    S, L = d.shape[0], d.shape[1]
    acc = E(np.zeros((S, 3)))
    prev = o + E(0.0)
    v = np.zeros((S, L, 3)); e = np.zeros((S, L, 3))
    for kk in range(L):
        acc = acc + E(d[:, kk])
        p = o + acc
        m = (p + prev) * E(0.5)
        v[:, kk], e[:, kk] = m.v, m.e
        prev = p
    return v, e


def strand_backward(d_xyz, direct):
    """gh_strand_backward_kernel: dL/dd_k = direct_k + 0.5 gx_k + sum_{j>k} gx_j; the suffix sum in any order (shuffle
    scan within 32-segment chunks, a carry across chunks) bounded by (terms - 1) u times the sum of its |terms|.
    d_xyz, direct: (S,L,3) float32 values -> (value, bound) (S,L,3)."""
    gx = np.asarray(d_xyz, np.float32).astype(np.float64)
    dd = np.asarray(direct, np.float32).astype(np.float64)
    L = gx.shape[1]
    rev = lambda a: np.flip(np.cumsum(np.flip(a, 1), 1), 1)  # noqa: E731
    suffix = rev(gx) - gx                                       # sum over j > k
    sabs = rev(np.abs(gx)) - np.abs(gx)
    cnt = (L - 1 - np.arange(L))[None, :, None]                 # terms of the suffix sum
    es = np.maximum(cnt - 1, 0) * U * sabs * (1.0 + 64 * U) + np.where(cnt > 0, TINY, 0.0)
    t1 = E(dd) + E(0.5 * gx)
    out = t1 + E(suffix, es)
    return out.v, out.e


# ------------------------------------------------------------------------------------------------ scenes
# Scenes shared by the host rehearsal (tests/test_project64_cpu.py) and the kernels' test (tests/test_gpu_project64.py):
# float32 numpy arrays, built from a seed.
GAUSSIAN_MODEL = dict(scale_act=1, opacity_act=1, label_act=1, conf_act=1, dir_mode=0, det_eps=1e-12)
HAIR_MODEL = dict(scale_act=0, opacity_act=2, label_act=2, conf_act=1, dir_mode=1, det_eps=1e-7)
HEAD_PRECOMP = dict(scale_act=0, opacity_act=0, label_act=3, conf_act=3, dir_mode=2, det_eps=1e-12)
IDENTITY_ACTS = dict(scale_act=0, opacity_act=0, label_act=0, conf_act=0, dir_mode=0, det_eps=1e-12)
HAIR_STRANDS = dict(HAIR_MODEL, strands=1)
CONFIGS = {"gaussian_model": GAUSSIAN_MODEL, "hair": HAIR_MODEL, "head": HEAD_PRECOMP, "identity": IDENTITY_ACTS,
           "strands": HAIR_STRANDS}


def ring_camera(k, W, H, focal_factor=1.2):
    """synth.make_camera's ring camera as float32 arrays: V, Pm (4,4) row-vector layout, campos, tan(fov/2)."""
    import math
    theta = 2.0 * math.pi * k / 64
    c = np.array([0.8 * math.sin(theta), 0.0, 0.8 * math.cos(theta)])
    zc = -c / np.linalg.norm(c)
    yc = np.array([0.0, 1.0, 0.0])
    xc = np.cross(yc, zc); xc /= np.linalg.norm(xc)
    R = np.stack([xc, yc, zc])
    w2c = np.eye(4); w2c[:3, :3] = R; w2c[:3, 3] = -R @ c
    focal = focal_factor * H
    tanx, tany = W / (2.0 * focal), H / (2.0 * focal)
    P = np.zeros((4, 4)); P[0, 0] = 1 / tanx; P[1, 1] = 1 / tany; P[3, 2] = 1.0
    P[2, 2] = 100.0 / (100.0 - 0.01); P[2, 3] = -(100.0 * 0.01) / (100.0 - 0.01)
    V = w2c.T
    return dict(W=W, H=H, V=V.astype(np.float32), Pm=(V @ P.T).astype(np.float32), campos=c.astype(np.float32),
                tanx=float(np.float32(tanx)), tany=float(np.float32(tany)))


def axis_camera(W, H, tanx=0.5, tany=0.25):
    """A camera at the origin looking down +z with V = identity: view-space positions are the positions themselves,
    and with power-of-two tan(fov/2) the clamp limits 1.3 tan are exact float32 products."""
    V = np.eye(4, dtype=np.float32)
    P = np.zeros((4, 4)); P[0, 0] = 1 / tanx; P[1, 1] = 1 / tany; P[3, 2] = 1.0
    P[2, 2] = 100.0 / (100.0 - 0.01); P[2, 3] = -(100.0 * 0.01) / (100.0 - 0.01)
    return dict(W=W, H=H, V=V, Pm=P.T.astype(np.float32), campos=np.zeros(3, np.float32), tanx=tanx, tany=tany)


def random_scene(P, seed, cfg_name, deg=3, mod=1.0, cam_k=5, W=640, H=480):
    """P Gaussians (or segments) in a ball in front of the ring camera; log-uniform scales, quaternions with |q| from
    1e-3 to 1e3, every 97th row behind the camera and every 89th near the near plane."""
    rng = np.random.default_rng(seed)
    cfg = CONFIGS[cfg_name]
    cam = ring_camera(cam_k, W, H)
    xyz = rng.uniform(-0.25, 0.25, (P, 3))
    xyz[::97] = 2.5 * cam["campos"] + rng.uniform(-0.05, 0.05, (len(xyz[::97]), 3))            # behind the camera
    fwd = -cam["campos"] / np.linalg.norm(cam["campos"])
    near = rng.uniform(0.15, 0.25, len(xyz[::89]))
    xyz[::89] = cam["campos"] + near[:, None] * fwd + rng.uniform(-0.01, 0.01, (len(near), 3))    # near plane 0.2
    s = np.exp(rng.uniform(np.log(1e-3), np.log(3e-2), (P, 3)))
    q = rng.normal(size=(P, 4))
    q *= (10.0 ** rng.uniform(-3, 3, (P, 1))) / np.linalg.norm(q, axis=1, keepdims=True)
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    sc = dict(P=P, cfg=cfg, deg=deg, mod=mod, cam=cam,
              xyz=f(xyz), f_dc=f(rng.normal(0, 0.6, (P, 3))), f_rest=f(rng.normal(0, 0.25, (P, 45))),
              opacity=f(rng.normal(0, 2, P)), label=f(rng.normal(0, 2, P)), conf=f(rng.normal(0, 1, P)),
              dirs=f(rng.normal(0, 1, (P, 3)) * 4e-3))
    if cfg.get("strands"):
        sc.update(scaling=f([1.5e-3]), rotation=None)
    else:
        sc.update(scaling=f(np.log(s) if cfg["scale_act"] == 1 else s), rotation=f(q))
    return sc


def inputs(sc):
    c = sc["cam"]
    return Inputs(sc["P"], c["W"], c["H"], sc["xyz"], sc["scaling"], sc["rotation"], sc["dirs"], sc["f_dc"], sc["f_rest"],
                  sc["opacity"], sc["label"], sc["conf"], c["V"], c["Pm"], c["campos"], c["tanx"], c["tany"], sc["mod"],
                  sc["deg"], sc["cfg"])


def random_grads(P, seed, conf_scale=1e-3):
    """incoming gradients: NDC mean (x, y), the public conic 3-vector [g00, 2 g01, g11] (with 2 g01 exact), colours
    (depth included) and opacity, float32"""
    rng = np.random.default_rng(seed)
    g01 = rng.normal(0, conf_scale, P).astype(np.float32)
    con = np.stack([rng.normal(0, conf_scale, P), 2.0 * g01.astype(np.float64), rng.normal(0, conf_scale, P)], 1)
    return dict(m2x=rng.normal(size=P).astype(np.float32), m2y=rng.normal(size=P).astype(np.float32),
                con=con.astype(np.float32), color=rng.normal(size=(P, 10)).astype(np.float32),
                opacity=rng.normal(size=P).astype(np.float32))


def neutralize(rp, gi):
    """Zero the incoming gradients whose result an ambiguous decision would change: a colour clamp zeroes its
    channel, an arg-max tie the two direction channels, a clamp decision the whole row."""
    gi = {k: v.copy() for k, v in gi.items()}
    for ch in range(3):
        gi["color"][rp.rows(f"color{ch}"), ch] = 0.0
    gi["color"][rp.rows("argmax"), 5:7] = 0.0
    whole = rp.rows("clamp")
    for k in gi:
        gi[k][whole] = 0.0
    return gi


def _up(x, n=1):
    x = np.float32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, np.float32(np.inf if n > 0 else -np.inf))
    return float(x)


def edge_scene():
    """Hand-built rows at the projection's decision edges, seen by `axis_camera(64, 32)` (tan 0.5 / 0.25, fx = fy =
    64): -> (scene, {name: row}).  Activated scales and identity activations (IDENTITY_ACTS), scale modifier 1.5."""
    cam = axis_camera(64, 32)
    mod = 1.5
    rows, names = [], {}

    def add(name, xyz, s=(1e-4, 1e-4, 1e-4), q=(1.0, 0.0, 0.0, 0.0)):
        names[name] = len(rows)
        rows.append((xyz, s, q))

    # near plane: view z one float32 step either side of 0.2, on it, and behind the camera
    for name, z in (("near_below", _up(0.2, -1)), ("near_on", _up(0.2, 0)), ("near_above", _up(0.2, 1)), ("behind", -1.0)):
        add(name, (0.0, 0.0, z), s=(1e-3, 1e-3, 1e-3))
    # the +-1.3 tan(fov/2) clamp at view z = 1: on, one step inside and one outside, both signs, both axes; large
    # footprints keep the rows visible, distinct scales keep the arg-max decided, and a tilted major axis gives the
    # direction channels a view-z component, so that the two branches' gradients differ by far more than the bound
    big = (0.3, 0.2, 0.25)
    for ax, lim in ((0, 0.65), (1, 0.325)):
        for sign in (1.0, -1.0):
            for name, t in (("on", lim), ("in", _up(lim, -1)), ("out", _up(lim, 1))):
                p = [0.0, 0.0, 1.0]
                p[ax] = sign * t
                add(f"clamp_{'xy'[ax]}{'+' if sign > 0 else '-'}_{name}", tuple(p), s=big, q=(0.9, 0.1, 0.3, -0.2))
    # tile rectangle empty by one tile at each image edge (and one half pixel inside): px = -2 / py = -2 and
    # px = 67 / py = 35 are the limits for a 3-pixel splat radius
    for name, ax, pix, vis in (("left", 0, -2.5, 0), ("left", 0, -1.5, 1), ("right", 0, 67.5, 0), ("right", 0, 66.5, 1),
                               ("top", 1, -2.5, 0), ("top", 1, -1.5, 1), ("bottom", 1, 35.5, 0), ("bottom", 1, 34.5, 1)):
        size = (64, 32)[ax]
        m = (2 * pix + 1) / size - 1
        p = [0.0, 0.0, 1.0]
        p[ax] = m * (1 + 1e-7) / (2.0, 4.0)[ax]
        add(f"tile_{name}_{'in' if vis else 'out'}", tuple(p))
    # near-singular 2-D covariances: a needle at 45 degrees in the image plane, ac - b^2 cancels
    c8, s8 = np.cos(np.pi / 8), np.sin(np.pi / 8)
    for kk, L in enumerate((0.05, 1.0, 4.0)):
        add(f"needle{kk}", (0.0, 0.0, 1.0), s=(L, 1e-5, 1e-5), q=(c8, 0.0, 0.0, s8))
    # equal scales (arg-max ties: first index), and scales equal only after the modifier
    add("tie01", (0.0, 0.0, 1.0), s=(0.01, 0.01, 0.005), q=(0.9, 0.1, 0.3, -0.2))
    add("tie12", (0.0, 0.0, 1.0), s=(0.005, 0.01, 0.01), q=(0.9, 0.1, 0.3, -0.2))
    add("tie012", (0.0, 0.0, 1.0), s=(0.01, 0.01, 0.01), q=(0.9, 0.1, 0.3, -0.2))
    m32 = np.float32(mod)
    for a in np.float32(0.015) + np.arange(64, dtype=np.float32) * np.float32(1e-6):
        b = np.nextafter(a, np.float32(1))
        if np.float32(a * m32) == np.float32(b * m32):
            break
    else:
        raise AssertionError("no scale pair that the modifier merges")
    add("tie_after_mod", (0.0, 0.0, 1.0), s=(float(a), float(b), 0.004), q=(0.9, 0.1, 0.3, -0.2))
    n = len(rows)
    rng = np.random.default_rng(11)
    f = lambda x: np.ascontiguousarray(x, dtype=np.float32)  # noqa: E731
    sc = dict(P=n, cfg=IDENTITY_ACTS, deg=3, mod=mod, cam=cam,
              xyz=f([r[0] for r in rows]), scaling=f([r[1] for r in rows]), rotation=f([r[2] for r in rows]),
              f_dc=f(rng.normal(0, 0.6, (n, 3))), f_rest=f(rng.normal(0, 0.25, (n, 45))),
              opacity=f(rng.normal(0, 2, n)), label=f(rng.normal(0, 2, n)), conf=f(rng.normal(0, 1, n)),
              dirs=f(rng.normal(0, 1, (n, 3))))
    return sc, names


def _solve(B, target):
    """a float32 r with fl(B * r) == target exactly, or None"""
    r = np.float32(np.float32(target) / B)
    for k in range(-64, 65):
        c = r
        for _ in range(abs(k)):
            c = np.nextafter(c, np.float32(np.inf if k > 0 else -np.inf))
        if np.float32(B * c) == np.float32(target):
            return c
    return None


def colour_tie_scene():
    """Three rows whose SH colour sums are exactly -0.5 (channel 0), one float32 step above (1) and one below (2).  The
    view direction is exactly +z and f_dc is 0, so the sum is one product acc = fl(B[k] * f_rest[k]) with a single
    rounding whether or not it is fused: B[2] = C1 (degree 1) or B[6] = 2 C22 (degree 2).
    -> (scene, the three sums, coefficient index k, B[k])"""
    for deg, kk, B in ((1, 2, np.float32(SH_C1)), (2, 6, np.float32(2) * np.float32(SH_C2[2]))):
        vals = [_solve(B, t) for t in (-0.5, _up(-0.5, 1), _up(-0.5, -1))]
        if all(v is not None for v in vals):
            break
    else:
        raise AssertionError("no f_rest values with exact SH sums at -0.5")
    cam = axis_camera(64, 32)
    P = 3
    rest = np.zeros((P, 45), np.float32)
    rest[:, 3 * (kk - 1):3 * kk] = vals                 # coefficient kk, channel ch -> acc_ch
    f = lambda x: np.ascontiguousarray(x, dtype=np.float32)  # noqa: E731
    sc = dict(P=P, cfg=IDENTITY_ACTS, deg=deg, mod=1.0, cam=cam, xyz=f([(0.0, 0.0, 4.0)] * P),
              scaling=f([(0.01, 0.02, 0.03)] * P), rotation=f([(1.0, 0.0, 0.0, 0.0)] * P), f_dc=np.zeros((P, 3), np.float32),
              f_rest=rest, opacity=f(np.zeros(P)), label=f(np.zeros(P)), conf=f(np.zeros(P)), dirs=f(np.ones((P, 3))))
    return sc, [float(np.float32(B * v)) for v in vals], kk, B


def strand_edge_scene():
    """Segment rows (HAIR_STRANDS): b.x close to -1, where 1 + b.x cancels, exactly -1, and zero-length segments,
    among random segments, seen by the ring camera."""
    sc = random_scene(64, 7, "strands", deg=2)
    d = sc["dirs"]
    L = 4e-3
    for i, eps in enumerate((0.0, 1e-7, 1e-5, 1e-3, 3e-2)):
        d[i] = np.float32([-L * np.sqrt(1 - eps * eps), L * eps, -L * eps * 0.5])
    d[5] = 0.0
    d[6] = 0.0
    sc["dirs"] = np.ascontiguousarray(d, np.float32)
    return sc


# ------------------------------------------------------------------------------------------------ checks
class Stats:
    """Per output: elements checked, unresolved elements (bound > 2^-10 |value|), largest |got - value| / bound."""

    def __init__(self):
        self.rows = {}

    def add(self, name, checked, unresolved, ratio):
        c, u, r = self.rows.get(name, (0, 0, 0.0))
        self.rows[name] = (c + checked, u + unresolved, max(r, ratio))

    def unresolved_fraction(self):
        c = sum(v[0] for v in self.rows.values())
        return sum(v[1] for v in self.rows.values()) / max(c, 1)

    def __str__(self):
        return "  ".join(f"{k}: n={c} unres={u} max err/bound={r:.3g}" for k, (c, u, r) in sorted(self.rows.items()))


def within(stats, name, got, e, rows=None):
    """assert |got - e.v| <= e.e element by element (on `rows`); exact zeros where the bound is zero"""
    got = np.asarray(got, dtype=np.float64)
    v, b = np.broadcast_to(e.v, got.shape), np.broadcast_to(e.e, got.shape)
    m = np.ones(got.shape, dtype=bool) if rows is None else np.broadcast_to(np.asarray(rows, bool).reshape(
        (-1,) + (1,) * (got.ndim - 1)), got.shape)
    err = np.abs(got - v)
    finite = np.isfinite(b)
    bad = m & finite & ~(err <= b)
    if bad.any():
        idx = np.argwhere(bad)[:5]
        det = "; ".join(f"{tuple(int(t) for t in i)}: got {got[tuple(i)]!r} replay {v[tuple(i)]!r} bound {b[tuple(i)]!r}" for i in idx)
        raise AssertionError(f"{name}: {int(bad.sum())} of {int((m & finite).sum())} elements outside the bound: {det}")
    unres = m & (~finite | (b > REL_UNRESOLVED * np.abs(v)))
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(m & finite & (b > 0), err / b, 0.0)
    stats.add(name, int(m.sum()), int(unres.sum()), float(ratio.max()) if ratio.size else 0.0)


def check_forward(rp, o, got, stats, P):
    """got: means2D (P,3), conic (P,3), colors (P,10), opacity (P,), visible (P,) bool, cov3D (P,6) or None"""
    full = lambda es: E(np.stack([np.broadcast_to(e.v, (P,)) for e in es], -1), np.stack([np.broadcast_to(e.e, (P,)) for e in es], -1))  # noqa: E731
    vis = np.asarray(got["visible"], bool)
    amb = rp.rows("vis")
    wrong = ~amb & (vis != o["visible"])
    assert not wrong.any(), f"visible differs from the replay on decided rows {np.flatnonzero(wrong)[:8].tolist()}"
    stats.add("visible", int((~amb).sum()), int(amb.sum()), 0.0)
    within(stats, "means2D", got["means2D"], full(o["means2D"]))
    within(stats, "conic", got["conic"], full(o["conic"]), rows=vis)
    assert float(np.abs(np.asarray(got["conic"])[~vis]).sum()) == 0.0, "a culled row has a non-zero conic"
    within(stats, "colors", got["colors"], full(o["color"]))
    within(stats, "opacity", np.asarray(got["opacity"]).reshape(P), E(np.broadcast_to(o["opacity"].v, (P,)), np.broadcast_to(o["opacity"].e, (P,))))
    if got.get("cov3D") is not None:
        within(stats, "cov3D", got["cov3D"], full(o["cov3D"]))


GRAD_KEYS = ("xyz", "scaling", "rotation", "dirs", "f_dc", "rest", "opacity", "label", "conf")


def check_backward(rp, go, cam, got, stats, P, cam_got=None):
    """got: dict of (P, k) arrays for the keys present (GRAD_KEYS); cam_got: the (37,) d_camera or None"""
    for key in GRAD_KEYS:
        if got.get(key) is None:
            continue
        val = go[key]
        es = val if isinstance(val, list) else [val]
        ref = E(np.stack([np.broadcast_to(e.v, (P,)) for e in es], -1), np.stack([np.broadcast_to(e.e, (P,)) for e in es], -1))
        within(stats, "d_" + key, np.asarray(got[key], np.float64).reshape(P, len(es)), ref)
    if cam_got is not None:
        v, b = camera_sum(cam)
        c = np.asarray(cam_got, np.float64).reshape(37)
        v37, b37 = cam37(v), cam37(b)
        within(stats, "d_camera", c, E(v37, b37))
