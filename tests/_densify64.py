"""TEST INFRASTRUCTURE ONLY -- a replay of `GaussianModel.densify_and_prune` (src/scene/gaussian_model.py:682-737) per
source row, in numpy, with no GPU and no reference sources: the fate decisions with their margins, the final row of
every original, clone and child, each child's sample slot, and each child's position and log-scale in float64 with a
first-order bound of a float32 evaluation.

Decisions.  The reference (and csrc/gh_densify.cu) decides per source row i
    g      = accum / denom, NaN -> 0                         one IEEE division: replayed exactly in float32
    clone  = |g| >= thr and smax <= dense                    smax = max_k exp(ls_k), NaN if any ls_k is NaN (torch.max)
    split  =  g  >= thr and smax >  dense
    prune  = op < min_opacity or (max_screen_size and smax > ws)      op = sigmoid(opacity logit)
    prune of a child: op < min_opacity or (max_screen_size and cmax > ws), cmax = max_k exp(log(exp(ls_k) * 0.625))
with thr = max_grad, dense = percent_dense * extent, ws = 0.1 * extent each rounded to float32 once (the comparison of
a float32 tensor with a Python float, and the ctypes argument).  smax, op and cmax go through expf / logf, whose float32
results are only known to within their documented CUDA error (expf 2 ulp, logf 1 ulp; division, addition and
multiplication correctly rounded): they are computed in float64 with an interval that contains every float32 result
those bounds allow.  A decision whose interval straddles its threshold is ambiguous, and a caller accepts either outcome
there.  A function value that is exact (exp(0) = 1, so sigmoid(0) = 1 / 2) has a point interval: those ties are decided.

Layout.  [kept originals | kept clones | first children | second children], each block in source order; a split
row's two children read samples[slot] and samples[n_split_all + slot], slot = its rank among ALL split rows (before the
final prune), because the reference draws one sample per split row and copy (stds.repeat(2, 1)).

Children.  position = R(q / |q|) sample + xyz, log-scale = log(exp(ls) * 0.625): torch on the device divides by the
Python scalar 0.8 * 2 as a multiplication by its float32 reciprocal, 1 / 1.6f = 0.625 exactly.  Bounds (units of
u = 2^-24, first order, every float32 operation rounding once to at most u times its result; a fused multiply-add
rounds less, and a different summation order is covered by bounding each sum by the sum of its absolute terms):
    |q|^2: 4 positive terms                                           <= 4 relative
    1 / sqrt(|q|^2) (or the quotient q / |q|): sqrt halves it, +1 +1  <= 4 relative
    q_k / |q|: one more product                                       <= 4 |q_k| / |q| + |q_k / |q||
    R entries 1 - 2 (b b + c c), 2 (a b -+ r c): the V arithmetic below, term by term (2 x is exact)
    position: the entries' errors times the exact samples, 3 products, 3 sums each <= sum |R_jk s_k| + |xyz_j|
    log-scale: expf 4 (2 ulp <= 4 u relative), the product 1, so 5 absolute after logf, plus logf's 1 ulp <= 2 |L|
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24
EXP_ULP_U = 4.0                 # expf: 2 ulp <= 4 u relative
LOG_ULP_U = 2.0                 # logf: 1 ulp <= 2 u relative
CHILD_SCALE = 0.625             # fl(1 / fl(0.8 * 2)): torch's reciprocal of the Python scalar
TINY = 2.0 ** -149              # one float32 denormal step: the absolute floor of any rounding


def f32(x):
    return np.float32(x)


class V:
    """float64 value `v` and a first-order bound `e` (units of u) of a float32 evaluation, elementwise."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = np.asarray(v, np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, np.float64)

    def _r(self, v, e):                       # one correctly rounded operation
        return V(v, e + np.abs(v))

    def __add__(a, b):
        b = b if isinstance(b, V) else V(np.full_like(a.v, b))
        return a._r(a.v + b.v, a.e + b.e)

    def __sub__(a, b):
        b = b if isinstance(b, V) else V(np.full_like(a.v, b))
        return a._r(a.v - b.v, a.e + b.e)

    def __rsub__(a, b):
        return V(np.full_like(a.v, b)) - a

    def __mul__(a, b):
        if not isinstance(b, V):
            if float(f32(b)) == float(b) and abs(np.log2(abs(b)) % 1.0) == 0.0:     # a power of two: exact
                return V(a.v * b, a.e * abs(b))
            b = V(np.full_like(a.v, b))
        return a._r(a.v * b.v, np.abs(a.v) * b.e + np.abs(b.v) * a.e)

    __rmul__ = __mul__


def v_exp(x: V) -> V:
    v = np.exp(x.v)
    return V(v, v * x.e + EXP_ULP_U * v)


def v_log(x: V) -> V:
    v = np.log(x.v)
    return V(v, x.e / np.abs(x.v) + LOG_ULP_U * np.abs(v))


def _exp_interval(x32):
    """[lo, hi] of every float32 expf(x) within 2 ulp; a point at x = 0 (expf(0) = 1 exactly)."""
    v = np.exp(x32.astype(np.float64))
    b = EXP_ULP_U * U * v + TINY
    b = np.where(x32 == 0, 0.0, b)
    return v - b, v + b, v


def _nanmax3(lo, hi, v):
    """torch.max over the 3 components: NaN if any component is NaN."""
    nan = np.isnan(v).any(axis=1)
    return (np.where(nan, np.nan, lo.max(axis=1)), np.where(nan, np.nan, hi.max(axis=1)),
            np.where(nan, np.nan, v.max(axis=1)))


def _decide(lo, hi, thr, op):
    """(decision, ambiguous, margin) of `x op thr` for x in [lo, hi]: NaN compares False, decided."""
    with np.errstate(invalid="ignore"):
        a, b = op(lo, thr), op(hi, thr)
    nan = np.isnan(lo) | np.isnan(hi)
    amb = (a != b) & ~nan
    return np.where(nan, False, a), amb


def thresholds(max_grad, min_opacity, extent, max_screen_size, percent_dense):
    ws = float(f32(0.1 * extent)) if max_screen_size else None
    return dict(thr=f32(max_grad), dense=float(f32(percent_dense * extent)), min_op=float(f32(min_opacity)), ws=ws)


def decide(accum, denom, log_scaling, opacity_logit, max_grad, min_opacity, extent, max_screen_size, percent_dense=0.01):
    """Per-row decisions.  Returns a dict of (P,) arrays:
        g (float32), hot_clone, hot_split, clone, split, prune_self, prune_child, and for each of dense / op / ws_self /
        ws_child the ambiguity flag `amb_*` and the margin `margin_*` = distance to the threshold over the half-width
        of the interval (inf where the value is exact, NaN where it is NaN)."""
    th = thresholds(max_grad, min_opacity, extent, max_screen_size, percent_dense)
    acc = np.asarray(accum, np.float32).reshape(-1)
    den = np.asarray(denom, np.float32).reshape(-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        g = acc / den
    g = np.where(np.isnan(g), np.float32(0), g).astype(np.float32)
    hot_clone = np.abs(g) >= th["thr"]
    hot_split = g >= th["thr"]

    ls = np.asarray(log_scaling, np.float32).reshape(-1, 3)
    lo, hi, v = _exp_interval(ls)
    smax_lo, smax_hi, smax = _nanmax3(lo, hi, v)
    le_dense, amb_dense = _decide(smax_lo, smax_hi, th["dense"], np.less_equal)
    gt_dense, _ = _decide(smax_lo, smax_hi, th["dense"], np.greater)

    # opacity: 1 / (1 + expf(-x)): expf 4 u * e / (1 + e), the sum and the quotient 1 u each; exact at x = 0
    x = np.asarray(opacity_logit, np.float32).reshape(-1).astype(np.float64)
    with np.errstate(over="ignore"):
        e = np.exp(-x)
        op = 1.0 / (1.0 + e)
        rel = EXP_ULP_U * (e / (1.0 + e)) + 2.0
    rel = np.where(np.isinf(e), 0.0, rel)              # expf(-x) = inf: the float32 sigmoid is 0, below any threshold
    ob = np.where(x == 0, 0.0, U * rel * op + TINY)
    op_lt, amb_op = _decide(op - ob, op + ob, th["min_op"], np.less)

    # the children's max scale: expf(logf(fl(expf(ls) * 0.625))), its own interval
    c = v_exp(v_log(v_exp(V(ls.astype(np.float64))) * CHILD_SCALE))
    cb = U * c.e + TINY
    cmax_lo, cmax_hi, cmax = _nanmax3(c.v - cb, c.v + cb, c.v)
    if th["ws"] is not None:
        ws_self, amb_ws_self = _decide(smax_lo, smax_hi, th["ws"], np.greater)
        ws_child, amb_ws_child = _decide(cmax_lo, cmax_hi, th["ws"], np.greater)
    else:
        ws_self = ws_child = amb_ws_self = amb_ws_child = np.zeros(g.shape, bool)

    def margin(val, lo_, hi_, t):
        half = (hi_ - lo_) / 2
        with np.errstate(divide="ignore", invalid="ignore"):
            m = (val - t) / half
            return np.where(half == 0, np.where(val == t, 0.0, np.sign(val - t) * np.inf), m)

    out = dict(g=g, hot_clone=hot_clone, hot_split=hot_split,
               clone=hot_clone & le_dense, split=hot_split & gt_dense,
               prune_self=op_lt | ws_self, prune_child=op_lt | ws_child,
               amb_dense=amb_dense & (hot_clone | hot_split), amb_op=amb_op, amb_ws_self=amb_ws_self & (th["ws"] is not None),
               amb_ws_child=amb_ws_child & (th["ws"] is not None),
               margin_dense=margin(smax, smax_lo, smax_hi, th["dense"]), margin_op=margin(op, op - ob, op + ob, th["min_op"]),
               smax=smax, cmax=cmax, opacity=op)
    if th["ws"] is not None:
        out["margin_ws_self"] = margin(smax, smax_lo, smax_hi, th["ws"])
        out["margin_ws_child"] = margin(cmax, cmax_lo, cmax_hi, th["ws"])
    return out


def flags_of(d) -> np.ndarray:
    """(P, 4) int32 in gh_densify_classify's layout: [original kept, clone kept, children kept, split]."""
    split, clone = d["split"], d["clone"]
    return np.stack([~split & ~d["prune_self"], clone & ~d["prune_self"], split & ~d["prune_child"], split], 1).astype(np.int32)


def ambiguous(d) -> np.ndarray:
    """(P,) rows with any ambiguous decision (their flags are taken from the kernel)."""
    return d["amb_dense"] | d["amb_op"] | d["amb_ws_self"] | d["amb_ws_child"]


def layout(flags) -> dict:
    """Destination rows (-1: none) of every source row, from (P, 4) flags:
    dst_orig, dst_clone, dst_child0, dst_child1, slot (sample rank among all split rows, -1 if not split),
    and the totals nA, nB, nC, n_split_all, P_new."""
    f = np.asarray(flags).astype(np.int64)
    inc = np.cumsum(f, axis=0)
    nA, nB, nC, nS = (int(inc[-1, k]) if len(f) else 0 for k in range(4))
    exc = inc - f
    none = -np.ones(len(f), np.int64)
    return dict(dst_orig=np.where(f[:, 0] == 1, exc[:, 0], none), dst_clone=np.where(f[:, 1] == 1, nA + exc[:, 1], none),
                dst_child0=np.where(f[:, 2] == 1, nA + nB + exc[:, 2], none),
                dst_child1=np.where(f[:, 2] == 1, nA + nB + nC + exc[:, 2], none),
                slot=np.where(f[:, 3] == 1, exc[:, 3], none), nA=nA, nB=nB, nC=nC, n_split_all=nS, P_new=nA + nB + 2 * nC)


def rotation_matrix(q) -> list:
    """build_rotation (src/utils/general_utils.py:79-109) of (P, 4) float32 quaternions as 3x3 nested V entries, R[j][k]."""
    q = np.asarray(q, np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / np.sqrt((q * q).sum(axis=1))
        # |q|^2 <= 4 u relative (4 positive terms), sqrt halves it and rounds once, the reciprocal (or the quotient
        # q / |q|) rounds once more: 4 u; the component product rounds once
        comps = [V(q[:, k] * inv, np.abs(q[:, k]) * 4.0 * inv + np.abs(q[:, k] * inv)) for k in range(4)]
    r, x, y, z = comps
    return [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y + r * z), 2.0 * (x * z - r * y)],
            [2.0 * (x * y - r * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z + r * x)],
            [2.0 * (x * z + r * y), 2.0 * (y * z - r * x), 1.0 - 2.0 * (x * x + y * y)]]


def children(xyz, log_scaling, rotation, samples, rows, slots, n_split_all):
    """Float64 children of the source `rows` with sample `slots`: (pos0, pos1, bound0, bound1, log_scale, ls_bound),
    positions (n, 3), bounds in absolute units (not u)."""
    rows = np.asarray(rows, np.int64)
    R = rotation_matrix(np.asarray(rotation)[rows])
    x = np.asarray(xyz, np.float32)[rows].astype(np.float64)
    s = np.asarray(samples, np.float32).astype(np.float64)
    out = []
    for off in (0, n_split_all):
        smp = s[np.asarray(slots, np.int64) + off] if len(rows) else np.zeros((0, 3))
        pos, bnd = [], []
        with np.errstate(invalid="ignore"):
            for j in range(3):
                terms = [R[j][k].v * smp[:, k] for k in range(3)]
                val = terms[0] + terms[1] + terms[2] + x[:, j]
                mag = sum(np.abs(t) for t in terms) + np.abs(x[:, j])
                # entry errors times the exact samples, 3 product roundings, 3 sums in any order (<= u * mag each)
                e = sum(R[j][k].e * np.abs(smp[:, k]) for k in range(3)) + sum(np.abs(t) for t in terms) + 3.0 * mag
                pos.append(val)
                bnd.append(U * e + TINY)
        out.append((np.stack(pos, 1), np.stack(bnd, 1)))
    ls = np.asarray(log_scaling, np.float32)[rows].astype(np.float64)
    L = v_log(v_exp(V(ls)) * CHILD_SCALE)
    return out[0][0], out[1][0], out[0][1], out[1][1], L.v, U * L.e + TINY


def replay(inputs: dict, samples, max_grad, min_opacity, extent, max_screen_size, percent_dense=0.01, flags=None) -> dict:
    """The full outcome for `inputs` (xyz, log_scaling, rotation, opacity_logit, accum, denom as float32 arrays).
    `flags`: take the (P, 4) flags from the kernel instead (the caller checks them against the decisions first).
    Returns decide()'s dict, layout()'s dict, `flags`, and the children (child rows, slots, positions, bounds)."""
    d = decide(inputs["accum"], inputs["denom"], inputs["log_scaling"], inputs["opacity_logit"], max_grad, min_opacity,
               extent, max_screen_size, percent_dense)
    f = flags_of(d) if flags is None else np.asarray(flags, np.int32)
    lay = layout(f)
    kept = np.nonzero(f[:, 2] == 1)[0]
    p0, p1, b0, b1, L, Lb = children(inputs["xyz"], inputs["log_scaling"], inputs["rotation"], samples, kept,
                                     lay["slot"][kept], lay["n_split_all"])
    return dict(decisions=d, flags=f, layout=lay, child_rows=kept, child_pos0=p0, child_pos1=p1, child_bound0=b0,
                child_bound1=b1, child_log_scale=L, child_log_scale_bound=Lb)


def expected_copies(src, lay) -> tuple:
    """(dst rows, src rows) of every bit-exact copy of a parameter row: kept originals, kept clones, and both children
    (which copy every parameter except position and scale)."""
    o = np.nonzero(lay["dst_orig"] >= 0)[0]
    c = np.nonzero(lay["dst_clone"] >= 0)[0]
    k = np.nonzero(lay["dst_child0"] >= 0)[0]
    return (np.concatenate([lay["dst_orig"][o], lay["dst_clone"][c], lay["dst_child0"][k], lay["dst_child1"][k]]),
            np.concatenate([o, c, k, k]))


def check_children(out_xyz, out_log_scale, rep) -> list:
    """Messages for every child element outside the replay's bound (NaN must sit where the replay has NaN)."""
    lay = rep["layout"]
    rows = rep["child_rows"]
    msgs = []
    for which, dst in ((0, lay["dst_child0"][rows]), (1, lay["dst_child1"][rows])):
        got = np.asarray(out_xyz, np.float64)[dst]
        want, bound = rep[f"child_pos{which}"], rep[f"child_bound{which}"]
        msgs += _bound_msgs(f"child{which} position", got, want, bound, rows)
        msgs += _bound_msgs(f"child{which} log-scale", np.asarray(out_log_scale, np.float64)[dst], rep["child_log_scale"],
                            rep["child_log_scale_bound"], rows)
    return msgs


def _bound_msgs(what, got, want, bound, rows) -> list:
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    msgs = []
    bad_nan = nan_g != nan_w
    if bad_nan.any():
        r = np.nonzero(bad_nan.any(axis=-1) if bad_nan.ndim > 1 else bad_nan)[0][:5]
        msgs.append(f"{what}: NaN positions differ at source rows {rows[r].tolist()}")
    with np.errstate(invalid="ignore"):
        err = np.abs(got - want)
        bad = (err > bound) & ~nan_g & ~nan_w
        bad |= np.isinf(want) & (got != want) & ~nan_g
    if bad.any():
        i = np.argwhere(bad)[0]
        msgs.append(f"{what}: {int(bad.sum())} elements outside the bound, e.g. source row {rows[i[0]]}: "
                    f"got {got[tuple(i)]!r} want {want[tuple(i)]!r} bound {bound[tuple(i)]!r}")
    return msgs


def special_rows(thr):
    """(log_scaling, opacity_logit, accum, denom, rotation) rows on the ties and the NaN / inf / degenerate inputs, for
    percent_dense * extent = 1, 0.1 * extent = 10."""
    big, half = math.log(20.0), math.log(5.0)
    q = [1.0, 0.0, 0.0, 0.0]
    two_thr = float(f32(2 * f32(thr)))
    rows = [
        ([0, 0, 0], 2.0, two_thr, 2, q),                    # smax = exp(0) = 1 = dense extent, g = thr: cloned
        ([0, -1, -2], 2.0, 1e-2, 1, q),                     # smax = 1 exactly, hot: cloned
        ([0.1, 0, 0], 2.0, two_thr, 2, q),                  # g = thr, smax > 1: split
        ([float("nan"), big, half], 2.0, 1e-2, 1, q),       # NaN scale: torch.max gives NaN, no clone / split / prune
        ([float("nan"), -3, -3], 2.0, 1e-2, 1, q),
        ([half, half, 0.2], float("nan"), 1e-2, 1, q),      # NaN opacity: split, never pruned on opacity
        ([0.3, 0.2, 0.1], 2.0, 0.0, 0, q),                  # 0 / 0 -> NaN -> 0: cold
        ([0.3, 0.2, 0.1], 2.0, 1e-5, 0, q),                 # x / 0 = inf: hot, split
        ([-2, -2, -3], 2.0, 1e-5, 0, q),                    # inf: hot, cloned
        ([0.5, 0.1, 0.2], 2.0, 1e-2, 1, [1e-3, 2e-4, -3e-4, 5e-4]),
        ([0.5, 0.1, 0.2], 2.0, 1e-2, 1, [-700.0, 300.0, 600.0, -100.0]),
        ([0.5, 0.1, 0.2], 2.0, 1e-2, 1, [-0.5, 0.5, -0.5, 0.5]),
        ([0.5, 0.1, 0.2], 2.0, 1e-2, 1, [0.0, 0.0, 0.0, 0.0]),     # zero quaternion: NaN children positions
        ([math.log(16.0), 0, 0], 2.0, 1e-2, 1, q),          # child max scale 0.625 * 16 = 10 = 0.1 * extent (within an ulp)
        ([math.log(10.0), 0, 0], 2.0, 1e-2, 1, q),          # parent on the world-size limit
        ([0, 0, 0], 0.0, 1e-2, 1, q),                       # sigmoid(0) = 0.5
    ]
    return rows
