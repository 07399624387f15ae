"""The densification replay (tests/_densify64.py) pinned three ways, with no GPU: decisions built by hand on exact ties,
the NaN / inf rules of the reference, and the reference's own `densify_and_prune` as run on an H100
(tests/golden/densify64.npz, tests/golden/make_golden_densify64.py): decisions and layout exactly, children within
the replay's bound."""
import math
import os

import numpy as np
import pytest

import _densify64 as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "densify64.npz")
SCENES = ("mixed", "no_screen", "tie_opacity", "max_grad_zero")
INPUTS = ("xyz", "log_scaling", "rotation", "opacity_logit", "accum", "denom")


def _decide(accum, denom, ls, op, max_grad=2e-4, min_opacity=0.005, extent=100.0, max_screen_size=20, percent_dense=0.01):
    f = lambda a: np.asarray(a, np.float32)  # noqa: E731
    return D.decide(f(accum), f(denom), f(ls).reshape(-1, 3), f(op), max_grad, min_opacity, extent, max_screen_size, percent_dense)


def test_gradient_tie_is_hot():
    thr = np.float32(2e-4)
    d = _decide([2 * thr, np.nextafter(2 * thr, np.float32(0))], [2, 2], [[1, 0, 0], [1, 0, 0]], [2, 2])
    assert d["g"][0] == thr and d["hot_clone"][0] and d["hot_split"][0]
    assert not d["hot_clone"][1] and not d["hot_split"][1]
    assert d["split"].tolist() == [True, False] and not D.ambiguous(d).any()


def test_dense_extent_tie_clones_and_is_decided():
    # exp(0) = 1 exactly and percent_dense * extent = 0.01 * 100 = 1: smax <= 1, a clone, not a split
    d = _decide([1e-2] * 4, [1] * 4, [[0, 0, 0], [0, -5, -1], [0, 1e-3, 0], [0, 1e-7, 0]], [2] * 4)
    assert d["clone"][:3].tolist() == [True, True, False] and d["split"][:3].tolist() == [False, False, True]
    assert not d["amb_dense"][:3].any() and d["margin_dense"][0] == 0.0
    assert d["amb_dense"][3]                         # exp(1e-7) lies within 2 ulp of 1: either answer is allowed


def test_opacity_tie_is_kept():
    # sigmoid(0) = 1 / (1 + exp(0)) = 0.5 exactly, not < min_opacity = 0.5
    d = _decide([0, 0, 0], [1, 1, 1], [[0, 0, 0]] * 3, [0, -1e-5, -1e-8], min_opacity=0.5)
    assert d["opacity"][0] == 0.5 and not d["prune_self"][0] and not d["amb_op"][0]
    assert d["prune_self"][1] and not d["amb_op"][1]
    assert d["amb_op"][2]                            # within the sigmoid's float32 bound of 0.5


def test_world_size_limit_only_with_a_screen_size():
    ls = [[math.log(30.0), 0, 0]]
    for mss, pruned in ((20, True), (None, False), (0, False)):
        d = _decide([1e-2], [1], ls, [2], max_screen_size=mss)
        assert d["split"][0] and bool(d["prune_self"][0]) == pruned
        # the children have max scale 30 * 0.625 = 18.75 > 10 as well
        assert bool(d["prune_child"][0]) == pruned
    d = _decide([1e-2], [1], [[math.log(12.0), 0, 0]], [2])            # parent 12 > 10, children 7.5
    assert d["prune_self"][0] and not d["prune_child"][0]
    assert D.flags_of(d).tolist() == [[0, 0, 1, 1]]


def test_nan_and_inf_gradients():
    d = _decide([0, 1e-5, -1e-5, np.nan, 1e-5], [0, 0, 0, 1, np.nan], [[1, 0, 0]] * 5, [2] * 5)
    assert d["g"][0] == 0 and d["g"][3] == 0 and d["g"][4] == 0           # 0/0, NaN/1, x/NaN -> NaN -> 0
    assert d["g"][1] == np.inf and d["g"][2] == -np.inf
    assert d["hot_split"].tolist() == [False, True, False, False, False]
    assert d["hot_clone"].tolist() == [False, True, True, False, False]   # torch.norm(-inf) = inf
    d = _decide([0], [0], [[1, 0, 0]], [2], max_grad=0.0)                  # max_grad = 0: g = 0 is hot
    assert d["split"][0]


def test_nan_scale_keeps_the_row_as_it_is():
    """torch.max propagates NaN, and NaN compares False: no clone, no split, no world-size prune."""
    big = math.log(20.0)
    d = _decide([1e-2, 1e-2, 1e-2], [1, 1, 1], [[np.nan, big, big], [big, np.nan, -3], [-3, -3, np.nan]], [2, 2, 2])
    assert np.isnan(d["smax"]).all() and np.isnan(d["cmax"]).all()
    assert not d["clone"].any() and not d["split"].any() and not d["prune_self"].any()
    assert D.flags_of(d).tolist() == [[1, 0, 0, 0]] * 3 and not D.ambiguous(d).any()


def test_nan_opacity_is_never_pruned():
    d = _decide([1e-2, 1e-2], [1, 1], [[1, 0, 0], [-3, -3, -3]], [np.nan, np.nan], min_opacity=0.5)
    assert not d["prune_self"].any() and not d["prune_child"].any()
    assert D.flags_of(d).tolist() == [[0, 0, 1, 1], [1, 1, 0, 0]]


def test_layout_order_and_sample_slots():
    # rows: kept, cloned, split + children kept, split + children pruned, pruned, split + children kept
    flags = np.array([[1, 0, 0, 0], [1, 1, 0, 0], [0, 0, 1, 1], [0, 0, 0, 1], [0, 0, 0, 0], [0, 0, 1, 1]], np.int32)
    lay = D.layout(flags)
    assert (lay["nA"], lay["nB"], lay["nC"], lay["n_split_all"], lay["P_new"]) == (2, 1, 2, 3, 7)
    assert lay["dst_orig"].tolist() == [0, 1, -1, -1, -1, -1]
    assert lay["dst_clone"].tolist() == [-1, 2, -1, -1, -1, -1]
    assert lay["dst_child0"].tolist() == [-1, -1, 3, -1, -1, 4]
    assert lay["dst_child1"].tolist() == [-1, -1, 5, -1, -1, 6]
    assert lay["slot"].tolist() == [-1, -1, 0, 1, -1, 2]          # ranks among ALL split rows: row 5 reads 2 and 3 + 2


def test_child_geometry_closed_forms():
    """Identity rotation, a quarter turn about z (unnormalised) and the zero quaternion."""
    xyz = np.array([[1, 2, 3]] * 3, np.float32)
    q = np.array([[1, 0, 0, 0], [3, 0, 0, 3], [0, 0, 0, 0]], np.float32)
    ls = np.zeros((3, 3), np.float32)
    samples = np.array([[0.5, 0.25, -1], [1, 0, 0], [1, 1, 1], [0, 0, 2], [0, 1, 0], [1, 1, 1]], np.float32)
    p0, p1, b0, b1, L, Lb = D.children(xyz, ls, q, samples, [0, 1, 2], [0, 1, 2], 3)
    assert np.allclose(p0[0], [1.5, 2.25, 2]) and np.allclose(p1[0], [1, 2, 5])
    # build_rotation's layout (R[1][0] = 2 (xy - rz)) sends e_x to -e_y and e_y to e_x for q = (1, 0, 0, 1)
    assert np.allclose(p0[1], [1, 1, 3], atol=1e-12) and np.allclose(p1[1], [2, 2, 3], atol=1e-12)
    assert np.isnan(p0[2]).all() and np.isnan(p1[2]).all()
    assert (b0[:2] < 1e-5).all() and (b0[:2] > 0).all()
    assert np.allclose(L, math.log(0.625)) and (Lb < 1e-6).all()


def _golden():
    if not os.path.isfile(GOLDEN):
        pytest.fail(f"missing {GOLDEN}")
    return np.load(GOLDEN)


def _golden_scene(z, sc):
    inp = {k: z[f"{sc}/{k}"] for k in INPUTS}
    mg, mo, ex, mss, pd = (float(v) for v in z[f"{sc}/params"])
    return inp, dict(max_grad=mg, min_opacity=mo, extent=ex, max_screen_size=None if mss < 0 else mss, percent_dense=pd)


@pytest.mark.parametrize("scene", SCENES)
def test_replay_matches_the_reference(scene):
    z = _golden()
    inp, prm = _golden_scene(z, scene)
    rep = D.replay(inp, z[f"{scene}/samples"], **prm)
    lay, d = rep["layout"], rep["decisions"]
    assert z[f"{scene}/samples"].shape[0] == 2 * lay["n_split_all"]
    assert z[f"{scene}/out_xyz"].shape[0] == lay["P_new"]
    # the layout, read off the row-index label and the moments (row + 0.25 / + 0.5 copied, zero for new rows)
    dst, src = D.expected_copies(None, lay)
    assert sorted(dst.tolist()) == list(range(lay["P_new"]))
    assert np.array_equal(z[f"{scene}/out_label"][dst, 0], src.astype(np.float32))
    kept = lay["dst_orig"] >= 0
    for n, off in (("exp_avg", 0.25), ("exp_avg_sq", 0.5)):
        for g in ("xyz", "scaling", "label"):
            m = z[f"{scene}/out_{g}_{n}"]
            assert np.array_equal(m[lay["dst_orig"][kept]], np.broadcast_to((np.nonzero(kept)[0] + off)[:, None], m[lay["dst_orig"][kept]].shape).astype(np.float32))
            new = np.setdiff1d(np.arange(lay["P_new"]), lay["dst_orig"][kept])
            assert (m[new] == 0).all(), (g, n)
    # copies of the geometry the children do not replace
    o = np.nonzero(kept)[0]
    for g, src_key in (("xyz", "xyz"), ("scaling", "log_scaling"), ("rotation", "rotation")):
        np.testing.assert_array_equal(z[f"{scene}/out_{g}"][lay["dst_orig"][o]], inp[src_key][o])
    c = np.nonzero(lay["dst_clone"] >= 0)[0]
    np.testing.assert_array_equal(z[f"{scene}/out_xyz"][lay["dst_clone"][c]], inp["xyz"][c])
    k = rep["child_rows"]
    np.testing.assert_array_equal(z[f"{scene}/out_rotation"][lay["dst_child1"][k]], inp["rotation"][k])
    assert D.check_children(z[f"{scene}/out_xyz"], z[f"{scene}/out_scaling"], rep) == []
    # the scenes reach what they were built for
    assert lay["nB"] > 0 and lay["nC"] > 0 and lay["n_split_all"] > lay["nC"]


def test_golden_reaches_the_ties_and_nan_rows():
    z = _golden()
    inp, prm = _golden_scene(z, "mixed")
    d = D.decide(inp["accum"], inp["denom"], inp["log_scaling"], inp["opacity_logit"], **prm)
    thr = np.float32(prm["max_grad"])
    assert (d["g"] == thr).any() and (d["clone"] & (d["margin_dense"] == 0)).any()
    assert np.isnan(inp["log_scaling"]).any(axis=1).sum() >= 2 and (d["hot_split"] & np.isnan(d["smax"])).any()
    assert np.isnan(inp["opacity_logit"]).any() and np.isinf(d["g"]).any()
    # NaN-scale rows stay in place, unchanged
    lay = D.layout(D.flags_of(d))
    nan_rows = np.nonzero(np.isnan(inp["log_scaling"]).any(axis=1))[0]
    assert (lay["dst_orig"][nan_rows] >= 0).all()
    out = z["mixed/out_scaling"][lay["dst_orig"][nan_rows]]
    np.testing.assert_array_equal(out, inp["log_scaling"][nan_rows])
    inp, prm = _golden_scene(z, "tie_opacity")
    d = D.decide(inp["accum"], inp["denom"], inp["log_scaling"], inp["opacity_logit"], **prm)
    assert ((d["opacity"] == 0.5) & ~d["prune_self"] & ~d["amb_op"]).sum() >= 10
