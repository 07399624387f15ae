"""CPU tests: pin the float64 blend replay (oracle/blend64.py) on the vectors the reference's CUDA build wrote
(tests/golden/make_golden.py), the way tests/test_oracle_cpu.py pins Oracle-B: n_contrib exactly, the image, final_T
and the four blend gradients within float32 rounding of the replay's per-element scale."""
import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import blend64  # noqa: E402

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "*_*.npz")))
GOLDEN = [g for g in GOLDEN if not os.path.basename(g).startswith(("pyref", "loss_"))]
# float32 rounding: the reference's outputs on these vectors sit within 2.4e-6 of the scale (worst: final_T of
# strands_render_hair); the blend tests on the GPU use the same measure
PIN_TOL = 1e-5
FLOOR = 1e-30


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_replay_matches_reference_cuda_build(path):
    d = np.load(path)
    W, H = int(d["W"]), int(d["H"])
    r = blend64.replay(d["st_means2D"], d["st_conic_opacity"], d["in_colors_precomp"], d["bg"], d["st_point_list"],
                       d["st_ranges"], W, H, d["dL_dout"])
    # every reached decision is farther from its threshold than float32 can move it
    for k in ("alpha_ratio", "power_ratio", "stop_ratio"):
        assert r[k] >= blend64.DECISION_SAFETY, f"{k} {r[k]}"
    assert np.array_equal(r["n_contrib"].numpy(), d["st_n_contrib"].astype(np.int64))
    assert int(r["n_contrib"].max()) > 0
    assert blend64.worst_ratio(d["out_color"], r["image"], r["image_scale"], FLOOR) <= PIN_TOL
    assert blend64.worst_ratio(d["st_final_T"], r["final_T"], r["final_T"], FLOOR) <= PIN_TOL
    for n in blend64.GRADS:
        assert blend64.worst_ratio(d["g_" + n], r[n], r["scale"][n], FLOOR) <= PIN_TOL, n


def test_replay_decisions_by_hand():
    """One pixel, four records at the centre of a 1x1 image, opacities chosen so that each of the reference's
    decisions happens once: a skip below 1/255, the 0.99 cap, a blend, and the stop on test_T < 1e-4."""
    P = 4
    xy = np.zeros((P, 2), np.float32)
    co = np.zeros((P, 4), np.float32)
    co[:, 0] = co[:, 2] = 1.0
    co[:, 3] = [0.003, 5.0, 0.5, 0.99]          # skipped, capped (T 1 -> 0.01), blended (-> 0.005), stop (test_T 5e-5)
    col = np.arange(P * 10, dtype=np.float32).reshape(P, 10)
    bg = np.ones(10, np.float32)
    r = blend64.replay(xy, co, col, bg, np.arange(P, dtype=np.uint32), np.array([[0, P]], np.uint32), 1, 1,
                       np.ones((10, 1, 1), np.float32))
    a1 = float(np.float32(0.99))
    T1 = 1.0 - a1
    assert int(r["n_contrib"][0]) == 3
    assert float(r["final_T"][0]) == pytest.approx(T1 * 0.5, rel=1e-15)
    img = a1 * col[1].astype(np.float64) + T1 * 0.5 * col[2].astype(np.float64) + T1 * 0.5 * bg
    np.testing.assert_allclose(r["image"][:, 0, 0].numpy(), img, rtol=1e-14)
    # dL/dcolour = alpha T_before dL; nothing for the skipped and the stopping record
    np.testing.assert_allclose(r["dL_dcolors"][:, 0].numpy(), [0.0, a1, T1 * 0.5, 0.0], rtol=1e-14)
    # dL/dopacity = G dL/dalpha, G = 1 at the mean; record 2: T_before (c . dL) - T_final / (1 - alpha) (bg . dL)
    d2 = T1 * col[2].sum() - (T1 * 0.5) / 0.5 * 10.0
    assert float(r["dL_dopacity"][2, 0]) == pytest.approx(d2, rel=1e-14)
