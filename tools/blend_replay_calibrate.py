"""Calibrate the tolerance of tests/test_gpu_blend_replay.py: run every scene of that file through the same checks with
the reference's own CUDA build (oracle/_ref) and with this repository's kernels, and print the worst ratio
|x - x64| / (scale + floor) per output for both.  The tests' TOL must leave the reference room to spare.

    python tools/blend_replay_calibrate.py OUT.json        (on a GPU, with oracle/_ref built)
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _util  # noqa: E402
import test_gpu_blend_replay as tb  # noqa: E402


def scenes():
    for W, H in ((33, 17), (47, 31)):
        yield f"border-{W}x{H}", tb.border_scene(W, H)
    yield "alpha-band", tb.band_scene()
    for n, k in tb.WINDOW_CASES:
        yield f"window-{n}" + (f"-stop{k}" if k else ""), tb.window_scene(n, k)
    yield "early-stop", tb.stop_scene()
    for a, b in tb.SORT_CASES:
        yield f"two-tiles-{a}-{b}", tb.two_tile_scene(a, b)
    for n in (1000, 3000):
        yield f"equal-depths-{n}", tb.equal_depth_scene(n)


def main(out_path):
    dev = torch.device("cuda:0")
    mods = {"reference": _util.ref_module()._C, "this": tb._mine()}
    res = {}
    for name, inp in scenes():
        res[name] = {k: tb.check(m, inp, dev)[0] for k, m in mods.items()}
        print(name, {k: f"{max(v.values()):.3g}" for k, v in res[name].items()}, flush=True)
    for k in mods:
        worst = max((max(r[k].values()), n) for n, r in res.items())
        print(f"{k}: worst ratio {worst[0]:.3g} ({worst[1]}); TOL = {tb.TOL}")
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1])
