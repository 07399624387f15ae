"""Measure how much of the replay's variance bound the orientation kernels use (TOL in tests/_orient_cases.py).

    python tools/orient_replay_calibrate.py [out.json]

For seeded images (noise, strand pictures, gratings, the non-default bank) it runs `orientation_maps` on the GPU and
the float64 replay (oracle/orient64.py) on the CPU, and reports the worst |var - var64| / var_scale over the pixels
whose index is a candidate, the pixel count outside the replay at TOL, and how many pixels the replay calls certain.
A ratio below 2^-24 = 5.96e-8 means the first-order float32 bound holds with room to spare.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _orient_cases as OC  # noqa: E402
import orient64  # noqa: E402


def main(out_path=None):
    import torch
    from gaussianhaircut_b200.orient import orientation_maps
    dev = torch.device("cuda:0")
    cases = [("noise 256x256", OC.noise(256, 256, 1), {}), ("strands 512x640", OC.strands(512, 640, 2), {}),
             ("strands RGBA 300x400", OC.strands(300, 400, 3, C=4), {}), ("grating 17deg", OC.grating(17), {}),
             ("grating 133deg", OC.grating(133), {}),
             ("strands 300x400, 2 sigma_x x 2 offsets", OC.strands(300, 400, 5), dict(num_sigmas_x=2, num_offsets=2))]
    rows = []
    for name, img, kw in cases:
        got = {k: v.cpu().numpy() for k, v in orientation_maps(torch.from_numpy(img).to(dev), **kw).items()}
        b, t, G = orient64.bank(**kw)
        rep = orient64.replay(orient64.dog64(img).astype(np.float32), b, t, G)
        res = orient64.check(got["orients"], got["var"], rep, OC.TOL)
        rows.append({"case": name, "pixels": res["n"], "certain": res["certain"], "outside_at_TOL": res["n_bad"],
                     "worst_ratio": res["worst_ratio"]})
        print(json.dumps(rows[-1]), flush=True)
    summary = {"TOL": OC.TOL, "worst_ratio": max(r["worst_ratio"] for r in rows), "cases": rows,
               "gpu": torch.cuda.get_device_name(dev)}
    print(json.dumps({"TOL": summary["TOL"], "worst_ratio": summary["worst_ratio"]}))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
