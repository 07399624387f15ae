"""Time the mesh signed distance at the FLAME filter's scale and print one JSON line (DESIGN §23).

    python tools/sdf_step.py [--gaussians 500000] [--reps 10]

For 500 k Gaussians (6 M icosahedron corners) against the ~10 k-face head of tests/_sdf_cases.py, and against a
~40 k-face version of it: the gh_sdf_query kernel time (CUDA events around each call after a warm-up, median),
`flame_filter_keep` end to end (corners + query + mask, median), the triangle-point pairs per second, the FP32-pipe
instructions per pair in the kernel's loop from `cuobjdump -sass`, and the card's name and power limit, read in the
same run.  There is no pysdf arm: pysdf is not part of this package's environment.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _sdf_cases as K  # noqa: E402
from gaussianhaircut_b200 import _capi, mesh as M  # noqa: E402

FP32 = ("FADD", "FMUL", "FFMA", "FMNMX", "FSETP", "FSEL", "FSET")


def sass_per_pair() -> dict:
    """Opcodes of the query kernel's hottest loop (the backward branch whose body holds the square roots), per pair:
    the loop body holds rsqrt count / 3 pairs."""
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                                         "cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", _capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    fn = out[out.index("gh_sdf_query_kernel"):]
    fn = fn[:fn.find("Function :", 10) if "Function :" in fn[10:] else len(fn)]
    ins = [(int(a, 16), op) for a, op in re.findall(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", fn)]
    addr = {a: i for i, (a, _) in enumerate(ins)}
    best = None
    for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?P\w+\s+)?BRA\s+(?:!?P\d+,\s*)?0x([0-9a-f]+)", fn):
        src, dst = int(m.group(1), 16), int(m.group(2), 16)
        if dst < src and dst in addr:
            body = [op for a, op in ins[addr[dst]:addr[src] + 1]]
            n_sqrt = sum(op.startswith("MUFU.RSQ") for op in body)
            if n_sqrt and (best is None or len(body) > len(best)):
                best = body
    if best is None:
        return {"error": "query loop not found in the SASS"}
    pairs = sum(op.startswith("MUFU.RSQ") for op in best) / 3
    count = lambda pred: sum(pred(op.split(".")[0]) for op in best) / pairs  # noqa: E731
    return {"pairs_per_loop_body": pairs, "fp32_per_pair": count(lambda o: o in FP32),
            "mufu_per_pair": count(lambda o: o == "MUFU"), "fp64_per_pair": count(lambda o: o in ("DADD", "DFMA")),
            "all_per_pair": len(best) / pairs}


def _median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def measure(verts, faces, P, reps, dev, label):
    mesh = M.MeshSDF(torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev))
    xyz, scaling, rotation, lab = (torch.from_numpy(a).to(dev) for a in K.gaussians(verts, faces, P, 5))
    corners = M.flame_corners(xyz, scaling, rotation)
    for _ in range(2):                                       # warm-up of both paths
        mesh(corners)
        M.flame_filter_keep(xyz, scaling, rotation, lab, mesh)
    torch.cuda.synchronize()
    k_med, k_min, k_max = _median_ms(lambda: mesh(corners), reps)
    e_med, _, _ = _median_ms(lambda: M.flame_filter_keep(xyz, scaling, rotation, lab, mesh), reps)
    pairs = corners.shape[0] * faces.shape[0]
    return {"mesh": label, "faces": int(faces.shape[0]), "gaussians": P, "corners": int(corners.shape[0]),
            "kernel_ms_median": round(k_med, 3), "kernel_ms_min": round(k_min, 3), "kernel_ms_max": round(k_max, 3),
            "filter_ms_median": round(e_med, 3), "pairs_per_s": pairs / (k_med * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=500_000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sdf_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rows = [measure(*K.head(), args.gaussians, args.reps, dev, "head ~10 k faces"),
            measure(*K.head(140, 144), args.gaussians, max(3, args.reps // 2), dev, "head ~40 k faces")]
    sass = sass_per_pair()
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    for r in rows:        # the FP32 pipe issues 128 lanes per SM per clock: the share of that rate the loop uses
        if "fp32_per_pair" in sass and smi:
            mhz = float(smi[0].split(",")[2].strip().split()[0])
            r["fp32_issue_share_at_max_clock"] = r["pairs_per_s"] * sass["fp32_per_pair"] / (sm * 128 * mhz * 1e6)
    print(json.dumps({"card": smi[0] if smi else torch.cuda.get_device_name(dev), "sm_count": sm, "sass": sass,
                      "rows": rows}))


if __name__ == "__main__":
    main()
