"""Time `simple_knn._C.distCUDA2` end to end (Morton codes, torch.sort, boxes, query) on the test distributions.

    python tools/knn_case.py [--sizes 100000,1000000,4000000] [--cases a,b,c] [--repeats 7] [--iters 5]
    python tools/knn_case.py --profile OUT_DIR      # per-kernel split from torch.profiler (a separate run)

Per (case, size): warm-up, then `repeats` windows of `iters` calls timed with CUDA events; the median window is
reported in ms per call.  The card's name and power limit are read in the same run.  One JSON line per row.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import _knn_cases as K  # noqa: E402
from simple_knn._C import distCUDA2  # noqa: E402

CASES = {"a": K.uniform, "b": K.head_shell, "c": K.strand_vertices}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def time_case(pts: torch.Tensor, repeats: int, iters: int) -> list:
    for _ in range(3):
        distCUDA2(pts)
    torch.cuda.synchronize()
    windows = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            distCUDA2(pts)
        e1.record()
        torch.cuda.synchronize()
        windows.append(e0.elapsed_time(e1) / iters)
    return windows


def profile(pts: torch.Tensor, out_dir: str) -> dict:
    from torch.profiler import ProfilerActivity, profile as tprofile
    for _ in range(3):
        distCUDA2(pts)
    torch.cuda.synchronize()
    n = 10
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            distCUDA2(pts)
        torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    split = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            split[ev.key[:80]] = round(t / n, 1)      # us per call
    return dict(sorted(split.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000,4000000")
    ap.add_argument("--cases", default="a,b,c")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--profile", metavar="OUT_DIR", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("knn_case: no CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    for c in a.cases.split(","):
        for P in (int(s) for s in a.sizes.split(",")):
            pts = torch.from_numpy(CASES[c](P, 1)).to(dev)
            row = dict(case=c, P=P, **info)
            if a.profile:
                row["us_per_call_by_kernel"] = profile(pts, a.profile)
                with open(os.path.join(a.profile, "knn_profile.jsonl"), "a") as f:
                    f.write(json.dumps(row) + "\n")
            else:
                w = time_case(pts, a.repeats, a.iters)
                row.update(ms_per_call=round(statistics.median(w), 4), windows_ms=[round(x, 4) for x in w])
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
