"""Time the orientation maps per image on the GPU and count the arithmetic the Gabor kernel does.

    python tools/orient_case.py [out.json]

Arms, at 1024x1024, 1920x1080 and 2048x2048 (seeded strand pictures):
  kernels     `orientation_maps` on a device tensor, CUDA events around 20 calls after warm-up (both stages, allocation);
  gabor       the Gabor stage alone (gh_orient_gabor), CUDA events, for the FMA rate;
  calc_orients the drop-in from numpy uint8 in to numpy out (host clock, includes copies and the device sync);
  ref tf32 / ref fp32  the reference's `calc_orients` from the staged copy with cuDNN TF32 on (its default) and off.
It also reports the FMAs per pixel the Gabor kernel computes (8 filters share a tap rectangle), the useful ones (each
filter's own support), the fraction of the card's FP32 FMA peak (SMs x 128 FMA/clock x the maximum SM clock), the
TF32-on disagreements with the kernels at 1080p, and the card's name, power limit and clocks.
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _orient_cases as OC  # noqa: E402
import orient64  # noqa: E402


def fma_counts(bank: np.ndarray, G: int):
    """(computed, useful) FMAs per pixel: the kernel runs every tap of the rectangle holding the non-zero taps of 8
    consecutive filters of a 64-filter chunk of one group; useful = each filter's own non-zero rectangle."""
    N, K, _ = bank.shape
    nf = N // G
    computed = useful = 0
    for g in range(G):
        for c0 in range(0, nf, 64):
            for w0 in range(c0, min(c0 + 64, nf), 8):
                js = range(w0, min(w0 + 8, nf))
                ys, xs = [], []
                for j in js:
                    yy, xx = np.nonzero(bank[j * G + g])
                    ys += [yy.min(), yy.max()]
                    xs += [xx.min(), xx.max()]
                    useful += (yy.max() - yy.min() + 1) * (xx.max() - xx.min() + 1)
                computed += 8 * (max(ys) - min(ys) + 1) * (max(xs) - min(xs) + 1)
    return computed, useful


def main(out_path=None):
    import torch
    from gaussianhaircut_b200 import _capi
    from gaussianhaircut_b200.orient import calc_orients, orientation_maps
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import orient_ref
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    props = torch.cuda.get_device_properties(dev)
    bank, thetas, G = orient64.bank()
    computed, useful = fma_counts(bank, G)
    try:
        max_mhz = float(q.split(",")[2].strip().split()[0])
    except (IndexError, ValueError):
        max_mhz = float("nan")
    peak_fma = props.multi_processor_count * 128 * max_mhz * 1e6
    ref = orient_ref.load()
    res = {"gpu": q, "sms": props.multi_processor_count, "fma_per_pixel_computed": computed,
           "fma_per_pixel_useful": useful, "fma_per_pixel_dense": 180 * 17 * 17, "peak_fma_per_s": peak_fma, "sizes": []}
    lib = _capi.load()
    for (W, H) in ((1024, 1024), (1920, 1080), (2048, 2048)):
        img = OC.strands(H, W, seed=W + H, n=int(1500 * H * W / 2e6) + 200)
        timg = torch.from_numpy(img).to(dev)
        for _ in range(3):
            orientation_maps(timg)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            out = orientation_maps(timg)
        e1.record()
        e1.synchronize()
        kernels_ms = e0.elapsed_time(e1) / 20
        # the Gabor stage alone, on the workspace the last call left its float32 DoG in
        c = next(iter(__import__("gaussianhaircut_b200.orient", fromlist=["_consts"])._consts.values()))
        nb = C.c_size_t()
        _capi.check(lib.gh_orient_workspace_size(H, W, c["N"], c["K"], c["nf"], C.byref(nb)))
        ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
        dog = torch.empty(H, W, dtype=torch.float64, device=dev)
        st = _capi._stream(dev)
        rl, rh = (c["w_low"].numel() - 1) // 2, (c["w_high"].numel() - 1) // 2
        _capi.check(lib.gh_orient_dog(H, W, 3, _capi._ptr(timg), _capi._ptr(c["w_low"]), rl, _capi._ptr(c["w_high"]), rh,
                                      _capi._ptr(dog), _capi._ptr(ws), nb.value, st))
        o, v = torch.empty(H, W, dtype=torch.int64, device=dev), torch.empty(H, W, device=dev)
        gab = lambda: _capi.check(lib.gh_orient_gabor(H, W, _capi._ptr(c["bank"]), c["N"], c["K"], c["nf"],  # noqa: E731
                                                      _capi._ptr(c["thetas"]), _capi._ptr(o), _capi._ptr(v),
                                                      _capi._ptr(ws), nb.value, st))
        gab()
        torch.cuda.synchronize()
        assert torch.equal(o, out["orients"]) and torch.equal(v, out["var"])
        e0.record()
        for _ in range(20):
            gab()
        e1.record()
        e1.synchronize()
        gabor_ms = e0.elapsed_time(e1) / 20
        calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 64)
        t0 = time.perf_counter()
        for _ in range(5):
            calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 64)
        drop_ms = (time.perf_counter() - t0) / 5 * 1e3
        row = {"W": W, "H": H, "kernels_ms": kernels_ms, "gabor_ms": gabor_ms, "calc_orients_ms": drop_ms,
               "gabor_fma_per_s": computed * H * W / (gabor_ms * 1e-3),
               "gabor_fraction_of_fp32_fma_peak": computed * H * W / (gabor_ms * 1e-3) / peak_fma}
        prev = torch.backends.cudnn.allow_tf32
        for arm, flag in (("ref_tf32_ms", True), ("ref_fp32_ms", False)):
            torch.backends.cudnn.allow_tf32 = flag
            ro, _, _ = ref.calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 64)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            reps = 2
            for _ in range(reps):
                ro, _, _ = ref.calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 64)
            row[arm] = (time.perf_counter() - t0) / reps * 1e3
            row[arm.replace("_ms", "_index_disagreements")] = int((ro != out["orients"].cpu().numpy()).sum())
        torch.backends.cudnn.allow_tf32 = prev
        res["sizes"].append(row)
        print(json.dumps(row, default=int), flush=True)
    print(json.dumps({k: v for k, v in res.items() if k != "sizes"}, default=int))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1, default=int)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
