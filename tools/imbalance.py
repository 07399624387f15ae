"""Measure the lock-step imbalance of the backward blend on a synthetic view (GPU tool).

The backward kernel walks the per-block lists of a warp in lock-step, so a warp spends
max(len over its blocks) steps per staged window.  This script rebuilds the per-block lists with
torch (exact alpha >= 1/255 test instead of the kernel's conservative span test, so it slightly
under-counts) and prints   sum(len)/8   vs   sum(max len)   for the current block->warp mapping and
for a per-tile mapping sorted by list length.

Forward: the kernel's lanes own vertical pixel pairs and walk the union of the pair's two lists; a warp covers
2 pair-rows x 16 columns (4 pixel rows) and a window holds 384 records.  The "forward PAIR" lines give its warp
steps (the product: window 384, 2 row pairs x 16 cols); the one-pixel-per-lane lines are kept for comparison.

    python tools/imbalance.py [--strands 5000] [--res 1920x1080]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strands", type=int, default=5000)
    ap.add_argument("--res", default="1920x1080")
    ap.add_argument("--max-tiles", type=int, default=600)
    args = ap.parse_args()
    from gaussianhaircut_b200 import _C
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import synth
    W, H = map(int, args.res.split("x"))
    dev = torch.device("cuda:0")
    scene = synth.make_strand_scene(args.strands, seed=0)
    cam = synth.make_camera(0, W, H)
    inp = synth.rasterizer_inputs(scene, cam, mode="native", device=dev)
    s, kw = inp["settings"], inp["kwargs"]
    e = torch.empty(0, device=dev)
    g = lambda k: kw[k] if kw.get(k) is not None else e
    fw = (s["bg"], kw["means3D"], kw["means2D"], g("colors_precomp"), kw["opacities"], g("scales"), g("rotations"),
          s["scale_modifier"], g("cov3D_precomp"), g("conic_precomp"), s["viewmatrix"], s["projmatrix"],
          s["tanfovx"], s["tanfovy"], s["image_height"], s["image_width"], e, s["sh_degree"], s["campos"],
          s["prefiltered"], False)
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fw)
    P = kw["means3D"].shape[0]
    d = _C.debug_export(P, W, H, R, geom, binning, img)
    ranges = d["ranges"].cpu()
    TX, TY = (W + 15) // 16, (H + 15) // 16
    ncon = d["n_contrib"].view(H, W)
    occupied = [t for t in range(TX * TY) if ranges[t, 1] > ranges[t, 0]]
    step = max(1, len(occupied) // args.max_tiles)
    sample = occupied[::step]
    tot_pairs = tot_cur = tot_sorted = tot_ideal = tot_pix = 0
    CH = (256, 384, 512, 1024, 4096)
    bsteps = {k: [0, 0] for k in CH}      # backward: [current mapping, sorted mapping]
    fsteps = {k: 0 for k in CH}           # forward: warp = 2 pixel rows, per-pixel lists
    SHAPES = ((2, 16), (4, 8), (8, 4))
    fshape = {(k, sh): 0 for k in (256, 384, 512) for sh in SHAPES}
    fpairs = 0
    inst_total = inst_contrib = inst_hit = inst_reached = 0
    ALT = ((4, 2), (2, 2), (2, 4), (8, 2), (4, 4))
    alt = {(bw, bh_, k): [0, 0] for (bw, bh_) in ALT for k in (256, 512)}
    alt_pix = {sh: 0 for sh in ALT}
    PSHAPES = ((2, 16), (4, 8))            # forward with a vertical pixel pair per lane: warp = row pairs x columns
    fpair_steps = {(k, sh): 0 for k in (256, 384, 512) for sh in PSHAPES}
    fpair_entries = 0
    for t in sample:
        ty, tx = divmod(t, TX)
        a, b = int(ranges[t, 0]), int(ranges[t, 1])
        ids = d["point_list"][a:b].long()
        xy = d["means2D"][ids]
        co = d["conic_opacity"][ids]
        ys, xs = torch.meshgrid(torch.arange(16, device=dev), torch.arange(16, device=dev), indexing="ij")
        px = (tx * 16 + xs).float().reshape(-1)
        py = (ty * 16 + ys).float().reshape(-1)
        dx = xy[:, 0:1] - px[None]
        dy = xy[:, 1:2] - py[None]
        power = -0.5 * (co[:, 0:1] * dx * dx + co[:, 2:3] * dy * dy) - co[:, 1:2] * dx * dy
        alpha = torch.clamp(co[:, 3:4] * torch.exp(power), max=0.99)
        hit = (power <= 0) & (alpha >= 1.0 / 255.0)                       # [L, 256]
        inside = ((tx * 16 + xs) < W) & ((ty * 16 + ys) < H)
        nc = torch.zeros(16, 16, dtype=torch.int32, device=dev)
        hh, ww = min(16, H - ty * 16), min(16, W - tx * 16)
        nc[:hh, :ww] = ncon[ty * 16: ty * 16 + hh, tx * 16: tx * 16 + ww]
        L = b - a
        pos = torch.arange(L, device=dev)[:, None]
        contributes = hit & (pos < nc.reshape(-1)[None]) & inside.reshape(-1)[None]
        tot_pix += int(contributes.sum())
        inst_total += L
        inst_contrib += int(contributes.any(1).sum())
        inst_hit += int((hit & inside.reshape(-1)[None]).any(1).sum())
        inst_reached += int(nc.max())
        blk = ((ys // 2) * 4 + (xs // 4)).reshape(-1)                     # [256] -> block id
        bh = torch.stack([hit[:, blk == k].any(1) for k in range(32)], 1)
        glast = torch.stack([nc.reshape(-1)[blk == k].max() for k in range(32)])
        bh &= pos < glast[None]
        nch = (L + 255) // 256
        pad = nch * 256 - L
        c = torch.nn.functional.pad(bh.int(), (0, 0, 0, pad)).view(nch, 256, 32).sum(1)     # [chunk, block]
        tot_pairs += int(c.sum())
        tot_cur += int(c.view(nch, 4, 8).max(2).values.sum())
        order = torch.argsort(c.sum(0))
        tot_sorted += int(c[:, order].view(nch, 4, 8).max(2).values.sum())
        tot_ideal += int(((c.sum(1) + 7) // 8).sum())
        # alternative block shapes (bw x bh pixels, lanes own vertical pixel pairs -> lanes per block = bw * bh / 2):
        # (block, G) pairs, pixels evaluated, warp steps of the lock-step walk with length-ranked block->warp assignment
        for (bw, bh_) in ALT:
            nbx, nby = 16 // bw, 16 // bh_
            bid = ((ys // bh_) * nbx + (xs // bw)).reshape(-1)
            nblk = nbx * nby
            lanes_per_block = bw * bh_ // 2
            per_warp = 32 // lanes_per_block
            hb = torch.stack([hit[:, bid == k].any(1) for k in range(nblk)], 1)
            gl2 = torch.stack([nc.reshape(-1)[bid == k].max() for k in range(nblk)])
            hb &= pos < gl2[None]
            for k in (256, 512):
                n = (L + k - 1) // k
                cb = torch.nn.functional.pad(hb.int(), (0, 0, 0, n * k - L)).view(n, k, nblk).sum(1)      # [chunk, block]
                order2 = torch.argsort(cb[-1])             # ranking from the last window, like the kernel
                steps = int(cb[:, order2].view(n, nblk // per_warp, per_warp).max(2).values.sum())
                a = alt[(bw, bh_, k)]
                a[0] += int(cb.sum()); a[1] += steps
            alt_pix[(bw, bh_)] += int(hb.sum()) * bw * bh_
        fh = hit & (pos < nc.reshape(-1).max())                             # forward: tile-wide early exit only
        fpairs += int(fh.sum())
        for k in CH:
            n = (L + k - 1) // k
            cb = torch.nn.functional.pad(bh.int(), (0, 0, 0, n * k - L)).view(n, k, 32).sum(1)
            bsteps[k][0] += int(cb.view(n, 4, 8).max(2).values.sum())
            bsteps[k][1] += int(cb[:, order].view(n, 4, 8).max(2).values.sum())
            cf = torch.nn.functional.pad(fh.int(), (0, 0, 0, n * k - L)).view(n, k, 8, 32).sum(1)   # [chunk, warp, lane]
            fsteps[k] += int(cf.max(2).values.sum())
            if k in (256, 384, 512):
                ph = fh.view(L, 8, 2, 16).any(2)                                   # [L, row pair, col]: union of the pair
                if k == 256:
                    fpair_entries += int(ph.sum())
                cpp = torch.nn.functional.pad(ph.reshape(L, 128).int(), (0, 0, 0, n * k - L)).view(n, k, 8, 16).sum(1)
                for (hh_, ww_) in PSHAPES:
                    m = cpp.view(n, 8 // hh_, hh_, 16 // ww_, ww_).amax(dim=(2, 4))
                    fpair_steps[(k, (hh_, ww_))] += int(m.sum())
                cpix = torch.nn.functional.pad(fh.int(), (0, 0, 0, n * k - L)).view(n, k, 16, 16).sum(1)   # [chunk, y, x]
                for (hh_, ww_) in SHAPES:
                    m = cpix.view(n, 16 // hh_, hh_, 16 // ww_, ww_).amax(dim=(2, 4))
                    fshape[(k, (hh_, ww_))] += int(m.sum())
    print(f"tiles sampled {len(sample)}/{len(occupied)}  R={R}")
    print(f"instances {inst_total}: before the tile's last contributor {inst_reached}, alpha>=1/255 somewhere in tile {inst_hit}, "
          f"blended by >=1 pixel {inst_contrib}")
    print(f"(pixel,G) contributing pairs      {tot_pix}")
    print(f"(block,G) pairs                   {tot_pairs}   -> pixel efficiency {tot_pix / max(1, tot_pairs * 8):.3f}")
    print(f"warp steps, current mapping       {tot_cur}   (lane efficiency {tot_pairs / 8 / tot_cur:.3f})")
    print(f"warp steps, length-sorted mapping {tot_sorted}   ({tot_pairs / 8 / tot_sorted:.3f})")
    print(f"warp steps, perfect balance       {tot_ideal}")
    for k in CH:
        print(f"backward lock-step window {k:5d}: steps {bsteps[k][0]} (eff {tot_pairs / 8 / bsteps[k][0]:.3f})   "
              f"sorted {bsteps[k][1]} (eff {tot_pairs / 8 / bsteps[k][1]:.3f})")
    for (bw, bh_) in ALT:
        for k in (256, 512):
            pairs, steps = alt[(bw, bh_, k)]
            lpb = bw * bh_ // 2
            print(f"backward blocks {bw}x{bh_} ({lpb} lanes/block, {32 // lpb} blocks/warp) window {k}: (block,G) pairs {pairs}, pixel eff "
                  f"{tot_pix / max(1, alt_pix[(bw, bh_)]):.3f}, warp steps {steps} (lane eff {pairs * lpb / 32 / max(1, steps):.3f}), "
                  f"pixel-pairs evaluated per contributing pixel {steps * 16 / max(1, tot_pix) * 2:.2f}")
    for k in CH:
        print(f"forward  lock-step window {k:5d}: warp steps {fsteps[k]} (lane eff {fpairs / 32 / fsteps[k]:.3f})")
    print(f"forward pixel entries {fpairs}; pixel-PAIR entries {fpair_entries} ({fpair_entries / fpairs:.3f} of single)")
    for (k, sh), v in fpair_steps.items():
        tag = "   <- product" if (k, sh) == (384, (2, 16)) else ""
        print(f"forward PAIR window {k} warp {sh[0]} row pairs x {sh[1]} cols: warp steps {v} (lane eff {fpair_entries / 32 / v:.3f}){tag}")
    for (k, sh), v in fshape.items():
        print(f"forward window {k} warp shape {sh[0]}x{sh[1]}: warp steps {v} (lane eff {fpairs / 32 / v:.3f})")


if __name__ == "__main__":
    main()
