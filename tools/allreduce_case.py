"""All-reduce of the gradient arena alone: NCCL vs gh_allreduce_p2p (peer ld/st, NVLS multimem), with a sweep over
the kernel's launch tunables (GH_ALLREDUCE_THREADS / _CTAS_PER_SM / _UNROLL, read per call).
   python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/allreduce_case.py [P] [--sweep]"""
import itertools, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch, torch.distributed as dist
from gaussianhaircut_b200 import dist as gd, _C
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = torch.device(f"cuda:{int(os.environ['LOCAL_RANK'])}")
torch.cuda.set_device(dev)
dist.init_process_group("nccl", device_id=dev)
argv = [a for a in sys.argv[1:] if not a.startswith("--")]
P = int(argv[0]) if argv else 500_000
sweep = "--sweep" in sys.argv
n = _C.trainable_floats(P)          # what travels per step in the native call shape (21 floats per Gaussian)
reps = 30

def timed(fn):
    for _ in range(5):
        fn()
    dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / reps], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item() * 1000

x = torch.randn(n, device=dev)
res = {"nccl": timed(lambda: dist.all_reduce(x))}
table = []
for name, mc in (("peer ld/st", False), ("multimem", True)):
    par = gd.PeerAllReduce(_C.arena_floats(P), dev, use_multicast=mc)
    if mc and not par.multicast:
        continue
    par.buffer.normal_()
    for k in ("GH_ALLREDUCE_THREADS", "GH_ALLREDUCE_CTAS_PER_SM", "GH_ALLREDUCE_UNROLL"):
        os.environ.pop(k, None)
    res[name] = timed(lambda: par.all_reduce(n_floats=n))
    assert par.ok()
    if sweep:
        if mc:      # the NVLS path likes few requests in flight: sweep downwards too (grid smaller than the SM count)
            grid = itertools.product((64, 128, 256, 512), (1, 2), (1, 2, 4, 8), (33, 66, 132, 1 << 20))
        else:
            grid = itertools.product((128, 256, 512), (1, 2, 4), (1,), (1 << 20,))
        for th, cps, un, mx in grid:
            if mx != 1 << 20 and cps > 1:
                continue
            os.environ.update(GH_ALLREDUCE_THREADS=str(th), GH_ALLREDUCE_CTAS_PER_SM=str(cps), GH_ALLREDUCE_UNROLL=str(un),
                              GH_ALLREDUCE_MAX_CTAS=str(mx))
            t = timed(lambda: par.all_reduce(n_floats=n))
            table.append({"path": name, "threads": th, "ctas_per_sm": cps, "unroll": un, "max_ctas": mx, "us": t})
        for k in ("GH_ALLREDUCE_THREADS", "GH_ALLREDUCE_CTAS_PER_SM", "GH_ALLREDUCE_UNROLL", "GH_ALLREDUCE_MAX_CTAS"):
            os.environ.pop(k, None)
    assert par.ok()
if rank == 0:
    mb = n * 4 / 1e6
    print(f"all-reduce of {mb:.0f} MB over {world} GPUs: " + ", ".join(f"{k} {v:.1f} us ({2 * (world - 1) / world * mb / v * 1e3:.0f} GB/s bus)" for k, v in res.items()))
    if sweep:
        for path in ("peer ld/st", "multimem"):
            rows = sorted((r for r in table if r["path"] == path), key=lambda r: r["us"])
            for r in rows[:6]:
                print(f"  {path}: threads {r['threads']} ctas/SM {r['ctas_per_sm']} unroll {r['unroll']} max CTAs {r['max_ctas']}: {r['us']:.1f} us")
        print(json.dumps({"world": world, "mb": mb, "defaults": res, "sweep": table}))
dist.destroy_process_group()
