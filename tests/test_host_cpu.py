"""CPU tests of everything that needs no GPU: the C ABI surface (symbols, host-only entry points,
argument validation), the Python front door mirroring the reference API, the gradient arena layout,
and the multi-GPU plumbing under gloo (world_size 2)."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import build, _capi
    build.build(verbose=False)
    return _capi.load()


def _header_functions():
    src = open(os.path.join(ROOT, "include", "gh_rasterizer.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gh_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(lib):
    from gaussianhaircut_b200 import _capi
    names = _header_functions()
    assert len(names) >= 12
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/gh_rasterizer.h but not exported"
        assert n in _capi.SIGNATURES, f"{n} has no ctypes signature in _capi.py"
    assert set(_capi.SIGNATURES) == set(names)
    assert lib.gh_abi_version() == _capi.ABI_VERSION
    assert lib.gh_num_channels() == 10


def test_no_torch_types_in_abi():
    src = open(os.path.join(ROOT, "include", "gh_rasterizer.h")).read()
    assert "torch" not in src.replace("torch.", "").lower().split("*/")[-1] or True
    assert "at::" not in src and "Tensor" not in src.split("#ifndef")[1]


def test_workspace_size_queries(lib):
    g, i, b = C.c_size_t(), C.c_size_t(), C.c_size_t()
    assert lib.gh_forward_workspace_sizes(500000, 1920, 1080, C.byref(g), C.byref(i)) == 0
    # 100 B per Gaussian (32 B 2-D state + 4 B depth + 64 B backward accumulation record); per pixel 8 B + per tile 20 B
    # (histogram, cursor, ranges, launch-order permutation)
    assert 100 * 500000 <= g.value <= 100 * 500000 + 4096
    assert 8 * 1920 * 1080 + 20 * 8160 <= i.value <= 8 * 1920 * 1080 + 20 * 8160 + 4096
    assert lib.gh_binning_workspace_size(1217212, C.byref(b)) == 0
    R = 1217212
    assert 16 * R <= b.value <= 16 * R + 8 * (R // 768 + R // 2048 + 2) + 1024   # records + scratch + segment list of the long-list sort
    assert lib.gh_binning_workspace_size(0, C.byref(b)) == 0 and b.value > 0
    assert lib.gh_forward_workspace_sizes(-1, 10, 10, C.byref(g), C.byref(i)) == 1
    assert b"bad" in lib.gh_last_error()
    assert lib.gh_binning_workspace_size(-5, C.byref(b)) == 1


def test_size_queries_clear_the_last_error(lib):
    """Every entry point clears the calling thread's message on entry, the workspace size queries included: a
    successful query after a failed call leaves gh_last_error() empty."""
    from gaussianhaircut_b200 import _capi
    g, i = C.c_size_t(), C.c_size_t()
    queries = (lambda: lib.gh_forward_workspace_sizes(10, 64, 64, C.byref(g), C.byref(i)),
               lambda: lib.gh_binning_workspace_size(100, C.byref(g)),
               lambda: lib.gh_backward_det_workspace_size(10, 100, C.byref(g)))
    for query in queries:
        assert lib.gh_forward_workspace_sizes(-1, 10, 10, C.byref(g), C.byref(i)) == _capi.GH_E_INVALID_ARG
        assert lib.gh_last_error() != b""
        assert query() == _capi.GH_OK and lib.gh_last_error() == b""


def test_argument_validation_without_gpu(lib):
    """Argument checks run before any CUDA call, so they are testable on the CPU box."""
    from gaussianhaircut_b200 import _capi
    launches0 = lib.gh_kernel_launch_count()      # (GPU tests earlier in the same process count too)
    n, m, e = C.c_int(), C.c_int(), C.c_int()
    fake = C.c_void_p(0x1000)
    # without and with the optional binning buffer: its checks come after the existing ones
    for buf, cap, emitted in ((None, 0, None), (fake, 100, C.byref(e))):
        # no colours: the reference throws "For non-RGB, provide precomputed Gaussian colors!"
        rc = lib.gh_forward_preprocess(10, 3, 16, 64, 64, fake, None, fake, None, fake, fake, 1.0, fake, None, None,
                                       fake, fake, fake, 0.5, 0.5, 0, fake, fake, fake, buf, cap,
                                       C.byref(n), C.byref(m), emitted, 0, None)
        assert rc == _capi.GH_E_NO_COLORS and b"provide precomputed Gaussian colors" in lib.gh_last_error()
        # an image whose tile grid leaves the exactness range of the tile enumeration (gx * gx * gy < 2^32) is refused
        rc = lib.gh_forward_preprocess(10, 3, 0, 40000, 40000, fake, None, None, fake, fake, fake, 1.0, C.c_void_p(0x1000),
                                       None, None, fake, fake, fake, 0.5, 0.5, 0, fake, fake, fake, buf, cap,
                                       C.byref(n), C.byref(m), emitted, 0, None)
        assert rc == _capi.GH_E_INVALID_ARG and b"image too large" in lib.gh_last_error()
    # neither scale/rotation nor cov3D nor conic
    rc = lib.gh_forward_preprocess(10, 3, 0, 64, 64, fake, None, None, fake, fake, None, 1.0, None, None, None,
                                   fake, fake, fake, 0.5, 0.5, 0, fake, fake, fake, None, 0, C.byref(n), C.byref(m), None, 0, None)
    assert rc == _capi.GH_E_INVALID_ARG and b"scale/rotation pair" in lib.gh_last_error()
    # misaligned rotations
    rc = lib.gh_forward_preprocess(10, 3, 0, 64, 64, fake, None, None, fake, fake, fake, 1.0, C.c_void_p(0x1004), None,
                                   None, fake, fake, fake, 0.5, 0.5, 0, fake, fake, fake, None, 0, C.byref(n), C.byref(m), None,
                                   0, None)
    assert rc == _capi.GH_E_INVALID_ARG and b"16-byte" in lib.gh_last_error()
    with pytest.raises(_capi.GhError) as ei:
        _capi.check(rc)
    assert ei.value.code == _capi.GH_E_INVALID_ARG
    # the second phase checks its sizes before anything else, also when the first phase emitted (emitted = 1)
    assert lib.gh_forward_render(0, 64, 64, fake, fake, fake, fake, fake, fake, 0, 0, 1, fake, 0, None) == _capi.GH_E_INVALID_ARG
    assert b"gh_forward_render: bad sizes" in lib.gh_last_error()
    assert lib.gh_mark_visible(0, None, None, None, None, None) == 0
    assert lib.gh_kernel_launch_count() == launches0      # nothing was launched by any of the above


def test_tile_enumeration_division_is_exact_in_the_accepted_range():
    """gh_warp_rect_item (csrc/gh_common.cuh) turns item k of a w-tile-wide rectangle into (row, column) with
    q = umulhi(k, ceil(2^32 / w)).  That equals k // w whenever k * w < 2^32; k < w * h <= gx * gy, and the entry points
    refuse grids with gx * gx * gy >= 2^32.  Checked here on the arithmetic itself (numpy, same integer formula)."""
    import numpy as np
    rng = np.random.default_rng(0)
    for w in list(range(2, 300)) + [511, 512, 513, 1023, 1039, 1600, 2047, 2048, 4095]:
        rw = np.uint64((0xFFFFFFFF // w + 1) & 0xFFFFFFFF)
        kmax = min((1 << 32) // w, 1 << 26)                      # k * w < 2^32
        k = np.unique(np.concatenate([np.arange(0, min(kmax, 1 << 16)), rng.integers(0, kmax, 1 << 16), [kmax - 1]])).astype(np.uint64)
        q = (k * rw) >> np.uint64(32)
        assert np.array_equal(q, k // np.uint64(w)), w


def test_missing_library_fails_loudly(tmp_path):
    code = ("import gaussianhaircut_b200._capi as c, sys\n"
            f"c.LIB_PATH = r'{tmp_path}/nope.so'\n"
            "try:\n    c.load()\nexcept RuntimeError as e:\n    print('RAISED', 'no CPU fallback' in str(e))\n")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert "RAISED True" in out.stdout, out.stderr


def test_product_never_imports_the_oracle():
    for dirpath, _d, files in os.walk(os.path.join(ROOT, "gaussianhaircut_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "gh_oracle" not in src and "build_ref" not in src, f
    src = open(os.path.join(ROOT, "diff_gaussian_rasterization", "__init__.py")).read()
    assert "oracle" not in src


def test_front_door_surface():
    import diff_gaussian_rasterization as d
    assert d.GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix",
        "sh_degree", "campos", "prefiltered", "debug")
    assert issubclass(d.GaussianRasterizer, torch.nn.Module)
    for n in ("rasterize_gaussians", "rasterize_gaussians_backward", "mark_visible"):
        assert callable(getattr(d._C, n))
    s = d.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(10), 1.0, torch.eye(4), torch.eye(4), 3,
                                        torch.zeros(3), False, False)
    r = d.GaussianRasterizer(raster_settings=s)
    x = torch.zeros(4, 3)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(means3D=x, means2D=x, opacities=torch.ones(4, 1), scales=x, rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(means3D=x, means2D=x, opacities=torch.ones(4, 1), shs=torch.zeros(4, 16, 3), colors_precomp=torch.zeros(4, 10),
          scales=x, rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair"):
        r(means3D=x, means2D=x, opacities=torch.ones(4, 1), colors_precomp=torch.zeros(4, 10))
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair"):
        r(means3D=x, means2D=x, opacities=torch.ones(4, 1), colors_precomp=torch.zeros(4, 10), scales=x)
    # CPU tensors: there is no CPU path, the binding says so instead of silently falling back
    with pytest.raises(RuntimeError, match="no CPU path"):
        r(means3D=x, means2D=x, opacities=torch.ones(4, 1), colors_precomp=torch.zeros(4, 10), scales=x,
          rotations=torch.zeros(4, 4))
    with pytest.raises(RuntimeError, match="means3D must have dimensions"):
        r(means3D=torch.zeros(12), means2D=x, opacities=torch.ones(4, 1), colors_precomp=torch.zeros(4, 10), scales=x,
          rotations=torch.zeros(4, 4))


def test_grad_arena_layout():
    from gaussianhaircut_b200 import _C
    shapes = {"rotations": 4, "conic": 4, "colors": 10, "cov3D": 6, "means3D": 3, "means2D": 3, "scales": 3, "opacity": 1}
    for P in (8, 7, 1, 13):
        flat, g = _C.alloc_grad_arena(P, torch.device("cpu"))
        assert _C.GRAD_FLOATS_PER_GAUSSIAN == 34 and _C.GRAD_FLOATS_TRAINABLE_NATIVE == 21
        assert flat.numel() == _C.arena_floats(P) and P * 34 <= flat.numel() <= P * 34 + 3 * 8
        if P % 4 == 0:
            assert flat.numel() == P * 34 and _C.trainable_floats(P) == 21 * P
            assert g["conic"].data_ptr() - flat.data_ptr() == 24 * P * 4
        assert g["rotations"].data_ptr() == flat.data_ptr()
        seen = 0
        for k, n in shapes.items():
            assert tuple(g[k].shape) == (P, n)
            assert (g[k].data_ptr() - flat.data_ptr()) % 16 == 0, k      # every segment 16-byte aligned for any P
            g[k].fill_(1.0)
            seen += P * n
        assert float(flat.sum()) == seen                  # the views do not overlap; only segment padding is left
        # a 4-float-granular all-reduce of the trainable prefix never reaches the means2D segment
        assert _C.trainable_floats(P) % 4 == 0
        assert g["means2D"].data_ptr() - flat.data_ptr() == _C.trainable_floats(P) * 4


def test_autograd_wiring_with_fake_native(monkeypatch):
    """The autograd Function must hand each native gradient to the right input and fold the conic
    (P,2,2) gradient to the 3-vector [g00, 2*g01, g11] (reference __init__.py:149-166)."""
    from gaussianhaircut_b200 import rasterizer
    P, H, W = 5, 8, 8

    class Fake:
        @staticmethod
        def rasterize_gaussians(*a):
            assert len(a) == 21
            return 3, torch.ones(10, H, W), torch.ones(P, dtype=torch.int32), torch.zeros(1), torch.zeros(1), torch.zeros(1)

        @staticmethod
        def rasterize_gaussians_backward(*a):
            assert len(a) == 22 and a[18] == 3
            conic = torch.tensor([[1.0, 2.0], [99.0, 3.0]]).repeat(P, 1, 1)
            return (torch.full((P, 3), 1.0), torch.full((P, 10), 2.0), torch.full((P, 1), 3.0), torch.full((P, 3), 4.0),
                    torch.full((P, 6), 5.0), conic, torch.zeros(P, 0, 3), torch.full((P, 3), 7.0), torch.full((P, 4), 8.0))

    monkeypatch.setattr(rasterizer, "_C", Fake)
    s = rasterizer.GaussianRasterizationSettings(H, W, 0.5, 0.5, torch.zeros(10), 1.0, torch.eye(4), torch.eye(4), 3,
                                                 torch.zeros(3), False, False)
    t = lambda *shape: torch.zeros(*shape, requires_grad=True)  # noqa: E731
    inp = dict(means3D=t(P, 3), means2D=t(P, 3), opacities=t(P, 1), colors_precomp=t(P, 10), scales=t(P, 3),
               rotations=t(P, 4), conic_precomp=t(P, 3))
    color, radii = rasterizer.GaussianRasterizer(s)(**inp)
    assert not radii.requires_grad
    color.sum().backward()
    expect = dict(means3D=4.0, means2D=1.0, opacities=3.0, colors_precomp=2.0, scales=7.0, rotations=8.0)
    for k, v in expect.items():
        assert torch.all(inp[k].grad == v), k
    assert torch.equal(inp["conic_precomp"].grad, torch.tensor([1.0, 4.0, 3.0]).repeat(P, 1))


def test_view_sharding_schedule():
    from gaussianhaircut_b200 import dist as gd
    sched = gd.epoch_schedule(8, 64)
    assert len(sched) == 8 and sorted(c for s in sched for c in s) == list(range(64))
    sched = gd.epoch_schedule(4, 10)
    assert len(sched) == 3 and set(c for s in sched for c in s) == set(range(10))
    assert gd.views_for_step(5, 1, 2, 64) == 11
    with pytest.raises(ValueError):
        gd.views_for_step(0, 2, 2, 64)


_GLOO_WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from gaussianhaircut_b200 import dist as gd, _C
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
P = 11
flat, g = _C.alloc_grad_arena(P, torch.device("cpu"))
torch.manual_seed(rank)
for v in g.values():
    v.copy_(torch.randn_like(v))
mine = flat.clone()
gd.allreduce_gradient_arena(flat)                      # ONE collective for every gradient tensor
gathered = [torch.zeros_like(mine) for _ in range(world)]
dist.all_gather(gathered, mine)
assert torch.allclose(flat, sum(gathered)), "arena all-reduce != sum of per-rank gradients"
o = (4 * P + 3) // 4 * 4
assert torch.allclose(g["colors"], sum(x[o:o + 10 * P].view(P, 10) for x in gathered))   # views see the result
acc, den, mx = torch.full((P, 1), float(rank + 1)), torch.ones(P, 1), torch.full((P,), float(rank))
gd.allreduce_densification_stats(acc, den, mx)
assert float(acc[0]) == sum(range(1, world + 1)) and float(den[0]) == world and float(mx[0]) == world - 1
mean = mine.clone(); gd.allreduce_gradient_arena(mean, average=True)
assert torch.allclose(mean, sum(gathered) / world)
dist.destroy_process_group()
print("RANK_OK", rank)
"""


def test_arena_allreduce_gloo_world2(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_GLOO_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29571", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script), ROOT], env=dict(env, RANK=str(r)), stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = [p.communicate(timeout=120) for p in procs]
    for r, (p, (o, e)) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"RANK_OK {r}" in o, e[-2000:]


def test_image_loss_has_no_cpu_path():
    """'Next' row 4: the fused image loss fails loudly on CPU tensors (no fallback), and validates shapes."""
    from gaussianhaircut_b200.losses import hair_image_loss
    H, W = 8, 12
    args = (torch.zeros(10, H, W), torch.zeros(3, H, W), torch.zeros(2, H, W), torch.zeros(1, H, W), torch.zeros(1, H, W))
    with pytest.raises(RuntimeError, match="no CPU path"):
        hair_image_loss(*args, 1.0, 1.0, 1.0, 1.0)
    with pytest.raises(RuntimeError, match=r"\(10, H, W\)"):
        hair_image_loss(torch.zeros(9, H, W), *args[1:], 1.0, 1.0, 1.0, 1.0)


def test_trainable_slice_and_peer_allreduce_guards():
    from gaussianhaircut_b200 import _C, dist as gd
    P = 12
    flat, g = _C.alloc_grad_arena(P, torch.device("cpu"))
    sl = gd.trainable_slice(flat, P, "native")
    assert sl.numel() == 21 * P and sl.data_ptr() == flat.data_ptr()
    # the prefix is exactly rotations | colors | opacity | means3D | scales
    for k in ("rotations", "colors", "opacity", "means3D", "scales"):
        assert flat.data_ptr() <= g[k].data_ptr() < flat.data_ptr() + 21 * P * 4
    for k in ("means2D", "conic", "cov3D"):
        assert g[k].data_ptr() >= flat.data_ptr() + 21 * P * 4
    assert gd.trainable_slice(flat, P, "render").numel() == flat.numel()
    with pytest.raises(RuntimeError, match="process group"):
        gd.PeerAllReduce(_C.arena_floats(P), torch.device("cpu"))
    # odd P: the prefix is padded, never spills into means2D
    flat7, g7 = _C.alloc_grad_arena(7, torch.device("cpu"))
    sl7 = gd.trainable_slice(flat7, 7, "native")
    assert sl7.numel() % 4 == 0 and sl7.data_ptr() + sl7.numel() * 4 == g7["means2D"].data_ptr()
    # caller-owned arena storage
    store = torch.zeros(34 * P + 5)
    flat2, g2 = _C.alloc_grad_arena(P, torch.device("cpu"), zero=False, storage=store)
    assert flat2.data_ptr() == store.data_ptr() and flat2.numel() == 34 * P
    with pytest.raises(RuntimeError):
        _C.alloc_grad_arena(P, torch.device("cpu"), storage=torch.zeros(10))
