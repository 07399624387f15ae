"""`simple_knn._C.distCUDA2` on the H100 (csrc/gh_knn.cu): bit-identical to the CPU oracle (oracle/knn_oracle.c) on
every test distribution, also at 4 M points of the head-like cloud with outliers; reproducible bit for bit, with and
without `torch.use_deterministic_algorithms`, and from a side stream; and driven by the reference's own
`GaussianModel.create_from_pcd`, imported unmodified."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

import _knn_cases as K

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(K.ROOT, "oracle"))
import knn_oracle  # noqa: E402
import ref_python  # noqa: E402

from simple_knn._C import distCUDA2  # noqa: E402


def _run(pts: np.ndarray, device) -> np.ndarray:
    out = distCUDA2(torch.from_numpy(pts).to(device))
    assert out.dtype == torch.float32 and out.shape == (pts.shape[0],) and out.device == device
    return out.cpu().numpy()


@pytest.mark.parametrize("name", list(K.CASES))
def test_bit_identical_to_the_oracle(cuda_device, name):
    gen, _, n_gpu = K.CASES[name]
    pts = gen(n_gpu, 5)
    K.assert_same_bits(_run(pts, cuda_device), knn_oracle.mean_dist3(pts), name)


@pytest.mark.parametrize("P", range(6))
def test_small_clouds(cuda_device, P):
    from gaussianhaircut_b200 import _capi
    pts = K.tiny(P, 7)
    n0 = _capi.load().gh_kernel_launch_count()
    got = _run(pts, cuda_device)
    if P == 0:
        assert _capi.load().gh_kernel_launch_count() == n0, "P = 0 launched a kernel"
    K.assert_same_bits(got, knn_oracle.mean_dist3(pts), f"P={P}")
    assert np.all(got == np.inf) if P <= 3 else np.all(np.isfinite(got))


def test_head_shell_at_4m(cuda_device):
    pts = K.head_shell(4_000_000, 9)
    K.assert_same_bits(_run(pts, cuda_device), knn_oracle.mean_dist3(pts), "b at 4M")


def test_one_point_all_zero(cuda_device):
    assert np.all(_run(K.one_point(10_000), cuda_device) == 0)


def test_reproducible_across_runs_modes_and_streams(cuda_device):
    pts = torch.from_numpy(K.head_shell(1_000_000, 4)).to(cuda_device)
    ref = distCUDA2(pts).cpu().numpy()
    K.assert_same_bits(distCUDA2(pts).cpu().numpy(), ref, "second call")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        K.assert_same_bits(distCUDA2(pts).cpu().numpy(), ref, "deterministic mode")
    finally:
        torch.use_deterministic_algorithms(prev)
    side = torch.cuda.Stream(cuda_device)
    side.wait_stream(torch.cuda.current_stream(cuda_device))
    with torch.cuda.stream(side):
        busy = torch.randn(4096, 4096, device=cuda_device)
        out = distCUDA2(pts)
        busy = busy @ busy
    side.synchronize()
    K.assert_same_bits(out.cpu().numpy(), ref, "side stream")


def test_input_conventions(cuda_device):
    pts = K.uniform(50_000, 6)
    want = knn_oracle.mean_dist3(pts)
    wide = torch.zeros(pts.shape[0], 5, device=cuda_device)
    wide[:, 1:4] = torch.from_numpy(pts).to(cuda_device)
    view = wide[:, 1:4]                                   # non-contiguous rows: made contiguous
    assert not view.is_contiguous()
    K.assert_same_bits(distCUDA2(view).cpu().numpy(), want, "strided")
    leaf = torch.from_numpy(pts).to(cuda_device).requires_grad_(True)
    out = distCUDA2(leaf)
    assert not out.requires_grad
    K.assert_same_bits(out.cpu().numpy(), want, "requires_grad input")
    for bad in (torch.zeros(10, 2, device=cuda_device), torch.zeros(10, 3, dtype=torch.float64, device=cuda_device),
                torch.zeros(3, device=cuda_device)):
        with pytest.raises(RuntimeError):
            distCUDA2(bad)
    with pytest.raises(RuntimeError, match="no CPU path"):
        distCUDA2(torch.from_numpy(pts))


def _reference_gaussian_model_module():
    """The reference's scene/gaussian_model.py, loaded unmodified under a private name with `simple_knn` bound to this
    repository's package (whatever an earlier test left in sys.modules)."""
    src = ref_python.ref_src_dir()
    if src is None:
        pytest.skip("reference Python sources not staged (python oracle/build_ref.py in the build container)")
    ref_python.install_stubs()
    for p in (src, K.ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    import simple_knn as pkg
    import simple_knn._C as mine
    saved = {k: sys.modules.get(k) for k in ("simple_knn", "simple_knn._C")}
    sys.modules["simple_knn"], sys.modules["simple_knn._C"] = pkg, mine
    try:
        spec = importlib.util.spec_from_file_location("gh_ref_gaussian_model_knn", os.path.join(src, "scene", "gaussian_model.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v
    return mod, mine


def test_reference_create_from_pcd_runs_on_the_drop_in(cuda_device):
    mod, mine = _reference_gaussian_model_module()
    from gaussianhaircut_b200.knn import mean_dist3
    assert mod.distCUDA2 is mine.distCUDA2 is mean_dist3
    from utils.graphics_utils import BasicPointCloud
    pts = K.head_shell(100_000, 8)
    rng = np.random.default_rng(8)
    pcd = BasicPointCloud(points=pts, colors=rng.random((pts.shape[0], 3)), normals=np.zeros_like(pts))
    gm = mod.GaussianModel(3)
    gm.create_from_pcd(pcd, 1.0)                          # the reference's method, as shipped
    torch.cuda.synchronize()
    dist2 = torch.clamp_min(torch.from_numpy(knn_oracle.mean_dist3(pts)).to(gm._scaling.device), 0.0000001)
    want = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
    assert gm._scaling.shape == (pts.shape[0], 3)
    assert torch.equal(gm._scaling.detach(), want)
    assert torch.equal(gm._xyz.detach().cpu(), torch.from_numpy(pts))
