"""CPU tests of the captured strand iteration: the two capturable strand entry points refuse bad arguments (row counts,
flag words, missing tan fov or status pointer, the capacity range, debug mode, the stage timer) before they launch
anything; the capture key of graphs.CapturedStrandStep and what changes it; the checks of the prior's `_dirs` gradient."""
import ctypes as C
import types

import pytest
import torch

import _util  # noqa: F401  (puts the repository root on sys.path)


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import _capi
    return _capi.load()


F = C.c_void_p(4096)        # never dereferenced: every call below is refused on the host


def _flags():
    from gaussianhaircut_b200 import projection as pj
    return pj.encode_flags(pj.HEAD_PRECOMP), pj.encode_flags(pj.HAIR_STRANDS)


def _forward(lib, n_head=64, S=8, L=16, tan=F, status=F, capacity=1024, debug=0, head_flags=None, flags=None):
    hf, sf = _flags()
    hf = hf if head_flags is None else head_flags
    sf = sf if flags is None else flags
    return lib.gh_hair_strands_forward_binned_capturable(
        n_head, S, L, 64, 48, F, F, F, F, F, F, hf, 1e-12, F, F, F, F, F, F, sf, 1e-7, F, F, F, tan, 1.0, 3, F,
        F, F, F, F, F, F, F, F, F, capacity, status, None, debug, None)


def _backward(lib, n_head=64, S=8, L=16, tan=F, debug=0, flags=None):
    sf = _flags()[1] if flags is None else flags
    return lib.gh_hair_strands_backward_capturable(
        n_head, S, L, 64, 48, F, F, F, F, F, F, sf, 1e-7, F, F, F, tan, 1.0, 3, F, F, F, F, F, F, F, None, debug, None)


CASES = [
    (lambda lib: _forward(lib, tan=None), "tan_fov"),
    (lambda lib: _forward(lib, status=None), "status"),
    (lambda lib: _forward(lib, capacity=-1), "capacity must lie in"),
    (lambda lib: _forward(lib, capacity=1 << 32), "capacity must lie in"),
    (lambda lib: _forward(lib, debug=1), "debug"),
    (lambda lib: _forward(lib, n_head=-1), "n_head must not be negative"),
    (lambda lib: _forward(lib, S=-2), "S and L must be non-negative"),
    (lambda lib: _forward(lib, S=1 << 16, L=1 << 15), "S * L overflows int"),
    (lambda lib: _forward(lib, n_head=(1 << 31) - 100, S=8, L=16), "n_head + S * L overflows int"),
    (lambda lib: _forward(lib, n_head=0, S=0, L=16), "nothing to render"),
    (lambda lib: _forward(lib, n_head=0, S=8, L=0), "nothing to render"),
    (lambda lib: _forward(lib, head_flags=_flags()[0] | (1 << 10)), "head_flags must not set the strand bit"),
    (lambda lib: _forward(lib, flags=_flags()[1] & ~(1 << 10)), "flags must set the strand bit"),
    (lambda lib: _backward(lib, tan=None), "tan_fov"),
    (lambda lib: _backward(lib, debug=1), "debug"),
    (lambda lib: _backward(lib, n_head=-1), "n_head must not be negative"),
    (lambda lib: _backward(lib, S=0), "S and L must be positive"),
    (lambda lib: _backward(lib, S=1 << 16, L=1 << 15), "S * L overflows int"),
    (lambda lib: _backward(lib, flags=_flags()[1] & ~(1 << 10)), "flags must set the strand bit"),
]


@pytest.mark.parametrize("call, message", CASES)
def test_strand_capturable_entry_points_refuse_bad_arguments_before_any_launch(lib, call, message):
    from gaussianhaircut_b200 import _capi
    n0 = lib.gh_kernel_launch_count()
    assert call(lib) == _capi.GH_E_INVALID_ARG
    assert message in lib.gh_last_error().decode()
    assert lib.gh_kernel_launch_count() == n0


@pytest.mark.parametrize("call", [lambda lib: _forward(lib), lambda lib: _backward(lib)])
def test_strand_capturable_entry_points_refuse_the_stage_timer(lib, call):
    from gaussianhaircut_b200 import _capi
    n0 = lib.gh_kernel_launch_count()
    lib.gh_stage_timing_enable(1)
    try:
        assert call(lib) == _capi.GH_E_INVALID_ARG
        assert "stage timer" in lib.gh_last_error().decode()
    finally:
        lib.gh_stage_timing_enable(0)
    assert lib.gh_kernel_launch_count() == n0


def _fake(S=6, L=5, n_head=7, sh=3):
    """(pc, pc_hair, optimizer) with CPU tensors: the attributes strand_capture_key reads."""
    pc = types.SimpleNamespace(xyz_precomp=torch.zeros(n_head, 3), scaling_precomp=torch.zeros(n_head, 3),
                               rotation_precomp=torch.zeros(n_head, 4), opacity_precomp=torch.zeros(n_head, 1),
                               shs_view=torch.zeros(n_head, 3, 16))
    hair = types.SimpleNamespace(_dirs=torch.zeros(S, L, 3), _features_dc=torch.zeros(S * L, 1, 3),
                                 _features_rest=torch.zeros(S * L, 15, 3), _orient_conf=torch.zeros(S * L, 1),
                                 pts_origins=torch.zeros(S, 1, 3), scale=torch.ones(1), active_sh_degree=sh)
    params = [hair._dirs, hair._features_dc, hair._features_rest, hair._orient_conf]
    opt = types.SimpleNamespace(param_groups=[{"params": [p]} for p in params],
                                state={p: {"exp_avg": torch.zeros_like(p), "exp_avg_sq": torch.zeros_like(p)} for p in params})
    return pc, hair, opt


def test_strand_capture_key():
    from gaussianhaircut_b200.graphs import strand_capture_key as key
    pc, hair, opt = _fake()
    k = key(pc, hair, opt, 64, 48)
    assert k[:3] == (6, 5, 7)
    assert key(pc, hair, opt, 64, 48) == k
    assert key(pc, hair, opt, 65, 48) != k and key(pc, hair, opt, 64, 47) != k
    assert key(pc, hair, opt, 64, 48, use_gt_orient_conf=False) != k
    assert key(pc, hair, opt, 64, 48, train_orient_conf=False) != k
    assert key(pc, hair, opt, 64, 48, dirs_grad=True) != k
    assert key(None, hair, opt, 64, 48)[2] == 0                     # hair only
    hair.active_sh_degree = 2
    assert key(pc, hair, opt, 64, 48) != k
    hair.active_sh_degree = 3
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(not prev)
    try:
        assert key(pc, hair, opt, 64, 48) != k
    finally:
        torch.use_deterministic_algorithms(prev)
    assert key(pc, hair, opt, 64, 48) == k
    # storage: origins, thickness, a moment, the head block (a new *_precomp tensor rebuilds the cached block)
    for attr in ("pts_origins", "scale"):
        old = getattr(hair, attr)
        setattr(hair, attr, old.clone())
        assert key(pc, hair, opt, 64, 48) != k
        setattr(hair, attr, old)
    assert key(pc, hair, opt, 64, 48) == k
    p = opt.param_groups[0]["params"][0]
    old = opt.state[p]["exp_avg_sq"]
    opt.state[p]["exp_avg_sq"] = torch.zeros_like(p)
    assert key(pc, hair, opt, 64, 48) != k
    opt.state[p]["exp_avg_sq"] = old
    pc.xyz_precomp = pc.xyz_precomp.clone()
    assert key(pc, hair, opt, 64, 48)[:10] == k[:10] and key(pc, hair, opt, 64, 48) != k
    # a different strand model size
    pc2, hair2, opt2 = _fake(S=9, L=4, n_head=3)
    assert key(pc2, hair2, opt2, 64, 48)[:3] == (9, 4, 3)


def test_dirs_grad_checks():
    from gaussianhaircut_b200.graphs import check_dirs_grad
    dirs = torch.zeros(6, 5, 3)
    check_dirs_grad(torch.zeros(6, 5, 3), dirs)
    for bad, msg in ((torch.zeros(30, 3), "shape of _dirs"), (torch.zeros(6, 5, 4), "shape of _dirs"),
                     (torch.zeros(5, 5, 3), "shape of _dirs"), (torch.zeros(6, 5, 3, dtype=torch.float64), "float32"),
                     ([0.0] * 90, "shape of _dirs")):
        with pytest.raises(RuntimeError, match=msg):
            check_dirs_grad(bad, dirs)
