"""CPU tests of the captured latent strand iteration: the two capturable segment entry points refuse bad arguments
(row counts, flag words, missing tan fov, status, xyz or dirs pointer, debug mode, the stage timer) before they launch
anything; the capture key of graphs.CapturedLatentStrandStep and what changes it; a backward that reaches the
gradients of an earlier step raises; making the optimizer optional in the shared base class leaves the other two
captured steps' keys and checks as they were."""
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


def _forward(lib, n_head=64, N=128, tan=F, status=F, xyz=F, dirs=F, capacity=1024, debug=0, head_flags=None,
             flags=None):
    hf, sf = _flags()
    hf = hf if head_flags is None else head_flags
    sf = sf if flags is None else flags
    return lib.gh_hair_segments_forward_binned_capturable(
        n_head, N, 64, 48, F, F, F, F, F, F, hf, 1e-12, xyz, dirs, F, F, F, F, sf, 1e-7, F, F, F, tan, 1.0, 3,
        F, F, F, F, F, F, F, F, F, capacity, status, None, debug, None)


def _backward(lib, n_head=64, N=128, tan=F, xyz=F, dirs=F, debug=0, flags=None):
    sf = _flags()[1] if flags is None else flags
    return lib.gh_hair_segments_backward_capturable(
        n_head, N, 64, 48, xyz, dirs, F, F, F, F, sf, 1e-7, F, F, F, tan, 1.0, 3, F, F, F, F, F, F, F, None, debug, None)


CASES = [
    (lambda lib: _forward(lib, tan=None), "tan_fov"),
    (lambda lib: _forward(lib, status=None), "status"),
    (lambda lib: _forward(lib, xyz=None), "xyz and dirs"),
    (lambda lib: _forward(lib, dirs=None), "xyz and dirs"),
    (lambda lib: _forward(lib, n_head=64, N=0, xyz=None), "xyz and dirs"),
    (lambda lib: _forward(lib, capacity=-1), "capacity must lie in"),
    (lambda lib: _forward(lib, capacity=1 << 32), "capacity must lie in"),
    (lambda lib: _forward(lib, debug=1), "debug"),
    (lambda lib: _forward(lib, n_head=-1), "n_head must not be negative"),
    (lambda lib: _forward(lib, N=-2), "N must be non-negative"),
    (lambda lib: _forward(lib, N=(1 << 30)), "N overflows int"),
    (lambda lib: _forward(lib, n_head=(1 << 31) - 100, N=128), "n_head + N overflows int"),
    (lambda lib: _forward(lib, n_head=0, N=0), "nothing to render"),
    (lambda lib: _forward(lib, head_flags=_flags()[0] | (1 << 10)), "head_flags must not set the strand bit"),
    (lambda lib: _forward(lib, flags=_flags()[1] & ~(1 << 10)), "flags must set the strand bit"),
    (lambda lib: _backward(lib, tan=None), "tan_fov"),
    (lambda lib: _backward(lib, xyz=None), "xyz and dirs"),
    (lambda lib: _backward(lib, dirs=None), "xyz and dirs"),
    (lambda lib: _backward(lib, debug=1), "debug"),
    (lambda lib: _backward(lib, n_head=-1), "n_head must not be negative"),
    (lambda lib: _backward(lib, N=0), "N must be positive"),
    (lambda lib: _backward(lib, N=-1), "N must be positive"),
    (lambda lib: _backward(lib, N=(1 << 30)), "N overflows int"),
    (lambda lib: _backward(lib, n_head=(1 << 31) - 100, N=128), "n_head + N overflows int"),
    (lambda lib: _backward(lib, flags=_flags()[1] & ~(1 << 10)), "flags must set the strand bit"),
]


@pytest.mark.parametrize("call, message", CASES)
def test_segment_capturable_entry_points_refuse_bad_arguments_before_any_launch(lib, call, message):
    from gaussianhaircut_b200 import _capi
    n0 = lib.gh_kernel_launch_count()
    assert call(lib) == _capi.GH_E_INVALID_ARG
    assert message in lib.gh_last_error().decode()
    assert lib.gh_kernel_launch_count() == n0


@pytest.mark.parametrize("call", [lambda lib: _forward(lib), lambda lib: _backward(lib)])
def test_segment_capturable_entry_points_refuse_the_stage_timer(lib, call):
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
    """(pc, pc_hair) with CPU tensors: the attributes latent_capture_key reads; N = S * L segment rows."""
    pc = types.SimpleNamespace(xyz_precomp=torch.zeros(n_head, 3), scaling_precomp=torch.zeros(n_head, 3),
                               rotation_precomp=torch.zeros(n_head, 4), opacity_precomp=torch.zeros(n_head, 1),
                               shs_view=torch.zeros(n_head, 3, 16))
    N = S * L
    hair = types.SimpleNamespace(_xyz=torch.zeros(N, 3), _dir=torch.zeros(N, 3), _features_dc=torch.zeros(N, 1, 3),
                                 _features_rest=torch.zeros(N, 15, 3), _orient_conf=torch.zeros(N, 1),
                                 scale=torch.ones(1), active_sh_degree=sh)
    return pc, hair


def test_latent_capture_key():
    from gaussianhaircut_b200.graphs import latent_capture_key as key
    pc, hair = _fake()
    k = key(pc, hair, 64, 48)
    assert k[:4] == (30, 7, 64, 48)
    assert key(pc, hair, 64, 48) == k
    assert key(pc, hair, 65, 48) != k and key(pc, hair, 64, 47) != k
    assert key(pc, hair, 64, 48, use_gt_orient_conf=False) != k
    assert key(pc, hair, 64, 48, train_orient_conf=False) != k
    assert key(None, hair, 64, 48)[1] == 0                      # hair only
    hair.active_sh_degree = 2
    assert key(pc, hair, 64, 48) != k
    hair.active_sh_degree = 3
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(not prev)
    try:
        assert key(pc, hair, 64, 48) != k
    finally:
        torch.use_deterministic_algorithms(prev)
    assert key(pc, hair, 64, 48) == k
    # the decoder's outputs are copied into the step's buffers: new tensors of the same shapes keep the key
    for name in ("_xyz", "_dir", "_features_dc", "_features_rest", "_orient_conf"):
        setattr(hair, name, getattr(hair, name).clone())
    assert key(pc, hair, 64, 48) == k
    # storage: the thickness, the head block (a new *_precomp tensor rebuilds the cached block)
    old = hair.scale
    hair.scale = old.clone()
    assert key(pc, hair, 64, 48) != k
    hair.scale = old
    assert key(pc, hair, 64, 48) == k
    pc.xyz_precomp = pc.xyz_precomp.clone()
    assert key(pc, hair, 64, 48)[:9] == k[:9] and key(pc, hair, 64, 48) != k
    # a different number of segment rows or head Gaussians
    pc2, hair2 = _fake(S=9, L=4, n_head=3)
    assert key(pc2, hair2, 64, 48)[:2] == (36, 3)


class _FakeStep:
    """The two attributes _StaticGradients reads from a CapturedLatentStrandStep."""

    def __init__(self, grads):
        self._grads, self._generation = grads, 1


def test_static_gradients_scale_with_grad_output_and_refuse_a_stale_step():
    from gaussianhaircut_b200.graphs import _StaticGradients
    gen = torch.Generator().manual_seed(3)
    shapes = ((12, 3), (12, 3), (12, 1, 3), (12, 15, 3), (12, 1))
    leaves = [torch.randn(sh, generator=gen, requires_grad=True) for sh in shapes]
    grads = tuple(torch.randn(sh, generator=gen) for sh in shapes)
    step = _FakeStep(grads)
    loss = _StaticGradients.apply(torch.tensor(1.5), step, 1, *[2.0 * t for t in leaves])
    assert loss.ndim == 0 and float(loss.detach()) == 1.5
    (loss * 3.0).backward()
    for leaf, g in zip(leaves, grads):
        assert torch.equal(leaf.grad, g * 3.0 * 2.0)
    # grad_output = 1: the gradients themselves, exactly
    for leaf in leaves:
        leaf.grad = None
    _StaticGradients.apply(torch.tensor(0.5), step, 1, *leaves).backward()
    for leaf, g in zip(leaves, grads):
        assert torch.equal(leaf.grad, g)
    # a later step overwrote the gradients: the earlier loss must not hand them out
    stale = _StaticGradients.apply(torch.tensor(0.5), step, 1, *leaves)
    step._generation = 2
    with pytest.raises(RuntimeError, match="overwritten by step 2"):
        stale.backward()
    step._grads = None                     # a step that failed before computing any gradient
    with pytest.raises(RuntimeError, match="call backward"):
        _StaticGradients.apply(torch.tensor(0.5), step, 2, *leaves).backward()


def test_the_base_class_still_requires_fused_adam_for_the_other_steps():
    from gaussianhaircut_b200 import graphs
    bg = torch.zeros(10)
    model = types.SimpleNamespace(_xyz=torch.zeros(4, 3))
    for opt in (None, types.SimpleNamespace(capturable=True), torch.optim.SGD([torch.zeros(1, requires_grad=True)], 0.1)):
        with pytest.raises(RuntimeError, match=r"CapturedTrainStep needs FusedAdam\(..., capturable=True\)"):
            graphs.CapturedTrainStep(model, opt, 64, 48, bg, (0.8, 0.2, 0.2, 0.1))
    pc, hair = _fake()
    strands = types.SimpleNamespace(_dirs=torch.zeros(6, 5, 3), scale=torch.ones(1))
    for opt in (None, types.SimpleNamespace(capturable=True)):
        with pytest.raises(RuntimeError, match=r"CapturedStrandStep needs FusedAdam\(..., capturable=True\)"):
            graphs.CapturedStrandStep(pc, strands, opt, 64, 48, bg, (0.8, 0.2, 0.2, 0.1))
    # the optimizer-free form is for the latent step alone: it takes no optimizer
    with pytest.raises(RuntimeError, match="no optimizer inside the graph"):
        graphs._CapturedStep("X", object(), 64, 48, bg, (1.0,), None, None, bg.device, needs_optimizer=False)
    with pytest.raises(RuntimeError, match="debug"):
        graphs.CapturedLatentStrandStep(pc, 64, 48, bg, (0.1, 1.0, 0.1), pipe=types.SimpleNamespace(debug=True))
    with pytest.raises(RuntimeError, match=r"\(l1, mask, orient\)"):
        graphs.CapturedLatentStrandStep(pc, 64, 48, bg, (0.8, 0.2, 0.2, 0.1))


def test_the_other_capture_keys_are_unchanged():
    """capture_key and strand_capture_key keep their layout (the optimizer-free base class does not touch them)."""
    from gaussianhaircut_b200.graphs import capture_key, strand_capture_key
    p = torch.zeros(4, 3)
    opt = types.SimpleNamespace(param_groups=[{"params": [p]}], state={p: {"exp_avg": torch.zeros(4, 3),
                                                                          "exp_avg_sq": torch.zeros(4, 3)}})
    model = types.SimpleNamespace(_xyz=p, active_sh_degree=3, xyz_gradient_accum=None, denom=None, max_radii2D=None)
    k = capture_key(model, opt, 64, 48)
    st = opt.state[p]
    assert k == (4, 64, 48, 3, torch.are_deterministic_algorithms_enabled(),
                 (p.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), 0, 0, 0), ())
    pc, _ = _fake()
    dirs = torch.zeros(6, 5, 3)
    strands = types.SimpleNamespace(_dirs=dirs, pts_origins=torch.zeros(6, 1, 3), scale=torch.ones(1), active_sh_degree=3)
    opt2 = types.SimpleNamespace(param_groups=[{"params": [dirs]}], state={})
    ks = strand_capture_key(pc, strands, opt2, 64, 48)
    assert ks[:10] == (6, 5, 7, 64, 48, 3, torch.are_deterministic_algorithms_enabled(), True, True, False)
    assert ks[10] == (dirs.data_ptr(), strands.pts_origins.data_ptr(), strands.scale.data_ptr())
