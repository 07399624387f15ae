"""CPU tests of the captured training iteration: the capturable C-ABI entry points refuse bad arguments (missing status
or tan fov pointer, a negative capacity, debug mode, the stage timer) before they launch anything, and the recapture key
and the capacity policy of graphs.CapturedTrainStep, as plain Python."""
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


def _project_forward(lib, tan=F, status=F, capacity=1024, debug=0, flags=None):
    from gaussianhaircut_b200 import projection as pj
    fl = pj.encode_flags(pj.GAUSSIAN_MODEL) if flags is None else flags
    return lib.gh_project_forward_binned_capturable(
        128, 64, 48, F, F, F, None, F, F, F, F, F, F, F, F, tan, 1.0, 3, fl, 1e-12,
        F, F, F, F, F, F, F, F, F, capacity, status, None, debug, None)


def _render(lib, capacity=1024, debug=0):
    return lib.gh_forward_render_capturable(128, 64, 48, capacity, F, F, F, F, F, F, debug, None)


def _backward(lib, capacity=1024, debug=0, det=None, det_bytes=0):
    return lib.gh_backward_capturable(128, 64, 48, capacity, F, F, F, F, F, F, F, debug, None, det, det_bytes)


def _project_backward(lib, tan=F, debug=0):
    from gaussianhaircut_b200 import projection as pj
    return lib.gh_project_backward_capturable(
        128, 64, 48, F, F, F, None, F, F, F, F, F, F, F, F, tan, 1.0, 3, pj.encode_flags(pj.GAUSSIAN_MODEL), 1e-12,
        F, F, None, None, None, None, F, F, F, None, F, F, F, F, F, F, None, None, None, debug, None)


def _adam(lib, lrs=F, step_state=F, debug=0):
    arr = (C.c_void_p * 1)(4096)
    return lib.gh_adam_step_capturable(1, arr, arr, arr, arr, (C.c_ulonglong * 1)(16), lrs, 0.9, 0.999, 1e-15,
                                       step_state, None, None, debug, None)


CASES = [
    (lambda lib: _project_forward(lib, tan=None), "tan_fov"),
    (lambda lib: _project_forward(lib, status=None), "status"),
    (lambda lib: _project_forward(lib, capacity=-1), "capacity must lie in"),
    (lambda lib: _project_forward(lib, capacity=1 << 32), "capacity must lie in"),
    (lambda lib: _project_forward(lib, debug=1), "debug"),
    (lambda lib: _project_forward(lib, flags=1 << 10), "strand mode"),
    (lambda lib: _render(lib, capacity=-1), "capacity must lie in"),
    (lambda lib: _render(lib, debug=1), "debug"),
    (lambda lib: _backward(lib, capacity=-5), "capacity must lie in"),
    (lambda lib: _backward(lib, debug=1), "debug"),
    (lambda lib: _backward(lib, det=F, det_bytes=16), "smaller than gh_backward_det_workspace_size"),
    (lambda lib: _backward(lib, det_bytes=16), "det_bytes given without a det_buffer"),
    (lambda lib: _project_backward(lib, tan=None), "tan_fov"),
    (lambda lib: _project_backward(lib, debug=1), "debug"),
    (lambda lib: _adam(lib, lrs=None), "lrs"),
    (lambda lib: _adam(lib, step_state=None), "step_state"),
    (lambda lib: _adam(lib, debug=1), "debug"),
]


@pytest.mark.parametrize("call, message", CASES)
def test_capturable_entry_points_refuse_bad_arguments_before_any_launch(lib, call, message):
    from gaussianhaircut_b200 import _capi
    n0 = lib.gh_kernel_launch_count()
    assert call(lib) == _capi.GH_E_INVALID_ARG
    assert message in lib.gh_last_error().decode()
    assert lib.gh_kernel_launch_count() == n0


@pytest.mark.parametrize("call", [lambda lib: _project_forward(lib), lambda lib: _render(lib), lambda lib: _backward(lib),
                                  lambda lib: _project_backward(lib), lambda lib: _adam(lib)])
def test_capturable_entry_points_refuse_the_stage_timer(lib, call):
    from gaussianhaircut_b200 import _capi
    n0 = lib.gh_kernel_launch_count()
    lib.gh_stage_timing_enable(1)
    try:
        assert call(lib) == _capi.GH_E_INVALID_ARG
        assert "stage timer" in lib.gh_last_error().decode()
    finally:
        lib.gh_stage_timing_enable(0)
    assert lib.gh_kernel_launch_count() == n0


def test_capacity_policy():
    from gaussianhaircut_b200 import _C
    from gaussianhaircut_b200.graphs import capacity_for
    assert capacity_for(0) == 256 and capacity_for(1000) == 1506 and capacity_for(4_000_003) == 5_000_259
    key = ("cpu-test", 7, 64, 48)
    for r in (100, 900, 300):
        _C.binning_record(key, r)
    assert _C.binning_capacity(key) == capacity_for(900) and _C.last_num_rendered(key) == 300
    _C._BIN_R.pop(key)


def _fake(P=16, sh=3):
    params = [torch.zeros(P, 3), torch.zeros(P, 1)]
    model = types.SimpleNamespace(_xyz=params[0], active_sh_degree=sh, xyz_gradient_accum=torch.zeros(P, 1),
                                  denom=torch.zeros(P, 1), max_radii2D=torch.zeros(P))
    opt = types.SimpleNamespace(param_groups=[{"params": [p]} for p in params],
                                state={p: {"exp_avg": torch.zeros_like(p), "exp_avg_sq": torch.zeros_like(p)} for p in params})
    return model, opt


def test_recapture_key():
    from gaussianhaircut_b200.graphs import capture_key
    model, opt = _fake()
    k = capture_key(model, opt, 64, 48)
    assert capture_key(model, opt, 64, 48) == k
    assert capture_key(model, opt, 65, 48) != k and capture_key(model, opt, 64, 47) != k
    model.active_sh_degree = 2
    assert capture_key(model, opt, 64, 48) != k
    model.active_sh_degree = 3
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(not prev)
    try:
        assert capture_key(model, opt, 64, 48) != k
    finally:
        torch.use_deterministic_algorithms(prev)
    # a densification replaces parameters, moments and statistics: new storage (and usually a new P)
    model.denom = torch.zeros(16, 1)
    assert capture_key(model, opt, 64, 48) != k
    model2, opt2 = _fake(P=20)
    assert capture_key(model2, opt2, 64, 48)[0] == 20
    p = opt.param_groups[1]["params"][0]
    opt.state[p]["exp_avg"] = torch.zeros_like(p)
    assert capture_key(model, opt, 64, 48)[:5] == k[:5]
