"""CPU tests of the first phase's optional binning buffer (gh_forward_preprocess, gh_project_forward_binned,
gh_forward_render) and of the capacity hint that sizes it (_C.binning_capacity): the ABI surface, and the refusal of
bad buffer arguments before anything is launched."""
import ctypes as C
import os
import re

import pytest

import _util  # noqa: F401  (puts the repository root on sys.path)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import _capi
    return _capi.load()


def _header_params(name):
    """Parameter names of `name` as declared in include/gh_rasterizer.h."""
    src = open(os.path.join(ROOT, "include", "gh_rasterizer.h")).read()
    decl = re.search(rf"\bint {name}\((.*?)\);", src, flags=re.S).group(1)
    return [p.split()[-1].lstrip("*") for p in decl.split(",")]


def test_abi_surface(lib):
    from gaussianhaircut_b200 import _capi
    # one entry point per forward phase since ABI 5 (the optional binning buffer is part of each signature); ABI 6 takes
    # the Adam betas as double
    assert lib.gh_abi_version() == _capi.ABI_VERSION == 6
    sig = _capi.SIGNATURES
    for name in ("gh_forward_preprocess_ex", "gh_forward_render_ex", "gh_project_forward_binned_ex"):
        assert name not in sig and not hasattr(lib, name), name
    for name, at in (("gh_forward_preprocess", 24), ("gh_project_forward_binned", 30)):
        params, args = _header_params(name), sig[name][1]
        assert len(params) == len(args), name
        assert params[at:at + 2] == ["binning_buffer", "binning_capacity"], name
        assert args[at:at + 2] == [C.c_void_p, C.c_longlong], name
        assert params.index("emitted") == params.index("max_tile_len") + 1 and args[params.index("emitted")] == C.POINTER(C.c_int)
    params, args = _header_params("gh_forward_render"), sig["gh_forward_render"][1]
    assert len(params) == len(args) and params[11] == "emitted" and args[11] is C.c_int


def _preprocess(lib, buf, cap, emitted=True):
    fake = C.c_void_p(0x1000)
    n, m, e = C.c_int(), C.c_int(), C.c_int(7)
    rc = lib.gh_forward_preprocess(10, 3, 0, 64, 64, fake, None, None, fake, fake, fake, 1.0, fake, None, None,
                                   fake, fake, fake, 0.5, 0.5, 0, fake, fake, fake, buf, cap,
                                   C.byref(n), C.byref(m), C.byref(e) if emitted else None, 0, None)
    return rc


def _project_binned(lib, buf, cap, emitted=True):
    from gaussianhaircut_b200 import projection as pj
    fake = C.c_void_p(4096)
    common = (128, 64, 48, fake, fake, fake, fake, fake, fake, None, None, fake, fake, fake, fake,
              0.5, 0.5, 1.0, 3, pj.encode_flags(pj.HAIR_MODEL), 1e-7)
    n, m, e = C.c_int(), C.c_int(), C.c_int(7)
    return lib.gh_project_forward_binned(*common, fake, fake, fake, fake, None, fake, fake, fake, fake, buf, cap,
                                         C.byref(n), C.byref(m), C.byref(e) if emitted else None, None)


@pytest.mark.parametrize("entry", [_preprocess, _project_binned])
def test_bad_binning_arguments_are_refused_before_any_launch(lib, entry):
    from gaussianhaircut_b200 import _capi
    launches0 = lib.gh_kernel_launch_count()
    buf = C.c_void_p(0x2000)
    cases = [
        (buf, -1, True, "binning_capacity must lie in [0, 2^32)"),
        (buf, 1 << 32, True, "binning_capacity must lie in [0, 2^32)"),
        (None, 100, True, "binning_capacity given without a binning_buffer"),
        (buf, 100, False, "needs the `emitted` output"),
    ]
    for b, cap, emitted, msg in cases:
        assert entry(lib, b, cap, emitted) == _capi.GH_E_INVALID_ARG, (b, cap, emitted)
        assert msg in lib.gh_last_error().decode(), (msg, lib.gh_last_error())
    assert lib.gh_kernel_launch_count() == launches0


def test_capacity_hint():
    from gaussianhaircut_b200 import _C
    key = ("test", 1000, 64, 48)
    _C._BIN_R.pop(key, None)
    assert _C.binning_capacity(key) == 0                                   # first call: no hint
    _C.binning_record(key, 1000)
    assert _C.binning_capacity(key) == 1000 + 250 + 256
    for R in (400, 2000, 900):
        _C.binning_record(key, R)
    assert _C.binning_capacity(key) == 2000 + 500 + 256                   # the largest R of the history
    for R in range(_C._BIN_HISTORY):
        _C.binning_record(key, 10 + R)
    assert len(_C._BIN_R[key]) == _C._BIN_HISTORY                          # only the last few are kept
    assert _C.binning_capacity(key) == 17 + 4 + 256
    _C._BIN_R.pop(key, None)


def test_capacity_hint_forgets_the_oldest_shape():
    from gaussianhaircut_b200 import _C
    saved = dict(_C._BIN_R)
    try:
        _C._BIN_R.clear()
        keys = [("test", P, 64, 48) for P in range(_C._BIN_KEYS + 5)]
        for k in keys:
            _C.binning_record(k, 100)
        assert len(_C._BIN_R) == _C._BIN_KEYS
        assert _C.binning_capacity(keys[0]) == 0 and _C.binning_capacity(keys[-1]) > 0
    finally:
        _C._BIN_R.clear()
        _C._BIN_R.update(saved)
