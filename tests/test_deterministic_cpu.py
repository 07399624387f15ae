"""CPU tests of the deterministic blend backward (gh_backward with a det_buffer): the C ABI surface, the argument checks
that run before any launch, the Gaussian-major row layout it writes its per-tile partials into, and the selection by
torch.use_deterministic_algorithms in _C._backward."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import build, _capi
    build.build(verbose=False)
    return _capi.load()


def _det_bytes(lib, P, R):
    n = C.c_size_t()
    assert lib.gh_backward_det_workspace_size(P, R, C.byref(n)) == 0
    return n.value


def test_abi_surface(lib):
    from gaussianhaircut_b200 import _capi
    assert _capi.ABI_VERSION == 4 and lib.gh_abi_version() == 4
    res, args = _capi.SIGNATURES["gh_backward_det_workspace_size"]
    assert res is C.c_int and args == [C.c_int, C.c_longlong, C.POINTER(C.c_size_t)]
    args = _capi.SIGNATURES["gh_backward"][1]
    assert len(args) == 38 and args[-2:] == [C.c_void_p, C.c_size_t]


def test_workspace_size(lib):
    # 64 B per instance + 4 B per Gaussian (+1) + the scan's per-CTA sums, each 256-byte aligned
    for P, R in ((1, 0), (1000, 1), (500000, 1217212), (2000000, 4900000)):
        b = _det_bytes(lib, P, R)
        lo = 64 * R + 4 * (P + 1) + 4 * ((P + 1023) // 1024)
        assert lo <= b <= lo + 4 * 256
    assert _det_bytes(lib, 500000, 1217212) < 80e6            # ~80 MB for the 1080p strand bench scene
    n = C.c_size_t()
    assert lib.gh_backward_det_workspace_size(-1, 5, C.byref(n)) == 1
    assert lib.gh_backward_det_workspace_size(5, -1, C.byref(n)) == 1


def _call_backward(lib, P, R, det_buffer, det_bytes):
    fake = C.c_void_p(0x1000)
    # conic_precomp call shape with all four 2-D outputs given: every pointer check passes
    return lib.gh_backward(P, 0, 0, R, 64, 48, fake, fake, None, fake, None, 1.0, None, None, fake,
                           fake, fake, fake, 0.5, 0.5, fake, fake, fake, fake, fake,
                           fake, fake, fake, fake, None, None, None, None, None, 0, None, det_buffer, det_bytes)


def test_backward_rejects_a_bad_det_buffer_before_launching(lib):
    from gaussianhaircut_b200 import _capi
    launches0 = lib.gh_kernel_launch_count()
    P, R = 1000, 5000
    need = _det_bytes(lib, P, R)
    assert _call_backward(lib, P, R, C.c_void_p(0x10000), need - 1) == _capi.GH_E_INVALID_ARG
    assert b"det_buffer smaller" in lib.gh_last_error()
    assert _call_backward(lib, P, R, None, need) == _capi.GH_E_INVALID_ARG
    assert b"without a det_buffer" in lib.gh_last_error()
    assert lib.gh_kernel_launch_count() == launches0


# ---- the row layout: a host restatement of gh_get_rect + gh_det_area + gh_det_row against brute-force enumeration
def _get_rect(px, py, r, gx, gy):
    """gh_get_rect in float32 with its rounding order: (p - r) * 1/16, ((p + r) + 16 - 1) * 1/16, truncation, clamp."""
    f = np.float32
    px, py, rf = f(px), f(py), f(r)
    t = lambda v: int(np.trunc(v))  # noqa: E731
    minx = min(gx, max(0, t(f(f(px - rf) * f(0.0625)))))
    miny = min(gy, max(0, t(f(f(py - rf) * f(0.0625)))))
    maxx = min(gx, max(0, t(f(f(f(f(px + rf) + f(16.0)) + f(-1.0)) * f(0.0625)))))
    maxy = min(gy, max(0, t(f(f(f(f(py + rf) + f(16.0)) + f(-1.0)) * f(0.0625)))))
    return minx, miny, maxx, maxy


def _slots(means, radii, gx, gy):
    rects = [_get_rect(x, y, r, gx, gy) if r > 0 else (0, 0, 0, 0) for (x, y), r in zip(means, radii)]
    area = np.array([(c - a) * (d - b) for a, b, c, d in rects], np.int64)
    off = np.concatenate([[0], np.cumsum(area)])
    return rects, off


def _check_layout(means, radii, W, H):
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rects, off = _slots(means, radii, gx, gy)
    R = 0
    seen = {}
    # brute force: every (Gaussian, tile) pair of the grid, emit's membership test, Gaussian-major then row-major
    for i, (a, b, c, d) in enumerate(rects):
        k = 0
        for ty in range(gy):
            for tx in range(gx):
                if radii[i] > 0 and a <= tx < c and b <= ty < d:
                    slot = off[i] + (ty - b) * (c - a) + (tx - a)
                    assert slot == R, (i, tx, ty)
                    assert slot not in seen
                    seen[slot] = (i, tx, ty)
                    R += 1
                    k += 1
        assert off[i + 1] - off[i] == k
    assert off[-1] == R == len(seen)
    return R


def test_row_layout_matches_brute_force_enumeration():
    W, H = 100, 70                                 # 7 x 5 tiles, last column / row partial
    rng = np.random.default_rng(0)
    n = 300
    means = np.stack([rng.uniform(-40, W + 40, n), rng.uniform(-40, H + 40, n)], axis=1).astype(np.float32)
    radii = rng.integers(0, 60, n)
    radii[:20] = 0                                             # not rendered
    means[20:30] = [[0.0, 0.0], [W - 1, H - 1], [0.0, H - 1], [W - 1, 0.0], [-5, 30], [W + 5, 30], [50, -5], [50, H + 5],
                    [15.99, 16.0], [16.0, 15.99]]           # rectangles clamped at every border and corner
    radii[20:30] = 9
    means[30], radii[30] = (W / 2, H / 2), 1000                # covers the whole grid
    R = _check_layout(means, radii, W, H)
    assert R > n
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rects, _ = _slots(means, radii, gx, gy)
    assert rects[30] == (0, 0, gx, gy)
    assert all(rects[i][0] == 0 or rects[i][2] == gx or rects[i][1] == 0 or rects[i][3] == gy for i in range(20, 28))


def test_row_layout_odd_image_and_nothing_rendered():
    _check_layout(np.array([[16.5, 8.0], [32.0, 16.0]], np.float32), np.array([4, 20]), 33, 17)
    assert _check_layout(np.zeros((5, 2), np.float32), np.zeros(5, np.int64), 33, 17) == 0


# ---- selection in _C._backward
class _FakeLib:
    def __init__(self):
        self.calls = []

    def gh_backward_det_workspace_size(self, P, R, out):
        out._obj.value = 64 * R + 4 * (P + 1) + 256
        return 0

    def gh_backward(self, *a):
        self.calls.append(a)
        return 0


@pytest.mark.parametrize("deterministic", [False, True])
def test_backward_selects_the_det_path_with_the_torch_switch(monkeypatch, deterministic):
    from gaussianhaircut_b200 import _C, _capi
    fake = _FakeLib()
    monkeypatch.setattr(_capi, "load", lambda: fake)
    monkeypatch.setattr(_C, "_stream", lambda device: None)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    P, R, H, W = 7, 40, 8, 12
    t = lambda *s: torch.zeros(*s)  # noqa: E731
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        _C._backward(t(10), t(P, 3), torch.ones(P, dtype=torch.int32), t(P, 10), None, None, 1.0, None, t(P, 3),
                     t(4, 4), t(4, 4), 0.5, 0.5, t(10, H, W), None, 0, t(3), t(100), R, t(100), t(100), False)
    finally:
        torch.use_deterministic_algorithms(prev)
    (args,) = fake.calls
    buf, nbytes = args[-2], args[-1]
    if deterministic:
        assert buf is not None and buf.value != 0 and nbytes == 64 * R + 4 * (P + 1) + 256
    else:
        assert buf is None and nbytes == 0
