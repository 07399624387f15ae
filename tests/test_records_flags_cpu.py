"""CPU tests of how the accumulation records of the blend backward are cleared: the forward's blend clears them
(GH_FLAG_ZERO_RECORDS) and marks its geometry workspace, the first backward on that workspace takes the mark and skips
its own clearing pass (GH_FLAG_RECORDS_ZEROED), and every other backward -- a second one on the same forward, or one
after a forward that did not clear -- clears the records itself.  The flags words are checked as they reach a stand-in
for the library; the library's own handling of the flags word is checked where it refuses a call before any launch."""
import contextlib
import ctypes as C
import inspect

import pytest
import torch

import _util  # noqa: F401  (puts the repository root on sys.path)


class _FakeLib:
    """Records the flags word of every gh_forward_render and gh_backward call."""

    def __init__(self):
        self.render_flags, self.backward_flags = [], []

    def gh_forward_render(self, *args):
        self.render_flags.append(args[13])
        return 0

    def gh_backward(self, *args):
        self.backward_flags.append(args[-4])
        return 0


@pytest.fixture
def fake(monkeypatch):
    from gaussianhaircut_b200 import _C, _capi
    lib = _FakeLib()
    monkeypatch.setattr(_capi, "_lib", lib)
    monkeypatch.setattr(_C, "_stream", lambda device: None)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    return lib


def _render(zero_records, geom=None):
    from gaussianhaircut_b200 import _C
    geom = torch.zeros(64, dtype=torch.uint8) if geom is None else geom
    t = torch.zeros(16)
    _C._render(t, torch.zeros(4, 10), torch.zeros(4, dtype=torch.int32), geom, torch.zeros(64, dtype=torch.uint8), 8, 4,
               torch.zeros(10, 2, 2), False, binned=torch.zeros(64, dtype=torch.uint8), stream=C.c_void_p(0),
               zero_records=zero_records)
    return geom


def test_first_backward_skips_the_clearing_and_a_second_one_clears(fake):
    from gaussianhaircut_b200 import _C, _capi
    geom = _render(True)
    assert fake.render_flags == [_capi.GH_FLAG_ZERO_RECORDS]
    assert _C._backward_flags(geom) == _capi.GH_FLAG_RECORDS_ZEROED
    # retain_graph=True: the records now hold the first backward's sums
    assert _C._backward_flags(geom) == 0
    assert _C._backward_flags(geom, debug=True) == _capi.GH_FLAG_DEBUG
    # a new forward on the same workspace clears them again
    _render(True, geom)
    assert _C._backward_flags(geom, debug=True) == _capi.GH_FLAG_RECORDS_ZEROED | _capi.GH_FLAG_DEBUG


def _backward(geom):
    from gaussianhaircut_b200 import _C
    P, R, H, W = 4, 40, 2, 2
    t = lambda *s: torch.zeros(*s)  # noqa: E731
    _C._backward(t(10), t(P, 3), torch.ones(P, dtype=torch.int32), t(P, 10), None, None, 1.0, None, t(P, 3),
                 t(4, 4), t(4, 4), 0.5, 0.5, t(10, H, W), None, 0, t(3), geom, R, t(100), t(100), False)


def test_backward_calls(fake):
    """What reaches gh_backward: the first backward after a clearing forward skips the clearing pass, a second one
    (retain_graph=True) does not."""
    from gaussianhaircut_b200 import _capi
    geom = _render(True)
    _backward(geom)
    _backward(geom)
    assert fake.backward_flags == [_capi.GH_FLAG_RECORDS_ZEROED, 0]
    _backward(_render(False))
    assert fake.backward_flags[-1] == 0


def test_forward_only_calls_do_not_clear(fake):
    from gaussianhaircut_b200 import _C, _capi
    geom = _render(False)
    assert fake.render_flags == [0]
    assert _C._backward_flags(geom) == 0
    # a forward that does not clear leaves an earlier forward's cleared records, and the mark, as they are: the blend
    # forward never writes the records otherwise
    _render(True, geom)
    _render(False, geom)
    assert fake.render_flags[-2:] == [_capi.GH_FLAG_ZERO_RECORDS, 0]
    assert _C._backward_flags(geom) == _capi.GH_FLAG_RECORDS_ZEROED


def test_forward_flags():
    from gaussianhaircut_b200 import _C, _capi
    geom = torch.zeros(8, dtype=torch.uint8)
    assert _C._forward_flags(geom, False, debug=True) == _capi.GH_FLAG_DEBUG
    assert not getattr(geom, "_gh_records_zeroed", False)
    assert _C._forward_flags(geom, True) == _capi.GH_FLAG_ZERO_RECORDS and geom._gh_records_zeroed


def test_defaults():
    """The `_C`-level forwards clear by default: a backward usually follows them."""
    from gaussianhaircut_b200 import _C
    for fn in (_C.rasterize_gaussians, _C.forward_render, _C.forward_render_capturable, _C._render):
        assert inspect.signature(fn).parameters["zero_records"].default is True, fn.__name__


@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import _capi
    return _capi.load()


F = C.c_void_p(4096)


def test_capturable_entry_points_take_the_records_bits(lib):
    """The capturable variants refuse GH_FLAG_DEBUG only: with a records bit set the call gets past that check and
    fails on the (deliberately bad) image size instead, before anything is launched."""
    from gaussianhaircut_b200 import _capi
    launches0 = lib.gh_kernel_launch_count()

    def render(flags, P=128):
        return lib.gh_forward_render_capturable(P, 64, 48, 1024, F, F, F, F, F, F, flags, None)

    def backward(flags, P=128):
        return lib.gh_backward_capturable(P, 64, 48, 1024, F, F, F, F, F, F, F, flags, None, None, 0)

    for call, bit in ((render, _capi.GH_FLAG_ZERO_RECORDS), (backward, _capi.GH_FLAG_RECORDS_ZEROED)):
        assert call(_capi.GH_FLAG_DEBUG | bit) == _capi.GH_E_INVALID_ARG
        assert "debug" in lib.gh_last_error().decode()
        assert call(bit, P=0) == _capi.GH_E_INVALID_ARG
        assert "bad sizes" in lib.gh_last_error().decode()
    assert lib.gh_kernel_launch_count() == launches0
