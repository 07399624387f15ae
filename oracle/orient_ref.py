"""TEST INFRASTRUCTURE ONLY -- runs the reference's `src/preprocessing/calc_orientation_maps.py` UNMODIFIED.

* `stage()` copies that one file from the reference sources (when present) to oracle/_ref/src/preprocessing/, next to
  the rest of the reference's Python that oracle/build_ref.py stages.  oracle/_ref is git-ignored build output; the
  copy travels to the GPU box with it, where the reference sources do not exist.  `__graft_entry__.build()` calls it.
* `load()` imports the script under a private module name.  It imports `gabor_kernel` and `difference_of_gaussians`
  from skimage.filters, which is not installed: for this one import `skimage` and `skimage.filters` resolve to a module
  carrying oracle/orient64.py's restatements of both (scikit-image 0.20 semantics).  Whatever sys.modules held for those
  names before (oracle/ref_python.py's stubs included) is restored afterwards, so every other caller sees what it saw.
Only tests/ and tools/ import this module; the product never does.
"""
from __future__ import annotations

import importlib.util
import os
import shutil
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REL = os.path.join("preprocessing", "calc_orientation_maps.py")
REF_SRC_LIVE = "/root/reference/src"
REF_SRC_STAGED = os.path.join(HERE, "_ref", "src")
MODULE_NAME = "gh_ref_calc_orientation_maps"


def stage(verbose: bool = False) -> str | None:
    """Copy the reference script into oracle/_ref/src; returns the staged path, or None without reference sources."""
    src = os.path.join(REF_SRC_LIVE, REL)
    if not os.path.isfile(src):
        return None
    dst = os.path.join(REF_SRC_STAGED, REL)
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    shutil.copyfile(src, dst)
    if verbose:
        print("[oracle/_ref] staged", dst, flush=True)
    return dst


def source_path() -> str | None:
    for d in (REF_SRC_LIVE, REF_SRC_STAGED):
        p = os.path.join(d, REL)
        if os.path.isfile(p):
            return p
    return None


def load():
    """The reference's calc_orientation_maps module (`calc_orients`, `main`, ...), imported as it is."""
    if MODULE_NAME in sys.modules:
        return sys.modules[MODULE_NAME]
    path = source_path()
    if path is None:
        raise RuntimeError("reference calc_orientation_maps.py not available (neither /root/reference/src nor "
                           "oracle/_ref/src; run __graft_entry__.build() where the reference sources exist)")
    if HERE not in sys.path:
        sys.path.insert(0, HERE)
    import orient64
    filters = orient64.skimage_filters_module()
    pkg = types.ModuleType("skimage")
    pkg.__path__ = []
    pkg.filters = filters
    saved = {k: sys.modules.get(k) for k in ("skimage", "skimage.filters")}
    sys.modules["skimage"], sys.modules["skimage.filters"] = pkg, filters
    try:
        spec = importlib.util.spec_from_file_location(MODULE_NAME, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v
            else:
                sys.modules.pop(k, None)
    sys.modules[MODULE_NAME] = mod
    return mod


if __name__ == "__main__":
    print(stage(verbose=True))
