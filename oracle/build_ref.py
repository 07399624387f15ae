"""TEST INFRASTRUCTURE ONLY -- builds Oracle-A (`oracle/_ref`).

Compiles the reference rasterizer **from its sources where they lie** under
/root/reference/ext/diff_gaussian_rasterization_hair (nothing is copied into
the tracked tree) into an importable package

    oracle/_ref/diff_gaussian_rasterization/{__init__.py, _C.<abi>.so}

exactly as the reference's own `setup.py` (setup.py:16-33) would install it,
with the two shims the container needs (SURVEY.md section 0.7):

  * `-I oracle/glm_shim`  -- glm (pinned 5c46b9c, install.sh:32-33) is not
    vendored and there is no network; the stand-in follows glm's evaluation
    order.
  * `-include cstdint`    -- gcc 13 (rasterizer_impl.h:24,40 use uintptr_t /
    uint32_t without the include).

Flags follow torch's CUDAExtension defaults (no fast-math, -fmad=true, IEEE
div/sqrt) plus `-gencode arch=compute_90a,code=sm_90a`.

`oracle/_ref/` is git-ignored (build output) but travels to the GPU box.
The reference has no CPU implementation of this path, so this CUDA build is
both the parity oracle on the GPU and the reported baseline
(BASELINE.json:north_star).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
REF_EXT = "/root/reference/ext/diff_gaussian_rasterization_hair"
OUT_PKG = os.path.join(HERE, "_ref", "diff_gaussian_rasterization")
OBJ_DIR = os.path.join(HERE, "_ref", "obj")
EXT_SUFFIX = sysconfig.get_config_var("EXT_SUFFIX")
SO_PATH = os.path.join(OUT_PKG, "_C" + EXT_SUFFIX)


REF_SRC = "/root/reference/src"
OUT_SRC = os.path.join(HERE, "_ref", "src")
# the reference's Python callers of the hot path (pure Python: "installing" them is a copy; oracle/_ref is
# git-ignored build output, so nothing of this enters the history) -- used by oracle/ref_python.py to run
# render() / render_hair() unmodified on the GPU box, where /root/reference does not exist
PY_STAGE = ("gaussian_renderer/__init__.py", "scene", "utils", "arguments/__init__.py")


def ref_available() -> bool:
    return os.path.isdir(REF_EXT)


def stage_python(verbose: bool = True) -> str:
    """Copy the reference's pure-Python render path next to the compiled extension (oracle/_ref/src)."""
    if not os.path.isdir(REF_SRC):
        return OUT_SRC
    for rel in PY_STAGE:
        src = os.path.join(REF_SRC, rel)
        dst = os.path.join(OUT_SRC, rel)
        if os.path.isdir(src):
            os.makedirs(dst, exist_ok=True)
            for f in sorted(os.listdir(src)):
                if f.endswith(".py"):
                    shutil.copyfile(os.path.join(src, f), os.path.join(dst, f))
        elif os.path.isfile(src):
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copyfile(src, dst)
    if verbose:
        print("[oracle/_ref] staged the reference's Python render path under", OUT_SRC, flush=True)
    return OUT_SRC


def is_built() -> bool:
    return os.path.isfile(SO_PATH) and os.path.isfile(os.path.join(OUT_PKG, "__init__.py"))


def _torch_paths():
    import torch
    tdir = os.path.dirname(torch.__file__)
    inc = [os.path.join(tdir, "include"),
           os.path.join(tdir, "include", "torch", "csrc", "api", "include")]
    lib = os.path.join(tdir, "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    return inc, lib, abi


def build(verbose: bool = True, force: bool = False) -> str:
    if not ref_available():
        if is_built():
            return SO_PATH
        raise RuntimeError("reference sources not present and oracle/_ref not prebuilt")
    srcs = [
        os.path.join(REF_EXT, "cuda_rasterizer", "rasterizer_impl.cu"),
        os.path.join(REF_EXT, "cuda_rasterizer", "forward.cu"),
        os.path.join(REF_EXT, "cuda_rasterizer", "backward.cu"),
        os.path.join(REF_EXT, "rasterize_points.cu"),
        os.path.join(REF_EXT, "ext.cpp"),
    ]
    stage_python(verbose=False)
    # this file holds the flags (target architecture): an oracle/_ref built with other flags is rebuilt
    deps = srcs + [os.path.join(HERE, "glm_shim", "glm", "glm.hpp"), os.path.abspath(__file__)]
    if is_built() and not force:
        newest = max(os.path.getmtime(p) for p in deps)
        if os.path.getmtime(SO_PATH) >= newest:
            return SO_PATH
    os.makedirs(OUT_PKG, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    inc, lib, abi = _torch_paths()
    pyinc = sysconfig.get_paths()["include"]
    common_inc = [f"-I{p}" for p in inc] + [f"-I{pyinc}", "-I/usr/local/cuda/include",
                                            f"-I{os.path.join(HERE, 'glm_shim')}",
                                            f"-I{REF_EXT}"]
    defs = ["-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
            f"-D_GLIBCXX_USE_CXX11_ABI={abi}"]
    nvcc_flags = ["-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
                  "-D__CUDA_NO_BFLOAT16_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__",
                  "--expt-relaxed-constexpr", "-std=c++17", "-O3",
                  "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
                  "--compiler-options", "-fPIC", "-include", "cstdint", "-w"]
    cxx_flags = ["-std=c++17", "-O2", "-fPIC", "-include", "cstdint", "-w"]

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJ_DIR, os.path.basename(src) + ".o")
        if src.endswith(".cu"):
            cmd = ["nvcc", "-c", src, "-o", obj] + nvcc_flags + defs + common_inc
        else:
            cmd = ["g++", "-c", src, "-o", obj] + cxx_flags + defs + common_inc
        if verbose:
            print("[oracle/_ref]", os.path.basename(src), flush=True)
        subprocess.run(cmd, check=True)
        return obj

    with ThreadPoolExecutor(max_workers=5) as ex:
        objs = list(ex.map(compile_one, srcs))
    link = ["g++", "-shared", "-o", SO_PATH] + objs + [
        f"-L{lib}", "-L/usr/local/cuda/lib64",
        "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
        "-lcudart", f"-Wl,-rpath,{lib}", "-Wl,-rpath,/usr/local/cuda/lib64"]
    subprocess.run(link, check=True)
    # "install" step of the reference's setup.py: the package's python front door
    shutil.copyfile(os.path.join(REF_EXT, "diff_gaussian_rasterization", "__init__.py"),
                    os.path.join(OUT_PKG, "__init__.py"))
    if verbose:
        print("[oracle/_ref] built", SO_PATH, flush=True)
    return SO_PATH


def load():
    """Import the reference package from oracle/_ref under a private module name
    (so it never shadows the product's `diff_gaussian_rasterization`)."""
    import importlib.util
    name = "gh_oracle_ref_diff_gaussian_rasterization"
    if name in sys.modules:
        return sys.modules[name]
    if not is_built():
        raise RuntimeError("oracle/_ref is not built (run python oracle/build_ref.py)")
    import torch  # noqa: F401  (libtorch must be loaded before the extension)
    spec = importlib.util.spec_from_file_location(
        name, os.path.join(OUT_PKG, "__init__.py"),
        submodule_search_locations=[OUT_PKG])
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    build(force="--force" in sys.argv)
