"""Recipe that compiles the UNMODIFIED reference extension (litegs/submodules/gaussian_raster) for sm_90a (H100).

TEST INFRASTRUCTURE ONLY.  The reference checkout is the one the environment variable LITEGS_REFERENCE names, else a LiteGS
checkout next to this repository (``../reference`` or ``../LiteGS``).  Sources are compiled where they lie (nothing is copied
into this repository); the outputs are ``oracle/_ref/litegs_fused_ref.so``, ``oracle/_ref/fused_ssim_cuda_ref.so`` and the
staged Python package under ``oracle/_ref/py`` (all git-ignored; a machine that runs the tests without the checkout needs
only a copy of ``oracle/_ref``).  They are the "reference itself"
whose outputs tests/golden/make_golden*.py store as the fixtures that pin the CPU oracle and our kernels, and the CUDA
baseline that ``bench.py --impl reference`` times next to ours ("ref_cuda").  Flags are the reference's own: -O3 --use_fast_math
(GR/setup.py:33-36) plus the arch.  The reference's build system (setup.py / CMake) is not run.
"""
from __future__ import annotations

import importlib.util
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")


def _find_reference() -> str:
    """$LITEGS_REFERENCE, else a LiteGS checkout beside the repository; "" when there is none."""
    env = os.environ.get("LITEGS_REFERENCE", "")
    if env:
        return env
    repo = os.path.dirname(HERE)
    for name in ("reference", "LiteGS"):
        cand = os.path.join(os.path.dirname(repo), name)
        if os.path.isdir(os.path.join(cand, "litegs", "submodules", "gaussian_raster")):
            return cand
    return ""


REF_ROOT = _find_reference()
REF_GR = os.path.join(REF_ROOT, "litegs", "submodules", "gaussian_raster") if REF_ROOT else ""
NAME = "litegs_fused_ref"
SOURCES = ["binning.cu", "compact.cu", "cuda_errchk.cpp", "ext_cuda.cpp", "raster.cu", "transform.cu"]


REF_SSIM = os.path.join(REF_ROOT, "litegs", "submodules", "fused_ssim") if REF_ROOT else ""
NOT_FOUND = ("[build_ref] no LiteGS checkout found (set LITEGS_REFERENCE, or place it at ../reference or ../LiteGS beside this "
             "repository): nothing is built or staged from it; what oracle/_ref already holds is used, and the tests that need the "
             "reference's own Python package skip without it")
SSIM_NAME = "fused_ssim_cuda_ref"
SSIM_SOURCES = ["ssim.cu", "ext.cpp"]


def so_path(name: str = NAME):
    if not os.path.isdir(OUT):
        return None
    for f in os.listdir(OUT):
        if f.startswith(name) and f.endswith(".so"):
            return os.path.join(OUT, f)
    return None


def build(quiet: bool = False):
    """Build oracle/_ref/litegs_fused_ref.so if the reference tree is present; returns the path or None."""
    if so_path() is not None:
        return so_path()
    if not REF_GR or not os.path.isdir(REF_GR):
        if not quiet:
            print(NOT_FOUND)
        return None
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ["CXX"] = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else os.environ.get("CXX", "g++")
    os.environ["CC"] = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else os.environ.get("CC", "gcc")
    from torch.utils import cpp_extension
    # the reference's own setup.py strips torch's "no half operators" defines (GR/setup.py:4-16)
    for flag in ("-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_BFLOAT16_CONVERSIONS__",
                 "-D__CUDA_NO_HALF2_OPERATORS__"):
        if flag in cpp_extension.COMMON_NVCC_FLAGS:
            cpp_extension.COMMON_NVCC_FLAGS.remove(flag)
    cpp_extension.load(
        name=NAME,
        sources=[os.path.join(REF_GR, s) for s in SOURCES],
        extra_cflags=["-O3"],
        extra_cuda_cflags=["-O3", "--use_fast_math", "-gencode", "arch=compute_90a,code=sm_90a"],
        build_directory=OUT,
        verbose=not quiet,
        is_python_module=True,
    )
    return so_path()


def build_ssim(quiet: bool = False):
    """Build oracle/_ref/fused_ssim_cuda_ref.so from the reference's fused_ssim/{ssim.cu,ext.cpp} with the reference's own
    nvcc flags (fused_ssim/setup.py:33: --maxrregcount=32 --use_fast_math) plus the arch; returns the path or None."""
    if so_path(SSIM_NAME) is not None:
        return so_path(SSIM_NAME)
    if not REF_SSIM or not os.path.isdir(REF_SSIM):
        if not quiet:
            print(NOT_FOUND)
        return None
    out = os.path.join(OUT, "ssim_build")
    os.makedirs(out, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ["CXX"] = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else os.environ.get("CXX", "g++")
    os.environ["CC"] = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else os.environ.get("CC", "gcc")
    from torch.utils import cpp_extension
    cpp_extension.load(
        name=SSIM_NAME,
        sources=[os.path.join(REF_SSIM, s) for s in SSIM_SOURCES],
        extra_cflags=["-O3"],
        extra_cuda_cflags=["-O3", "--maxrregcount=32", "--use_fast_math", "-gencode", "arch=compute_90a,code=sm_90a"],
        build_directory=out,
        verbose=not quiet,
        is_python_module=True,
    )
    import shutil
    for f in os.listdir(out):
        if f.startswith(SSIM_NAME) and f.endswith(".so"):
            shutil.copy2(os.path.join(out, f), os.path.join(OUT, f))
    return so_path(SSIM_NAME)


PY_OUT = os.path.join(OUT, "py")


def stage_python(quiet: bool = False):
    """Stage the UNMODIFIED reference Python package (``litegs/`` without its native submodules, plus the example scripts)
    under ``oracle/_ref/py`` (git-ignored) so that the drop-in test
    (tests/test_gpu_dropin.py) and the ``ref_cuda`` bench leg can import the reference's own ``wrapper.py`` /
    ``render/__init__.py`` / ``training/trainer.py`` on a machine the reference checkout is not copied to.  Files are byte
    copies (checked by the test against a manifest of SHA-256 digests written here); nothing is copied into tracked paths."""
    import hashlib
    import json
    import shutil
    if not REF_ROOT or not os.path.isdir(os.path.join(REF_ROOT, "litegs")):
        if not quiet:
            print(NOT_FOUND)
        return PY_OUT if os.path.isdir(PY_OUT) else None
    os.makedirs(PY_OUT, exist_ok=True)
    manifest = {}
    for top in ("litegs", "example_train.py", "example_metrics.py"):
        src = os.path.join(REF_ROOT, top)
        if os.path.isfile(src):
            shutil.copy2(src, os.path.join(PY_OUT, top))
            manifest[top] = hashlib.sha256(open(src, "rb").read()).hexdigest()
            continue
        for d, dirs, files in os.walk(src):
            dirs[:] = [x for x in dirs if x not in ("submodules", "__pycache__")]
            rel = os.path.relpath(d, REF_ROOT)
            os.makedirs(os.path.join(PY_OUT, rel), exist_ok=True)
            for f in files:
                if f.endswith(".py"):
                    shutil.copy2(os.path.join(d, f), os.path.join(PY_OUT, rel, f))
                    manifest[os.path.join(rel, f)] = hashlib.sha256(open(os.path.join(d, f), "rb").read()).hexdigest()
    json.dump(manifest, open(os.path.join(PY_OUT, "MANIFEST.json"), "w"), indent=1, sort_keys=True)
    return PY_OUT


def reference_python_path():
    """Directory to put on sys.path to import the reference's ``litegs`` package: the checkout if present, else the
    staged copy, else None."""
    if REF_ROOT and os.path.isdir(os.path.join(REF_ROOT, "litegs")):
        return REF_ROOT
    return PY_OUT if os.path.isdir(os.path.join(PY_OUT, "litegs")) else None


def _load(name: str):
    p = so_path(name)
    if p is None:
        return None
    import torch  # noqa: F401  (registers the ATen symbols the extension links against)
    spec = importlib.util.spec_from_file_location(name, p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load():
    """Import the prebuilt reference module (needs torch). Returns None if absent."""
    return _load(NAME)


def load_ssim():
    """Import the prebuilt reference fused_ssim_cuda module (fusedssim, fusedssim_backward, fusedl1ssim_loss,
    fusedl1ssim_loss_backward). Returns None if absent."""
    return _load(SSIM_NAME)


if __name__ == "__main__":
    print(build(quiet="-q" in sys.argv))
    print(build_ssim(quiet="-q" in sys.argv))
    print(stage_python(quiet="-q" in sys.argv))
