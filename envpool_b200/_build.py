"""In-tree build of the CUDA engine and the pybind11 host modules.

    python -m envpool_b200._build            # build everything that is out of date

Produces (all git-ignored):
  envpool_b200/lib/libenvpool_b200.so      C-ABI engine (include/envpool_b200.h), sm_90a
  envpool_b200/<family>_envpool*.so        pybind11 host modules (classic_control_envpool,
                                           toy_text_envpool, jumanji_envpool,
                                           mujoco_gym_envpool, pgx_envpool)
nvcc cross-compiles for sm_90a without a GPU, so this runs on a machine without one.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
OBJDIR = os.path.join(PKG, "lib", "obj")
ENGINE_SO = os.path.join(LIBDIR, "libenvpool_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_COMMON = ["-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC"] + ARCH

# translation unit -> extra flags.  classic.cu: no FMA contraction, the reference's double
# arithmetic is plain x86-64 mul/add (see the file header).
CUDA_UNITS = {
    "classic.cu": ["-fmad=false"],
    "toytext.cu": [],
    "jumanji.cu": [],
    "mujoco.cu": [],
    "pgx.cu": [],
    "go.cu": [],
    "chess.cu": [],
    "capi.cu": [],
}
PY_MODULES = {
    # module name and location as in the reference (envpool/classic_control/
    # classic_control_envpool, envpool/toy_text/toy_text_envpool,
    # envpool/jumanji/jumanji_envpool, envpool/mujoco/mujoco_gym_envpool,
    # envpool/pgx/pgx_envpool) ->
    # (sub-directory, family macro)
    "classic_control_envpool": ("classic_control", "EPB_FAMILY_CLASSIC_CONTROL"),
    "toy_text_envpool": ("toy_text", "EPB_FAMILY_TOY_TEXT"),
    "jumanji_envpool": ("jumanji", "EPB_FAMILY_JUMANJI"),
    "mujoco_gym_envpool": ("mujoco", "EPB_FAMILY_MUJOCO_GYM"),
    "pgx_envpool": ("pgx", "EPB_FAMILY_PGX"),
}


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA engine cannot be built")


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(ROOT, "include", "envpool_b200.h"))
    return hs


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build step failed:\n  " + " ".join(cmd) + "\n" + r.stdout)
    return r.stdout


def module_path(name: str) -> str:
    suffix = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    return os.path.join(PKG, PY_MODULES[name][0], name + suffix)


def build_engine(verbose: bool = False) -> str:
    os.makedirs(OBJDIR, exist_ok=True)
    nvcc = _nvcc()
    hdrs = _headers()
    jobs = []
    objs = []
    for unit, extra in CUDA_UNITS.items():
        src = os.path.join(CSRC, unit)
        obj = os.path.join(OBJDIR, unit.replace(".cu", ".o"))
        objs.append(obj)
        if _newer(obj, [src] + hdrs):
            jobs.append([nvcc] + NVCC_COMMON + extra + ["-c", src, "-o", obj])
    if jobs:
        with ThreadPoolExecutor(max_workers=len(jobs)) as ex:
            for out in ex.map(_run, jobs):
                if verbose and out.strip():
                    print(out)
    if jobs or _newer(ENGINE_SO, objs):
        _run([nvcc, "-shared", "-o", ENGINE_SO] + objs + ARCH + ["-cudart", "static"])
    return ENGINE_SO


def build_pymodules(verbose: bool = False):
    import pybind11

    src = os.path.join(CSRC, "py_module.cc")
    if not os.path.exists(src):
        return []
    inc = [
        "-I" + pybind11.get_include(),
        "-I" + sysconfig.get_paths()["include"],
        "-I" + os.path.join(ROOT, "include"),
    ]
    outs = []
    jobs = []
    for name, (_subdir, macro) in PY_MODULES.items():
        out = module_path(name)
        outs.append(out)
        if _newer(out, [src, os.path.join(ROOT, "include", "envpool_b200.h"), ENGINE_SO]):
            jobs.append(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fvisibility=hidden",
                         "-D" + macro, "-DEPB_MODULE_NAME=" + name] + inc +
                        [src, "-o", out, "-L" + LIBDIR, "-lenvpool_b200",
                         "-Wl,-rpath,$ORIGIN/../lib"])
    if jobs:
        with ThreadPoolExecutor(max_workers=len(jobs)) as ex:
            for o in ex.map(_run, jobs):
                if verbose and o.strip():
                    print(o)
    return outs


def build_all(verbose: bool = False):
    so = build_engine(verbose)
    mods = build_pymodules(verbose)
    return [so] + mods


if __name__ == "__main__":
    for path in build_all(verbose="-v" in sys.argv):
        print("built", os.path.relpath(path, ROOT))
