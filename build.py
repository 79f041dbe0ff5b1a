#!/usr/bin/env python
"""In-tree native build for gloo_b200 (C++17 + CUDA sm_90a).

Generates build/build.ninja and runs ninja. Produces:
  gloo_b200/_C.<abi>.so          python extension: whole library + pybind11 bindings
  gloo_b200/lib/libglb.so        the C++ library on its own (for C++ consumers)
  gloo_b200/bin/glb_benchmark    C++ benchmark CLI (host + CUDA collectives)
  gloo_b200/bin/glb_selftest     C++ self-test binary (threads-as-ranks)

Everything CUDA is compiled with  -gencode arch=compute_90a,code=sm_90a -lineinfo.
cudart is linked statically and the driver API / NCCL are resolved at run time
(cudaGetDriverEntryPoint / dlopen), so the extension imports on a CPU-only box.

Usage: python build.py [-j N] [--verbose] [--clean] [--sanitize thread|address|undefined]

--sanitize X builds only gloo_b200/bin/glb_benchmark_<X> (host code instrumented with
-fsanitize=X, objects under build/san-X) - the reference's -DSANITIZE=<x> switch.
"""
from __future__ import annotations

import argparse
import os
import shutil
import subprocess
import sys
import sysconfig
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
BUILD = ROOT / "build"
PKG = ROOT / "gloo_b200"

CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")
# The image exports CXX=/opt/gcc/bin/g++, a relocated compiler whose link step
# silently drops libstdc++.so (exceptions then crash inside CPython). Use the
# system compiler unless GLB_CXX overrides it.
CXX = os.environ.get("GLB_CXX") or ("/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def ext_suffix() -> str:
    return sysconfig.get_config_var("EXT_SUFFIX") or ".so"


def collect():
    lib_cc, lib_cu, py_cc, bins = [], [], [], {}
    for p in sorted((CSRC / "glb").rglob("*")):
        if p.suffix not in (".cc", ".cu"):
            continue
        rel = p.relative_to(CSRC)
        parts = rel.parts
        if "python" in parts:
            py_cc.append(p)
        elif "benchmark" in parts and p.name.endswith("_main.cc"):
            bins[p.name[: -len("_main.cc")]] = p
        elif p.suffix == ".cu":
            lib_cu.append(p)
        else:
            lib_cc.append(p)
    return lib_cc, lib_cu, py_cc, bins


def write_ninja(verbose: bool, sanitize: str = "") -> Path:
    import pybind11

    global BUILD
    if sanitize:
        BUILD = ROOT / "build" / f"san-{sanitize}"
    BUILD.mkdir(parents=True, exist_ok=True)
    (PKG / "lib").mkdir(parents=True, exist_ok=True)
    (PKG / "bin").mkdir(parents=True, exist_ok=True)
    lib_cc, lib_cu, py_cc, bins = collect()

    py_inc = sysconfig.get_paths()["include"]
    common_inc = f"-I{CSRC} -I{CUDA_HOME}/include"
    have_mpi = os.path.exists("/usr/include/mpi.h") or bool(shutil.which("mpicxx"))
    mpi_def = "-DGLB_USE_MPI=1 " if have_mpi else "-DGLB_USE_MPI=0 "
    cxxflags = (
        mpi_def + "-std=c++17 -O2 -g1 -fPIC -Wall -Wextra -Wno-unused-parameter -Wno-missing-field-initializers "
        "-pthread -DGLB_USE_CUDA=1 " + common_inc
    )
    nvccflags = (
        " ".join(ARCH_FLAGS)
        + f" -ccbin {CXX}"
        + " -std=c++17 -O3 -lineinfo --expt-relaxed-constexpr -Xcompiler -fPIC,-Wall "
        + "-DGLB_USE_CUDA=1 "
        + common_inc
    )
    if verbose:
        nvccflags += " -Xptxas -v"
    if sanitize:
        cxxflags = cxxflags.replace("-O2 -g1", "-O1 -g") + f" -fsanitize={sanitize} -fno-omit-frame-pointer"
    pyflags = f"-I{py_inc} -I{pybind11.get_include()}"
    ldflags = (
        f"-L{CUDA_HOME}/lib64 -lcudart_static -ldl -lrt -pthread -Wl,--exclude-libs,libcudart_static.a"
    )
    if sanitize:
        ldflags += f" -fsanitize={sanitize}"

    out = []
    w = out.append
    w("ninja_required_version = 1.5")
    w(f"builddir = {BUILD}")
    w(f"cxx = {CXX}")
    w(f"nvcc = {NVCC}")
    w(f"cxxflags = {cxxflags}")
    w(f"nvccflags = {nvccflags}")
    w(f"pyflags = {pyflags}")
    w(f"ldflags = {ldflags}")
    w("")
    w("rule cxx")
    w("  command = $cxx -MMD -MF $out.d $cxxflags $extra -c $in -o $out")
    w("  depfile = $out.d")
    w("  deps = gcc")
    w("  description = CXX $in")
    w("rule nvcc")
    w("  command = $nvcc -MD -MF $out.d $nvccflags -c $in -o $out")
    w("  depfile = $out.d")
    w("  deps = gcc")
    w("  description = NVCC $in")
    w("rule link_shared")
    # link to a temporary name and rename: a reader (an importing process, a snapshot of
    # the tree) sees either the old or the new file, never a half-written one
    w("  command = $cxx -shared -o $out.tmp $in $ldflags $extra && mv -f $out.tmp $out")
    w("  description = LINK $out")
    w("rule link_exe")
    w("  command = $cxx -o $out.tmp $in $ldflags $extra && mv -f $out.tmp $out")
    w("  description = LINK $out")
    w("")

    def obj(p: Path) -> str:
        rel = p.relative_to(CSRC)
        return str(BUILD / "obj" / (str(rel).replace("/", "__") + ".o"))

    lib_objs = []
    for p in lib_cc:
        o = obj(p)
        lib_objs.append(o)
        w(f"build {o}: cxx {p}")
    for p in lib_cu:
        o = obj(p)
        lib_objs.append(o)
        w(f"build {o}: nvcc {p}")
    py_objs = []
    for p in py_cc:
        o = obj(p)
        py_objs.append(o)
        w(f"build {o}: cxx {p}")
        w("  extra = $pyflags -fvisibility=hidden")

    targets = []
    if not sanitize:
        ext = PKG / f"_C{ext_suffix()}"
        w(f"build {ext}: link_shared {' '.join(lib_objs + py_objs)}")
        targets.append(str(ext))
        lib = PKG / "lib" / "libglb.so"
        w(f"build {lib}: link_shared {' '.join(lib_objs)}")
        targets.append(str(lib))
    for name, p in bins.items():
        o = obj(p)
        w(f"build {o}: cxx {p}")
        exe = PKG / "bin" / (f"glb_{name}_{sanitize}" if sanitize else f"glb_{name}")
        w(f"build {exe}: link_exe {o} {' '.join(lib_objs)}")
        targets.append(str(exe))
    w("")
    w("default " + " ".join(targets))
    path = BUILD / "build.ninja"
    path.write_text("\n".join(out) + "\n")
    return path


def build(jobs: int | None = None, verbose: bool = False, clean: bool = False, sanitize: str = "") -> None:
    if clean and BUILD.exists():
        shutil.rmtree(BUILD)
    ninja_file = write_ninja(verbose, sanitize)
    cmd = [shutil.which("ninja") or "ninja", "-f", str(ninja_file)]
    if jobs:
        cmd += ["-j", str(jobs)]
    if verbose:
        cmd.append("-v")
    subprocess.check_call(cmd, cwd=str(ROOT))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("-j", type=int, default=None)
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--clean", action="store_true")
    ap.add_argument("--sanitize", default="", help="thread | address | undefined: build glb_benchmark_<x> only")
    a = ap.parse_args()
    build(a.j, a.verbose, a.clean, a.sanitize)
