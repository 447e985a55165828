"""Build libslb200.so in-tree with nvcc for sm_90a (H100) (no JIT cache, the .so travels with the repo).

Every translation unit is compiled to an object file concurrently (the GP tile kernel is one unit
per input dimension and tile size, ``gp_tile_inst.cu`` with ``-DSLB_TILE_DIN=k -DSLB_TP=t``), then linked; only units whose
sources changed are recompiled.
"""

from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJDIR = os.path.join(CSRC, "build")
OUTPUT = os.path.join(HERE, "libslb200.so")
HEADER = os.path.join(HERE, "..", "include", "slb200.h")

# (object name, source, extra flags, headers it depends on besides common.cuh / exp2_tab64.h / slb200.h)
UNITS = [("gp_tile_%d_%d.o" % (d, tp), "gp_tile_inst.cu", ["-DSLB_TILE_DIN=%d" % d, "-DSLB_TP=%d" % tp],
          ["gp_tile.cuh", "gp_args.h"]) for d in range(1, 7) for tp in (64, 32)]
UNITS += [("gp_sweep.o", "gp_sweep.cu", [], ["gp_args.h"]),
          ("filter.o", "filter.cu", [], ["bulk_copy.cuh", "exp2_tab512.cuh", "gp_mean_staged.cuh", "gp_mean_grid.cuh",
                                         "gp_args.h"]),
          ("light.o", "light.cu", [], ["bulk_copy.cuh", "exp2_tab512.cuh", "gp_mean_staged.cuh", "bellman.cuh"]),
          ("bellman_tile.o", "bellman_tile.cu", [], []),
          ("rollout.o", "rollout.cu", [], ["bulk_copy.cuh", "exp2_tab512.cuh", "gp_mean_staged.cuh", "bellman.cuh"]),
          ("value_opt.o", "value_opt.cu", [], ["bulk_copy.cuh", "exp2_tab512.cuh", "gp_mean_staged.cuh",
                                               "bellman.cuh"]),
          ("network_grad.o", "network_grad.cu", [], []),
          ("triangulation_grad.o", "triangulation_grad.cu", [], []),
          ("gp_grad.o", "gp_grad.cu", [], []),
          ("gp_hyper.o", "gp_hyper.cu", [], []),
          ("no_shrink.o", "no_shrink.cu", [], [])]
SOURCES = sorted({u[1] for u in UNITS})

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


def _mtime(path):
    return os.path.getmtime(path) if os.path.exists(path) else 0.0


def _unit_stale(unit):
    obj, src, _, headers = unit
    built = _mtime(os.path.join(OBJDIR, obj))
    deps = [os.path.join(CSRC, src), os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "exp2_tab64.h"),
            HEADER, os.path.abspath(__file__)]
    deps += [os.path.join(CSRC, h) for h in headers]
    return built == 0.0 or any(_mtime(d) > built for d in deps)


def _stale():
    if not os.path.exists(OUTPUT):
        return True
    built = os.path.getmtime(OUTPUT)
    return any(_unit_stale(u) or _mtime(os.path.join(OBJDIR, u[0])) > built for u in UNITS)


def _run(cmd, verbose):
    proc = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or proc.returncode != 0:
        sys.stderr.write(proc.stdout)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed (%s):\n%s" % (" ".join(cmd), proc.stdout))
    return proc.stdout


def build_library(force=False, verbose=False, jobs=None):
    """Compile csrc/*.cu -> libslb200.so.  Returns the output path."""
    if not force and not _stale():
        return OUTPUT
    nvcc = os.environ.get("NVCC", "nvcc")
    os.makedirs(OBJDIR, exist_ok=True)
    todo = [u for u in UNITS if force or _unit_stale(u)]
    extra = ["-Xptxas", "-v"] if verbose else []

    def compile_unit(unit):
        obj, src, flags, _ = unit
        return _run([nvcc] + CFLAGS + extra + flags + ["-c", src, "-o", os.path.join(OBJDIR, obj)],
                    verbose)

    jobs = jobs or min(len(todo) or 1, os.cpu_count() or 1)
    with ThreadPoolExecutor(max_workers=jobs) as pool:
        list(pool.map(compile_unit, todo))
    _run([nvcc, "-shared"] + ARCH + ["-o", OUTPUT] + [os.path.join(OBJDIR, u[0]) for u in UNITS],
         verbose)
    return OUTPUT


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
