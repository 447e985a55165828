"""Resources of the decision filter's closed-form kernels (no GPU): ``cuobjdump -res-usage`` on the built
library.  Stage 1's factored grid kernel (``filter_grid_mean_kernel<2>``) and the head stage behind it
(``filter_head_kernel<3, 2>``) keep every per-point operand in registers instead of a stack frame (local
memory goes to L2 in these kernels: they give almost all of L1 to shared memory).  The grid kernel has no
stack at all and stays within 128 registers, so that two of its 256-thread CTAs fit on an SM.  The head
kernel keeps one 8-byte spill slot: a value held across the 72-DMMA chain of its sigma bound at the 128
registers of a 512-thread CTA.  The head stage of the fp32 screening scheme runs the same closed form at every
(d_in, D) it is compiled for, within a 64-byte frame (the fp64 scheme's ``filter_head_kernel<DIN, 0>``: 480 B)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "safe_learning_b200", "libslb200.so")


def _cuobjdump():
    found = shutil.which("cuobjdump")
    if found:
        return found
    path = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    return path if os.path.exists(path) else None


@pytest.fixture(scope="module")
def usage():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs the built libslb200.so and cuobjdump")
    out = subprocess.run([tool, "-res-usage", LIB], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, check=True).stdout
    kernels = {}
    name = None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name is not None and "REG:" in line:
            kernels[name] = {k: int(v) for k, v in re.findall(r"(\w+(?:\[\d+\])?):(\d+)", line)}
            name = None
    return kernels


def _one(usage, pattern):
    hits = [v for k, v in usage.items() if re.search(pattern, k)]
    assert len(hits) == 1, "expected one kernel matching %r, found %d" % (pattern, len(hits))
    return hits[0]


def test_grid_kernel_has_no_stack_and_fits_two_ctas_per_sm(usage):
    res = _one(usage, r"filter_grid_mean_kernelILi2EE")
    assert res["STACK"] == 0 and res["LOCAL"] == 0, res
    assert res["REG"] <= 128, res


def test_closed_form_head_kernel_keeps_its_entries_in_registers(usage):
    res = _one(usage, r"filter_head_kernelILi3ELi2EE")
    assert res["STACK"] <= 8 and res["LOCAL"] == 0, res


def test_screened_head_kernels_keep_their_entries_in_registers(usage):
    shapes = {}
    for name, res in usage.items():
        m = re.search(r"filter_head_kernelILi(\d)ELi([1-9])EE", name)
        if m:
            shapes[(int(m.group(1)), int(m.group(2)))] = res
    # D = d_in - m outputs, m = 1, 2, D <= 4
    assert sorted(shapes) == [(2, 1), (3, 1), (3, 2), (4, 2), (4, 3), (5, 3), (5, 4), (6, 4)]
    for shape, res in shapes.items():
        assert res["STACK"] <= 64 and res["LOCAL"] == 0, (shape, res)
