"""Resources of the LML gradient's tile kernels (no GPU): ``cuobjdump -res-usage`` on the built library.  Both
instantiations, the one-column ``gp_lml_grad_tile_kernel<DIN, false>`` and the k-column ``<DIN, true>``, run
without a stack or local memory at every d_in, and stay within the 255 registers that
``__launch_bounds__(128, 2)`` allows.  The k-column kernel stages SLB_MAX_OUT alpha columns per panel where the
one-column kernel stages one: 5 KB more shared memory, nothing else."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "safe_learning_b200", "libslb200.so")


@pytest.fixture(scope="module")
def usage():
    tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                                     "cuobjdump")
    if not os.path.exists(tool) or not os.path.exists(LIB):
        pytest.skip("needs the built libslb200.so and cuobjdump")
    out = subprocess.run([tool, "-res-usage", LIB], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, check=True).stdout
    kernels, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name is not None and "REG:" in line:
            kernels[name] = {k: int(v) for k, v in re.findall(r"(\w+(?:\[\d+\])?):(\d+)", line)}
            name = None
    return kernels


def _one(usage, din, cols):
    pattern = r"gp_lml_grad_tile_kernelILi%dELb%dE" % (din, int(cols))
    hits = [v for k, v in usage.items() if re.search(pattern, k)]
    assert len(hits) == 1, "expected one kernel matching %r, found %d" % (pattern, len(hits))
    return hits[0]


@pytest.mark.parametrize("din", range(1, 7))
def test_tile_kernels_have_no_stack(usage, din):
    one, cols = _one(usage, din, False), _one(usage, din, True)
    for res in (one, cols):
        assert res["STACK"] == 0 and res["LOCAL"] == 0, res
        assert res["REG"] <= 255, res
    # the k-column kernel stages 6 alpha columns per panel where the one-column kernel stages 1
    assert cols["SHARED"] - one["SHARED"] == 2 * 64 * (6 - 1) * 8, (one, cols)
