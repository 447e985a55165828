"""Resources of the refine pass on the filter's closed form (no GPU: ``cuobjdump -res-usage`` on the built
library).  ``gp_tile_closed_kernel<3, 2, TP>`` takes its per-point terms from stage 1's list A entries and
finishes its tiles with the register-only evaluators, so neither the interpreter nor its stack frame is linked
into it: no stack and no local memory at either tile size (the generic ``gp_tile_kernel`` keeps its frame)."""
import pytest

from test_stage_kernel_resources_host import _one, usage  # noqa: F401


@pytest.mark.parametrize("tp", [32, 64])
def test_closed_form_refine_kernel_has_no_stack(usage, tp):  # noqa: F811
    res = _one(usage, r"gp_tile_closed_kernelILi3ELi2ELi%dEE" % tp)
    assert res["STACK"] == 0 and res["LOCAL"] == 0, res
