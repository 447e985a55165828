"""Worker for the multi-GPU test of optimize_value_function: one process per GPU (NCCL).  Every
rank assembles and solves the whole system; the tables must be identical on all ranks."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

local_rank = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local_rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
rank, world = dist.get_rank(), dist.get_world_size()

import safe_learning_b200 as sl  # noqa: E402
import value_opt_oracle as V  # noqa: E402

rl, grid = V.gp55_objects(sl, "product")
assert (rl._begin, rl._end) != (0, grid.nindex)           # the grid is sharded for the sweeps
for _ in range(2):
    values = rl.optimize_value_function()
    table = torch.as_tensor(values, device="cuda").reshape(-1)
    gathered = [torch.empty_like(table) for _ in range(world)]
    dist.all_gather(gathered, table)
    for other in gathered:
        assert torch.equal(other, table), rank
    assert np.array_equal(rl.value_function.parameters[0], values)

dist.barrier()
if rank == 0:
    print("value_opt dist worker ok, world", world)
dist.destroy_process_group()
