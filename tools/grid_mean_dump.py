"""Dump the factored grid mean of stage 1 (filter_grid_mean_kernel) as raw bytes, to compare two builds.

For C2 (256 x 256 pendulum grid, two M=500 GPs on distinct factors), C2 with one shared factor, and a
70 x 83 grid whose tiles are mixed (policy gain x 3), swept over a range that starts and ends mid-row,
writes every point's probed mean mu and bound dm (slb_debug_screening_probe) and the flags to
OUT/<case>.npz.  With --compare A B it checks that two such dumps are equal byte for byte.

    python tools/grid_mean_dump.py OUT
    python tools/grid_mean_dump.py --compare A B
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

CASES = ["c2", "c2_shared", "mixed_range"]


def _case(name):
    import bench
    import bench_workloads as W
    if name == "c2":
        par = W.make_pendulum(num_points=bench.GRID, M=bench.M_TRAIN)
    elif name == "c2_shared":
        par = W.make_pendulum(num_points=bench.GRID, M=bench.M_TRAIN, shared_hypers=True)
    else:
        par = W.make_pendulum(num_points=[70, 83], M=300, tau_scale=1 / 16., seed=5)
        par["K"] = np.asarray(par["K"]) * 3.0
    gpu = W.build_product(par)
    n = gpu.sweep_descriptor().grid.nindex
    begin, end = (0, n) if name != "mixed_range" else (83 * 5 + 7, n - 40)
    return gpu, begin, end


def dump(out):
    import torch
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    os.makedirs(out, exist_ok=True)
    for name in CASES:
        gpu, begin, end = _case(name)
        assert lib.slb_filter_mean_scheme(gpu.sweep_descriptor()) == nat.MEAN_GRID_FACTORED
        n = end - begin
        mu = torch.zeros((n, 2), dtype=torch.float64, device="cuda")
        dm = torch.full((n, 2), -1.0, dtype=torch.float64, device="cuda")
        lib.slb_debug_screening_probe(mu.data_ptr(), dm.data_ptr())
        try:
            flags = gpu.compute_negative_range(begin, end).cpu().numpy().copy()
            torch.cuda.synchronize()
        finally:
            lib.slb_debug_screening_probe(None, None)
        np.savez(os.path.join(out, name + ".npz"), mu=mu.cpu().numpy(), dm=dm.cpu().numpy(), flags=flags)
        print(name, n, "points, dm finite: %.4f" % np.isfinite(dm.cpu().numpy()).mean())


def compare(a, b):
    ok = True
    for name in CASES:
        x, y = np.load(os.path.join(a, name + ".npz")), np.load(os.path.join(b, name + ".npz"))
        for key in ("mu", "dm", "flags"):
            same = x[key].tobytes() == y[key].tobytes()
            ok &= same
            print("%-12s %-6s %s" % (name, key, "identical bytes" if same else
                                     "DIFFERENT (%d of %d)" % (int((x[key] != y[key]).sum()), x[key].size)))
    return ok


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    dump(args.out)
