"""CPU-side tests (no GPU): the C-ABI library loads and exports every symbol the header
declares, the ctypes mirror matches the C layout, host-side logic agrees with the oracle, the
packed-factor index arithmetic of the sweep kernel is right (numpy emulation of the kernel's
addressing), compute calls fail loudly without a device, and the sharded (world_size 2, gloo)
prefix reduction equals the unsharded oracle."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from safe_learning_b200 import _native
    return _native.load()


def test_header_symbols_exported(lib):
    header = open(os.path.join(ROOT, "include", "slb200.h")).read()
    declared = set(re.findall(r"\b(slb_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 18
    from safe_learning_b200 import _native
    assert declared == set(_native.SIGNATURES), "binding and header disagree"
    nm = subprocess.run(["nm", "-D", "--defined-only", _native.LIB_PATH], stdout=subprocess.PIPE,
                        text=True, check=True).stdout
    exported = set(re.findall(r"\bT (slb_[a-z0-9_]+)", nm))
    assert declared <= exported, "missing exports: %s" % sorted(declared - exported)


def test_struct_layout_and_version(lib):
    from safe_learning_b200 import _native
    assert lib.slb_abi_version() == _native.ABI_VERSION == 6
    _native._check_layout(lib)
    assert lib.slb_packed_len(500) == 63 * 64 * 32
    assert lib.slb_packed_len(8) == 2 * 32
    assert lib.slb_packed_len(0) == 0
    assert lib.slb_first_fail_workspace(10 ** 6) >= 1024 * 32


def test_sm90a_tensor_instructions_in_binary(lib):
    """The GP kernel must be built for sm_90a and use the fp64 tensor pipe (DMMA)."""
    from safe_learning_b200 import _native
    out = subprocess.run(["cuobjdump", "-lelf", _native.LIB_PATH], stdout=subprocess.PIPE,
                         text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out
    # one disassembly pass, counted with grep (the text is ~350 MB: 75 kernels, 25 of them
    # instantiations of the GP tile kernel)
    counts = subprocess.run(
        "cuobjdump -sass %s | grep -o -E 'DMMA|UBLKCP.S.G|SYNCS.ARRIVE.TRANS64|"
        "SYNCS.PHASECHK.TRANS64.TRYWAIT' | sort | uniq -c" % _native.LIB_PATH, shell=True,
        stdout=subprocess.PIPE, text=True).stdout
    found = {line.split()[1]: int(line.split()[0]) for line in counts.strip().splitlines()}
    assert found.get("DMMA", 0) >= 80
    # the filter stages bring their tables into shared memory with TMA bulk copies tracked by
    # mbarrier transaction counts (cp.async.bulk -> UBLKCP, expect_tx / try_wait -> SYNCS)
    for mnemonic in ("UBLKCP.S.G", "SYNCS.ARRIVE.TRANS64", "SYNCS.PHASECHK.TRANS64.TRYWAIT"):
        assert found.get(mnemonic, 0) >= 6, (mnemonic, found)


def test_no_cpu_fallback_without_device(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    import safe_learning_b200 as sl
    from safe_learning_b200 import _native
    with pytest.raises(_native.NativeLibraryError):
        sl.QuadraticFunction(np.eye(2))(np.zeros((3, 2)))
    with pytest.raises(_native.NativeLibraryError):
        sl.Lyapunov(sl.GridWorld([[-1, 1]], 3), sl.QuadraticFunction(np.array([[1.0]])),
                    sl.LinearSystem(np.array([[1, 1.]])), 0.4, 0.3, 0.5,
                    sl.LinearSystem(np.array([[-.1]])))
    assert lib.slb_device_count() < 0 and b"no CPU fallback" in lib.slb_last_error()


def test_product_sources_never_import_oracle():
    pkg = os.path.join(ROOT, "safe_learning_b200")
    for dirpath, _, files in os.walk(pkg):
        for name in files:
            if name.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, name)).read()
                assert not re.search(r"^\s*(import|from)\s+oracle\b", text, re.M), name


def test_gridworld_host_helpers_match_oracle(lib):
    import safe_learning_b200 as sl
    rng = np.random.default_rng(0)
    for limits, num in ([[[-1.1, 1.5], [2.2, 2.4]], [7, 8]], [[[-1, 1]] * 3, [5, 9, 4]],
                        [[[0, 1]], 3]):
        a, b = sl.GridWorld(limits, num), O.GridWorld(limits, num)
        assert a.nindex == b.nindex and a.nrectangles == b.nrectangles and a.ndim == b.ndim
        assert_array_equal(a.unit_maxes, b.unit_maxes)
        assert_array_equal(a.all_points, b.all_points)
        idx = rng.integers(0, a.nindex, 50)
        assert_array_equal(a.index_to_state(idx), b.index_to_state(idx))
        lo, hi = a.limits[:, 0], a.limits[:, 1]
        pts = rng.uniform(lo - 0.2, hi + 0.2, (200, a.ndim))
        assert_array_equal(a.state_to_index(pts), b.state_to_index(pts))
        assert_array_equal(a.state_to_rectangle(pts), b.state_to_rectangle(pts))
        rect = np.arange(a.nrectangles)
        assert_array_equal(a.rectangle_to_state(rect), b.rectangle_to_state(rect))
        assert_array_equal(a.rectangle_corner_index(rect), b.rectangle_corner_index(rect))
        d = a.descriptor()
        assert d.ndim == a.ndim and d.nindex == a.nindex
        assert [d.num_points[c] for c in range(a.ndim)] == list(a.num_points)
    with pytest.raises(sl.DimensionError):
        sl.GridWorld([[0, 1]], 1)
    tri_a = sl.functions._TriangulationTables(sl.GridWorld([[-1, 1], [0, 2]], [4, 5]))
    tri_b = O.Triangulation(O.GridWorld([[-1, 1], [0, 2]], [4, 5]))
    assert_array_equal(tri_a.unit_simplices, tri_b.unit_simplices)
    assert_array_equal(tri_a.hyperplanes, tri_b.hyperplanes)


def test_utilities_match_oracle():
    from safe_learning_b200 import utilities
    k, p = utilities.dlqr(1., 1., 1., 1.)
    assert_allclose(k, 0.5 * (np.sqrt(5) - 1))
    assert_allclose(p, 0.5 * (np.sqrt(5) + 1))
    arr = np.arange(23)
    got = [(i, [v.copy() for v in views]) for i, views in utilities.batchify((arr, arr * 2), 5)]
    want = [(i, [v.copy() for v in views]) for i, views in O.batchify((arr, arr * 2), 5)]
    assert [g[0] for g in got] == [w[0] for w in want]
    for g, w in zip(got, want):
        assert_array_equal(g[1][0], w[1][0])


# ----------------------------------------------------------------- kernel addressing emulation
def _pack_factor(linv):
    """numpy twin of pack_factor_kernel (gp_sweep.cu): k-steps paired, 2 doubles per lane."""
    M = linv.shape[0]
    nrb = (M + 7) // 8
    out = np.zeros(nrb * (nrb + 1) * 32)
    for b in range(nrb):
        for kp in range(b + 1):
            base = (b * (b + 1) // 2 + kp) * 64
            for lane in range(32):
                for half in range(2):
                    row, col = 8 * b + lane // 4, 8 * kp + 4 * half + lane % 4
                    if row < M and col <= row:
                        out[base + 2 * lane + half] = linv[row, col]
    return out


def _emulate_tile(wpack, M, K):
    """Replays gp_tile_kernel's loop structure and fragment addressing (8 warps x 4 row blocks,
    panels of 256 rows/cols, bottom-up row-block dealing, per-block limits in PAIRS of k-steps)
    on the host; returns a = W k [M_pad, P] accumulated exactly where the kernel accumulates."""
    nrb, nk4 = (M + 7) // 8, (M + 3) // 4
    npan = (nrb + 31) // 32
    P = K.shape[1]
    Kpad = np.zeros((npan * 256 + 8, P))
    Kpad[:M] = K
    a = np.zeros((nrb * 8, P))
    lanes = np.arange(32)
    for ip in range(npan):
        pbeg, pend = 32 * ip, min(32 * ip + 32, nrb)
        for wslot in range(8):
            for q in range(4):
                b = pend - 1 - wslot - 8 * (3 - q)
                if b < pbeg:
                    continue
                for jp in range(ip + 1):
                    nkp = min(64, nk4 - 64 * jp)
                    npairs = (nkp + 1) // 2
                    mend = min(npairs, b - pbeg + 1) if jp == ip else npairs
                    for m in range(mend):
                        frag = wpack[(b * (b + 1) // 2 + 32 * jp + m) * 64:][:64].reshape(32, 2)
                        for half in range(2):
                            A = np.zeros((8, 4))
                            A[lanes // 4, lanes % 4] = frag[:, half]
                            r0 = 256 * jp + 8 * m + 4 * half
                            a[8 * b: 8 * b + 8] += A @ Kpad[r0:r0 + 4]
    return a


@pytest.mark.parametrize("M", [1, 5, 8, 33, 255, 256, 257, 500, 530])
def test_packed_factor_addressing(M):
    rng = np.random.default_rng(M)
    L = np.tril(rng.normal(size=(M, M))) + 3 * np.eye(M)
    linv = np.linalg.inv(L)
    linv = np.tril(linv)
    K = rng.normal(size=(M, 5))
    a = _emulate_tile(_pack_factor(linv), M, K)
    assert_allclose(a[:M], linv @ K, rtol=1e-8, atol=1e-10)
    assert np.all(a[M:] == 0)


# ----------------------------------------------------------------- sharded prefix rule (gloo)
def _numpy_first_fail(values, ok, begin):
    """numpy twin of slb_first_fail on one shard -> the int64[4] slb_fail_key row."""
    def key(v):
        v = np.where(v == 0.0, 0.0, v)
        b = v.view(np.uint64)
        return np.where(b >> np.uint64(63) == 1, ~b, b | np.uint64(1 << 63))
    kv = key(values.copy())
    fail = np.nonzero(~ok)[0]
    row = np.zeros(4, dtype=np.int64)
    row[2] = ok.sum()
    if len(fail) == 0:
        row[0], row[1] = -1, np.iinfo(np.int64).max
    else:
        order = np.lexsort((fail + begin, kv[fail]))
        row[0] = kv[fail][order[0]].astype(np.uint64).view(np.int64)
        row[1] = fail[order[0]] + begin
    return row, kv


_WORKER = r"""
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, {root!r})
sys.path.insert(0, os.path.join({root!r}, "tests"))
from test_host_and_abi import _numpy_first_fail
from safe_learning_b200 import _device as dev
from safe_learning_b200.lyapunov import combine_fail_keys, combine_prefix_stats
import oracle as O
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:{port}", rank=int(sys.argv[1]), world_size=2)
rng = np.random.default_rng(123)
for trial in range(30):
    n = int(rng.integers(3, 400))
    values = rng.integers(-2, 5, n).astype(float)
    neg = rng.random(n) < 0.97
    init = rng.random(n) < 0.1
    begin, end = dev.shard_range(n)
    row, kv = _numpy_first_fail(values[begin:end], (neg | init)[begin:end], begin)
    rows = dev.allgather_rows(torch.from_numpy(row))
    best, (kstar_v, kstar_i, n_ok) = combine_fail_keys(rows.numpy())
    idx = np.arange(begin, end)
    below = (kv < np.uint64(kstar_v)) | ((kv == np.uint64(kstar_v)) & (idx < kstar_i))
    safe_local = below | init[begin:end]
    stats = np.array([safe_local.sum(), below.sum(), 0, 0], dtype=np.int64)
    n_safe, n_below, _, _ = combine_prefix_stats(dev.allgather_rows(torch.from_numpy(stats)).numpy())
    safe_ref, p = O.prefix_rule(values, neg | init, init)
    assert np.array_equal(safe_local, safe_ref[begin:end]), (trial, "safe set")
    assert n_below == p and n_safe == safe_ref.sum() and n_ok == (neg | init).sum(), trial
dist.barrier()
dist.destroy_process_group()
print("rank", sys.argv[1], "ok")
"""


def test_sharded_prefix_rule_world2_gloo(tmp_path, lib):
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    script = tmp_path / "worker.py"
    script.write_text(_WORKER.format(root=ROOT, port=port))
    procs = [subprocess.Popen([sys.executable, str(script), str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=300)[0] for p in procs]
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d failed:\n%s" % (r, out)
        assert "ok" in out


def test_shard_ranges_cover_grid():
    from safe_learning_b200 import _device as dev
    for n in (1, 7, 64, 65536, 16777216, 101):
        for world in (1, 2, 3, 4, 8):
            spans = [dev.shard_range(n, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            for (b0, e0), (b1, e1) in zip(spans, spans[1:]):
                assert e0 == b1 and b0 <= e0


def test_kernel_algebra_normal_form_and_descriptor():
    """Host side of the covariance expressions: sums of products expand to the normal form the
    device evaluates, the descriptor carries active_dims as zero weights, and the torch
    evaluation used for the Cholesky refit equals the oracle's gpflow restatement."""
    import torch
    import oracle as O
    import bench_workloads as W
    import safe_learning_b200 as sl
    from safe_learning_b200 import _native as nat

    spec = ('["prod", ["add", ["rbf", 2, {"variance": 0.7, "lengthscales": [0.8, 1.3], "active_dims": [0, 2], '
            '"ARD": true}], ["linear", 3, {"variance": [0.1, 0.2, 0.3], "ARD": true}]], '
            '["add", ["matern32", 1, {"lengthscales": 0.6, "active_dims": [1]}], ["white", 3, {"variance": 0.01}]]]')
    k_prod, k_orc = W.build_kernel(sl, spec), W.build_kernel(O, spec)
    terms = k_prod.terms()
    assert [[type(p).__name__ for p in t] for t in terms] == [
        ["RBF", "Matern32"], ["RBF", "White"], ["Linear", "Matern32"], ["Linear", "White"]]
    X = np.random.default_rng(0).normal(size=(7, 3))
    X2 = np.random.default_rng(1).normal(size=(4, 3))
    Xt, X2t = torch.as_tensor(X), torch.as_tensor(X2)
    assert np.allclose(k_prod.K_device(Xt).numpy(), k_orc.K(X), rtol=1e-13, atol=1e-15)
    assert np.allclose(k_prod.K_device(Xt, X2t).numpy(), k_orc.K(X, X2), rtol=1e-13, atol=1e-15)
    assert np.allclose(k_prod.Kdiag_device(Xt).numpy(), k_orc.Kdiag(X), rtol=1e-13, atol=1e-15)

    desc = nat.SlbKernel()
    with pytest.raises(NotImplementedError):           # 8 primitives > SLB_MAX_KPRIM
        k_prod.fill(desc, 3)
    nb = W.build_kernel(sl, W.notebook_pendulum_kernels([[0.1, 0.2, 0.3]])[0])
    nb.fill(desc, 3)
    assert desc.num_prims == 3
    prims = [desc.prims[i] for i in range(3)]
    assert [(p.kind, p.term) for p in prims] == [(nat.K_LINEAR, 0), (nat.K_MATERN32, 1), (nat.K_LINEAR, 1)]
    assert list(prims[0].w)[:3] == [0.1, 0.2, 0.3]
    assert list(prims[1].w)[:3] == [1.0, 0.0, 0.0] and prims[1].variance == 1.0
    assert list(prims[2].w)[:3] == [0.2, 0.0, 0.0]
    with pytest.raises(sl.DimensionError):
        sl.Matern32(1, active_dims=[4]).fill(desc, 3)
    assert sl.RBF(3, lengthscales=[1., 2., 3.]).is_plain_rbf(3)
    assert not sl.RBF(2, active_dims=[0, 2]).is_plain_rbf(3)


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the CPU arm timed beside ours) prints one JSON line
    with the result keys, without touching CUDA or the reference sources."""
    import json
    import subprocess
    proc = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference",
                           "--steps", "1", "--warmup", "0"], stdout=subprocess.PIPE,
                          stderr=subprocess.PIPE, text=True, timeout=600, cwd=ROOT)
    assert proc.returncode == 0, proc.stderr[-2000:]
    line = json.loads(proc.stdout.strip().splitlines()[-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step",
                "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "e2e",
                "cpu_baseline", "impl"):
        assert key in line, key
    assert line["impl"] == "reference" and line["steps"] == 1 and line["warmup"] == 0
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["value"] == line["value"]
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["value"] > 0 and "workload" in line["config"]


def test_host_array_helpers():
    """utilities.py:252-296, 496-516 as shipped with the product (pure numpy, no GPU)."""
    from safe_learning_b200 import utilities as U
    assert_array_equal(U.combinations([np.array([1, 2]), np.array([5, 6, 7])]),
                       np.array([[1, 5], [1, 6], [1, 7], [2, 5], [2, 6], [2, 7]]))
    grid = U.linearly_spaced_combinations([(-1, 1), (0, 2)], [3, 2])
    assert_array_equal(grid, np.array([[-1, 0], [-1, 2], [0, 0], [0, 2], [1, 0], [1, 2]], dtype=float))
    assert U.linearly_spaced_combinations([(-1, 1)], 5).shape == (5, 1)
    a = np.array([[1, 1], [1, 2], [1, 3], [1, 2], [1, 3], [1, 4], [2, 3]])
    assert_array_equal(U.unique_rows(a), O.unique_rows(a))
    assert_array_equal(U.unique_rows(a), np.array([[1, 1], [1, 2], [1, 3], [1, 4], [2, 3]]))


# ----------------------------------------------------------------- adaptive branch, as written
@pytest.mark.parametrize("tau_scale,max_refinement,safety_factor,batch",
                         [(1 / 30., 4, 2.0, 64), (1 / 60., 12, 4.0, 100), (1 / 30., 8, 1.0, 10000)])
def test_adaptive_as_written_loop_matches_oracle(tau_scale, max_refinement, safety_factor, batch):
    """The host replay of lyapunov.py:540-582 (refinement_mode="reference") over per-point arrays
    equals the oracle running the reference loop state by state."""
    import bench_workloads as W
    from safe_learning_b200.lyapunov import adaptive_as_written
    par = W.make_pendulum(num_points=[26, 21], M=40, tau_scale=tau_scale)
    old = O.config.gp_batch_size
    O.config.gp_batch_size = batch
    try:
        grid, dyn = W._build(O, par, "oracle")
        policy = O.Saturation(O.LinearSystem(-par["K"]), -1., 1.)
        cpu = O.Lyapunov(grid, O.QuadraticFunction(par["P"]), dyn, par["L_dyn"],
                         O.AbsFunction(O.LinearSystem((2 * par["P"],))), par["tau"], policy,
                         initial_set=par["initial"], adaptive=True)
        states = grid.all_points
        decrease, threshold = cpu.decrease_and_threshold(states)
        coef = cpu.threshold(states, 1.0).ravel()
        with np.errstate(invalid="ignore"):
            negative = (decrease < threshold).ravel()
        safe, refinement, position = adaptive_as_written(
            cpu.values, negative, decrease.ravel(), np.ascontiguousarray(threshold).ravel(), coef,
            par["initial"], par["tau"], batch, max_refinement, max(safety_factor, 1.))
        cpu.update_safe_set(max_refinement=max_refinement, safety_factor=safety_factor,
                            refinement_mode="reference")
        assert_array_equal(safe, cpu.safe_set)
        assert_array_equal(refinement, cpu._refinement)
        assert cpu.values[O.stable_value_order(cpu.values)[position]] == cpu.c_max
    finally:
        O.config.gp_batch_size = old


def test_filter_bounds_are_certified_on_the_oracle():
    """The two facts the decision filter (csrc/filter.cu) rests on, checked with the oracle's own
    arithmetic: (1) the variance given the first R training rows is the first R rows of the same
    triangular solve and bounds the full posterior variance from above; (2) the mean through
    gamma = L^-T alpha equals a . alpha.  Also records how much of the C2 workload each stage
    decides (the numbers quoted in DESIGN.md)."""
    import scipy.linalg as sla
    import bench_workloads as W
    par = W.make_pendulum(num_points=64, M=200, shared_hypers=False)
    cpu = W.build_oracle(par)
    states = cpu.discretization.all_points
    z = np.hstack([states, cpu.policy(states)])
    mean, err = cpu.dynamics(states, cpu.policy(states))
    for j, f in enumerate(cpu.dynamics.functions):
        gp = f.gaussian_process
        L, X, s = np.asarray(gp.cholesky), np.asarray(gp.X), gp._scale
        Kx = s ** 2 * gp.kern.K(X, z)
        a = sla.solve_triangular(L, Kx, lower=True)
        full = (s ** 2 * gp.kern.Kdiag(z) - np.sum(a * a, axis=0)) / s ** 2
        assert_allclose(f.beta * np.sqrt(full), err[:, j], rtol=1e-9)
        prev = gp.kern.Kdiag(z)
        for R in (16, 64, 128, 200):
            head = (s ** 2 * gp.kern.Kdiag(z) - np.sum(a[:R] * a[:R], axis=0)) / s ** 2
            a_head = sla.solve_triangular(L[:R, :R], Kx[:R], lower=True)
            assert_allclose(a_head, a[:R], rtol=1e-7, atol=1e-12)     # same rows of the solve
            assert np.all(head <= prev * (1 + 1e-12)) and np.all(head >= full * (1 - 1e-12))
            prev = head
        gamma = sla.solve_triangular(L.T, np.asarray(gp.alpha), lower=False)
        m_gamma = (Kx.T.dot(gamma) + s * gp._mean(z)) / s
        assert_allclose(m_gamma[:, 0], mean[:, j], rtol=1e-7, atol=1e-12)


def test_filter_stage1_selection_is_host_logic():
    """slb_filter_stage1 (which first stage the filtered sweep runs) is decided on the host from the
    descriptor alone: the fp32 screening kernel needs plain RBF factors, V = QUADRATIC on at most four
    outputs (optional scale), L_V constant or LINEAR with abs / 1-norm / scale, and room for every
    factor's tables in the head stage's shared memory; everything else keeps the fp64 mean kernel."""
    from safe_learning_b200 import _native as nat
    lib = nat.load()

    def sweep(D=2, M=500, factors=None, v_kind=nat.FN_QUADRATIC, v_flags=0, l_kind=nat.FN_LINEAR,
              l_flags=nat.FLAG_ABS, l_out=None, prims=0):
        cfg = nat.SlbSweep()
        factors = D if factors is None else factors
        cfg.gp.num_outputs, cfg.gp.num_factors, cfg.gp.input_dim = D, factors, D + 1
        for f in range(factors):
            cfg.gp.factors[f].M = M
            cfg.gp.factors[f].kernel.num_prims = prims
        for o in range(D):
            cfg.gp.outputs[o].factor = min(o, factors - 1)
        cfg.lyapunov.kind, cfg.lyapunov.in_dim, cfg.lyapunov.out_dim = v_kind, D, 1
        cfg.lyapunov.flags = v_flags
        cfg.lipschitz_v.kind, cfg.lipschitz_v.in_dim = l_kind, D
        cfg.lipschitz_v.out_dim = D if l_out is None else l_out
        cfg.lipschitz_v.flags = l_flags
        return cfg

    assert lib.slb_filter_stage1(sweep()) == 32                                   # the C2 composition
    assert lib.slb_filter_stage1(sweep(l_kind=nat.FN_NONE)) == 32                 # constant L_V
    assert lib.slb_filter_stage1(sweep(l_flags=nat.FLAG_NORM1, l_out=2)) == 32
    assert lib.slb_filter_stage1(sweep(v_flags=nat.FLAG_SCALE, l_flags=nat.FLAG_ABS | nat.FLAG_SCALE)) == 32
    assert lib.slb_filter_stage1(sweep(D=4, factors=1, M=100)) == 32
    assert lib.slb_filter_stage1(sweep(v_kind=nat.FN_TRIANGULATION)) == 64        # no closed-form slack
    assert lib.slb_filter_stage1(sweep(v_flags=nat.FLAG_ABS)) == 64
    assert lib.slb_filter_stage1(sweep(l_flags=nat.FLAG_SATURATE)) == 64
    assert lib.slb_filter_stage1(sweep(l_flags=nat.FLAG_MAXABS)) == 64
    assert lib.slb_filter_stage1(sweep(prims=2)) == 64                            # covariance expression
    assert lib.slb_filter_stage1(sweep(D=5, factors=1, M=100)) == 64              # slack written out for <= 4
    assert lib.slb_filter_stage1(sweep(D=4, factors=4, M=100)) == 64              # four head factors fill the CTA
    assert lib.slb_filter_stage1(sweep(M=5000)) == 64                             # tables do not fit
    empty = nat.SlbSweep()
    assert lib.slb_filter_stage1(empty) == 0                                      # no GP
    try:
        lib.slb_debug_filter_stages(7)
        assert lib.slb_filter_stage1(sweep()) == 64                               # forced fp64 mean stage
    finally:
        lib.slb_debug_filter_stages(3)


def test_screening_bound_holds_in_a_c_restatement(tmp_path):
    """tools/screening_bound_check.c restates the fp32 screening mean of gp_mean_staged.cuh with C floats
    (worst-sign 2^-22 perturbation for ex2.approx) and holds it to the certified bound against long-double
    sums over sixteen magnitude regimes (centre up to 300 length scales from the origin, |z - centre| up to
    7): the derivation of the bound, checked without a GPU (the GPU test holds the kernel itself to it)."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    exe = str(tmp_path / "sbc")
    subprocess.run(["gcc", "-O2", "-o", exe, os.path.join(ROOT, "tools", "screening_bound_check.c"), "-lm"],
                   check=True)
    proc = subprocess.run([exe], stdout=subprocess.PIPE, text=True, timeout=300)
    assert proc.returncode == 0, proc.stdout[-2000:]
    assert "ok: every mean inside its bound" in proc.stdout


def test_screening_slack_inequalities():
    """The closed-form slack of the screening stage (filter.cu: screening_slack) rests on two inequalities
    over the box mu +- dm:  |V(mu + e) - V(mu)| <= sum_i |((P + P^T) mu)_i| dm_i + sum_ij |P_ij| dm_i dm_j
    for V = x^T P x (P need not be symmetric), and | |A (mu + e)|_j - |A mu|_j | <= sum_i |A_ji| dm_i (summed
    over j for the 1-norm form).  Checked at the corners and at random interior points of random boxes."""
    rng = np.random.default_rng(17)
    for n in (1, 2, 3, 4):
        for _ in range(50):
            P = rng.standard_normal((n, n))
            A = rng.standard_normal((n, n))
            mu = rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 1)
            dm = np.abs(rng.standard_normal(n)) * 10.0 ** rng.uniform(-8, 0)
            dv = np.abs((P + P.T) @ mu) @ dm + dm @ np.abs(P) @ dm
            rows = np.abs(A) @ dm
            corners = np.array(np.meshgrid(*[[-1.0, 1.0]] * n)).reshape(n, -1).T
            samples = np.vstack((corners, rng.uniform(-1, 1, size=(64, n)))) * dm
            for e in samples:
                x = mu + e
                # (the difference of two fp64 evaluations carries their rounding: a few ulps of |V|)
                round_off = 8e-16 * n * (abs(x) @ abs(P) @ abs(x) + abs(mu) @ abs(P) @ abs(mu))
                assert abs(x @ P @ x - mu @ P @ mu) <= dv * (1 + 1e-12) + round_off
                diff = np.abs(np.abs(A @ x) - np.abs(A @ mu))
                assert (diff <= rows * (1 + 1e-12) + 8e-16 * n * (abs(A) @ (abs(x) + abs(mu)))).all()
                assert abs(np.abs(A @ x).sum() - np.abs(A @ mu).sum()) <= (
                    rows.sum() * (1 + 1e-12) + 8e-16 * n * (abs(A) @ (abs(x) + abs(mu))).sum())
