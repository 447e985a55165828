"""Small driver for ncu: builds the C2 workload and runs a few full update_safe_set steps."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench_workloads as W

shared = "--shared" in sys.argv
M = 500
for a in sys.argv:
    if a.startswith("--M="):
        M = int(a[4:])
par = W.make_pendulum(num_points=256, M=M, shared_hypers=shared)
lyap = W.build_product(par)
if "--filtered" not in sys.argv:
    lyap.filter = False        # the full posterior for every point (the round-1 kernel profile)
for _ in range(3):
    lyap.update_safe_set()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    lyap.compute_negative()
e1.record(); e1.synchronize()
print("kernel ms", e0.elapsed_time(e1) / 5, "safe", int(lyap.safe_set.sum()))

if "--phases" in sys.argv:
    import time
    import numpy as np
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    ntiles = (lyap._end - lyap._begin + 63) // 64
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    buf = torch.zeros((ntiles, 8, 8), dtype=torch.int64, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for label, pre in (("back-to-back", lambda: lyap.compute_negative()),
                       ("after 256MB fill", lambda: flush.fill_(1)),
                       ("after 5 ms idle", lambda: (torch.cuda.synchronize(), time.sleep(0.005)))):
        for _ in range(3):
            pre()
            lib.slb_debug_phase_timing(buf.data_ptr())
            lyap.compute_negative()
            torch.cuda.synchronize()
            lib.slb_debug_phase_timing(None)
        t = buf.cpu().numpy().astype(float)
        cyc, ns = t[:, 0, 3], t[:, 0, 5] - t[:, 0, 4]
        order = np.argsort(t[:, 0, 4])
        mhz = 1e3 * cyc / ns
        print(label, "| kernel span ms %.3f" % ((t[:, :, 5].max() - t[:, :, 4].min()) * 1e-6),
              "| SM MHz by tile start order: first wave %.0f, middle %.0f, last wave %.0f"
              % (mhz[order[:sms]].mean(), mhz[order[400:600]].mean(), mhz[order[-sms:]].mean()),
              "| cycles/tile %.0f" % cyc.mean(),
              "| by start decile", [int(cyc[order[i * len(order) // 10:(i + 1) * len(order) // 10]].mean() / 1000)
                                    for i in range(10)])
    print("per-tile cycles, mean over tiles, per warp: [gen, mma, epi, total, barrier-wait]")
    print(np.round(t.mean(axis=0)[:, [0, 1, 2, 3, 6]]).astype(int))

if "--flush" in sys.argv:
    import time
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    small = torch.empty(8 << 20, dtype=torch.uint8, device="cuda")
    def timed(pre, n=10):
        out = []
        for _ in range(n):
            pre()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); lyap.compute_negative(); e1.record(); e1.synchronize()
            out.append(e0.elapsed_time(e1))
        return ["%.3f" % v for v in out]
    print("no flush        ", timed(lambda: None))
    print("flush 256MB fill", timed(lambda: flush.fill_(1)))
    print("flush + sync    ", timed(lambda: (flush.fill_(1), torch.cuda.synchronize())))
    print("flush+sync+5ms  ", timed(lambda: (flush.fill_(1), torch.cuda.synchronize(), time.sleep(0.005))))
    print("sleep 5ms only  ", timed(lambda: (torch.cuda.synchronize(), time.sleep(0.005))))
    print("small 8MB fill  ", timed(lambda: small.fill_(1)))
    rd = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print("flush by read   ", timed(lambda: rd.sum()))
    print("flush, 1 untimed sweep, then timed", timed(lambda: (flush.fill_(1), lyap.compute_negative())))
    print("flush 64MB      ", timed(lambda: flush[:64 << 20].fill_(1)))
    print("flush 128MB     ", timed(lambda: flush[:128 << 20].fill_(1)))
    A64 = torch.randn(2048, 2048, dtype=torch.float64, device="cuda")
    print("fill + fp64 matmul 2048^3 (cuBLAS DMMA)", timed(lambda: (flush.fill_(1), torch.matmul(A64, A64))))
    print("fp64 matmul only (no fill)", timed(lambda: torch.matmul(A64, A64)))
    warm = torch.zeros(1 << 20, dtype=torch.float64, device="cuda")
    print("fill + 8MB elementwise compute", timed(lambda: (flush.fill_(1), warm.mul_(1.0001).add_(1.0))))
