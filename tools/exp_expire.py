"""Cost of mm_expire (search timeout on the device) against today's way of doing the same: mm_pool_read (the whole
pool over PCIe, sorted on the host), a numpy filter on the waits, then mm_remove of the ids it finds.

State measured: config3 (10 M players, 32 groups, 5v5, rating order) with enqueue stamps i and now = N, so a
max_wait of N - k + 1 expires the k oldest players.  Every measured call starts from the same state (mm_snapshot once,
mm_restore before each call, not timed).  Prints one JSON line per expired fraction with the card's name and power
limit, read in the same run.

    python tools/exp_expire.py [--fractions 0,0.01,0.5,1] [--calls 20]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
H100_HBM_GBS = 3350.0  # NVIDIA H100 SXM data sheet, HBM3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        name, plim = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit_w": float(plim)}
    except Exception:
        return {"name": None, "power_limit_w": None}


def call_expire(eng, now, max_wait, ids, seq):
    n = C.c_uint32(0)
    rc = eng.lib.mm_expire(eng.h, now, max_wait, ids.ctypes.data, seq.ctypes.data, len(ids), C.byref(n))
    assert rc == 0, rc
    return n.value


def kernel_us(eng, now, max_wait, ids, seq, calls):
    """Device time of k_expire per call (torch.profiler, CUDA activities), in µs."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            eng.restore()
            call_expire(eng, now, max_wait, ids, seq)
        torch.cuda.synchronize()
    tot, cnt = 0.0, 0
    for ev in prof.events():
        if "k_expire" in ev.name and ev.device_time_total > 0:
            tot += ev.device_time_total
            cnt += 1
    return (tot / cnt if cnt else None), cnt


def today(eng, now, max_wait):
    """mm_pool_read + numpy + mm_remove: the same players leave the pool and the active set."""
    from importlib import import_module
    en = import_module("microservice-matchmaking_b200.engine")
    pr = eng.pool_read()
    gone = pr["id"][en.wait_of(now, pr["enq_ts"]) >= max_wait]
    if len(gone):
        eng.remove(gone)
    return len(gone)


def run(pkg, fraction, calls, warmup, today_calls):
    import torch
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n + 65536)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    k = int(round(fraction * n))
    now, max_wait = n, n - k + 1  # stamps i: wait n - i >= n - k + 1  <=>  i <= k - 1
    out_ids = np.empty(n, np.uint64)
    out_seq = np.empty(n, np.uint32)
    with pkg.Engine(cfg) as eng:
        assert eng.enqueue(ids, rating, mode, ts).all()
        eng.snapshot()
        for _ in range(warmup):
            eng.restore()
            assert call_expire(eng, now, max_wait, out_ids, out_seq) == k
        torch.cuda.synchronize()
        call_us = []
        for _ in range(calls):
            eng.restore()
            t0 = time.perf_counter()
            got = call_expire(eng, now, max_wait, out_ids, out_seq)
            call_us.append((time.perf_counter() - t0) * 1e6)
        assert got == k and np.array_equal(np.sort(out_ids[:got]), np.sort(ids[:k]))
        k_us, k_cnt = kernel_us(eng, now, max_wait, out_ids, out_seq, calls)
        today_us = []
        for _ in range(today_calls):
            eng.restore()
            t0 = time.perf_counter()
            assert today(eng, now, max_wait) == k
            today_us.append((time.perf_counter() - t0) * 1e6)
    bytes_read = 5 * n + 14 * k  # mode + stamp per slot; id, seq and bin per expired player (active-set probes aside)
    return {
        "workload": name, "players": n, "expired": k, "fraction": fraction,
        "expire_call_us": {"median": float(np.median(call_us)), "p10": float(np.percentile(call_us, 10)),
                           "p90": float(np.percentile(call_us, 90)), "calls": calls,
                           "timing": "host clock around mm_expire with cap = pool size (ends in a stream synchronise; "
                                     "includes copying the ids and seq to the host)"},
        "expire_kernel_us": k_us, "kernel_launches_profiled": k_cnt,
        "min_bytes_read": bytes_read,
        "datasheet_bound_us": bytes_read / (H100_HBM_GBS * 1e9) * 1e6,
        "pool_read_numpy_remove_us": {"median": float(np.median(today_us)), "calls": today_calls},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fractions", default="0,0.01,0.5,1")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--today-calls", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    gpu = card()
    for f in args.fractions.split(","):
        r = run(pkg, float(f), args.calls, args.warmup, args.today_calls)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
