"""Cost of mm_queue_stats (per-queue depth + wait histograms on the device) against today's way of getting the same
numbers: mm_pool_read (the whole pool over PCIe, sorted on the host) + numpy.

State measured: a pool of N players is ticked (the match section then covers the N players that tick read), and N
fresh players are enqueued (the waiting section covers them), so both sections stream N slots each.  Prints one JSON
line per workload with the card's name and power limit, read in the same run.

    python tools/exp_queue_stats.py [--workloads config3_10m_g32_5v5,config2_1m_g8_1v1] [--calls 200]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PKG = "microservice-matchmaking_b200"
H100_HBM_GBS = 3350.0  # NVIDIA H100 SXM data sheet, HBM3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        name, plim = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit_w": float(plim)}
    except Exception:
        return {"name": None, "power_limit_w": None}


def kernel_us(eng, now, calls):
    """Device time of k_queue_stats per call (torch.profiler, CUDA activities), in µs: (waiting + match) launch."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            eng.queue_stats(now)
        torch.cuda.synchronize()
    tot, cnt = 0.0, 0
    for ev in prof.events():
        if "k_queue_stats" in ev.name and ev.device_time_total > 0:  # the kernel's own (device-side) event
            tot += ev.device_time_total
            cnt += 1
    return (tot / cnt if cnt else None), cnt


def today(eng, cfg, now):
    """The same per-queue numbers from mm_pool_read + numpy (waiting section only: nothing else exposes the last tick)."""
    en = importlib.import_module(PKG + ".engine")
    pr = eng.pool_read()
    g = np.full(len(pr["rating"]), cfg.default_group, np.int64)
    for k in reversed(range(cfg.n_groups)):
        g[(pr["rating"] >= cfg.group_lo[k]) & (pr["rating"] <= cfg.group_hi[k])] = k
    cut = pr["mode"].astype(np.int64) * cfg.n_groups + g
    w = en.wait_of(now, pr["enq_ts"])
    n_cut = cfg.n_modes * cfg.n_groups
    cnt = np.bincount(cut, minlength=n_cut)
    mx = np.zeros(n_cut, np.int64)
    np.maximum.at(mx, cut, w)
    hist = np.bincount(cut * 120 + en.wait_bucket(w), minlength=n_cut * 120).reshape(n_cut, 120)
    return cnt, mx, hist


def run(pkg, name, calls, warmup, today_calls):
    import torch
    abi = pkg.abi
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, abi.MM_ORDER_RATING, n + 65536)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    ids2, rating2, mode2, ts2 = pkg.synth.gen_pool(2, n, first=n, mode=mode_idx)
    ts2 = ts2 + np.uint32(n)
    with pkg.Engine(cfg) as eng:
        assert eng.enqueue(ids, rating, mode, ts).all()
        now_tick = 2 * n
        _l, _m, _s, st = eng.tick(now_tick)
        assert eng.enqueue(ids2, rating2, mode2, ts2).all()
        now = 3 * n
        for _ in range(warmup):
            q = eng.queue_stats(now)
        torch.cuda.synchronize()
        host_us = []
        for _ in range(calls):
            t0 = time.perf_counter()
            q = eng.queue_stats(now)
            host_us.append((time.perf_counter() - t0) * 1e6)
        k_us, k_cnt = kernel_us(eng, now, calls)
        slots = (eng.pool_size(), st.pool_before)
        bytes_moved = 5 * sum(slots) + st.pool_before // 8  # mode 1 + ts 4 per slot and section, 1 bit per matched slot
        # today: mm_pool_read + numpy (also the check that the device numbers are right)
        cnt, mx, hist = today(eng, cfg, now)
        assert np.array_equal(q["n_waiting"], cnt) and np.array_equal(q["max_wait"], mx)
        assert np.array_equal(q["wait_hist"], hist)
        assert int(q["n_matched"].sum()) == st.n_matched and int(q["n_lobbies"].sum()) == st.n_lobbies
        today_us = []
        for _ in range(today_calls):
            t0 = time.perf_counter()
            today(eng, cfg, now)
            today_us.append((time.perf_counter() - t0) * 1e6)
    host_us = np.array(host_us)
    return {
        "workload": name, "players_waiting": slots[0], "players_last_tick": slots[1], "queues": len(q),
        "tick_device_us": st.device_us,
        "queue_stats_call_us": {"median": float(np.median(host_us)), "p10": float(np.percentile(host_us, 10)),
                                "p90": float(np.percentile(host_us, 90)), "calls": calls,
                                "timing": "host clock around mm_queue_stats (it ends in a stream synchronise)"},
        "queue_stats_kernel_us": k_us, "kernel_launches_profiled": k_cnt,
        "bytes_per_call": bytes_moved,
        "achieved_gbs": (bytes_moved / (k_us * 1e-6) / 1e9) if k_us else None,
        "datasheet_bound_us": bytes_moved / (H100_HBM_GBS * 1e9) * 1e6,
        "pool_read_plus_numpy_us": {"median": float(np.median(today_us)), "calls": today_calls,
                                    "note": "waiting section only"},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="config3_10m_g32_5v5,config2_1m_g8_1v1")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--today-calls", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    gpu = card()
    for name in args.workloads.split(","):
        r = run(pkg, name, args.calls, args.warmup, args.today_calls)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
