"""Cost of a queue move (mm_export_queues on the source, mm_merge on the target) against today's way of doing the
same: mm_pool_read of the whole source pool (sorted on the host), a numpy filter on the moved groups, mm_remove of
those ids on the source and mm_enqueue of them on the target.

State measured: config3 (10 M players, 32 groups, 5v5, rating order), 1/8 of the groups moved (groups 12..15, the
centre of the rating range).  Every measured move starts from the same state: the source is restored from one
mm_snapshot and the target is recreated empty, neither timed.  Host clock over the blocking calls; device time of the
kernels each call launches from torch.profiler.  Prints one JSON line with the card's name and power limit, read in
the same run.

    python tools/exp_move.py [--calls 5] [--today-calls 2]
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

EXPORT_KERNELS = ("k_img_tiles", "k_scan_small", "k_expire")
MERGE_KERNELS = ("k_img_tiles", "k_mrg_order", "k_mrg_dups", "k_enq_", "k_mrg_rejects", "k_rehash")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        name, plim = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit_w": float(plim)}
    except Exception:
        return {"name": None, "power_limit_w": None}


def stats(us):
    return {"median": float(np.median(us)), "min": float(np.min(us)), "max": float(np.max(us)), "calls": len(us)}


def kernel_us(prof, names):
    """Device time per call of the kernels whose names contain one of `names`, summed over one call."""
    tot = 0.0
    for ev in prof.events():
        if ev.device_time_total > 0 and any(k in ev.name for k in names):
            tot += ev.device_time_total
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--today-calls", type=int, default=2)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    shard = __import__("importlib").import_module("microservice-matchmaking_b200.shard")
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n + 65536)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    G = cfg.n_groups
    moved = np.arange(12, 12 + G // 8)
    mask = np.zeros((cfg.n_modes, G), bool)
    mask[:, moved] = True
    sel = np.isin(shard.group_of_rating(cfg, rating), moved)
    k = int(sel.sum())
    res = {"workload": name, "players": n, "groups_moved": len(moved), "moved_players": k}
    with pkg.Engine(cfg) as src:
        assert src.enqueue(ids, rating, mode, ts).all()
        src.snapshot()
        exp_us, mrg_us, img_bytes = [], [], 0
        for _ in range(args.calls + 1):  # the first move warms up
            src.restore()
            with pkg.Engine(cfg) as dst:
                t0 = time.perf_counter()
                img = src.export_queues(mask)
                t1 = time.perf_counter()
                rej = dst.merge_queues(img)
                t2 = time.perf_counter()
                assert len(rej) == 0 and dst.pool_size() == k
            exp_us.append((t1 - t0) * 1e6)
            mrg_us.append((t2 - t1) * 1e6)
            img_bytes = len(img)
        src.restore()
        with pkg.Engine(cfg) as dst:
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as p_exp:
                img = src.export_queues(mask)
                torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as p_mrg:
                dst.merge_queues(img)
                torch.cuda.synchronize()
        res["export_queues_us"] = stats(exp_us[1:])
        res["merge_us"] = stats(mrg_us[1:])
        res["export_kernels_us"] = kernel_us(p_exp, EXPORT_KERNELS)
        res["merge_kernels_us"] = kernel_us(p_mrg, MERGE_KERNELS)
        res["image_bytes"] = img_bytes
        res["timing"] = ("host clock around the blocking Engine.export_queues / Engine.merge_queues calls (host buffer "
                         "allocation, PCIe copies and the kernels); kernels: torch.profiler device time of one call")
        today_us = []
        for _ in range(args.today_calls):
            src.restore()
            with pkg.Engine(cfg) as dst:
                t0 = time.perf_counter()
                pr = src.pool_read()
                pick = np.isin(shard.group_of_rating(cfg, pr["rating"]), moved)
                src.remove(pr["id"][pick])
                acc = dst.enqueue(pr["id"][pick], pr["rating"][pick], pr["mode"][pick], pr["enq_ts"][pick])
                today_us.append((time.perf_counter() - t0) * 1e6)
                assert int(pick.sum()) == k and acc.all()
        res["pool_read_numpy_remove_enqueue_us"] = stats(today_us)
    res["gpu"] = card()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
