"""Cost of deploying another config without dropping the queue: mm_import_regroup of a config3 image (10 M queued
players, 32 equal-width rating groups, 5v5, rating order) into engines with
  (a) 24 equal-width groups, (b) 32 groups cut at the population's quantiles, (c) the 32 groups and one more mode,
beside mm_export, mm_import of the same image under the same config, and the host alternative (mm_pool_read of the
whole pool and mm_enqueue into a fresh engine, which gives every player a new sequence number), run once.

Host clock around the blocking calls; every engine is created before its clock starts.  The regrouped pools are checked
against the host alternative's (pool_read: ids, ratings, modes and stamps in the same order) and every repeated call
against the first (the export's bytes).  --profile runs, in a process of its own, one call of each with torch.profiler
and prints the device time per kernel.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_regroup.py [--calls 5] [--profile]
"""
import argparse
import json
import os
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, stats  # noqa: E402


def configs(pkg, cfg, rating):
    def copy(**groups):
        c = type(cfg).from_buffer_copy(cfg)
        if groups:
            g = groups["groups"]
            c.n_groups = len(g)
            for k, (lo, hi) in enumerate(g):
                c.group_lo[k], c.group_hi[k] = lo, hi
            c.default_group = len(g) // 2 + 1 if len(g) // 2 + 1 < len(g) else -1
        return c
    los, his = pkg.synth.equal_width_groups(24)
    cuts = np.unique(np.clip(np.quantile(rating, np.linspace(0, 1, 33)[1:-1]).astype(np.int64), 1, 4999))
    balanced = list(zip(np.r_[0, cuts[:-1] + 1].tolist(), cuts.tolist())) + [(int(cuts[-1]) + 1, 5000)]
    c = copy()
    c.modes[c.n_modes].teams, c.modes[c.n_modes].team_size = 2, 1
    c.n_modes += 1
    return {"a_24_equal": copy(groups=list(zip(los, his))), "b_balanced": copy(groups=balanced), "c_mode_added": c}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n + 65536)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    targets = configs(pkg, cfg, rating)
    out = {"workload": name, "players": n, "groups": {k: int(c.n_groups) for k, c in targets.items()}}
    with pkg.Engine(cfg) as src:
        assert src.enqueue(ids, rating, mode, ts).all()
        img = src.export_state()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            prof = {}
            for k, c in [("regroup_same_config", cfg)] + list(targets.items()):
                with pkg.Engine(c) as e:
                    e.import_regroup(img)  # warm-up: module load, first launches
                with pkg.Engine(c) as e:
                    torch.cuda.synchronize()
                    with profile(activities=[ProfilerActivity.CUDA]) as p:
                        e.import_regroup(img)
                        torch.cuda.synchronize()
                    per = {}
                    for ev in p.events():
                        if ev.device_time_total > 0:
                            per[ev.name] = per.get(ev.name, 0.0) + ev.device_time_total
                    prof[k] = {kk: round(v, 1) for kk, v in sorted(per.items(), key=lambda kv: -kv[1])}
            out["kernels_us"] = prof
            out["gpu"] = card()
            print(json.dumps(out), flush=True)
            return
        exp_us = []
        for _ in range(args.calls + 1):
            t0 = time.perf_counter()
            again = src.export_state()
            exp_us.append((time.perf_counter() - t0) * 1e6)
            assert np.array_equal(again, img)
        out["mm_export_us"] = stats(exp_us[1:])
        out["image_bytes"] = int(len(img))

    def timed(c, call):
        us, digest = [], None
        for _ in range(args.calls + 1):  # the first call warms up
            with pkg.Engine(c) as e:
                t0 = time.perf_counter()
                call(e)
                us.append((time.perf_counter() - t0) * 1e6)
                d = zlib.crc32(e.export_state().tobytes())
                assert digest in (None, d)
                digest = d
        return stats(us[1:])

    out["mm_import_same_config_us"] = timed(cfg, lambda e: e.import_state(img))
    for k, c in targets.items():
        out[f"mm_import_regroup_{k}_us"] = timed(c, lambda e: e.import_regroup(img))
    # the host alternative, once, into (a): the whole pool read back and enqueued (new sequence numbers)
    c = targets["a_24_equal"]
    with pkg.Engine(cfg) as src2:
        src2.import_state(img)
        with pkg.Engine(c) as e:
            t0 = time.perf_counter()
            rd = src2.pool_read()
            assert e.enqueue(rd["id"], rd["rating"], rd["mode"], rd["enq_ts"]).all()
            out["host_pool_read_enqueue_us"] = (time.perf_counter() - t0) * 1e6
            host = e.pool_read()
    with pkg.Engine(c) as e:
        assert len(e.import_regroup(img)) == 0
        got = e.pool_read()
        for f in ("id", "rating", "mode", "enq_ts"):
            assert np.array_equal(got[f], host[f]), f
    out["checked"] = "repeated calls give the same export; regroup (a) pool_read == host alternative's"
    out["timing"] = "host clock around the blocking call (image upload, kernels, counter read, load), engine created before"
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
