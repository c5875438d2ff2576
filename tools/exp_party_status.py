"""Cost of the party search status calls (mm_party_queue_stats, mm_party_locate) against what they replace.

config3 (32 groups, 5v5, rating order), 10 M resident solos, queued parties of 2-4 members making up 1 % and 10 % of
the players.  Per party share:
  - mm_party_queue_stats against SearchPool.party_status's fallback path: mm_party_read (the whole table to the host)
    and its per-(mode, group) aggregation in Python;
  - mm_party_locate of 1, 1 000 and 10 000 random party members against the mm_party_match dry run (zero
    capacities: MM_E_CAP after the plan, nothing taken), which runs the same compaction, sort and plan.
Each number is the median host-clock time of the blocking call and the median device time of the same call from CUDA
events recorded on the engine's stream around it.  Prints one JSON line with the card's name and power limit, read in
the same run.  --profile instead runs each call once under torch.profiler and prints the device time per kernel (a
separate run: tracing slows the host).

    python tools/exp_party_status.py [--calls 7] [--plan-calls-10pct 1] [--profile]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, stats  # noqa: E402


def timed(stream, calls, fn):
    import torch
    host, dev = [], []
    for _ in range(calls + 1):  # the first call warms up
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record(stream)
        fn()
        b.record(stream)
        host.append((time.perf_counter() - t0) * 1e6)
        b.synchronize()
        dev.append(a.elapsed_time(b) * 1e3)
    return {"call_us": stats(host[1:]), "device_us": stats(dev[1:])}


def party_read_path(e, cfg):
    """SearchPool.party_status's fallback: the whole table to the host, then the per-queue aggregation."""
    pr = e.party_read()
    out = {}
    for m, g, s in zip(pr["mode"].tolist(), pr["group"].tolist(), pr["size"].tolist()):
        d = out.setdefault((m, g), [0, 0])
        d[0] += 1
        d[1] += s
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7)
    ap.add_argument("--plan-calls-10pct", type=int, default=1,
                    help="timed calls of the plan-bound calls at 10 %% (each runs the whole plan, seconds there)")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    abi = pkg.abi
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, abi.MM_ORDER_RATING, n)
    cfg.active_capacity = 12_000_000
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    md = int(np.asarray(mode).reshape(-1)[0])
    stream = torch.cuda.Stream()
    now = 10_000_000
    rules = {(md, g): (30, 10, 5, 5, 100) for g in range(cfg.n_groups)}
    out = {"workload": name, "solos": n}
    for share in (0.01, 0.10):
        rng = np.random.default_rng(2)
        members_want = int(n * share)
        sizes = rng.integers(2, 5, members_want // 3 + 1).astype(np.uint8)
        sizes = sizes[np.cumsum(sizes) <= members_want]
        k, m = len(sizes), int(sizes.sum())
        pid = np.arange(m, dtype=np.uint64) + np.uint64(1 << 41)
        prat = np.clip(np.repeat(rng.integers(0, 3000, k), sizes) + rng.integers(-30, 31, m), 0, 2999).astype(np.int32)
        pts = (now - rng.integers(0, 100, k)).astype(np.uint32)
        res = {"parties": k, "members": m}
        with pkg.Engine(cfg) as e:
            e.set_stream(stream.cuda_stream)
            e.set_option("party_capacity", m + 1024)
            assert e.enqueue(ids, rating, mode, ts).all()
            assert (e.enqueue_party(sizes, pid, prat, np.full(k, md, np.uint8), pts) == 1).all()
            wr = e.widen_rules(rules)
            st = abi.PartyStats()
            dry = lambda: e.lib.mm_party_match(e.h, now, wr.ctypes.data, None, 0, None, 0, C.byref(st))  # noqa: E731
            sels = {q: pid[rng.permutation(m)[:q]] for q in (1, 1000, 10_000)}
            if args.profile:
                from torch.profiler import ProfilerActivity, profile
                for label, fn in [("party_queue_stats", lambda: e.party_queue_stats(now)), ("party_match_dry", dry)] + \
                        [(f"party_locate_{q}", lambda s=s: e.party_locate(s, now, rules)) for q, s in sels.items()]:
                    fn()
                    torch.cuda.synchronize()
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        fn()
                        torch.cuda.synchronize()
                    res[label] = {ev.key: round(ev.device_time_total, 1) for ev in prof.key_averages()
                                  if ev.device_time_total > 0}
            else:
                res["party_queue_stats"] = timed(stream, args.calls, lambda: e.party_queue_stats(now))
                res["party_read_path"] = timed(stream, args.calls, lambda: party_read_path(e, cfg))
                pc = args.calls if share < 0.05 else args.plan_calls_10pct
                res["party_match_dry"] = timed(stream, pc, lambda: dry() == abi.MM_E_CAP or 1 / 0)
                for q, s in sels.items():
                    res[f"party_locate_{q}"] = timed(stream, pc, lambda s=s: e.party_locate(s, now, rules))
        out[f"parties_{int(share * 100)}pct"] = res
    out["timing"] = ("profile: device us per kernel over one call (torch.profiler)" if args.profile else
                     "call_us: host clock around the blocking call; device_us: CUDA events on the engine's stream "
                     "around the same call")
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
