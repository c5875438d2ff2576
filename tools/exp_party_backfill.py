"""Cost of a party backfill (mm_backfill_party: open team slots of running lobbies filled with whole queued parties,
then the nearest solos) beside mm_backfill on the same requests with the parties left out.

config3 (32 groups, 5v5, rating order), 10 M resident solos and 200 k queued parties of 2-4 members, no tick.  Cases:
1 000 and 10 000 requests over all queues, each with 1-5 open slots on each team.  Every measured call starts from the
same state: mm_restore of one mm_snapshot of the solos, then mm_merge_parties(MM_PARTY_KEEP_SEQ) of one party image
(not timed); mm_backfill runs on the restored solos alone, with count = the request's open slots.  Host clock over the
blocking calls (median of --calls); the device time of the kernels one call launches from torch.profiler in a separate
run, split into the table (compaction and the (bin, age) sort: k_pt_keep, k_scan_small, k_pt_move, k_pt_count,
k_pt_scatter), the plan (k_pbf_plan or k_bf_plan, k_bf_keys), the take (the band pipeline) and the output (k_bf_out,
k_pbf_pos, k_pt_out).  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_party_backfill.py [--calls 7]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, kernel_us, stats  # noqa: E402

PARTS = {"table": ("k_pt_keep", "k_scan_small", "k_pt_move", "k_pt_count", "k_pt_scatter"),
         "plan": ("k_pbf_plan", "k_bf_plan", "k_bf_keys"),
         "take": ("k_band_prep", "k_band_count", "k_band_scan", "k_band_limit", "k_band_place"),
         "out": ("k_bf_out", "k_pbf_pos", "k_pt_out")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    rng = np.random.default_rng(1)
    G = cfg.n_groups
    T, S = cfg.modes[mode_idx].teams, cfg.modes[mode_idx].team_size

    def reqs(k):
        g = rng.integers(0, G, k)
        lo = np.array([cfg.group_lo[x] for x in g])
        hi = np.array([cfg.group_hi[x] for x in g])
        room = [rng.integers(1, S + 1, T).tolist() for _ in range(k)]
        return np.full(k, mode_idx, np.int64), g, rng.integers(lo, hi + 1), room, np.full(k, -1)

    cases = {"1000": reqs(1000), "10000": reqs(10_000)}
    out = {"workload": name, "players": n}
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        e.set_option("party_capacity", 1_000_000)
        k = 200_000
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        pid = np.arange(m, dtype=np.uint64) + np.uint64(1 << 41)
        g = rng.integers(0, G, k)
        base = rng.integers([cfg.group_lo[x] for x in g], [cfg.group_hi[x] + 1 for x in g])
        prat = np.repeat(base, sizes).astype(np.int32)
        assert (e.enqueue_party(sizes, pid, prat, np.full(k, mode_idx, np.uint8),
                                np.zeros(k, np.uint32)) == 1).all()
        pimg = e.export_parties()
        e.snapshot()
        out["parties"] = k

        def fresh(parties):
            e.restore()
            if parties:
                assert (e.merge_parties(pimg, keep_seq=True) == 1).all()
            torch.cuda.synchronize()

        for label, (md, gr, tg, room, win) in cases.items():
            count = np.array([sum(r) for r in room], np.int64)
            res = {}
            for what, parties, fn in (("backfill_party", True, lambda: e.backfill_party(md, gr, tg, room, win)),
                                      ("backfill", False, lambda: e.backfill(md, gr, tg, count, win))):
                us = []
                for _ in range(args.calls + 1):  # the first call warms up
                    fresh(parties)
                    t0 = time.perf_counter()
                    r = fn()
                    us.append((time.perf_counter() - t0) * 1e6)
                fresh(parties)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn()
                    torch.cuda.synchronize()
                taken = sum(sum(f) for f in r[0]) if what == "backfill_party" else int(r[0].sum())
                res[what] = {"players_taken": int(taken), "call_us": stats(us[1:]),
                             "kernels_us": {p: kernel_us(prof, v) for p, v in PARTS.items()}}
            out[label] = res
    out["timing"] = ("host clock around the blocking calls (request upload, kernels, the counter read, the member copy); "
                     "kernels: torch.profiler device time of one call")
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
