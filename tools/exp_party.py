"""Cost of a party match (mm_party_match: lobbies around the parties that waited longest, the other parties of the window
placed team by team, the open slots filled with solos).

config3 (32 groups, 5v5, rating order): 10 M solos, then parties of 2 - 4 members near one rating making up 1 % and
10 % of all players, every party an anchor (min_wait 0), window 10 + 5 per 50 of wait, at most 200.  Every measured
call starts from the same state: mm_restore of one mm_snapshot of the solos (which empties the party table), then the
parties are enqueued again (not timed).  Host clock over the blocking call (median of --calls, after one warm-up call)
and the call's own device time (mm_party_stats.device_us); the kernels of one call from torch.profiler in a separate
run, split into the compaction and sort, the plan, the gather / take and the output.  The plan serves each queue's
anchors one after another in one warp, so the queue with the most anchors bounds the call.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_party.py [--calls 5]
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

PARTS = {"table": ("k_pt_keep", "k_scan_small", "k_pt_move", "k_pt_count", "k_pt_scatter", "k_pt_binsort"),
         "plan": ("k_pt_plan", "k_bf_keys"),
         "take": ("k_band_prep", "k_band_count", "k_band_scan", "k_band_limit", "k_band_place"),
         "out": ("k_wd_bases", "k_wd_hdr", "k_bf_out", "k_pt_out")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
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
    rng = np.random.default_rng(2)
    now = int(ts.max()) + 1
    out = {"workload": name, "solos": n, "card": card()}
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        e.snapshot()
        e.set_option("party_capacity", n // 4)
        rules = e.widen_rules({(mode_idx, g): (0, 10, 50, 5, 200) for g in range(cfg.n_groups)})
        dense = bool(cfg.flags & pkg.abi.MM_F_DENSE_IDS)
        for share in (0.01, 0.1):
            k = int(n * share / 0.99 / 3)  # parties of 3 on average
            sizes = rng.integers(2, 5, k).astype(np.uint8)
            m = int(sizes.sum())
            x = np.arange(n, n + m, dtype=np.uint64)
            pid = x if dense else pkg.synth.mix64(x + np.uint64(9 << 40))
            prat = np.clip(np.repeat(rng.integers(0, 5001, k), sizes) + rng.integers(-20, 21, m), 0, 5000).astype(np.int32)
            pts = (now - rng.integers(0, 60, k)).astype(np.uint32)

            def fresh():
                e.restore()
                assert (e.enqueue_party(sizes, pid, prat, np.full(k, mode_idx, np.uint8), pts) == 1).all()
                torch.cuda.synchronize()

            host_us, dev_us = [], []
            for _ in range(args.calls + 1):  # the first call warms up
                fresh()
                t0 = time.perf_counter()
                lob, mem, st = e.party_match(now, rules, lobby_cap=1 << 21, member_cap=1 << 24)
                host_us.append((time.perf_counter() - t0) * 1e6)
                dev_us.append(st.device_us)
            fresh()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                e.party_match(now, rules, lobby_cap=1 << 21, member_cap=1 << 24)
                torch.cuda.synchronize()
            out[f"parties_{share:g}"] = {
                "parties": k, "members": m, "anchors": st.n_anchors, "absorbed": st.n_absorbed,
                "lobbies": st.n_lobbies, "matched": st.n_matched, "parties_placed": st.n_parties,
                "call_us": stats(host_us[1:]), "device_us": stats(dev_us[1:]),
                "kernels_us": {kk: kernel_us(prof, v) for kk, v in PARTS.items()}}
        e.restore()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
