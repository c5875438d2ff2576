"""Cost of a party requeue (mm_requeue_party: matched parties back into the party table at their age position).

config3 (32 groups, 5v5, rating order): 10 M solos, then parties of 2 - 4 members near one rating making up 1 % of all
players, matched by one mm_party_match (every party an anchor, window 10 + 5 per 50 of wait, at most 200).  Then 1,
1 000 and 10 000 of the matched parties are requeued in one call, with the columns the caller kept (party_read before
the match).  Every measured call starts from the same state: mm_restore of one mm_snapshot of the solos (which empties
the party table), the parties enqueued again and matched (not timed).  Host clock over the blocking call and CUDA
events recorded on the default stream around it (median of --calls, after one warm-up call); the kernels of one call
from torch.profiler in a separate run.  Prints one JSON line with the card's name and power limit, read in the same
run.

    python tools/exp_party_requeue.py [--calls 5]
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

KERNELS = ("k_pq_check", "k_pq_party", "k_scan_small", "k_pt_keep", "k_pq_seat", "k_pq_move", "k_pq_write")


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
        k = int(n * 0.01 / 0.99 / 3)  # parties of 3 on average
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        x = np.arange(n, n + m, dtype=np.uint64)
        pid = x if dense else pkg.synth.mix64(x + np.uint64(9 << 40))
        prat = np.clip(np.repeat(rng.integers(0, 5001, k), sizes) + rng.integers(-20, 21, m), 0, 5000).astype(np.int32)
        pts = (now - rng.integers(0, 60, k)).astype(np.uint32)
        out["parties"], out["members"] = k, m

        def matched():
            """restore, enqueue, match -> the matched parties' columns as the caller kept them, in age order"""
            e.restore()
            assert (e.enqueue_party(sizes, pid, prat, np.full(k, mode_idx, np.uint8), pts) == 1).all()
            pr = e.party_read()
            _lob, mem, _st = e.party_match(now, rules, lobby_cap=1 << 21, member_cap=1 << 24)
            placed = set(mem.tolist())
            sel = [j for j, (mi, _mr) in enumerate(pr["members"]) if int(mi[0]) in placed]
            torch.cuda.synchronize()
            return pr, sel

        for want in (1, 1000, 10_000):
            host_us, ev_us = [], []
            for _ in range(args.calls + 1):  # the first call warms up
                pr, sel = matched()
                sel = sel[:want]
                cols = (pr["size"][sel], np.concatenate([pr["members"][j][0] for j in sel]),
                        np.concatenate([pr["members"][j][1] for j in sel]), pr["mode"][sel], pr["enq_ts"][sel],
                        pr["seq"][sel])
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                t0 = time.perf_counter()
                codes = e.requeue_party(*cols)
                host_us.append((time.perf_counter() - t0) * 1e6)
                b.record()
                torch.cuda.synchronize()
                ev_us.append(a.elapsed_time(b) * 1000.0)
                assert (codes == 1).all() and len(codes) == want
            rows = len(e.party_read()["size"])
            pr, sel = matched()
            sel = sel[:want]
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                e.requeue_party(pr["size"][sel], np.concatenate([pr["members"][j][0] for j in sel]),
                                np.concatenate([pr["members"][j][1] for j in sel]), pr["mode"][sel],
                                pr["enq_ts"][sel], pr["seq"][sel])
                torch.cuda.synchronize()
            out[f"requeue_{want}"] = {"table_rows_after": rows, "call_us": stats(host_us[1:]),
                                      "event_us": stats(ev_us[1:]), "kernels_us": kernel_us(prof, KERNELS)}
        e.restore()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
