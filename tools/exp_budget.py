"""Cost of the lobby budget (mm_set_lobby_budget) on config3 (10 M players, 32 groups, 5v5, rating order).

Every tick starts from the same restored snapshot with L2 flushed (a 256 MiB write), as bench.py does; warm-up ticks
first; device time from mm_tick_stats.device_us, phase times from its stamps.  Measured, S0 and max_spread 2:
  budget    the tick with no budget set and with a per-mode budget of 50 %, 10 % and 0 of the candidate lobbies (0 =
            every player is a leftover of its row: the row compaction moves the whole pool)
  calls     host time of mm_lobby_candidates and mm_set_lobby_budget
  requeue   the alternative at a 50 % budget: an unbudgeted mm_tick, then mm_requeue of the surplus lobbies' members
            (host clock over both blocking calls; S0 only)
The comparison of the unbudgeted tick with the previous build is made with bench.py itself (run both builds
alternately in one session and compare their --dump-outputs files).  Prints one JSON line with the card's name and
power limit, read in the same run.

    python tools/exp_budget.py [--steps 10] [--warmup 3]
"""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    shard = importlib.import_module(pkg.__name__ + ".shard")
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, 2 * n)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, bell=True, mode=mode_idx)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out = {"workload": name, "players": n, "card": card(), "steps": args.steps}
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()  # sequence numbers = the input index
        e.snapshot()
        for policy, spread in (("S0", -1), ("S1_w2", 2)):
            e.set_option("max_spread", spread)
            cand = int(e.lobby_candidates().sum())
            res = {"candidate_lobbies": cand}
            for label, share in (("none", None), ("50%", 0.5), ("10%", 0.1), ("0", 0.0)):
                e.set_lobby_budget(per_mode=None if share is None else [int(cand * share)])
                us, ph = [], []
                for k in range(args.warmup + args.steps):
                    e.restore()
                    flush.fill_(1)
                    torch.cuda.synchronize()
                    st = e.tick_device(0)
                    if k >= args.warmup:
                        us.append(st.device_us)
                        ph.append((st.hist_us, st.scan_us, st.place_us, st.epilogue_us))
                ph = np.median(np.array(ph), axis=0)
                res[label] = {"lobbies": int(st.n_lobbies), "held_players": int(st.n_residual), "device_us": stats(us),
                              "hist_scan_place_epilogue_us": [float(x) for x in ph]}
            base, zero = res["none"], res["0"]
            held = zero["held_players"] - base["held_players"]
            res["us_per_million_held_players"] = (zero["device_us"]["median"] - base["device_us"]["median"]) / held * 1e6
            out[policy] = res
        # call times
        e.set_option("max_spread", -1)
        e.restore()
        t_c, t_s = [], []
        half = [int(e.lobby_candidates().sum()) // 2]
        for _ in range(20):
            t0 = time.perf_counter(); e.lobby_candidates(); t1 = time.perf_counter()
            e.set_lobby_budget(per_mode=half); t2 = time.perf_counter()
            t_c.append((t1 - t0) * 1e6); t_s.append((t2 - t1) * 1e6)
        out["calls_host_us"] = {"lobby_candidates": stats(t_c[5:]), "set_lobby_budget": stats(t_s[5:])}
        # the alternative: tick everything, requeue the surplus half
        alt, bud = [], []
        for k in range(2 + 3):
            e.restore()
            e.set_lobby_budget()
            t0 = time.perf_counter()
            lob, mem, _, st = e.tick(0, want_emit_seq=False)
            cand_q = np.bincount(lob["group"], minlength=cfg.n_groups)
            allot = shard.apportion(half[0], cand_q)
            q = lob["group"].astype(np.int64)
            surplus = np.arange(len(q)) - np.searchsorted(q, q, "left") >= allot[q]
            back = mem[np.repeat(surplus, 10)]
            order = np.argsort(ids)
            idx = order[np.searchsorted(ids[order], back)]
            e.requeue(back, rating[idx], mode[idx], ts[idx], idx.astype(np.uint32))
            t1 = time.perf_counter()
            e.restore()
            e.set_lobby_budget(per_mode=half)
            t2 = time.perf_counter()
            e.tick(0, want_emit_seq=False)
            t3 = time.perf_counter()
            if k >= 2:
                alt.append((t1 - t0) * 1e6); bud.append((t3 - t2) * 1e6)
        out["half_budget_host_us"] = {"tick_then_requeue_surplus": stats(alt), "budgeted_tick": stats(bud),
                                      "note": "host clock, results copied to the host in both; the requeue path includes "
                                              "finding the surplus members' columns on the host"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
