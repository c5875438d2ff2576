"""Cost of the off-tick budget (mm_set_offtick_budget, DESIGN §5): a budgeted mm_widen / mm_party_match runs one
single-CTA allowance kernel after its plan, and when an allowance falls short of its queue's lobbies the plan runs
again, capped.

config3 (32 groups, 5v5, rating order), 10 M solos:
  - no budget: tools/exp_widen.py and tools/exp_party.py on two trees in one session, alternating them (--parent, a
    checkout of the parent commit with its library built, and this tree); widen at 1 % anchors, parties making up 1 %
    of the players (the setups of DESIGN §5 "Widening search cost" and "Party match cost");
  - on this tree, the same two setups under a per-queue budget that binds (half of every queue's lobbies) and a
    per-mode budget that binds (a third of the mode's lobbies): host clock over the blocking call and the call's
    device_us, median of --calls after one warm-up call, every call from the same state; then the kernels of one call
    of each from torch.profiler in a separate run.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_offtick_budget.py --parent DIR [--rounds 2] [--calls 5]
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
from exp_offtick import run  # noqa: E402

PARTS = {"plan": ("k_wd_plan", "k_pt_plan"), "allot": ("k_wd_allot",), "keys": ("k_bf_keys",),
         "take": ("k_band_prep", "k_band_count", "k_band_scan", "k_band_limit", "k_band_place"),
         "out": ("k_wd_bases", "k_wd_hdr", "k_bf_out", "k_pt_out")}


def budgets(pkg, e, source, cfg, reset, call):
    """{variant: (per_queue, per_mode)} from an unbudgeted call's per-queue counts."""
    reset()
    call()
    cand, _ = e.offtick_budget_report(source)
    return {"none": (None, None), "queue_binding": (cand // 2, None),
            "mode_binding": (None, [int(cand.sum()) // 3] * cfg.n_modes)}


def measure(e, source, variants, reset, call, calls):
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for key, (pq, pm) in variants.items():
        print(f"source {source}: {key}", file=sys.stderr, flush=True)
        e.set_offtick_budget(source, per_queue=pq, per_mode=pm)
        host_us, dev_us = [], []
        for _ in range(calls + 1):  # the first call warms up
            reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            lob, _mem, st = call()
            host_us.append((time.perf_counter() - t0) * 1e6)
            dev_us.append(st.device_us)
        cand, emitted = e.offtick_budget_report(source)
        reset()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        out[key] = {"candidates": int(cand.sum()), "lobbies": len(lob), "call_us": stats(host_us[1:]),
                    "device_us": stats(dev_us[1:]), "kernels_us": {k: kernel_us(prof, v) for k, v in PARTS.items()}}
    e.set_offtick_budget(source)
    return out


def budgeted(pkg, calls):
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    now = int(ts.max()) + 1
    out = {}
    with pkg.Engine(cfg) as e:  # widen: exp_widen.py's setup at 1 % anchors
        assert e.enqueue(ids, rating, mode, ts).all()
        e.set_option("max_spread", 2)
        e.set_lobby_budget(per_queue=[1000] * cfg.n_groups)
        e.tick(now)
        wait = now - e.pool_read()["enq_ts"].astype(np.int64)
        e.snapshot()
        rules = e.widen_rules({(mode_idx, g): (int(np.quantile(wait, 0.99)), 3, 50, 5, 400)
                               for g in range(cfg.n_groups)})
        call = lambda: e.widen(now, rules, lobby_cap=1 << 20, member_cap=1 << 23)  # noqa: E731
        src = pkg.abi.MM_OFFTICK_WIDEN
        out["widen"] = measure(e, src, budgets(pkg, e, src, cfg, e.restore, call), e.restore, call, calls)
    rng = np.random.default_rng(2)
    with pkg.Engine(cfg) as e:  # party_match: exp_party.py's setup, parties making up 1 % of the players
        assert e.enqueue(ids, rating, mode, ts).all()
        e.snapshot()
        e.set_option("party_capacity", n // 4)
        k = int(n * 0.01 / 0.99 / 3)
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        x = np.arange(n, n + m, dtype=np.uint64)
        pid = x if cfg.flags & pkg.abi.MM_F_DENSE_IDS else pkg.synth.mix64(x + np.uint64(9 << 40))
        prat = np.clip(np.repeat(rng.integers(0, 5001, k), sizes) + rng.integers(-20, 21, m), 0, 5000).astype(np.int32)
        pts = (now - rng.integers(0, 60, k)).astype(np.uint32)
        pmode = np.full(k, mode_idx, np.uint8)

        def reset():  # mm_restore empties the party table; the parties go in again
            e.restore()
            assert (e.enqueue_party(sizes, pid, prat, pmode, pts) == 1).all()

        rules = e.widen_rules({(mode_idx, g): (0, 10, 50, 5, 200) for g in range(cfg.n_groups)})
        call = lambda: e.party_match(now, rules, lobby_cap=1 << 21, member_cap=1 << 24)  # noqa: E731
        src = pkg.abi.MM_OFFTICK_PARTY_MATCH
        out["party_match"] = measure(e, src, budgets(pkg, e, src, cfg, reset, call), reset, call, calls)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="a checkout of the parent commit with its library built")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--calls", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    trees = {"parent": os.path.abspath(args.parent), "branch": ROOT}
    runs = {k: {"widen": [], "party_match": []} for k in trees}
    for _ in range(args.rounds):
        for key, tree in trees.items():  # alternating: parent, branch, parent, branch, ...
            w = run(tree, "exp_widen.py", args.calls)["anchors_0.01"]
            p = run(tree, "exp_party.py", args.calls)["parties_0.01"]
            runs[key]["widen"].append({"lobbies": w["lobbies"], "device_us": w["device_us"]["median"],
                                       "call_us": w["call_us"]["median"]})
            runs[key]["party_match"].append({"lobbies": p["lobbies"], "device_us": p["device_us"]["median"],
                                             "call_us": p["call_us"]["median"]})
            print(f"{key}: widen {w['device_us']['median']:.0f} us, party_match {p['device_us']['median']:.0f} us",
                  file=sys.stderr, flush=True)
    out = {"card": card(), "rounds": args.rounds, "no_budget": {}}
    for call in ("widen", "party_match"):
        med = {k: float(np.median([r["device_us"] for r in runs[k][call]])) for k in trees}
        out["no_budget"][call] = {"parent_device_us": med["parent"], "branch_device_us": med["branch"],
                                  "delta_pct": 100.0 * (med["branch"] / med["parent"] - 1.0),
                                  "runs": {k: runs[k][call] for k in trees}}
    out["budgeted"] = budgeted(pkg, args.calls)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
