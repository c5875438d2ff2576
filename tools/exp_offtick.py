"""Cost of the off-tick report's capture (mm_offtick_report, DESIGN §5): mm_widen and mm_party_match capture their
lobbies' waits and rating quality on the device, so their device_us grows by the capture; mm_offtick_report itself is
device-to-host copies.

Runs tools/exp_widen.py and tools/exp_party.py (config3, 10 M solos; widen at min_wait so that 1 % of the players
left are anchors, about the 99th percentile of the waits; parties making up 1 % of the players) on two trees in one
session, alternating them: --parent, a checkout of the parent commit with its library built, and this tree.  Then,
on this tree, the host time of mm_offtick_report after each call (median of --calls, report with the per-lobby
array).  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_offtick.py --parent DIR [--rounds 2] [--calls 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, stats  # noqa: E402


def run(tree, script, calls):
    out = subprocess.run([sys.executable, os.path.join(tree, "tools", script), "--calls", str(calls)], cwd=tree,
                         capture_output=True, text=True, check=True).stdout
    return json.loads(out.strip().splitlines()[-1])


def report_us(pkg, calls):
    """Host time of mm_offtick_report (waits, quality and per-lobby records) after one widen and one party call."""
    import torch
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    rng = np.random.default_rng(2)
    now = int(ts.max()) + 1
    out = {}
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        e.set_option("party_capacity", n // 4)
        k = int(n * 0.01 / 0.99 / 3)
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        x = np.arange(n, n + m, dtype=np.uint64)
        pid = x if cfg.flags & pkg.abi.MM_F_DENSE_IDS else pkg.synth.mix64(x + np.uint64(9 << 40))
        prat = np.clip(np.repeat(rng.integers(0, 5001, k), sizes) + rng.integers(-20, 21, m), 0, 5000).astype(np.int32)
        assert (e.enqueue_party(sizes, pid, prat, np.full(k, mode_idx, np.uint8),
                                (now - rng.integers(0, 60, k)).astype(np.uint32)) == 1).all()
        rules = e.widen_rules({(mode_idx, g): (0, 10, 50, 5, 200) for g in range(cfg.n_groups)})
        lob, _, _ = e.party_match(now, rules, lobby_cap=1 << 21, member_cap=1 << 24)
        wait = now - e.pool_read()["enq_ts"].astype(np.int64)
        min_wait = int(np.quantile(wait, 0.99))
        rules = e.widen_rules({(mode_idx, g): (min_wait, 3, 50, 5, 400) for g in range(cfg.n_groups)})
        wlob, _, _ = e.widen(now, rules, lobby_cap=1 << 20, member_cap=1 << 23)
        for key, src, nl in (("party_match", pkg.abi.MM_OFFTICK_PARTY_MATCH, len(lob)),
                             ("widen", pkg.abi.MM_OFFTICK_WIDEN, len(wlob))):
            us = []
            for _ in range(calls + 1):  # the first call warms up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e.offtick_report(src, want_lobbies=True)
                us.append((time.perf_counter() - t0) * 1e6)
            out[key] = {"lobbies": nl, "report_us": stats(us[1:])}
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
            runs[key]["widen"].append({"lobbies": w["lobbies"], "device_us": w["device_us"]["median"]})
            runs[key]["party_match"].append({"lobbies": p["lobbies"], "device_us": p["device_us"]["median"]})
    out = {"card": card(), "rounds": args.rounds}
    for call in ("widen", "party_match"):
        med = {k: float(np.median([r["device_us"] for r in runs[k][call]])) for k in trees}
        out[call] = {"lobbies": runs["branch"][call][0]["lobbies"], "parent_device_us": med["parent"],
                     "branch_device_us": med["branch"], "delta_pct": 100.0 * (med["branch"] / med["parent"] - 1.0),
                     "runs": {k: runs[k][call] for k in trees}}
    out["report"] = report_us(pkg, args.calls)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
