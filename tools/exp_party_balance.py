"""Cost and effect of balanced party lobbies (mm_set_option("party_balance"): each party lobby of a masked two-team mode
split into its most even teams, every party kept whole).

The workload of tools/exp_party.py: config3 (32 groups, 5v5, rating order), 10 M solos, then parties of 2 - 4 members
near one rating making up 1 % and 10 % of all players, every party an anchor.  Every call starts from the same state
(mm_restore of one mm_snapshot of the solos, the parties enqueued again, not timed) and runs with the 5v5 mask off and
on, alternating.  Reported per share: mm_party_stats.device_us of both (median of --calls, after one warm-up call each),
the kernel time of the balance pass alone (k_tb_pieces, k_tb_parties, k_tb_lobby) from torch.profiler in a separate
run, and the summed imbalance before and after.  "before" is computed here from the unbalanced call's members and this
tool's own ratings; "after" is sum_imbalance, checked against the same computation on the balanced call's members.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_party_balance.py [--calls 5]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, kernel_us, stats  # noqa: E402

BALANCE = ("k_tb_pieces", "k_tb_parties", "k_tb_lobby")


def imbalance(lob, mem, key, val, lo, hi, S):
    """per lobby |sum of team 1 - sum of team 2| of c = the member's own rating clamped to [lo, hi]"""
    idx = lob["first_member"].astype(np.int64)[:, None] + np.arange(2 * S)[None, :]
    c = np.clip(val[np.searchsorted(key, mem[idx])], lo, hi)
    return np.abs(c[:, :S].sum(1) - c[:, S:].sum(1))


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
    S = cfg.modes[mode_idx].team_size
    lo = min(cfg.group_lo[g] for g in range(cfg.n_groups)) - 1
    hi = max(cfg.group_hi[g] for g in range(cfg.n_groups)) + 1
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
            allid = np.concatenate([ids.astype(np.uint64), pid])
            order = np.argsort(allid)
            key, val = allid[order], np.concatenate([rating, prat]).astype(np.int64)[order]

            def call(mask):
                e.restore()
                assert (e.enqueue_party(sizes, pid, prat, np.full(k, mode_idx, np.uint8), pts) == 1).all()
                e.set_option("party_balance", mask)
                torch.cuda.synchronize()
                return e.party_match(now, rules, lobby_cap=1 << 21, member_cap=1 << 24)

            dev = {0: [], 1: []}
            res = {}
            for _ in range(args.calls + 1):  # the first call of each warms up
                for mask in (0, 1 << mode_idx):
                    res[mask] = call(mask)
                    dev[bool(mask)].append(res[mask][2].device_us)
            (lb, mb, sb), (la, ma, sa) = res[0], res[1 << mode_idx]
            assert np.array_equal(la, lb) and sb.sum_imbalance == 0
            idx = lb["first_member"].astype(np.int64)[:, None] + np.arange(2 * S)[None, :]
            assert np.array_equal(np.sort(ma[idx], 1), np.sort(mb[idx], 1))  # the same players in every lobby
            before = imbalance(lb, mb, key, val, lo, hi, S)
            after = imbalance(la, ma, key, val, lo, hi, S)
            assert int(after.sum()) == sa.sum_imbalance and (after <= before).all()
            e.restore()
            assert (e.enqueue_party(sizes, pid, prat, np.full(k, mode_idx, np.uint8), pts) == 1).all()
            e.set_option("party_balance", 1 << mode_idx)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                e.party_match(now, rules, lobby_cap=1 << 21, member_cap=1 << 24)
                torch.cuda.synchronize()
            out[f"parties_{share:g}"] = {
                "parties": k, "members": m, "lobbies": sa.n_lobbies, "parties_placed": sa.n_parties,
                "device_us_off": stats(dev[False][1:]), "device_us_on": stats(dev[True][1:]),
                "balance_kernels_us": kernel_us(prof, BALANCE),
                "sum_imbalance_before": int(before.sum()), "sum_imbalance_after": int(sa.sum_imbalance),
                "lobbies_changed": int((after < before).sum())}
        e.set_option("party_balance", 0)
        e.restore()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
