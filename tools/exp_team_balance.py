"""Cost and effect of balanced teams (mm_set_option("team_balance")) on config3 (10 M players, 32 groups, 5v5).

Cases: both orders; rating order with and without max_spread 25 (max_spread needs rating order).  Per case the pool is
enqueued once and kept by mm_snapshot; every rep restores it and runs one host-buffer mm_tick, alternating the mask
off and on, so both settings see the same pool and the same machine state.  Reported per case:
  tick_us_off / tick_us_on   median host clock around the whole Engine.tick (kernels, balance pass, result copies)
  pass_us                    torch.profiler device time of the balance kernels (k_tb_*, and in arrival order the
                             live-slot count and scan they use) per tick, in a separate profiled run with the mask on
  sum_imbalance_off / _on    sum over all lobbies of mm_match_quality's sum_imbalance
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_team_balance.py [--reps 5]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, stats  # noqa: E402

WORKLOAD = "config3_10m_g32_5v5"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    out = {"workload": WORKLOAD, "cases": []}
    n = pkg.synth.WORKLOADS[WORKLOAD]["n"]
    for order, spread in ((pkg.abi.MM_ORDER_RATING, -1), (pkg.abi.MM_ORDER_RATING, 25), (pkg.abi.MM_ORDER_ARRIVAL, -1)):
        cfg, mode_idx = pkg.synth.workload_config(WORKLOAD, order, n)
        ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx, bell=True)
        mask = 1 << mode_idx
        rec = {"order": "rating" if order else "arrival", "max_spread": spread}
        with pkg.Engine(cfg) as e:
            if spread >= 0:
                e.set_option("max_spread", spread)
            assert e.enqueue(ids, rating, mode, ts).all()
            e.snapshot()
            host = {0: [], mask: []}
            imb = {}
            for rep in range(2 * (args.reps + 1)):  # the first pair warms up (and allocates the scratch)
                m = mask if rep & 1 else 0
                e.restore()
                e.set_option("team_balance", m)
                t0 = time.perf_counter()
                lob, _mem, _seq, st = e.tick(10_000, want_emit_seq=False)
                dt = (time.perf_counter() - t0) * 1e6
                if rep >= 2:
                    host[m].append(dt)
                q, _ = e.match_quality()
                imb[m] = (int(q["sum_imbalance"].sum()), int(q["n_lobbies"].sum()))
                rec["lobbies"] = st.n_lobbies
            assert imb[0][1] == imb[mask][1] == rec["lobbies"]
            rec["tick_us_off"], rec["tick_us_on"] = stats(host[0]), stats(host[mask])
            rec["sum_imbalance_off"], rec["sum_imbalance_on"] = imb[0][0], imb[mask][0]
            from torch.profiler import ProfilerActivity, profile
            e.set_option("team_balance", mask)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    e.restore()
                    e.tick_device(10_000)
                torch.cuda.synchronize()
            kern = {ev.key: round(ev.device_time_total / args.reps, 1) for ev in prof.key_averages()
                    if ev.device_time_total > 0 and ("k_tb_" in ev.key or "k_img_tiles" in ev.key or
                                                      "k_scan_small" in ev.key)}
            rec["pass_kernels_us"] = kern
            rec["pass_us"] = round(sum(kern.values()), 1)
        out["cases"].append(rec)
        print(json.dumps(rec), file=sys.stderr, flush=True)
    out["timing"] = ("tick_us: median host clock around a blocking Engine.tick (all 10 M member ids copied to the host), "
                     "mask off and on alternating on the same restored pool; pass_us: torch.profiler device time of "
                     "the balance kernels per tick in a separate run")
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
