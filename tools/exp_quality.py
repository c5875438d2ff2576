"""Cost of the match-quality report (mm_match_quality) after one tick.

config2 (1 M players, 8 groups, 1v1) and config3 (10 M players, 32 groups, 5v5), both orders, S0 and S1 (rating
order only, max_spread 25).  Per case: one tick, then the median host-clock time of the blocking call (records only,
and records plus every per-lobby record) over --calls calls after one warm-up call.  With --profile, a separate run of
the same calls under torch.profiler writes the kernel times (per kernel name, averaged over the calls) to the JSON
line, and with --trace-dir one Chrome trace per case into that directory.  Prints one JSON line with the card's name
and power limit, read in the same run.

    python tools/exp_quality.py [--calls 9] [--profile [--trace-dir DIR]]
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


def cases(pkg):
    for name in ("config2_1m_g8_1v1", "config3_10m_g32_5v5"):
        for order in (pkg.abi.MM_ORDER_RATING, pkg.abi.MM_ORDER_ARRIVAL):
            for spread in ((-1, 25) if order == pkg.abi.MM_ORDER_RATING else (-1,)):
                yield name, order, spread


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=9)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--trace-dir", default=None, help="with --profile: write one Chrome trace per case here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    out = {"cases": []}
    kern = {}
    for name, order, spread in cases(pkg):
        n = pkg.synth.WORKLOADS[name]["n"]
        cfg, mode_idx = pkg.synth.workload_config(name, order, n)
        ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx, bell=True)
        with pkg.Engine(cfg) as e:
            if spread >= 0:
                e.set_option("max_spread", spread)
            assert e.enqueue(ids, rating, mode, ts).all()
            st = e.tick_device(10_000)
            rec = {"workload": name, "order": "rating" if order else "arrival", "max_spread": spread,
                   "lobbies": st.n_lobbies, "tick_us": round(st.device_us, 1)}
            for want in (False, True):
                host = []
                for _ in range(args.calls + 1):  # the first call warms up (and allocates the scratch)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    q, _l = e.match_quality(want_lobbies=want)
                    host.append((time.perf_counter() - t0) * 1e6)
                assert int(q["n_lobbies"].sum()) == st.n_lobbies
                rec["call_us_lobbies" if want else "call_us"] = stats(host[1:])
            if args.profile:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.calls):
                        e.match_quality()
                    torch.cuda.synchronize()
                key = f"{name}/{rec['order']}/{spread}"
                kern[key] = {ev.key: round(ev.device_time_total / args.calls, 1)
                             for ev in prof.key_averages() if ev.device_time_total > 0}
                if args.trace_dir:
                    os.makedirs(args.trace_dir, exist_ok=True)
                    prof.export_chrome_trace(os.path.join(args.trace_dir,
                                                          f"quality_{key.replace('/', '_')}.pt.trace.json"))
        out["cases"].append(rec)
        print(json.dumps(rec), file=sys.stderr, flush=True)
    if args.profile:
        out["kernel_us_per_call"] = kern
    out["timing"] = ("call_us: median host clock around the blocking Engine.match_quality (kernels and record copies); "
                     "kernel_us_per_call: torch.profiler device time per kernel in a separate run")
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
