"""Cost of the cross-group boundary pass: shard.boundary_pass (the host path: mm_pool_read of the whole pool, numpy
band selection, one band engine per boundary, np.isin + mm_take) against shard.boundary_pass_device
(mm_band_candidates / mm_band_match on the device).

Geometry of config3: 32 groups, 5v5, rating order, W = 2, 10 M players, K = 1 or K engines on one GPU (one thread per
rank, LocalComm).  Two states, each restored from one mm_snapshot per rank before every measured pass:
  tick    the pool left after a local S1 tick (max_spread = W) of the 10 M players;
  notick  the 10 M players with no tick first: about 2W/157 of the pool (~250 k players) are band candidates.
Host clock over the whole pass (all ranks); device time of the band kernels from torch.profiler over one device pass.
Prints one JSON line per (state, K) with the card's name and power limit, read in the same run.

    python tools/exp_boundary.py [--ks 1,4] [--calls 3] [--host-calls 1]
"""
import argparse
import importlib
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.exp_move import card, stats  # noqa: E402

BAND_KERNELS = ("k_band_",)


def run_ranks(K, fn):
    out, errs = [None] * K, []

    def work(r):
        try:
            out[r] = fn(r)
        except BaseException as ex:  # noqa: BLE001
            errs.append(ex)

    th = [threading.Thread(target=work, args=(r,)) for r in range(K)]
    [t.start() for t in th]
    [t.join() for t in th]
    if errs:
        raise errs[0]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--ks", default="1,4")
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--host-calls", type=int, default=1)
    ap.add_argument("--states", default="tick,notick")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    import __graft_entry__
    pkg = __graft_entry__.build()
    shard = importlib.import_module("microservice-matchmaking_b200.shard")
    W, n = 2, args.n
    cfg = pkg.synth.make_config(n_groups=32, modes=(("5v5", 2, 5),), order=pkg.abi.MM_ORDER_RATING, capacity=n)
    ids, rating, mode, ts = pkg.synth.gen_pool(3, n)
    info = card()
    for state in args.states.split(","):
        for K in [int(k) for k in args.ks.split(",")]:
            owner = shard.route(cfg, rating, K)
            engines = []
            for r in range(K):
                mine = owner == r
                c = type(cfg).from_buffer_copy(cfg)
                c.capacity = int(mine.sum()) + 16
                eng = pkg.Engine(c)
                eng.set_option("max_spread", W)
                eng.enqueue(ids[mine], rating[mine], mode[mine], ts[mine])
                if state == "tick":
                    eng.tick()
                eng.snapshot()
                engines.append(eng)

            def one(device):
                for e in engines:
                    e.restore()
                torch.cuda.synchronize()
                comm = shard.LocalComm()
                fn = shard.boundary_pass_device if device else shard.boundary_pass
                t0 = time.perf_counter()
                res = run_ranks(K, lambda r: fn(pkg, cfg, W, K, r, engines[r], comm))
                return (time.perf_counter() - t0) * 1e6, res

            host_us, dev_us = [], []
            for _ in range(args.host_calls):
                us, host_res = one(False)
                host_us.append(us)
            for _ in range(args.calls):
                us, dev_res = one(True)
                dev_us.append(us)
            same = all(
                (h["hdr"] is None and d["hdr"] is None or np.array_equal(h["hdr"], d["hdr"]))
                and np.array_equal(h["member_ids"], d["member_ids"])
                and all(h[k] == d[k] for k in ("sent", "received", "matched", "lobbies"))
                for h, d in zip(host_res, dev_res))
            for e in engines:
                e.restore()
            torch.cuda.synchronize()
            pcomm = shard.LocalComm()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run_ranks(K, lambda r: shard.boundary_pass_device(pkg, cfg, W, K, r, engines[r], pcomm))
                torch.cuda.synchronize()
            kern = {}
            for ev in prof.key_averages():
                if ev.device_time_total > 0 and any(k in ev.key for k in BAND_KERNELS):
                    name = ev.key.split("(")[0].split("<")[0].replace("void ", "").replace("mm::", "")
                    kern[name] = kern.get(name, 0.0) + ev.device_time_total
            for e in engines:
                e.close()
            print(json.dumps({"experiment": "boundary_pass", "card": info, "state": state, "n": n, "K": K, "W": W,
                              "groups": 32, "sent": int(sum(d["sent"] for d in dev_res)),
                              "matched": int(sum(d["matched"] for d in dev_res)),
                              "lobbies": int(sum(d["lobbies"] for d in dev_res)), "equal": bool(same),
                              "host_pass_us": stats(host_us), "device_pass_us": stats(dev_us),
                              "band_kernels_us": kern}), flush=True)


if __name__ == "__main__":
    main()
