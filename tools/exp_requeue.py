"""Cost of a requeue (mm_requeue: the members of K lobbies back into their queues at their enqueue position) against
the nearest existing path, mm_remove + mm_enqueue of the same players with their old stamps (which puts them behind
every later arrival and gives them new sequence numbers).

States measured, config3 (32 groups, 5v5, rating order): S0 after a tick of 10 M players (each queue holds fewer than
L players); S1 (max_spread 2) after a tick of 10 M players and another 10 M enqueued, so that 10 M players are
resident.  K = 1 000 and 100 000 lobbies of the tick, chosen at random.  Every measured call starts from the same state
(mm_restore of one mm_snapshot, not timed).  Host clock over the blocking calls; device time of the kernels the call
launches from torch.profiler; the C call alone (mm_requeue on columns already in age order) beside Engine.requeue, which
sorts them first.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_requeue.py [--calls 5]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, kernel_us, stats  # noqa: E402

REQUEUE_KERNELS = ("k_rq_", "k_img_tiles", "k_scan_small", "k_img_load", "k_restamp")
TODAY_KERNELS = ("k_remove", "k_enq_", "k_scan_small", "k_rehash")


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
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, 3 * n)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    ids2, rating2, mode2, ts2 = pkg.synth.gen_pool(2, n, mode=mode_idx)
    order = np.argsort(ids)
    out = {"workload": name, "players": n}
    rng = np.random.default_rng(1)
    for policy, spread in (("S0", -1), ("S1", 2)):
        with pkg.Engine(cfg) as e:
            if spread >= 0:
                e.set_option("max_spread", spread)
            assert e.enqueue(ids, rating, mode, ts).all()  # sequence numbers 0 .. n-1 = the input index
            lob, mem, _, st = e.tick(100)
            if spread >= 0:
                assert e.enqueue(ids2, rating2, mode2, ts2).all()
            e.snapshot()
            res = {"lobbies_of_the_tick": int(st.n_lobbies), "resident": e.pool_size()}
            for K in (1000, 100_000):
                pick = rng.choice(st.n_lobbies, K, replace=False)
                first, cnt = lob["first_member"][pick].astype(np.int64), lob["n_members"][pick].astype(np.int64)
                back = np.concatenate([mem[f:f + c] for f, c in zip(first.tolist(), cnt.tolist())])
                idx = order[np.searchsorted(ids[order], back)]
                cols = (back, rating[idx], mode[idx], ts[idx], idx.astype(np.uint32))
                # the C call alone, on columns already in age order (Engine.requeue sorts them first)
                o = np.argsort(cols[4])
                raw = [np.ascontiguousarray(c[o]) for c in cols]
                codes_buf, k_out = np.empty(len(back), np.uint8), C.c_uint32(0)
                rq_us, today_us, raw_us = [], [], []
                for _ in range(args.calls + 1):
                    e.restore()
                    t0 = time.perf_counter()
                    rc = e.lib.mm_requeue(e.h, len(back), *(x.ctypes.data_as(C.c_void_p) for x in raw[:4]),
                                          raw[4].ctypes.data_as(C.c_void_p), codes_buf.ctypes.data_as(C.c_void_p),
                                          C.byref(k_out))
                    raw_us.append((time.perf_counter() - t0) * 1e6)
                    assert rc == 0 and k_out.value == len(back)
                for _ in range(args.calls + 1):  # the first call warms up
                    e.restore()
                    t0 = time.perf_counter()
                    codes = e.requeue(*cols)
                    rq_us.append((time.perf_counter() - t0) * 1e6)
                    assert (codes == 1).all()
                for _ in range(args.calls + 1):
                    e.restore()
                    t0 = time.perf_counter()
                    e.remove(back)
                    acc = e.enqueue(back, cols[1], cols[2], cols[3])
                    today_us.append((time.perf_counter() - t0) * 1e6)
                    assert acc.all()
                e.restore()
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as p_rq:
                    e.requeue(*cols)
                    torch.cuda.synchronize()
                e.restore()
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as p_today:
                    e.remove(back)
                    e.enqueue(back, cols[1], cols[2], cols[3])
                    torch.cuda.synchronize()
                res[f"K{K}"] = {"players": len(back), "requeue_us": stats(rq_us[1:]), "mm_requeue_us": stats(raw_us[1:]),
                                "requeue_kernels_us": kernel_us(p_rq, REQUEUE_KERNELS),
                                "remove_enqueue_us": stats(today_us[1:]),
                                "remove_enqueue_kernels_us": kernel_us(p_today, TODAY_KERNELS)}
            out[policy] = res
    out["timing"] = ("host clock around the blocking calls (host-to-device copies, kernels, the counter reads); kernels: "
                     "torch.profiler device time of one call")
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
