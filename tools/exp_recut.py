"""Cost of re-cutting a sharded deployment (shard.recut, mm_import_regroup_many): config3 (10 M queued players, 5v5,
rating order, 32 equal-width groups) on K = 4 engines of one GPU, groups owned by balanced_owners of the queue depths,
re-cut into (a) 24 equal-width groups and (b) 32 groups cut at the population's quantiles, new owners by
balanced_owners again.  Beside it, the host alternative: every rank reads its pool back (mm_pool_read) and the players
are enqueued into the new ranks' engines by route(), which gives every player a new sequence number.

Host clock around shard.recut (the four ranks as threads over LocalComm: export, exchange, new engines, import, status
exchange, swap); the source engines are rebuilt from their images before each call, outside the clock.  --profile
runs one re-cut per target under torch.profiler and prints the device time per kernel and of the host-to-device
copies.  Every re-cut is checked against the first (the new ranks' export bytes).  Prints one JSON line with the
card's name and power limit, read in the same run.

    python tools/exp_recut.py [--calls 3] [--profile]
"""
import argparse
import importlib
import json
import os
import sys
import threading
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, stats  # noqa: E402

K = 4


def targets(pkg, cfg, rating):
    def copy(groups):
        c = type(cfg).from_buffer_copy(cfg)
        c.n_groups = len(groups)
        for k, (lo, hi) in enumerate(groups):
            c.group_lo[k], c.group_hi[k] = lo, hi
        c.default_group = -1
        return c
    los, his = pkg.synth.equal_width_groups(24)
    cuts = np.unique(np.clip(np.quantile(rating, np.linspace(0, 1, 33)[1:-1]).astype(np.int64), 1, 4999))
    balanced = list(zip(np.r_[0, cuts[:-1] + 1].tolist(), cuts.tolist())) + [(int(cuts[-1]) + 1, 5000)]
    return {"a_24_equal": copy(list(zip(los, his))), "b_quantile": copy(balanced)}


def on_ranks(fn):
    out, errs = [None] * K, []

    def one(r):
        try:
            out[r] = fn(r)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=one, args=(r,)) for r in range(K)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errs:
        raise errs[0]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    shard = importlib.import_module(ge.PKG + ".shard")
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n + 65536)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    grp = shard.group_of_rating(cfg, rating)
    old_own = shard.balanced_owners(np.bincount(grp, minlength=cfg.n_groups), K)
    to = old_own[grp]
    images = []
    for r in range(K):
        with pkg.Engine(cfg) as e:
            s = to == r
            assert e.enqueue(ids[s], rating[s], mode[s], ts[s]).all()
            images.append(e.export_state())
    out = {"workload": name, "players": n, "ranks": K, "image_bytes": [int(len(i)) for i in images]}

    def sources():
        engines = [pkg.Engine(cfg) for _ in range(K)]
        for e, img in zip(engines, images):
            e.import_state(img)
        torch.cuda.synchronize()
        return engines

    def recut(new, new_own, engines):
        comm = shard.LocalComm()
        return on_ranks(lambda r: shard.recut(pkg, cfg, new, old_own, new_own, r, engines[r], comm))

    tg = targets(pkg, cfg, rating)
    owners = {k: shard.balanced_owners(np.bincount(shard.group_of_rating(c, rating), minlength=c.n_groups), K)
              for k, c in tg.items()}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        prof = {}
        for k, c in tg.items():
            for warm in (True, False):
                engines = sources()
                torch.cuda.synchronize()
                if warm:  # module load, first launches
                    res = recut(c, owners[k], engines)
                else:
                    with profile(activities=[ProfilerActivity.CUDA]) as p:
                        res = recut(c, owners[k], engines)
                        torch.cuda.synchronize()
                    per = {}
                    for ev in p.events():
                        if ev.device_time_total > 0:
                            per[ev.name] = per.get(ev.name, 0.0) + ev.device_time_total
                    prof[k] = {kk: round(v, 1) for kk, v in sorted(per.items(), key=lambda kv: -kv[1])}
                for x in res:
                    x["engine"].close()
        out["device_us"] = prof
        out["gpu"] = card()
        print(json.dumps(out), flush=True)
        return
    for k, c in tg.items():
        us, digest = [], None
        for _ in range(args.calls + 1):  # the first call warms up
            engines = sources()
            t0 = time.perf_counter()
            res = recut(c, owners[k], engines)
            us.append((time.perf_counter() - t0) * 1e6)
            assert all(x["ok"] for x in res)
            d = zlib.crc32(b"".join(x["engine"].export_state().tobytes() for x in res))
            assert digest in (None, d)
            digest = d
            out.setdefault(f"recut_{k}_sizes", [int(x["engine"].pool_size()) for x in res])
            for x in res:
                x["engine"].close()
        out[f"recut_{k}_us"] = stats(us[1:])
    # the host alternative, once, into (a): every rank's pool read back and enqueued on the new owners
    c = tg["a_24_equal"]
    engines = sources()
    news = [pkg.Engine(c) for _ in range(K)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()

    def host_rank(r):
        rd = engines[r].pool_read()
        return rd, shard.route(c, rd["rating"], K, owners=owners["a_24_equal"])
    reads = on_ranks(host_rank)
    for d in range(K):
        for rd, dest in reads:
            s = dest == d
            assert news[d].enqueue(rd["id"][s], rd["rating"][s], rd["mode"][s], rd["enq_ts"][s]).all()
    torch.cuda.synchronize()
    out["host_pool_read_enqueue_us"] = (time.perf_counter() - t0) * 1e6
    for e in engines + news:
        e.close()
    out["checked"] = "every repeated re-cut gives the same new-rank exports"
    out["timing"] = "host clock around shard.recut on 4 thread ranks (export, LocalComm exchange, create, import, swap)"
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
