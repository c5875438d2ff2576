"""Cost of re-cutting a sharded deployment with parties queued (shard.recut, mm_import_regroup_many_parties): config3
(10 M queued solos, 5v5, rating order, 32 equal-width groups) on K = 4 engines of one GPU, owners by balanced_owners,
re-cut into (a) 24 equal-width groups and (b) 32 quantile groups, with 0 and with 200 k parties of 2 .. 5 members
(delivered to the rank that owns their group, as routing would).

Host clock around shard.recut (the four ranks as threads over LocalComm), median of --calls after one warm-up call; the
source engines are rebuilt from their images before each call, outside the clock.  --profile runs one re-cut per
target with 200 k parties under torch.profiler and prints the device time per kernel.  Prints one JSON line with the
card's name and power limit, read in the same run.

    python tools/exp_recut_parties.py [--calls 3] [--profile]
"""
import argparse
import importlib
import json
import os
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, stats  # noqa: E402
from exp_recut import K, on_ranks, targets  # noqa: E402

PARTIES = 200_000


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
    rng = np.random.default_rng(7)
    tsz = cfg.modes[int(mode[0])].team_size
    sizes = rng.integers(2, tsz + 1, PARTIES).astype(np.uint8)
    moff = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
    pids = (np.uint64(1) << np.uint64(40)) + np.arange(moff[-1], dtype=np.uint64)
    prat = rng.integers(0, 5001, moff[-1]).astype(np.int32)
    R = np.floor_divide(np.add.reduceat(prat.astype(np.int64), moff[:-1]), sizes.astype(np.int64))
    pg = shard.group_of_rating(cfg, R)
    pto = np.where(pg >= 0, old_own[np.maximum(pg, 0)], -1)
    images, pimages = [], []
    for r in range(K):
        with pkg.Engine(cfg) as e:
            s = to == r
            assert e.enqueue(ids[s], rating[s], mode[s], ts[s]).all()
            e.set_option("party_capacity", 2_000_000)
            mine = np.flatnonzero(pto == r)
            take = np.concatenate([np.arange(moff[j], moff[j + 1]) for j in mine])
            code = e.enqueue_party(sizes[mine], pids[take], prat[take], np.full(len(mine), mode[0], np.uint8),
                                   (1000 + mine % 977).astype(np.uint32))
            assert (code == 1).all()
            pimages.append(np.array(e.export_parties(), copy=True))
            images.append(np.array(e.export_state(), copy=True))
    out = {"workload": name, "players": n, "parties": int((pto >= 0).sum()), "ranks": K,
           "party_image_bytes": [int(len(p)) for p in pimages]}

    def sources(with_parties):
        engines = [pkg.Engine(cfg) for _ in range(K)]
        for e, img, p in zip(engines, images, pimages):
            e.import_state(img)
            if with_parties:
                e.set_option("party_capacity", 2_000_000)
                e.merge_parties(p, keep_seq=True)
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
                engines = sources(True)
                if warm:
                    res = recut(c, owners[k], engines)
                else:
                    with profile(activities=[ProfilerActivity.CUDA]) as p:
                        res = recut(c, owners[k], engines)
                        torch.cuda.synchronize()
                    per = {}
                    for ev in p.events():
                        if ev.device_time_total > 0:
                            per[ev.name] = per.get(ev.name, 0.0) + ev.device_time_total
                    prof[k] = {kk: round(v, 1) for kk, v in sorted(per.items(), key=lambda kv: -kv[1])
                               if "rp_" in kk or "rc_" in kk or "rg_" in kk or "Memcpy" in kk}
                for x in res:
                    x["engine"].close()
        out["device_us"] = prof
        out["gpu"] = card()
        print(json.dumps(out), flush=True)
        return
    for k, c in tg.items():
        for with_parties in (False, True):
            us, digest = [], None
            for _ in range(args.calls + 1):  # the first call warms up
                engines = sources(with_parties)
                t0 = time.perf_counter()
                res = recut(c, owners[k], engines)
                us.append((time.perf_counter() - t0) * 1e6)
                assert all(x["ok"] for x in res)
                d = zlib.crc32(b"".join(x["engine"].pool_read()["id"].tobytes() for x in res))
                assert digest in (None, d)
                digest = d
                if with_parties:
                    out.setdefault(f"recut_{k}_parties_loaded", [len(x["engine"].party_read()["size"]) for x in res])
                for x in res:
                    x["engine"].close()
            out[f"recut_{k}_{'200k_parties' if with_parties else 'no_parties'}_us"] = stats(us[1:])
    out["timing"] = "host clock around shard.recut on 4 thread ranks (release, export, exchange, create, import, swap)"
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
