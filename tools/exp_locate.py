"""Cost of a search-status lookup (mm_locate) against the host alternative, mm_pool_read + a numpy restatement.

config3 (32 groups, 5v5, rating order), 10 M resident players, no tick.  Lookups of 1, 1 000, 100 000 and every
queued player (random queued ids).  Per size: the median host-clock time of the blocking call (id upload, the three
kernels, the record copy) and the median device time of the same call from CUDA events recorded on the engine's
stream around it.  The host alternative reads the pool (mm_pool_read) and restates ahead / depth in numpy
(tests/test_locate.py's restatement, which needs the sequence numbers: the ids' enqueue order stands in for them here,
as nothing was requeued).  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/exp_locate.py [--calls 7]
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

from exp_move import card, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, pkg.abi.MM_ORDER_RATING, n)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    rng = np.random.default_rng(1)
    stream = torch.cuda.Stream()
    out = {"workload": name, "players": n}
    with pkg.Engine(cfg) as e:
        e.set_stream(stream.cuda_stream)
        assert e.enqueue(ids, rating, mode, ts).all()
        for k in (1, 1000, 100_000, n):
            q = ids[rng.permutation(n)[:k]] if k < n else ids
            host, dev = [], []
            for _ in range(args.calls + 1):  # the first call warms up
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                a.record(stream)
                rec = e.locate(q, 10_000_000)
                b.record(stream)
                host.append((time.perf_counter() - t0) * 1e6)
                b.synchronize()
                dev.append(a.elapsed_time(b) * 1e3)
            assert (rec["state"] == 1).all()
            out[f"locate_{k}"] = {"call_us": stats(host[1:]), "device_us": stats(dev[1:])}
        from tests.test_locate import restate
        t0 = time.perf_counter()
        p = e.pool_read()
        t1 = time.perf_counter()
        restate(cfg, p["id"], p["rating"], p["mode"], np.arange(len(p["id"]), dtype=np.uint32), len(p["id"]))
        t2 = time.perf_counter()
        out["host_alternative_us"] = {"pool_read": (t1 - t0) * 1e6, "restate": (t2 - t1) * 1e6, "total": (t2 - t0) * 1e6}
    out["timing"] = ("call_us: host clock around the blocking Engine.locate; device_us: CUDA events on the engine's "
                     "stream around the same call (id upload, kernels, record copy)")
    out["gpu"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
