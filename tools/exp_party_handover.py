"""Cost of carrying parties through a hand-over (mm_export_parties / mm_merge_parties, SearchPool.checkpoint).

config3 (32 groups, 5v5, rating order): 10 M solos, then parties of 2 - 4 members making up 0 %, 1 % and 10 % of all
players.  For each share, from the same state every time (mm_restore of one snapshot of the solos, the parties enqueued
again, not timed):
  - export: Engine.export_parties() of every queue (the release included);
  - merge_keep_seq: Engine.merge_parties(image, keep_seq=True) back into the engine it came from;
  - merge_new: Engine.merge_parties(image) into a second engine holding the same solos;
  - checkpoint_engine: the engine part of SearchPool.checkpoint() — release, Engine.export_state(), merge back with
    keep_seq (share 0: export_state alone, what a pool without party capacity runs);
  - search_pool_checkpoint: the whole SearchPool.checkpoint() of a pool over the same engine, with a host state of one
    small document per player and the party_of map (share 0: a pool without party capacity).
Each call is timed by CUDA events recorded on the engine's stream around it (the engine runs on a stream of this
process, mm_set_stream; every call returns with its work done, so the events bracket all of its device work and the
copies) and by the host clock; the kernels' own time comes from torch.profiler in a separate run.  Medians of --calls
after one warm-up (the whole SearchPool.checkpoint: one call per share).  Prints one JSON line with the card's name and
power limit, read in the same run.

    python tools/exp_party_handover.py [--calls 5]
"""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exp_move import card, kernel_us, stats  # noqa: E402

EXPORT = ("k_pt_sel", "k_scan_small", "k_pt_export")
MERGE = ("k_pt_keep", "k_pt_move", "k_pt_claim", "k_pt_resolve", "k_scan_small", "k_pt_commit", "k_pt_members")


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
    out = {"workload": name, "solos": n, "card": card()}
    stream = torch.cuda.Stream()
    sw = importlib.import_module(pkg.__name__ + ".search_worker")
    with pkg.Engine(cfg) as e, pkg.Engine(cfg) as t:
        for x in (e, t):  # both on one stream of this process: the events below bracket their work
            x.set_stream(stream.cuda_stream)
        for x in (e, t):
            assert x.enqueue(ids, rating, mode, ts).all()
            x.snapshot()
            x.set_option("party_capacity", n // 4)
        dense = bool(cfg.flags & pkg.abi.MM_F_DENSE_IDS)
        doc = {"id": "player"}
        for share in (0.0, 0.01, 0.1):
            k = int(n * share / 0.99 / 3)  # parties of 3 on average
            sizes = rng.integers(2, 5, k).astype(np.uint8)
            m = int(sizes.sum())
            x = np.arange(n, n + m, dtype=np.uint64)
            pid = x if dense else pkg.synth.mix64(x + np.uint64(9 << 40))
            prat = np.clip(np.repeat(rng.integers(0, 5001, k), sizes) + rng.integers(-20, 21, m), 0, 5000).astype(np.int32)
            pts = (now - rng.integers(0, 60, k)).astype(np.uint32)

            def fresh():
                e.restore()
                t.restore()
                if k:
                    assert (e.enqueue_party(sizes, pid, prat, np.full(k, mode_idx, np.uint8), pts) == 1).all()
                torch.cuda.synchronize()

            def checkpoint():
                if not k:
                    return e.export_state()
                img = e.export_parties()
                try:
                    return e.export_state()
                finally:
                    e.merge_parties(img, keep_seq=True)

            steps = {"export": lambda st: st.__setitem__("img", e.export_parties()),
                     "merge_keep_seq": lambda st: e.merge_parties(st["img"], keep_seq=True),
                     "merge_new": lambda st: t.merge_parties(st["img"]),
                     "checkpoint_engine": lambda st: checkpoint()}

            def timed(f, st, on=stream):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(on)
                t0 = time.perf_counter()
                f(st)
                host = (time.perf_counter() - t0) * 1e6
                b.record(on)
                b.synchronize()
                return host, a.elapsed_time(b) * 1e3

            host = {s: [] for s in steps}
            dev = {s: [] for s in steps}
            for _ in range(args.calls + 1):  # the first round warms up
                fresh()
                st = {}
                for s, f in steps.items():
                    if s == "checkpoint_engine":
                        fresh()
                    h, d = timed(f, st)
                    host[s].append(h)
                    dev[s].append(d)
            fresh()
            st = {}
            kern = {}
            for s, f in steps.items():
                if s == "checkpoint_engine":
                    fresh()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    f(st)
                    torch.cuda.synchronize()
                kern[s] = kernel_us(prof, EXPORT + MERGE)
            # the whole SearchPool.checkpoint over this engine: one document per player, the parties' party_of
            fresh()
            pool = sw.SearchPool(e, [f"mode{i}" for i in range(cfg.n_modes)], [f"g{g}" for g in range(cfg.n_groups)],
                                 party_capacity=n // 4 if k else None)
            pool.players = dict.fromkeys(range(n + m), doc)
            pool.handles.id_of = list(range(n + m))
            off = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))]) + n
            pool.party_of = {h: tuple(range(int(off[j]), int(off[j + 1]))) for j in range(k)
                             for h in range(int(off[j]), int(off[j + 1]))}
            ph, pd = timed(lambda _st: pool.checkpoint(), None)
            del pool
            out[f"parties_{share:g}"] = {
                "parties": k, "members": m, "image_bytes": int(len(st["img"])),
                "call_us": {s: stats(v[1:]) for s, v in host.items()},
                "events_us": {s: stats(v[1:]) for s, v in dev.items()}, "kernels_us": kern,
                "search_pool_checkpoint": {"call_us": ph, "events_us": pd}}
        e.restore()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
