"""Cost of the pool hand-over: mm_export of config3 with 10 M resident players into a host buffer, and mm_import of
that image into a fresh engine, against mm_pool_read of the same pool (the only way to read the queued players out
before mm_export, and only part of what a hand-over needs).

State measured: config3 (10 M players, 32 groups, 5v5) in the given order, MM_F_DENSE_IDS, 10 M queued players plus
the active-set entries of the members of one earlier tick's lobbies.  Every call is timed with the host clock around
the blocking call, after a warm-up; the import runs into a new engine each time (engine creation not timed).  The host
buffer is ordinary pageable memory, as a caller's would be.  Prints one JSON line per order with the card's name and
power limit, read in the same run.

    python tools/exp_checkpoint.py [--orders rating,arrival] [--calls 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        name, plim = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit_w": float(plim)}
    except Exception:
        return {"name": None, "power_limit_w": None}


def spread(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "calls": len(xs)}


def kernel_us(fn, calls):
    """Device time per call of the kernels the call launches (torch.profiler, CUDA activities; copies and memsets
    excluded), in µs."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    tot, names = 0.0, set()
    for ev in prof.events():
        if ev.name.startswith(("void mm::", "mm::")) and ev.device_time_total > 0:
            tot += ev.device_time_total
            names.add(ev.name.split("(")[0])
    return {"us": tot / calls, "kernels": sorted(names)}


def import_once(pkg, cfg, buf):
    with pkg.Engine(cfg) as dst:
        assert dst.lib.mm_import(dst.h, buf.ctypes.data_as(C.c_void_p), len(buf)) == 0


def run(pkg, order, calls, warmup):
    n = 10_000_000
    cfg = pkg.synth.make_config(n_groups=32, modes=[("5v5", 2, 5)], order=order, capacity=n + 65536, active_capacity=2 * n,
                                flags=pkg.abi.MM_F_DENSE_IDS)
    _, rating, _, _ = pkg.synth.gen_pool(1, n)
    key = pkg.Engine.pack_key(rating, np.zeros(n, np.uint8))
    ts = (np.arange(n) % 977).astype(np.uint32)
    with pkg.Engine(cfg) as src:
        assert (src.enqueue_packed(np.arange(n, dtype=np.uint32), key, ts) == 1).all()
        src.tick_packed(1000)  # its members stay in the active set
        assert (src.enqueue_packed(np.arange(n, 2 * n, dtype=np.uint32), key, ts) == 1).all()
        size = C.c_uint64(0)
        assert src.lib.mm_export(src.h, None, 0, C.byref(size)) == 0
        buf = np.empty(size.value, np.uint8)
        buf.fill(0)  # the pages exist before the first timed call

        def export():
            t0 = time.perf_counter()
            assert src.lib.mm_export(src.h, buf.ctypes.data_as(C.c_void_p), len(buf), C.byref(size)) == 0
            return time.perf_counter() - t0

        for _ in range(warmup):
            export()
        exp_s = [export() for _ in range(calls)]
        h, _ = pkg.engine.read_image(buf)

        def pool_read():
            t0 = time.perf_counter()
            src.pool_read()
            return time.perf_counter() - t0

        read_s = [pool_read() for _ in range(max(1, calls // 2))]
        exp_kernel_us = kernel_us(lambda: export(), calls)
        imp_s = []
        for k in range(warmup + calls):
            with pkg.Engine(cfg) as dst:
                t0 = time.perf_counter()
                assert dst.lib.mm_import(dst.h, buf.ctypes.data_as(C.c_void_p), len(buf)) == 0
                dt = time.perf_counter() - t0
                if k >= warmup:
                    imp_s.append(dt)
                if k == warmup + calls - 1:
                    assert dst.active_size() == src.active_size() and dst.pool_size() == h.n_players
        imp_kernel_us = kernel_us(lambda: import_once(pkg, cfg, buf), 1)
    return {
        "workload": "config3_10m_g32_5v5", "order": "rating" if order == pkg.abi.MM_ORDER_RATING else "arrival",
        "queued_players": h.n_players, "active_not_queued": h.n_active, "image_bytes": int(len(buf)),
        "bytes_per_queued_player": len(buf) / h.n_players,
        "export_ms": {k: (v * 1e3 if k != "calls" else v) for k, v in spread(exp_s).items()},
        "import_ms": {k: (v * 1e3 if k != "calls" else v) for k, v in spread(imp_s).items()},
        "pool_read_ms": {k: (v * 1e3 if k != "calls" else v) for k, v in spread(read_s).items()},
        "export_kernels_us": exp_kernel_us, "import_kernels_us": imp_kernel_us,
        "export_gb_per_s": len(buf) / np.median(exp_s) / 1e9, "import_gb_per_s": len(buf) / np.median(imp_s) / 1e9,
        "timing": "host clock around the blocking call, pageable host buffer, after warm-up",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--orders", default="rating,arrival")
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import __graft_entry__ as ge
    pkg = ge.build()
    gpu = card()
    for o in args.orders.split(","):
        r = run(pkg, pkg.abi.MM_ORDER_RATING if o == "rating" else pkg.abi.MM_ORDER_ARRIVAL, args.calls, args.warmup)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
