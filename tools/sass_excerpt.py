#!/usr/bin/env python
"""profiles/rNN_sass_k_tick.txt: static instruction mix of the tick / ingest kernels and every TMA / mbarrier /
shared-memory-atomic line of k_tick, from `cuobjdump -sass` of the in-tree library (no GPU needed)."""
import collections, os, re, subprocess, sys
so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "microservice-matchmaking_b200", "csrc", "libmm_engine.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
funcs, cur = collections.OrderedDict(), None
for ln in out.splitlines():
    m = re.search(r"Function : (\S+)", ln)
    if m: cur = m.group(1); funcs[cur] = []; continue
    if cur and re.search(r"/\*[0-9a-f]{4,}\*/\s+\S", ln): funcs[cur].append(ln.rstrip())
KEYS = ("UBLKCP", "SYNCS", "ATOMS", "ATOMG", "REDG", "REDUX", "BAR", "VOTE", "MATCH", "SHFL", "LDS", "STS", "LDG", "STG", "WARPSYNC", "POPC", "MEMBAR", "FENCE", "HMMA", "UTCMMA")
print("cuobjdump -sass libmm_engine.so (sm_90a), instruction mix of the tick and ingest kernels (static counts) and the TMA / mbarrier / shared-memory-atomic lines of k_tick\n")
for name, lines in funcs.items():
    if not re.search(r"k_tick|k_place|k_hist|k_enq_append|k_enq_claim", name): continue
    c = collections.Counter()
    for ln in lines:
        op = re.sub(r"^\s*/\*[0-9a-f]+\*/\s+(@!?U?P\d+\s+)?", "", ln).split()[0].split(".")[0]
        if op in KEYS: c[op] += 1
    print(name); print(f"  {len(lines)} SASS instructions; {dict((k, c[k]) for k in KEYS if c[k])}")
print("\n--- k_tick: every UBLKCP / SYNCS / ATOMS / RED / MATCH line")
for name, lines in funcs.items():
    if "k_tick" in name:
        for ln in lines:
            if re.search(r"\b(UBLKCP|SYNCS|ATOMS|REDG|MATCH)\b", ln): print(ln)
