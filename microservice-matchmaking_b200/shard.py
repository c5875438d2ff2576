"""Rating-group sharding across the GPUs of one box (SURVEY §8e).

(rating group, game-mode) partitions never interact in the reference: one queue +
exchange per group (search/worker.ex:46-66), workers per group (application.ex:26-40),
one Mnesia table per group (models/lobby_state.ex:15-29).  So the pool shards by group
with NO data-path collective: the Generic stage's routing rule
(generic/worker.ex:46-69) decides, on the host at ingest, which rank's engine receives a
player; every rank ticks independently; the job's result is the per-rank results merged
back into canonical (mode, group, emission) order.  Pure host logic, no compute.
"""
import numpy as np


def owner_of_group(g, n_groups, world):
    """Contiguous rating ranges per GPU: group g -> rank floor(g * P / G)."""
    return (np.asarray(g, np.int64) * world) // n_groups


def groups_of_rank(rank, n_groups, world, owners=None):
    """owners: optional owner rank per group (balanced_owners); default floor(g * P / G)."""
    g = np.arange(n_groups)
    own = owner_of_group(g, n_groups, world) if owners is None else np.asarray(owners, np.int64)
    return g[own == rank]


def balanced_owners(load, world):
    """Contiguous owner ranks (non-decreasing in the group) that minimise the largest per-rank load; load[g] >= 0, e.g.
    the queue depths of mm_queue_stats summed over the modes.  Among the optimal splits, every rank takes as many
    groups as it can, lowest rank first (the lexicographically smallest owner array), so every rank computes the same
    answer.  -> int64[G]"""
    load = np.asarray(load, np.float64)
    G = len(load)
    if G == 0:
        return np.zeros(0, np.int64)
    if world < 1 or (load < 0).any():
        raise ValueError("balanced_owners needs world >= 1 and loads >= 0")
    pre = np.concatenate([[0.0], np.cumsum(load)])

    def greedy(cap):  # every rank takes the longest run of groups that stays within cap; None if P ranks do not do
        own = np.empty(G, np.int64)
        r, start = 0, 0
        for g in range(G):
            if pre[g + 1] - pre[g] > cap:
                return None
            if pre[g + 1] - pre[start] > cap:
                r, start = r + 1, g
                if r >= world:
                    return None
            own[g] = r
        return own

    cands = np.unique((pre[None, :] - pre[:, None])[np.triu_indices(G + 1, 1)])  # every run's load: one is optimal
    lo, hi = 0, len(cands) - 1
    while lo < hi:
        mid = (lo + hi) // 2
        if greedy(cands[mid]) is None:
            lo = mid + 1
        else:
            hi = mid
    return greedy(cands[lo])


def group_of_rating(cfg, rating):
    """Vectorised generic/worker.ex:46-53 (first match in list order, else default)."""
    rating = np.asarray(rating, np.int64)
    grp = np.full(rating.shape, cfg.default_group, np.int64)
    unset = np.ones(rating.shape, bool)
    for g in range(cfg.n_groups):
        hit = unset & (rating >= cfg.group_lo[g]) & (rating <= cfg.group_hi[g])
        grp[hit] = g
        unset &= ~hit
    return grp


def route(cfg, rating, world, owners=None):
    """-> owner rank of every player (-1: unroutable, no default group).  owners: optional owner rank per group
    (balanced_owners, or the `new` array of a move_queues); default floor(g * P / G)."""
    grp = group_of_rating(cfg, rating)
    g0 = np.maximum(grp, 0)
    own = owner_of_group(g0, cfg.n_groups, world) if owners is None else np.asarray(owners, np.int64)[g0]
    return np.where(grp < 0, -1, own)


def merge_results(cfg, per_rank):
    """per_rank[r] = (lobbies, member_ids[, emit_seq]) of rank r, each already in canonical
    (mode, group, emission) order and covering disjoint groups.  -> the whole job's
    (lobbies, member_ids[, emit_seq]) in canonical order with first_member re-based."""
    lobs = [np.asarray(x[0]) for x in per_rank]
    has_seq = all(len(x) > 2 and x[2] is not None for x in per_rank)
    parts_l, parts_m, parts_s = [], [], []
    off = 0
    for m in range(cfg.n_modes):
        for r, lob in enumerate(lobs):  # ranks own increasing group ranges
            sel = lob["mode"] == m
            if not sel.any():
                continue
            sub = lob[sel].copy()
            L = int(sub["n_members"][0])
            a = int(sub["first_member"][0])
            mem = np.asarray(per_rank[r][1])[a:a + L * len(sub)]
            sub["first_member"] = off + np.arange(len(sub), dtype=np.uint32) * L
            off += len(mem)
            parts_l.append(sub); parts_m.append(mem)
            if has_seq:
                parts_s.append(np.asarray(per_rank[r][2])[sel])
    if not parts_l:
        z = lobs[0][:0] if lobs else np.zeros(0)
        return (z, np.zeros(0, np.uint64)) + ((np.zeros(0, np.uint32),) if has_seq else ())
    out = (np.concatenate(parts_l), np.concatenate(parts_m))
    return out + ((np.concatenate(parts_s),) if has_seq else ())


# ======================================================================================================================
# EXTENSION (SURVEY F3 / §8e, BASELINE configs[3]-[4]): the boundary pass.
#
# Not reference behaviour: the reference never lets a player leave its rating group (requeue -> generic -> same
# group queue, search/worker.ex:239-248).  Under the rating-window policy S1 (mm_set_option "max_spread" = W) a
# player near a group boundary may have no partner inside its own group while a neighbour W points away sits in the
# next group — on another GPU when the boundary coincides with a shard boundary.  After every rank's local tick:
#
#   for every pair of adjacent groups (g, g+1) and every mode: the still-queued players of g with rating > hi_g - W
#   and those of g+1 with rating <= hi_g + W form ONE band; the band is matched by the same windowed walk as a
#   partition (policy S1, oracle: orc_run_windowed on the band), candidates of g first then of g+1, each in enqueue
#   order (the tie-break inside a rating); a lobby formed in the band belongs to the LOWER group g and is emitted by the
#   rank that owns g; band players that stay unmatched simply remain queued at home.
#
# Bands must be disjoint (every group at least 2 W wide), so all boundaries are independent and every rank works in
# parallel.  Data path when g and g+1 live on different ranks: the upper rank SENDS its band candidates (id, rating,
# mode columns) to the lower one, which matches the band and sends back the ids it consumed; point-to-point over the
# process group — NCCL send/recv over NVLink on GPUs, gloo in the CPU tests.  Matched players leave their home pool
# through mm_take (they stay in the active set like any matched player).
# ======================================================================================================================
def check_bands(cfg, W):
    """Adjacent groups must be contiguous ascending rating ranges, each at least 2 W wide."""
    for g in range(cfg.n_groups):
        if cfg.group_hi[g] - cfg.group_lo[g] + 1 < 2 * W:
            raise ValueError(f"rating group {g} is narrower than 2 x max_spread: boundary bands would overlap")
        if g and cfg.group_lo[g] != cfg.group_hi[g - 1] + 1:
            raise ValueError("the boundary pass needs contiguous ascending rating groups")


def band_config(pkg, cfg, g, W, capacity):
    """One-group engine configuration covering the band around the boundary of groups g | g+1."""
    hi = int(cfg.group_hi[g])
    modes = [(f"m{m}", int(cfg.modes[m].teams), int(cfg.modes[m].team_size)) for m in range(cfg.n_modes)]
    c = pkg.synth.make_config(groups=[(hi - W + 1, hi + W)], modes=modes, order=pkg.abi.MM_ORDER_RATING,
                              capacity=max(int(capacity), 1), default_group=-1, device=int(cfg.device))
    return c


class LocalComm:
    """In-process stand-in for the point-to-point exchange (GPU tests where K engines share one process, one thread
    per rank): a blocking queue per (src, dst)."""

    def __init__(self):
        import collections
        import queue
        self.box = collections.defaultdict(queue.Queue)
        self.bytes_sent = 0

    def send(self, src, dst, arrays):
        arrays = [np.array(a, copy=True) for a in arrays]
        self.bytes_sent += sum(a.nbytes for a in arrays)
        self.box[(src, dst)].put(arrays)

    def recv(self, src, dst):
        return self.box[(src, dst)].get(timeout=120)


class DistComm:
    """torch.distributed point-to-point: a count, then the columns as tensors (on the GPU for NCCL)."""
    DTYPES = ("int64", "int32", "uint8")

    def __init__(self, device=None):
        import torch
        import torch.distributed as dist
        self.torch, self.dist, self.device = torch, dist, device
        self.bytes_sent = 0

    def send(self, src, dst, arrays):
        t, d = self.torch, self.dist
        n = len(arrays[0])
        d.send(t.tensor([n, len(arrays)], dtype=t.int64, device=self.device), dst)
        for a, dt in zip(arrays, self.DTYPES):
            if n:
                x = t.from_numpy(np.ascontiguousarray(a).view(getattr(np, dt) if dt != "int64" else np.int64))
                d.send(x.to(self.device) if self.device is not None else x, dst)
                self.bytes_sent += x.numel() * x.element_size()

    def recv(self, src, dst):
        t, d = self.torch, self.dist
        hdr = t.zeros(2, dtype=t.int64, device=self.device)
        d.recv(hdr, src)
        n, k = int(hdr[0].item()), int(hdr[1].item())
        out = []
        for dt in self.DTYPES[:k]:
            x = t.zeros(n, dtype=getattr(t, dt), device=self.device)
            if n:
                d.recv(x, src)
            out.append(x.cpu().numpy())
        if out:
            out[0] = out[0].view(np.uint64)
        return out


def boundary_pass(pkg, cfg, W, world, rank, engine, comm, make_engine=None, cache=None):
    """Run this rank's share of the boundary pass (see above).  `engine` has just ticked.
    cache: dict kept by the caller across ticks — the band engines are reused instead of re-created.
    -> dict(hdr, member_ids, sent, received, matched, lobbies) — hdr: mm_lobby_hdr records (first_member into member_ids)
    carrying the LOWER group's index; sent / received / matched: players; lobbies: count."""
    check_bands(cfg, W)
    make_engine = make_engine or pkg.Engine
    G = cfg.n_groups
    mine = groups_of_rank(rank, G, world)
    res = engine.pool_read()
    ids, rating, mode = res["id"], res["rating"], res["mode"]
    grp = group_of_rating(cfg, rating)
    stats = {"sent": 0, "received": 0, "matched": 0, "lobbies": 0}
    if len(mine) == 0:
        return dict(hdr=None, member_ids=np.zeros(0, np.uint64), **stats)
    a, b = int(mine[0]), int(mine[-1])
    if rank > 0:  # my lowest group's low-side band goes down to the owner of group a-1
        sel = (grp == a) & (rating <= cfg.group_hi[a - 1] + W)
        comm.send(rank, rank - 1, (ids[sel], rating[sel], mode[sel]))
        stats["sent"] += int(sel.sum())
    lob_parts, mem_parts, off = [], [], 0
    for g in range(a, min(b, G - 2) + 1):
        lo_sel = (grp == g) & (rating > cfg.group_hi[g] - W)
        low = (ids[lo_sel], rating[lo_sel], mode[lo_sel])
        remote = g + 1 > b
        if remote:
            high = comm.recv(rank + 1, rank)
            stats["received"] += len(high[0])
        else:
            hi_sel = (grp == g + 1) & (rating <= cfg.group_hi[g] + W)
            high = (ids[hi_sel], rating[hi_sel], mode[hi_sel])
        n_band = len(low[0]) + len(high[0])
        took_remote = np.zeros(0, np.uint64)
        if n_band:
            band = cache.get(g) if cache is not None else None
            if band is None or band.cfg.capacity < n_band:
                if band is not None:
                    band.close()
                band = make_engine(band_config(pkg, cfg, g, W, max(n_band, 1 << 16 if cache is not None else 1)))
                band.set_option("max_spread", W)
                if cache is not None:
                    cache[g] = band
            for part in (low, high):  # the lower group's candidates first: tie-break inside a rating
                if len(part[0]):
                    acc = band.enqueue(part[0], part[1], part[2])
                    assert (np.asarray(acc) == 1).all()
            lob, mem, _seq, st = band.tick()
            if cache is None:
                band.close()
            else:  # leave the band engine empty for the next tick: the unmatched candidates went back home
                band.remove(np.concatenate([low[0], high[0]]))
            if len(lob):
                lob = lob.copy()
                lob["group"] = g
                lob["first_member"] = lob["first_member"] + off
                off += len(mem)
                lob_parts.append(lob); mem_parts.append(mem)
                stats["matched"] += len(mem); stats["lobbies"] += len(lob)
                own = np.isin(mem, ids)
                if own.any():
                    assert engine.take(mem[own]) == int(own.sum())
                took_remote = mem[~own]
        if remote:
            comm.send(rank, rank + 1, (took_remote,))
    if rank > 0:  # what the lower rank consumed of my candidates leaves my pool
        (gone,) = comm.recv(rank - 1, rank)
        if len(gone):
            assert engine.take(gone) == len(gone)
    hdr = np.concatenate(lob_parts) if lob_parts else None
    members = np.concatenate(mem_parts) if mem_parts else np.zeros(0, np.uint64)
    return dict(hdr=hdr, member_ids=members, **stats)


def boundary_pass_device(pkg, cfg, W, world, rank, engine, comm):
    """boundary_pass on the device: the same bands, lobbies, takes, messages and result dict, but the candidates are
    gathered and the bands matched inside `engine` (mm_band_candidates / mm_band_match, DESIGN §6) — the pool is never
    read to the host and no band engine exists.  Only the candidate columns sent down, the lobby headers, the members
    and the consumed ids cross PCIe.  `engine` is a pkg.Engine that has just ticked; boundary_pass stays the reference
    (and the only path for engines without the device calls)."""
    check_bands(cfg, W)
    G = cfg.n_groups
    mine = groups_of_rank(rank, G, world)
    stats = {"sent": 0, "received": 0, "matched": 0, "lobbies": 0}
    if len(mine) == 0:
        return dict(hdr=None, member_ids=np.zeros(0, np.uint64), **stats)
    a, b = int(mine[0]), int(mine[-1])
    if rank > 0:  # my lowest group's low-side band goes down to the owner of group a-1
        cand = engine.band_candidates(W, a)
        comm.send(rank, rank - 1, cand)
        stats["sent"] += len(cand[0])
    hdr, members = None, np.zeros(0, np.uint64)
    g_last = min(b, G - 2)
    if a <= g_last:
        remote = g_last + 1 > b
        upper = None
        if remote:
            upper = comm.recv(rank + 1, rank)
            stats["received"] += len(upper[0])
        lob, mem, taken, _st = engine.band_match(W, a, g_last, upper)
        if remote:
            comm.send(rank, rank + 1, (np.asarray(upper[0], np.uint64)[taken],))
        if len(lob):
            hdr, members = lob, mem
            stats["matched"] += len(mem); stats["lobbies"] += len(lob)
    if rank > 0:  # what the lower rank consumed of my candidates leaves my pool
        (gone,) = comm.recv(rank - 1, rank)
        if len(gone):
            assert engine.take(gone) == len(gone)
    return dict(hdr=hdr, member_ids=members, **stats)


# ======================================================================================================================
# Moving rating groups between ranks (mm_export_queues / mm_merge).  A group's queues, all modes, go from the rank that
# owns it to another one while both keep running: scale out / in, or a rebalance by balanced_owners() when the
# rating distribution leaves one rank with most of the pool.
# ======================================================================================================================
def _status(x):
    return int(np.asarray(x).view(np.int64).reshape(-1)[0])


def _party_members(engine, g=None):
    """Members of the parties queued in `engine` (of group g only, unless None); 0 for an engine without parties."""
    if not getattr(engine, "party_capacity", 0):
        return 0
    pr = engine.party_read()
    return int(pr["size"][pr["group"] == g].sum() if g is not None else pr["size"].sum())


def can_take(cfg, engine, g, n, n_party=0):
    """Would a merge of n players and n_party party members of group g into `engine` pass mm_merge's and
    mm_merge_parties' checks?  No live player in any of the group's queues, n more pool slots within the capacity (the
    slots in use count dead ones until the next tick), n_party more members within the party capacity, and for a
    hashed active set n + n_party more entries within its 3/4 load.  Conservative: rejected ids would need no room."""
    if int(engine.queue_stats(0)["n_waiting"].reshape(cfg.n_modes, cfg.n_groups)[:, g].sum()):
        return False
    if engine.pool_size() + n > engine.cfg.capacity:
        return False
    if n_party and _party_members(engine) + n_party > getattr(engine, "party_capacity", 0):
        return False
    from .engine import active_set_limit
    limit = active_set_limit(engine.cfg)  # a hashed active set: its 3/4 load
    if limit is not None and engine.active_size() + n + n_party > limit:
        return False
    return True


def _merge_with_parties(engine, img, pimg=None):
    """merge_queues(img) into an engine that may hold parties: mm_merge refuses while a party is queued, so the
    engine's own parties step aside (export_parties) and come back, with their numbers when the queue image took
    none (else renumbered in their order); then the party image pimg merges if the queue image went in.  Every step
    is caught.  -> (True if img merged, [party images that did not go back in])"""
    own, left = None, []
    if getattr(engine, "party_capacity", 0):
        try:
            own = np.ascontiguousarray(engine.export_parties(), np.uint8)
            seq0 = engine.seq_next()
        except Exception:  # a refused export changes nothing
            return False, []
    try:
        engine.merge_queues(img)
        ok = True
    except Exception:
        ok = False
    if own is not None:
        try:
            engine.merge_parties(own, keep_seq=engine.seq_next() == seq0)
        except Exception:
            left.append(own)
    if ok and pimg is not None:
        try:
            engine.merge_parties(pimg)
        except Exception:
            left.append(pimg)
    return ok, left


def move_queues(pkg, cfg, old, new, rank, engine, comm):
    """Move every group g with old[g] != new[g] from rank old[g] to rank new[g]; every rank of the job calls this with
    the same arrays.  Moves run in ascending group order on every rank; each involves exactly two ranks, and every
    message below is answered whatever fails, so blocking point-to-point calls can neither deadlock nor wait forever.
    One move, all messages int64 arrays:

      1. source -> target: [n], the group's live players here (mm_queue_stats), or [-1] if they cannot be counted;
         [n, m] when m members of the group's queued parties go along;
      2. target -> source: [0] if it can take them (can_take: no live player of the group, room in the pool, the party
         table and the active set), else [1] — the source has released nothing yet, so a refusal here changes nothing;
      3. source -> target: the queue image (Engine.export_queues: the players are released in the same call) as one
         int64 array (an image is a multiple of 8 bytes and at least its 624-byte header), or [-1] if the export failed.
         With parties, the group's party image (Engine.export_parties) follows the queue image in the same array;
      4. target -> source: [0] if Engine.merge_queues took it, else [1].

    mm_export_queues and mm_merge refuse while a party is queued, so an engine with parties releases the others around
    them (export_parties) and merges them back (merge_parties: with their numbers where the sequence did not move).
    The target merges the moved parties after the solos.

    Every engine call of a move is caught, so the peer always gets its next message.  If step 4 fails anyway (a CUDA
    error, an active set that filled in between), the source merges the image back, and the party image (new numbers
    there).  Should that fail too (the released players' dead slots still count in the source's pool until its next
    tick), the image is kept in `stranded` instead of being lost: merge it into the source (Engine.merge_queues) after
    its next tick.  With parties, stranded[g] is a tuple of the images this rank could not put back: queue images
    (magic MM_QUEUE_IMAGE_MAGIC) go to Engine.merge_queues, party images (MM_PARTY_IMAGE_MAGIC) to Engine.merge_parties
    — on the target, a moved party image that did not merge after its solos did, or the target's own parties.
    -> dict(moved=[groups], failed=[groups], stranded={group: image or tuple of images}) as seen by this rank.

    Routing is the caller's job: new deliveries of a moved group must go to its new owner (route(..., owners=new))
    on every rank from the move on, and those of a failed move to the old one."""
    old, new = np.asarray(old, np.int64), np.asarray(new, np.int64)
    out = {"moved": [], "failed": [], "stranded": {}}
    for g in range(cfg.n_groups):
        src, dst = int(old[g]), int(new[g])
        if src == dst or rank not in (src, dst):
            continue
        if rank == src:
            try:
                n = int(engine.queue_stats(0)["n_waiting"].reshape(cfg.n_modes, cfg.n_groups)[:, g].sum())
                m = _party_members(engine, g)
            except Exception:
                n, m = -1, 0
            comm.send(src, dst, (np.array([n, m] if m else [n], np.int64),))
            (reply,) = comm.recv(dst, src)
            ok = n >= 0 and _status(reply) == 0
            left = []  # images that could not go back into this engine
            if ok:
                mask = np.zeros((cfg.n_modes, cfg.n_groups), bool)
                mask[:, g] = True
                pimg = rest = img = None
                try:  # a refused export (e.g. a staged packed batch) changes nothing; the target still gets a message
                    if getattr(engine, "party_capacity", 0):
                        pimg = np.ascontiguousarray(engine.export_parties(mask), np.uint8)
                        rest = np.ascontiguousarray(engine.export_parties(~mask), np.uint8)
                    img = np.ascontiguousarray(engine.export_queues(mask), np.uint8)
                except Exception:
                    img = None
                for b, keep in ((rest, True), (pimg if img is None else None, False)):
                    if b is not None:
                        try:
                            engine.merge_parties(b, keep_seq=keep)
                        except Exception:
                            left.append(b)
                if img is None:
                    pimg = None
                msg = np.array([-1], np.int64)
                if img is not None:
                    msg = img.view(np.int64) if pimg is None else np.concatenate([img, pimg]).view(np.int64)
                comm.send(src, dst, (msg,))
                (status,) = comm.recv(dst, src)
                ok = img is not None and _status(status) == 0
                if img is not None and not ok:  # the group's queues hold only dead slots here now: the images go back
                    back, rest_left = _merge_with_parties(engine, img, pimg)
                    left += rest_left if back else [img] + ([pimg] if pimg is not None else []) + rest_left
            if left:
                out["stranded"][g] = left[0] if len(left) == 1 and left[0] is img else tuple(left)
        else:
            (prop,) = comm.recv(src, dst)
            n = _status(prop)
            n_party = int(np.asarray(prop).reshape(-1)[1]) if np.asarray(prop).size > 1 else 0
            try:
                ok = n >= 0 and can_take(cfg, engine, g, n, n_party)
            except Exception:
                ok = False
            comm.send(dst, src, (np.array([0 if ok else 1], np.int64),))
            if ok:
                (arr,) = comm.recv(src, dst)
                arr = np.ascontiguousarray(arr).view(np.uint8)
                ok = len(arr) > 8
                if ok:
                    q = int(arr[16:24].view(np.uint64)[0])  # the queue image's total_bytes; its party image follows
                    img, pimg = arr[:q], (arr[q:] if len(arr) > q else None)
                    ok, left = _merge_with_parties(engine, img, pimg)
                    if left:  # taken: what did not merge here is kept (the source has released it)
                        out["stranded"][g] = tuple(left)
                comm.send(dst, src, (np.array([0 if ok else 1], np.int64),))
        out["moved" if ok else "failed"].append(g)
    return out


# ======================================================================================================================
# Re-cut: a new rating-group table and owner array for every rank at once (mm_import_regroup_many).  Every old rank
# exports its engine; each new rank loads the images of the old ranks whose players can map to a queue it owns under
# the new table, keeps those queues, and takes its own active section.  The world size does not change.
# ======================================================================================================================
def recut_sends(old_cfg, new_cfg, old_owners, new_owners, world):
    """-> bool [world, world]: send[s, d] = an image of old rank s can hold a player that new rank d keeps (s != d).
    Every rating behaves like one of the clamped domain [min(rmin) - 1, max(rmax) + 1] of the two configs."""
    lo = min(min(c.group_lo[g] for g in range(c.n_groups)) for c in (old_cfg, new_cfg)) - 1
    hi = max(max(c.group_hi[g] for g in range(c.n_groups)) for c in (old_cfg, new_cfg)) + 1
    r = np.arange(lo, hi + 1, dtype=np.int64)
    go, gn = group_of_rating(old_cfg, r), group_of_rating(new_cfg, r)
    ok = (go >= 0) & (gn >= 0)
    send = np.zeros((world, world), bool)  # a mode both configs have maps a rating to the same groups in every mode
    send[np.asarray(old_owners, np.int64)[go[ok]], np.asarray(new_owners, np.int64)[gn[ok]]] = True
    np.fill_diagonal(send, False)
    return send


def _exchange(rank, world, comm, out, want):
    """Point-to-point with every other rank in ascending pair order (every rank's pairs come in one global order, so
    blocking calls cannot deadlock): out(d) -> the arrays for d or None; want(s) -> whether s sends to me.
    -> {s: arrays received}"""
    got = {}
    for other in range(world):
        if other == rank:
            continue
        for step in ((0, 1) if rank < other else (1, 0)):
            if step == 0:
                arrays = out(other)
                if arrays is not None:
                    comm.send(rank, other, arrays)
            elif want(other):
                got[other] = comm.recv(other, rank)
    return got


def recut(pkg, old_cfg, new_cfg, old_owners, new_owners, rank, engine, comm, make_engine=None, party_capacity=None):
    """Re-cut a deployment sharded by rating group to a new group table and owner array; every rank of the job calls
    this with the same arguments.  world = 1 + the largest rank in either owner array, and every rank below it calls.
      1. every rank exports its engine (export_state: the old engine is never changed);
      2. every rank computes the same send matrix (recut_sends) and old rank s sends its image, as one int64 array,
         to every rank d with send[s, d] (or [-1] if its export failed); a rank always keeps its own image;
      3. every rank creates an engine under new_cfg (make_engine, default pkg.Engine) and calls import_regroup_many
         with the images in old-rank order, keep = the queues of the groups new_owners gives it, active_image = its
         own image;
      4. every rank sends its status ([0] ok, [1] failed) to every other rank.  Only if all succeeded does each rank
         keep its new engine and close the old one; otherwise every rank closes its new engine and keeps the old one,
         untouched: a failure anywhere loses no player.
    Parties (an engine with party_capacity): mm_export refuses while a party is queued, so in step 1 the rank first
    releases its parties (export_parties) and then exports its engine: both images come from the same stop.  The party
    image follows the engine image in the array of step 2 (the send matrix is unchanged: a party's R is a rating of the
    clamped domain), the new engine gets party_capacity (default: the old engine's) and loads both kinds with
    import_regroup_many_parties.  On failure anywhere every rank merges its own party image back into its old engine
    with keep_seq (valid right after the release: nothing else is queued as a party and seq_next has not moved), which
    leaves it as it was; a party image that cannot go back is returned as `stranded` (merge it with
    Engine.merge_parties).  Engines without party capacity take the path above unchanged.
    Preconditions: no ingest or tick on any rank during the call, and routing switches to route(new_cfg, ...,
    owners=new_owners) after it.  While it runs, each rank holds its old engine, its new one and the images it loads.
    With more than one old image a rank's players and parties are renumbered (include/mm_engine.h): requeue records
    of players and parties matched before the re-cut do not carry over.
    -> dict(ok, engine: the engine this rank uses from now on, dropped: ids of this rank's own players that have no
    queue under new_cfg (they left: answer them), elsewhere: players skipped here because another rank owns them,
    bytes_sent: bytes this rank sent; with parties also dropped_parties: the member ids of this rank's own parties that
    have no queue under new_cfg, parties_elsewhere, stranded: this rank's party image if it could not go back, else
    None)."""
    make_engine = make_engine or pkg.Engine
    old_owners, new_owners = np.asarray(old_owners, np.int64), np.asarray(new_owners, np.int64)
    world = int(max(old_owners.max(initial=0), new_owners.max(initial=0))) + 1
    send = recut_sends(old_cfg, new_cfg, old_owners, new_owners, world)
    sent = [0]
    parties = bool(getattr(engine, "party_capacity", 0))
    if party_capacity is None:
        party_capacity = getattr(engine, "party_capacity", 0)

    def counted(arrays):
        sent[0] += sum(np.asarray(a).nbytes for a in arrays)
        return arrays

    pimg = img = None
    try:
        if parties:
            pimg = np.ascontiguousarray(engine.export_parties(), np.uint8)
        img = np.ascontiguousarray(engine.export_state(), np.uint8)
    except Exception:
        img = None
    if img is None:
        mine = np.array([-1], np.int64)
    else:
        mine = img.view(np.int64) if not parties else np.concatenate([img, pimg]).view(np.int64)
    got = _exchange(rank, world, comm, lambda d: counted((mine,)) if send[rank, d] else None,
                    lambda s: bool(send[s, rank]))
    images, pimages, own = [], [], None
    for s in range(world):
        if s == rank:
            own = len(images)
            images.append(img)
            pimages.append(pimg)
        elif send[s, rank]:
            arr = np.ascontiguousarray(got[s][0]).view(np.uint8)
            if len(arr) <= 8:
                images.append(None)
                pimages.append(None)
                continue
            q = int(arr[16:24].view(np.uint64)[0])  # the engine image's total_bytes; its party image follows
            images.append(arr[:q])
            pimages.append(arr[q:] if len(arr) > q else None)
    new, dropped, elsewhere = None, np.zeros(0, np.uint64), 0
    dropped_parties, p_else = np.zeros(0, np.uint64), 0
    ok = all(x is not None for x in images)
    use_parties = parties or any(p is not None for p in pimages)
    if ok:
        try:
            new = make_engine(new_cfg)
            keep = np.broadcast_to(new_owners == rank, (new_cfg.n_modes, new_cfg.n_groups))
            if use_parties:
                if party_capacity:
                    new.set_option("party_capacity", party_capacity)
                rejected, elsewhere, prej, p_else = new.import_regroup_many_parties(images, pimages, keep=keep,
                                                                                    active_image=own)
                if pimg is not None and len(prej):
                    _h, c = pkg.engine.read_party_image(pimg.tobytes())
                    off = np.concatenate([[0], np.cumsum(c["size"].astype(np.int64))])
                    mine_rej = prej[prej[:, 0] == own, 1]
                    dropped_parties = np.concatenate(
                        [np.zeros(0, np.uint64)] + [np.asarray(c["id"][off[j]:off[j + 1]], np.uint64) for j in mine_rej])
            else:
                rejected, elsewhere = new.import_regroup_many(images, keep=keep, active_image=own)
            ids = pkg.engine.read_image(images[own])[1]["id"]
            dropped = np.asarray(ids[rejected[rejected[:, 0] == own, 1]], np.uint64)
        except Exception:
            ok = False
    status = np.array([0 if ok else 1], np.int64)
    got = _exchange(rank, world, comm, lambda d: counted((status,)), lambda s: True)
    ok = ok and all(_status(got[s][0]) == 0 for s in got)
    if ok:
        engine.close()
        out = dict(ok=True, engine=new, dropped=dropped, elsewhere=int(elsewhere), bytes_sent=sent[0])
        if parties:
            out.update(dropped_parties=dropped_parties, parties_elsewhere=int(p_else), stranded=None)
        return out
    if new is not None:
        new.close()
    out = dict(ok=False, engine=engine, dropped=np.zeros(0, np.uint64), elsewhere=0, bytes_sent=sent[0])
    if parties:
        stranded = None
        if pimg is not None:
            try:
                engine.merge_parties(pimg, keep_seq=True)
            except Exception:
                stranded = pimg
        out.update(dropped_parties=np.zeros(0, np.uint64), parties_elsewhere=0, stranded=stranded)
    return out


# ======================================================================================================================
# One lobby budget per game mode over several engines (mm_set_lobby_budget, include/mm_engine.h).  A mode's budget is
# apportioned over ALL its rating groups by their candidate lobbies; sharded by group, no engine sees all of them.  Every
# engine reports its own (Engine.lobby_candidates, a dry run that changes nothing), the counts are gathered, every rank
# computes the same apportionment and sets the per-queue budgets of its own engine: K engines under one mode budget then
# emit exactly what a single engine with per_mode would.
# ======================================================================================================================
UNLIMITED = 0xFFFFFFFF


def apportion(budget, cand):
    """Largest-remainder apportionment of `budget` lobbies over queues with cand[g] candidate lobbies each, the rule
    of mm_set_lobby_budget in 64-bit integers: everything if sum(cand) <= budget, else floor(budget * cand[g] / sum)
    each and one more for the budget - sum(floors) queues with the largest (budget * cand[g]) mod sum, ties to the
    lower index.  -> int64[len(cand)], never above cand."""
    c = np.asarray(cand, np.uint64)
    total, budget = int(c.sum(dtype=np.uint64)), int(budget)
    if total <= budget:
        return c.astype(np.int64)
    prod = c * np.uint64(budget)  # budget < total <= 2^32 and cand < 2^32: the product fits 64 bits
    a, rem = (prod // np.uint64(total)).astype(np.int64), prod % np.uint64(total)
    extra = budget - int(a.sum())
    first = np.lexsort((np.arange(len(c)), np.uint64(total) - rem))  # remainder descending, then index ascending
    a[first[:extra]] += 1
    return a


def queue_budgets(cfg, per_mode, cand):
    """Per-queue budgets (u32[n_modes * n_groups], queue_stats() record order) that make engines holding parts of a
    pool emit what one engine with `per_mode` would: cand = the candidate lobbies of every queue over the whole pool."""
    cand = np.asarray(cand, np.int64).reshape(cfg.n_modes, cfg.n_groups)
    out = np.empty((cfg.n_modes, cfg.n_groups), np.int64)
    for m in range(cfg.n_modes):
        b = int(per_mode[m])
        out[m] = cand[m] if b >= UNLIMITED else apportion(b, cand[m])
    return out.reshape(-1).astype(np.uint32)


def set_mode_budget(engines, per_mode, comm=None, rank=0, world=1):
    """Put the engines of a job under one lobby budget per game mode for the next tick.  engines: all of the job's
    engines when they share this process, or this rank's engine (with comm, rank, world: every rank calls this with the
    same per_mode; the counts travel as int64 arrays over comm.send / comm.recv, ranks pairing up in a fixed order so
    that blocking calls cannot deadlock).  Call it before every tick: the candidates change with the pool.
    -> the per-queue budgets that were set."""
    engines = list(engines) if isinstance(engines, (list, tuple)) else [engines]
    cfg = engines[0].cfg
    cand = sum(np.asarray(e.lobby_candidates(), np.int64) for e in engines)
    if comm is not None:
        mine = cand.copy()
        for peer in range(world):
            if peer == rank:
                continue
            if rank < peer:
                comm.send(rank, peer, (mine,))
                (theirs,) = comm.recv(peer, rank)
            else:
                (theirs,) = comm.recv(peer, rank)
                comm.send(rank, peer, (mine,))
            cand = cand + np.asarray(theirs).view(np.int64)
    budgets = queue_budgets(cfg, per_mode, cand)
    for e in engines:
        e.set_lobby_budget(per_queue=budgets)
    return budgets
