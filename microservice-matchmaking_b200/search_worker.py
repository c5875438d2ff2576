"""Host-side mirror of the reference search stage's worker interface.

Reference: matchmaking/lib/search/worker.ex (`Matchmaking.Search.Worker`), a GenServer
per (rating group, worker id).  The BEAM toolchain is absent in this environment
(SURVEY F5), so the host side above the C ABI is mirrored in Python with the same
names, argument meaning and error behaviour:

    start_link(opts)                 worker.ex:68-71     opts: group_name (required), channel_name
    configure(channel_name, opts)    worker.ex:73-76     declares/consumes the group queue
    consume(channel_name, group_name, tag, headers, payload)   worker.ex:291-324
    ack / nack(channel_name, tag)    worker.ex:81-90
    status()                         worker.ex:115-117,326-334
    handle_info(msg)                 worker.ex:337-368

What changed behind the interface: consume/5 no longer pops a partial lobby from Mnesia
and asks the strategist per request (worker.ex:295-321).  It stages the player in the
shared `SearchPool` (the GPU-resident pool, `Matchmaking.Search.Engine` in
INTEGRATION.md); `SearchPool.flush()` ingests a batch through mm_enqueue and acks the
deliveries once the players are resident (manual ack after processing, worker.ex:323);
`SearchPool.tick()` runs one search tick and publishes every emitted lobby as the same
JSON document, to the same exchange/routing key, with the same publish options as
prepare_game_lobby/4 (worker.ex:250-261, 315-319).  A player that is not matched is not
re-published to the requeue exchange (worker.ex:239-248): it simply stays resident.

The AMQP connection is duck-typed (declare_exchange / declare_queue / bind / qos /
basic_consume / basic_publish / basic_ack / basic_nack / queue_status) so the same code
drives a real client or the in-memory broker used by the tests.
"""
import heapq
import json
import math

import numpy as np

from . import abi

# module attributes of the reference (worker.ex:23-40)
DEFAULT_EXCHANGE_PATH = "open-matchmaking.matchmaking"
DEFAULT_EXCHANGE_TYPE = "direct"
DEFAULT_QUEUE_PATH = "matchmaking.queues"
QUEUE_OPTIONS = {"durable": True}
EXCHANGE_OPTIONS = {"type": "direct", "durable": True}
QOS_OPTIONS = {"prefetch_count": 10}
EXCHANGE_FORWARD = "open-matchmaking.matchmaking.game-lobby.direct"
QUEUE_FORWARD = "matchmaking.queues.lobbies"
EXCHANGE_REQUEUE = "open-matchmaking.matchmaking.requeue.direct"
QUEUE_REQUEUE = "matchmaking.games.requeue"
EXCHANGE_RESPONSE = "open-matchmaking.responses.direct"  # game-lobby/worker.ex:27
TIMEOUT_DETAILS = "No opponents were found within the search time limit."


def prepare_timeout_response(player):
    """The error response of game-lobby/worker.ex:63-71 with the search timeout as its cause."""
    return json.dumps({"error": {"type": "MatchmakingError", "details": TIMEOUT_DETAILS},
                       "event-name": player.get("event-name")})


def generate_queue_name(suffix):  # worker.ex:46-48
    return f"{DEFAULT_QUEUE_PATH}.{suffix}"


def generate_exchange_name(suffix):  # worker.ex:50-52
    return f"{DEFAULT_EXCHANGE_PATH}.{suffix}.{DEFAULT_EXCHANGE_TYPE}"


def prepare_config(opts):  # worker.ex:54-66
    """opts["prefetch_count"] overrides the reference's QoS (worker.ex:29: 10).  The batched worker acks a delivery only
    once its player is resident in the pool (SearchPool.flush), so a prefetch of 10 would cap the ingest at 10
    players per worker per flush: start_link passes the pool's batch size instead (INTEGRATION.md §3)."""
    if not opts.get("group_name"):
        raise RuntimeError("You need to configure group_name in options.")
    queue_name = generate_queue_name(opts["group_name"])
    qos = dict(QOS_OPTIONS)
    if opts.get("prefetch_count"):
        qos["prefetch_count"] = int(opts["prefetch_count"])
    return {
        "queue": dict(name=queue_name, routing_key=queue_name, **QUEUE_OPTIONS),
        "exchange": dict(name=generate_exchange_name(opts["group_name"]), **EXCHANGE_OPTIONS),
        "qos": qos,
    }


class HandleTable:
    """Host-side player id <-> dense device handle table (SURVEY §7.3 "dense slot index").

    Reference ids are UUID strings (active_user.ex:7); the device stores a small integer.  A table — not a hash of
    the id — so that two players can never collide into "You are already in the queue." and so that the Elixir and
    Python hosts need not agree on a hash function; handles are recycled when the player leaves the active set
    (ActiveUser.remove_user/1).  With an MM_F_DENSE_IDS engine the handle indexes the device's active set directly."""

    def __init__(self, capacity=None):
        self.capacity = capacity
        self.handle_of = {}
        self.id_of = []
        self.free = []

    def acquire(self, player_id):
        """-> (handle, is_new).  None when the handle range is exhausted."""
        h = self.handle_of.get(player_id)
        if h is not None:
            return h, False
        if self.free:
            h = self.free.pop()
            self.id_of[h] = player_id
        else:
            if self.capacity is not None and len(self.id_of) >= self.capacity:
                return None, False
            h = len(self.id_of)
            self.id_of.append(player_id)
        self.handle_of[player_id] = h
        return h, True

    def lookup(self, player_id):
        return self.handle_of.get(player_id)

    def release(self, player_id):
        h = self.handle_of.pop(player_id, None)
        if h is not None:
            self.id_of[h] = None
            self.free.append(h)
        return h

    def __len__(self):
        return len(self.handle_of)


class WindowSchedule:
    """EXTENSION beyond the reference (SURVEY F3 / §8f-3): time-expanded search window.

    The reference stamps `created_at` on every queued player (active_user.ex:47) and never
    reads it; its strategist decides without a notion of waiting time.  This schedule turns
    the wait of the LONGEST-waiting queued player into the tick's maximum lobby spread
    (strategist policy S1, mm_set_option("max_spread")):

        W(now) = min(w_max, w0 + growth_per_s * (now - enqueue_time(oldest queued player)))

    so a sparse pool relaxes until its oldest player can be matched and tightens again once
    it has left.  One window per tick for the whole pool; per-player windows run after the
    tick (SearchPool(widen=...), Engine.widen)."""

    def __init__(self, w0, growth_per_s, w_max):
        self.w0, self.growth_per_s, self.w_max = int(w0), float(growth_per_s), int(w_max)

    def spread(self, now, oldest_enqueued_at):
        wait = 0.0 if oldest_enqueued_at is None else max(0.0, float(now) - float(oldest_enqueued_at))
        return int(min(self.w_max, self.w0 + self.growth_per_s * wait))


class SearchPool:
    """Owner of the GPU pool shared by every search worker of this node.

    engine: an object with the `Engine` API (enqueue / tick / remove / in_queue /
    pool_size / set_option); mode_names: index -> "1v1", ...; group_names: index -> "bronze", ...
    max_batch: deliveries staged before an ingest (also the QoS prefetch every worker asks the broker for: a
    delivery is acked only once its player is resident, so the broker must be allowed that many unacked messages);
    flush_every_s: an ingest also happens when the oldest staged delivery has waited this long (and at every tick);
    window: optional WindowSchedule (extension; needs MM_ORDER_RATING); clock: () -> seconds.
    timeout_ms: optional search time limit (extension): after each tick's lobbies are published, every player still
    queued who has waited at least this long leaves the pool (Engine.expire) and gets the error response of
    game-lobby/worker.ex:63-71 on its "response-queue".  None (the default) never expires anyone.
    lobby_budget: optional flow control (extension): a callable () -> {mode name: lobbies} asked before every tick —
    the free game-server slots, what the lobby stage would otherwise find out per lobby (calculate_required_slots,
    game-lobby/worker.ex:118-141); a mode it does not name is unlimited.  The tick emits at most that many lobbies of
    the mode (Engine.set_lobby_budget), shared over the rating groups in proportion to what each could emit; the rest
    stay ordinary queued players (timeout_ms, requeue, move_out, checkpoint treat them as such).  pause() / resume_queues()
    set single queues to 0 / unlimited.  A checkpoint does not carry budgets or pauses: resume() starts unlimited.
    widen: optional per-player search windows (extension; needs MM_ORDER_RATING): {mode name: (min_wait_ms, w0,
    step_ms, inc, w_max)}.  After each tick's lobbies are published, and before timeout_ms expires anyone, every player
    of the mode who has waited at least min_wait_ms anchors a lobby in a rating window of w0 points either side, plus
    inc per whole step_ms waited past min_wait_ms, at most w_max (Engine.widen, every rating group of the mode).  Its
    lobbies are published like the tick's; stats["widened"] counts them.
    balance_teams: optional list of mode names (extension; two-team modes of at most 8 players a team): every lobby of
    those modes, from the tick and from widen, is split into the two teams with the least rating difference
    (mm_set_option("team_balance")).  Membership and lobby order are unchanged; team t is still members
    [t * team_size, (t + 1) * team_size).  resume() sets it again on the new engine.
    balance_parties: optional list of mode names (extension; two-team modes of at most 8 players a team): every
    party_match lobby of those modes is split into its most even teams that keep every party whole
    (mm_set_option("party_balance")); the published "teams" follow that order.  Independent of balance_teams, which
    never splits party lobbies.  resume() sets it again on the new engine.
    parties / party_capacity: optional parties (extension; needs MM_ORDER_RATING): players who queue together, staged
    with stage_party() and acked or nacked as one delivery, are matched into one lobby and one team.  party_capacity
    sets how many party members the engine holds (mm_set_option("party_capacity")); parties = {mode name: (min_wait_ms,
    w0, step_ms, inc, w_max)} is the party window of the mode, as widen takes it.  Every tick runs Engine.party_match
    before the tick itself, so parties get the first pick of the solos; its lobbies are published like the tick's and
    stats["party_lobbies"] counts them.  A party member removed with remove_user() takes its whole party out; a matched
    member's requeue() answers "gone" (the caller enqueues the party again).
    budget_offtick: with lobby_budget, one step's budget covers every lobby the step publishes (extension,
    Engine.set_offtick_budget): party_match runs under the callable's per-mode budget F, the tick under F minus the
    step's party lobbies of each mode, widen under what is left; paused queues emit nothing from any of the three, and
    held_back() reports each source.  Off (the default), party_match and widen run without a budget.
    requeue_parties: with parties, requeue() puts matched parties back as parties (extension, Engine.requeue_party):
    the pool keeps a book of every queued party (members, ratings, mode, stamp and enqueue sequence number) and moves a
    party's entry aside when party_match places it, until remove_user or a requeue.  Off (the default), requeue() of a
    matched party member answers "gone" as described above.

    Every ingest batch is stamped with now_ms(), the clock in milliseconds since the pool was created (u32, wraps
    after 49 days), and every tick passes the same clock as its `now`: the engine's per-queue waits
    (Engine.queue_stats, SearchWorker.status) are in milliseconds.
    """

    def __init__(self, engine, mode_names, group_names, max_batch=65536, window=None, clock=None, flush_every_s=0.005,
                 handle_capacity=None, timeout_ms=None, wall_clock=None, lobby_budget=None, widen=None,
                 balance_teams=None, parties=None, party_capacity=None, requeue_parties=False, balance_parties=None,
                 budget_offtick=False):
        import time
        if widen and engine.cfg.order_mode != abi.MM_ORDER_RATING:
            raise ValueError("widen needs an MM_ORDER_RATING engine: windows are rating distances")
        if (parties or party_capacity) and engine.cfg.order_mode != abi.MM_ORDER_RATING:
            raise ValueError("parties need an MM_ORDER_RATING engine: party windows are rating distances")
        self.window = window
        self.widen = {(i, g): tuple(int(x) for x in widen[m]) for i, m in enumerate(mode_names) if m in (widen or {})
                      for g in range(len(group_names))}
        self.party_rules = {(i, g): tuple(int(x) for x in parties[m]) for i, m in enumerate(mode_names)
                            if m in (parties or {}) for g in range(len(group_names))}
        self.party_capacity = int(party_capacity or 0)
        if party_capacity:
            engine.set_option("party_capacity", int(party_capacity))
        self.party_of = {}  # handle -> the handles of its queued party (remove_user takes the whole party out)
        # requeue_parties: handle -> the record of its party ({"members", "rating", "mode", "ts", "seq"}, one dict shared
        # by the members), while the party is queued (party_book) and once party_match has placed it (matched_parties)
        self.requeue_parties = bool(requeue_parties)
        self.party_book = {}
        self.matched_parties = {}
        self._staged_parties = []  # (worker, tag, [player documents], game mode)
        self.timeout_ms = timeout_ms
        self.lobby_budget = lobby_budget
        self.budget_offtick = bool(budget_offtick)
        self.paused = set()  # queues (mode * n_groups + group) that emit nothing until resume_queues()
        self.clock = clock or time.monotonic
        self.wall_clock = wall_clock or time.time  # seconds since the epoch: checkpoint() / resume() bridge the downtime
        self._t0 = self.clock()
        self.enqueued_at = {}  # handle -> clock() when the player became resident (insertion = enqueue order)
        self.matched_at = {}   # window: the enqueued_at of players matched and not yet removed (requeue() puts it back)
        self.last_spread = None
        self.engine = engine
        self.mode_names = list(mode_names)
        self.mode_index = {m: i for i, m in enumerate(self.mode_names)}
        self.group_names = list(group_names)
        for arg, option, names in (("balance_teams", "team_balance", balance_teams),
                                   ("balance_parties", "party_balance", balance_parties)):
            if names:
                unknown = [m for m in names if m not in self.mode_index]
                if unknown:
                    raise ValueError(f"{arg} names unknown modes {unknown}")
                engine.set_option(option, sum(1 << self.mode_index[m] for m in set(names)))
        self.max_batch = max_batch
        self.flush_every_s = flush_every_s
        self.handles = HandleTable(handle_capacity)
        self.players = {}   # handle -> decoded player document (without "game-mode")
        # handle -> [rating, mode, enq_ts, seq] at its enqueue: what requeue() hands the engine back (kept from flush()
        # until remove_user, for engines with seq_next())
        self.queued = {}
        self.moved_out = set()  # queues (mode * n_groups + group) released by move_out() and not moved back in
        self.workers = {}   # group name -> worker that publishes the group's lobbies
        self._staged = []   # (player id, rating, mode, player, worker, tag)
        self._staged_since = None
        self.stats = {"enqueued": 0, "duplicates": 0, "invalid": 0, "lobbies": 0, "failed_batches": 0}
        if timeout_ms is not None:
            self.stats["timed_out"] = 0
        if self.widen:
            self.stats["widened"] = 0
        if self.party_rules or party_capacity:
            self.stats["party_lobbies"] = 0

    def now_ms(self):
        """The pool's clock: milliseconds since the pool was created, modulo 2^32 (the engine's enq_ts / now)."""
        return int((self.clock() - self._t0) * 1000.0) & 0xFFFFFFFF

    # -- models/active_user.ex mirrors ---------------------------------------------------
    def in_queue(self, player_id):  # ActiveUser.in_queue?/1
        h = self.handles.lookup(player_id)
        return h is not None and bool(self.engine.in_queue([h])[0])

    def remove_user(self, player_id):  # ActiveUser.remove_user/1 -> {:ok, :removed}
        self.flush()
        h = self.handles.lookup(player_id)
        if h is not None:
            self.engine.remove([h])  # a queued party member: the engine removes its whole party
            for x in self.party_of.pop(h, (h,)):
                self.party_of.pop(x, None)
                self.party_book.pop(x, None)
                self.matched_parties.pop(x, None)
                self.handles.release(self.handles.id_of[x])
                self.players.pop(x, None)
                self.enqueued_at.pop(x, None)
                self.matched_at.pop(x, None)
                self.queued.pop(x, None)
        return ("ok", "removed")

    def requeue(self, players):
        """Put the members of a lobby that did not start (a declined ready check, no game server) back into their
        queue at their enqueue position (Engine.requeue): their wait and the search timeout go on from their first
        enqueue.  players: the lobby's player documents, as the lobby stage has them.  -> one outcome per player:
        "requeued" (queued again; its document is back in the pool), "queued" (still queued: nothing changed) or
        "gone" (not in this pool's active set — removed, timed out, never queued — its queue has moved to another pool,
        or its rating or mode has no queue under this pool's config after a resume(regroup=True): answer it as today,
        remove_user and an error response).  With requeue_parties, the matched party members among `players` go back by
        party: two or more members of one party as one party with the party's stamp and number (Engine.requeue_party;
        the members not among `players` stay out of it), a lone member as a solo with its own rating and the party's
        stamp and number.  The parties go first; if the engine refuses them (the party table is full), they answer
        "gone" and the solos go on.  A lone member whose co-member went back the same way and is still queued in the
        same (mode, group) queue answers "gone": the engine holds one player of a party number per partition."""
        self.flush()
        out = ["gone"] * len(players)
        n_modes = self.engine.cfg.n_modes
        pos, hs, solo_rec, by_party = {}, [], {}, {}
        for i, doc in enumerate(players):
            h = self.handles.lookup(doc.get("id"))
            if h is None or h in pos:
                continue
            if h in self.party_book:  # a member of a queued party: nothing to put back
                pos[h] = i
                out[i] = "queued"
                continue
            party = self.matched_parties.get(h) if self.requeue_parties else None
            if party is not None:
                pos[h] = i
                by_party.setdefault(id(party), (party, set()))[1].add(h)
                continue
            rec = self.queued.get(h)
            if rec is None or rec[1] >= n_modes:
                continue
            q = self._queue_of(rec[0], rec[1])
            if q < 0 or q in self.moved_out:
                continue
            pos[h] = i
            hs.append(h)
        parties = []  # (member handles, ratings, record) of the parties that go back whole
        for party, asked in by_party.values():
            mem = [x for x in party["members"] if x in asked]
            rat = [party["rating"][party["members"].index(x)] for x in mem]
            if party["mode"] >= n_modes:
                continue
            q = self._queue_of(rat[0] if len(mem) == 1 else sum(rat) // len(rat), party["mode"])
            if q < 0 or q in self.moved_out:
                continue
            if len(mem) == 1:  # a lone member goes back as a solo with the party's number
                # ... which a co-member sent back the same way and still queued in this queue holds already: mm_requeue
                # would refuse the whole call, so this one is answered "gone"
                if any(x != mem[0] and x in self.queued and x in self.players and
                       self._queue_of(self.queued[x][0], self.queued[x][1]) == q for x in party["members"]):
                    continue
                solo_rec[mem[0]] = [rat[0], party["mode"], party["ts"], party["seq"]]
                hs.append(mem[0])
            else:
                parties.append((mem, rat, party))
        if parties:  # first: a refused call (the table is full) changes nothing, and its parties answer "gone"
            sizes = np.array([len(m) for m, _r, _p in parties], np.uint8)
            try:
                codes = self.engine.requeue_party(
                    sizes, np.array([x for m, _r, _p in parties for x in m], np.uint64),
                    np.array([x for _m, r, _p in parties for x in r], np.int32),
                    np.array([p["mode"] for _m, _r, p in parties], np.uint8),
                    np.array([p["ts"] for _m, _r, p in parties], np.uint32),
                    np.array([p["seq"] for _m, _r, p in parties], np.uint32))
            except Exception:
                codes = np.full(len(parties), 4, np.uint8)
                self.stats["failed_requeues"] = self.stats.get("failed_requeues", 0) + 1
            for (mem, rat, party), c in zip(parties, codes.tolist()):
                if c == 1:
                    rec = dict(party, members=tuple(mem), rating=tuple(rat))
                    for h in mem:
                        out[pos[h]] = "requeued"
                        self.players[h] = players[pos[h]]
                        self.matched_parties.pop(h, None)
                        self.party_of[h] = tuple(mem)
                        self.party_book[h] = rec
                elif c == 0:
                    for h in mem:
                        out[pos[h]] = "queued"
        back = []  # window: (clock value, handle) of the requeued players
        if hs:
            rec = np.array([self.queued[h] if h in self.queued else solo_rec[h] for h in hs], np.int64)
            codes = self.engine.requeue(np.array(hs, np.uint64), rec[:, 0].astype(np.int32), rec[:, 1].astype(np.uint8),
                                        rec[:, 2].astype(np.uint32), rec[:, 3].astype(np.uint32))
            for h, c in zip(hs, codes.tolist()):
                if c == 1:
                    out[pos[h]] = "requeued"
                    self.players[h] = players[pos[h]]
                    if h in solo_rec:  # a solo from now on
                        self.queued[h] = solo_rec[h]
                        self.matched_parties.pop(h, None)
                    at = self.matched_at.pop(h, None)
                    if self.window and at is not None:
                        back.append((at, h))
                elif c == 0:
                    out[pos[h]] = "queued"
        if back:  # into the oldest-first order the window reads: one merge of two sorted runs
            back.sort()
            self.enqueued_at = dict(heapq.merge(self.enqueued_at.items(), ((h, at) for at, h in back),
                                                key=lambda kv: kv[1]))
        for i, doc in enumerate(players):  # a repeated document shares its first copy's outcome
            h = self.handles.lookup(doc.get("id"))
            if h in pos and pos[h] != i:
                out[i] = out[pos[h]]
        self.stats["requeued"] = self.stats.get("requeued", 0) + out.count("requeued")
        return out

    def backfill(self, requests):
        """Fill the open slots of running lobbies from their queues (Engine.backfill): a lobby that lost members asks
        for players instead of being disbanded.  requests: (game-mode name, group name, target rating, count) or
        (..., count, window) tuples, served in order; each takes up to `count` queued players of its queue, nearest to
        the target rating first within `window` (the oldest first on an arrival-order engine).  -> per request, the
        player documents taken (fewer than count when the queue runs short).  Taken players leave the pool as matched
        players do: requeue() puts them back, remove_user() forgets them."""
        self.flush()
        if not requests:
            return []
        cols = [(self.mode_index[r[0]], self.group_names.index(r[1]), int(r[2]), int(r[3]),
                 -1 if len(r) < 5 or r[4] is None else int(r[4])) for r in requests]
        mode, group, target, count, window = (np.array(c, np.int64) for c in zip(*cols))
        _n_taken, members = self.engine.backfill(mode, group, target, count, window)
        out = []
        for ids in members:
            out.append([self.players.pop(int(x)) for x in ids])
            if self.window:  # kept aside until remove_user: requeue() puts it back
                for x in ids:
                    at = self.enqueued_at.pop(int(x), None)
                    if at is not None:
                        self.matched_at[int(x)] = at
        self.stats["backfilled"] = self.stats.get("backfilled", 0) + sum(len(d) for d in out)
        return out

    def backfill_teams(self, requests):
        """Fill the open team slots of running lobbies with whole queued parties, then the nearest solos
        (Engine.backfill_party; needs party_capacity): a lobby that lost a premade can take another party on one team.
        requests: (game-mode name, group name, target rating, [open slots per team]) or (..., slots, window) tuples,
        served in order.  -> per request, one list of player documents per team: the team's parties first, each party's
        members together, then its solos (fewer than the open slots when the queue runs short: requeue() hands a short
        fill back).  Taken players leave the pool as matched players do; a placed party is kept aside as party_match's
        are, so requeue() with requeue_parties puts it back whole."""
        self.flush()
        if not requests:
            return []
        mode = [self.mode_index[r[0]] for r in requests]
        group = [self.group_names.index(r[1]) for r in requests]
        target = [int(r[2]) for r in requests]
        room = [[int(x) for x in r[3]] for r in requests]
        window = [-1 if len(r) < 5 or r[4] is None else int(r[4]) for r in requests]
        _filled, members = self.engine.backfill_party(np.array(mode, np.int64), np.array(group, np.int64),
                                                      np.array(target, np.int64), room, np.array(window, np.int64))
        out = []
        for teams in members:
            docs = []
            for ids in teams:
                docs.append([self.players.pop(int(x)) for x in ids])
                for x in ids.tolist():
                    if x in self.party_of:  # a placed party's member: its record moves aside, as after party_match
                        self.party_of.pop(x, None)
                        rec = self.party_book.pop(x, None)
                        if rec is not None:
                            self.matched_parties[x] = rec
                    if self.window:  # kept aside until remove_user: requeue() puts it back
                        at = self.enqueued_at.pop(x, None)
                        if at is not None:
                            self.matched_at[x] = at
            out.append(docs)
        self.stats["backfilled_teams"] = self.stats.get("backfilled_teams", 0) + sum(
            len(d) for teams in out for d in teams)
        return out

    def search_status(self, player_ids):
        """Where each player's search stands (Engine.locate at now_ms()), without ingesting the staged deliveries.
        -> one dict per player id: "state" is "searching" (queued), "matched" (placed in a lobby, or taken by backfill,
        and not yet removed), "staged" (received, not yet ingested: only its "game_mode" and "group" are known) or
        "unknown"; "game_mode" and "group" name its queue; "wait_ms" is its wait; "position" counts the players of its
        queue that the tick feeds before it and "queue_size" the players of the queue; "next_tick" is {"lobby": ordinal
        among the queue's lobbies of the next tick, "team": team index} or None if the next tick leaves it queued.
        The prediction holds for the engine as it is set now.  A pool with a WindowSchedule or a lobby_budget callable
        sets max_spread and the budgets again before each tick, so its prediction is "under the current spread and
        budget" — the next tick may use others.  Fields that do not apply to a state are None."""
        empty = dict(state="unknown", game_mode=None, group=None, wait_ms=None, position=None, queue_size=None,
                     next_tick=None)
        out = [dict(empty) for _ in player_ids]
        known = [(i, h) for i, pid in enumerate(player_ids) for h in [self.handles.lookup(pid)] if h is not None]
        if known:
            rec = self.engine.locate(np.array([h for _i, h in known], np.uint64), self.now_ms())
            for (i, _h), r in zip(known, rec):
                if r["state"] == 2:
                    out[i]["state"] = "matched"
                elif r["state"] == 1:
                    m = int(r["mode"])
                    nxt = None
                    if int(r["lobby"]) != 0xFFFFFFFF:
                        nxt = {"lobby": int(r["lobby"]), "team": int(r["member"]) // self.engine.cfg.modes[m].team_size}
                    out[i].update(state="searching", game_mode=self.mode_names[m], group=self.group_names[int(r["group"])],
                                  wait_ms=int(r["wait"]), position=int(r["ahead"]), queue_size=int(r["depth"]),
                                  next_tick=nxt)
        staged = {}
        for s in self._staged:  # the first delivery of a player names its queue
            staged.setdefault(s[0], s)
        for i, pid in enumerate(player_ids):
            s = staged.get(pid)
            if out[i]["state"] != "unknown" or s is None:
                continue
            mode = self.mode_index.get(s[2]) if isinstance(s[2], str) else None
            q = self._queue_of(s[1], mode) if mode is not None else -1
            out[i].update(state="staged", game_mode=s[2] if mode is not None else None,
                          group=self.group_names[q % len(self.group_names)] if q >= 0 else None)
        return out

    def party_search_status(self, player_ids):
        """Where each party member's search stands (Engine.party_locate at now_ms() under the pool's party rules),
        without ingesting the staged deliveries.  -> one dict per player id: "state" is "searching" (queued in a party),
        "matched" (placed in a lobby, or taken, and not yet removed), "staged" (its party was received, not yet
        ingested: only "game_mode", "group" and "party_size" are known) or "unknown" (anything else, a queued solo
        included: see search_status); "game_mode" and "group" name its party's queue; "party_size" counts the party;
        "wait_ms" is the party's wait; "position" counts the parties of the queue older than its party and
        "queue_size" the queue's parties; "anchor" says whether the party has waited long enough to anchor a lobby and
        "window" is then its rating window; "next_match" is {"lobby": ordinal among the queue's lobbies of the next
        party_match, "team": team index} or None if its party stays queued.  The prediction holds for the engine and
        the off-tick budget as they are set now.  Fields that do not apply to a state are None."""
        empty = dict(state="unknown", game_mode=None, group=None, party_size=None, wait_ms=None, position=None,
                     queue_size=None, anchor=None, window=None, next_match=None)
        out = [dict(empty) for _ in player_ids]
        known = [(i, h) for i, pid in enumerate(player_ids) for h in [self.handles.lookup(pid)] if h is not None]
        if known and self.party_capacity and hasattr(self.engine, "party_locate"):
            rec = self.engine.party_locate(np.array([h for _i, h in known], np.uint64), self.now_ms(), self.party_rules)
            for (i, _h), r in zip(known, rec):
                if r["state"] == 2:
                    out[i]["state"] = "matched"
                elif r["state"] == 3:
                    m = int(r["mode"])
                    nxt = None
                    if int(r["lobby"]) != 0xFFFFFFFF:
                        nxt = {"lobby": int(r["lobby"]), "team": int(r["member"]) // self.engine.cfg.modes[m].team_size}
                    out[i].update(state="searching", game_mode=self.mode_names[m], group=self.group_names[int(r["group"])],
                                  party_size=int(r["size"]), wait_ms=int(r["wait"]), position=int(r["ahead"]),
                                  queue_size=int(r["depth"]), anchor=bool(r["anchor"]),
                                  window=int(r["window"]) if r["anchor"] else None, next_match=nxt)
        staged = {}
        for (_w, _t, players, game_mode) in self._staged_parties:  # the first delivery of a player names its queue
            for doc in players:
                staged.setdefault(doc.get("id") if isinstance(doc, dict) else None, (players, game_mode))
        for i, pid in enumerate(player_ids):
            s = staged.get(pid)
            if out[i]["state"] != "unknown" or s is None:
                continue
            players, game_mode = s
            mode = self.mode_index.get(game_mode) if isinstance(game_mode, str) else None
            q = -1
            if mode is not None and players:
                q = self._queue_of(sum(int(d["rating"]) for d in players) // len(players), mode)
            out[i].update(state="staged", game_mode=game_mode if mode is not None else None,
                          group=self.group_names[q % len(self.group_names)] if q >= 0 else None,
                          party_size=len(players))
        return out

    def party_queue_status(self, group_name):
        """The engine's view of one rating group's queued parties (Engine.party_queue_stats at now_ms()), per mode name:
        parties and their players, the oldest / p50 / p99 party wait in ms, and "sizes" = {party size: parties} (15
        counts every size from 15 up).  Quantiles are the upper bounds of histogram buckets (at most 25 % high).  {}
        for a group the pool does not know or a pool without party capacity."""
        from .engine import wait_quantile
        if group_name not in self.group_names or not self.party_capacity:
            return {}
        g = self.group_names.index(group_name)
        out = {}
        for r in self.engine.party_queue_stats(self.now_ms()):
            if int(r["group"]) != g or int(r["mode"]) >= len(self.mode_names):
                continue
            out[self.mode_names[int(r["mode"])]] = {
                "parties": int(r["n_parties"]),
                "players": int(r["n_members"]),
                "oldest_wait_ms": int(r["max_wait"]),
                "p50_wait_ms": wait_quantile(r["wait_hist"], 0.50),
                "p99_wait_ms": wait_quantile(r["wait_hist"], 0.99),
                "sizes": {k: int(v) for k, v in enumerate(r["size_hist"].tolist()) if v},
            }
        return out

    def _queue_of(self, rating, mode):
        """(mode, group) queue index of a rating: the first group that holds it, else the default group (-1: none)."""
        cfg = self.engine.cfg
        for g in range(cfg.n_groups):
            if cfg.group_lo[g] <= rating <= cfg.group_hi[g]:
                return int(mode) * cfg.n_groups + g
        return int(mode) * cfg.n_groups + cfg.default_group if cfg.default_group >= 0 else -1

    # -- ingest -----------------------------------------------------------------------------
    def stage(self, worker, tag, player, game_mode, rating):
        if not self._staged:
            self._staged_since = self.clock()
        self._staged.append((player["id"], int(rating), game_mode, player, worker, tag))
        if len(self._staged) >= self.max_batch or self.clock() - self._staged_since >= self.flush_every_s:
            self.flush()

    def stage_party(self, worker, tag, players, game_mode):
        """One delivery that queues several players together: players = their documents (each with "id" and
        "rating").  Ingested at the next flush, after the staged solos; acked once the party is queued (or a member was
        already queued), nacked if it is invalid or the party table is full."""
        if not self._staged and not self._staged_parties:
            self._staged_since = self.clock()
        self._staged_parties.append((worker, tag, list(players), game_mode))
        if len(self._staged) + len(self._staged_parties) >= self.max_batch or \
                self.clock() - self._staged_since >= self.flush_every_s:
            self.flush()

    def _flush_parties(self):
        """mm_enqueue_party the staged parties; ack or nack each party's delivery by its code."""
        staged, self._staged_parties = self._staged_parties, []
        if not staged:
            return 0
        fresh, ids, rating, sizes, mode = [], [], [], [], []
        for (_w, _t, players, game_mode) in staged:
            sizes.append(len(players))
            mode.append(self.mode_index.get(game_mode, 255) if isinstance(game_mode, str) else 255)
            for doc in players:
                h, is_new = self.handles.acquire(doc["id"])
                if h is None:
                    h = 2 ** 64 - 1
                elif is_new:
                    fresh.append(doc["id"])
                ids.append(h)
                rating.append(int(doc["rating"]))
        sizes = np.minimum(np.array(sizes, np.int64), 255).astype(np.uint8)  # a longer list is invalid (code 2)
        ids = np.array(ids, np.uint64)
        rating = np.clip(np.array(rating, np.int64), -(2 ** 31), 2 ** 31 - 1).astype(np.int32)
        try:
            if np.any(sizes.astype(np.int64) != [len(s[2]) for s in staged]):
                raise ValueError("a party of more than 255 players")
            seq0 = self.engine.seq_next() if self.requeue_parties else 0  # party j of the batch gets seq0 + j
            stamp = self.now_ms()
            codes = self.engine.enqueue_party(sizes, ids, rating, np.array(mode, np.uint8),
                                              np.full(len(staged), stamp, np.uint32))
        except Exception:  # nothing was enqueued
            for pid in fresh:
                self.handles.release(pid)
            for (worker, tag, _p, _m) in staged:
                worker.nack(worker.channel_name, tag)
            self.stats["failed_batches"] += 1
            return 0
        fresh, off = set(fresh), 0
        for j, (code, (worker, tag, players, _m)) in enumerate(zip(codes.tolist(), staged)):
            hs = ids[off:off + len(players)].tolist()
            rec = dict(members=tuple(hs), rating=tuple(rating[off:off + len(players)].tolist()), mode=int(mode[j]),
                       ts=stamp, seq=(seq0 + j) & 0xFFFFFFFF)
            off += len(players)
            if code == 1:
                for h, doc in zip(hs, players):
                    self.players[h] = doc
                    self.party_of[h] = tuple(hs)
                    if self.requeue_parties:
                        self.party_book[h] = rec
                self.stats["enqueued"] += len(players)
                worker.ack(worker.channel_name, tag)
            elif code == 0:  # a member is already queued
                self.stats["duplicates"] += 1
                worker.ack(worker.channel_name, tag)
            else:  # invalid, or the party table is full
                for h, doc in zip(hs, players):
                    if doc["id"] in fresh and self.handles.lookup(doc["id"]) == h and h not in self.players:
                        self.handles.release(doc["id"])
                self.stats["invalid"] += 1
                worker.nack(worker.channel_name, tag)
        return len(staged)

    def party_status(self, group_name):
        """Queued parties of one rating group, per mode name with at least one: {"parties", "players"}.  From
        Engine.party_queue_stats (only the per-queue records cross PCIe); an engine without it is read with
        Engine.party_read."""
        if group_name not in self.group_names:
            return {}
        g = self.group_names.index(group_name)
        out = {}
        if self.party_capacity and hasattr(self.engine, "party_queue_stats"):
            for r in self.engine.party_queue_stats(self.now_ms()):
                if int(r["group"]) == g and int(r["mode"]) < len(self.mode_names) and int(r["n_parties"]):
                    out[self.mode_names[int(r["mode"])]] = {"parties": int(r["n_parties"]),
                                                             "players": int(r["n_members"])}
            return out
        if not hasattr(self.engine, "party_read"):
            return {}
        pr = self.engine.party_read()
        for m, grp, size in zip(pr["mode"].tolist(), pr["group"].tolist(), pr["size"].tolist()):
            if grp == g and m < len(self.mode_names):
                d = out.setdefault(self.mode_names[m], {"parties": 0, "players": 0})
                d["parties"] += 1
                d["players"] += size
        return out

    def flush(self):
        """mm_enqueue the staged deliveries; ack each one once its player is resident.  Never raises: a batch the
        engine refuses (active set full, CUDA error) is nacked as a whole — the broker redelivers it.  Staged parties
        follow (_flush_parties)."""
        staged, self._staged = self._staged, []
        if self._staged_parties and not staged:
            return self._flush_parties()
        if not staged:
            return 0
        try:
            return self._flush_solos(staged)
        finally:
            self._flush_parties()

    def _flush_solos(self, staged):
        fresh = []
        ids = np.empty(len(staged), np.uint64)
        for i, s in enumerate(staged):
            h, is_new = self.handles.acquire(s[0])
            if h is None:                      # handle range exhausted: an id the engine rejects as invalid
                h = 2 ** 64 - 1
            elif is_new:
                fresh.append(s[0])
            ids[i] = h
        rating = np.clip(np.array([s[1] for s in staged], np.int64), -(2 ** 31), 2 ** 31 - 1).astype(np.int32)
        mode = np.array([self.mode_index.get(s[2], 255) if isinstance(s[2], str) else 255 for s in staged], np.uint8)
        stamp = self.now_ms()
        # every offered entry of an accepted batch takes one sequence number: entry i gets seq0 + i
        seq0 = self.engine.seq_next() if hasattr(self.engine, "seq_next") else None
        try:
            acc = self.engine.enqueue(ids, rating, mode, np.full(len(staged), stamp, np.uint32))
        except Exception:                       # nothing was enqueued (mm_enqueue refuses a batch as a whole)
            for pid in fresh:
                self.handles.release(pid)
            for (_pid, _r, _m, _player, worker, tag) in staged:
                worker.nack(worker.channel_name, tag)
            self.stats["failed_batches"] += 1
            return 0
        t_resident = self.clock() if self.window else None
        fresh = set(fresh)
        for i, (code, h, (pid, _r, _m, player, worker, tag)) in enumerate(zip(acc, ids.tolist(), staged)):
            if code == 1:
                self.players[h] = player
                if seq0 is not None:
                    self.queued[h] = [int(rating[i]), int(mode[i]), stamp, (seq0 + i) & 0xFFFFFFFF]
                if self.window:
                    self.enqueued_at[h] = t_resident
                self.stats["enqueued"] += 1
                worker.ack(worker.channel_name, tag)       # worker.ex:323
            elif code == 0:                                 # "You are already in the queue."
                self.stats["duplicates"] += 1
                worker.ack(worker.channel_name, tag)
            else:                                           # unknown mode / unroutable rating / full
                if pid in fresh and self.handles.lookup(pid) == h and h not in self.players:
                    self.handles.release(pid)
                self.stats["invalid"] += 1
                worker.nack(worker.channel_name, tag)
        return len(staged)

    # -- the tick ---------------------------------------------------------------------------
    def tick(self, now=None):
        """One search tick; publishes each lobby like prepare_game_lobby/4. -> lobbies emitted.  now: the engine tick's
        clock (default now_ms(), the clock the ingest stamps)."""
        self.flush()
        if now is None:
            now = self.now_ms()
        if self.window:  # the oldest queued player is the first key: dicts keep insertion (= enqueue) order
            oldest = next(iter(self.enqueued_at.values()), None)
            self.last_spread = self.window.spread(self.clock(), oldest)
            self.engine.set_option("max_spread", self.last_spread)
        left = None  # budget_offtick: the step's per-queue and per-mode budgets, less what the step published
        if self.lobby_budget is not None:
            if self.budget_offtick:
                left = self._budget_arrays(self.lobby_budget())
            else:
                self._set_budget(self.lobby_budget())
        n_lob = 0
        if self.party_rules:  # before the tick: parties get the first pick of the solos
            if left is not None:
                self.engine.set_offtick_budget(abi.MM_OFFTICK_PARTY_MATCH, *left)
            plob, pmem, _st = self.engine.party_match(now, self.party_rules)
            left = self._budget_less(left, plob)
            for x in pmem.tolist():
                self.party_of.pop(x, None)
                rec = self.party_book.pop(x, None)
                if rec is not None:  # requeue() can put the party back whole
                    self.matched_parties[x] = rec
            self._publish(plob, pmem)
            self.stats["party_lobbies"] += len(plob)
            n_lob += len(plob)
        if left is not None:
            self.engine.set_lobby_budget(*left)
        lob, mem, _seq, _st = self.engine.tick(now)
        left = self._budget_less(left, lob)
        self._publish(lob, mem)
        self.stats["lobbies"] += len(lob)
        n_lob += len(lob)
        if self.widen:  # before the timeout: a player who waited long gets its widest window before it is dropped
            if left is not None:
                self.engine.set_offtick_budget(abi.MM_OFFTICK_WIDEN, *left)
            wlob, wmem, _st = self.engine.widen(now, self.widen)
            self._publish(wlob, wmem)
            self.stats["widened"] += len(wlob)
            n_lob += len(wlob)
        if self.timeout_ms is not None:  # after the lobbies: a player this tick matched is never timed out
            self._expire(now)
        return n_lob

    def _publish(self, lob, mem):
        """Publish each lobby like prepare_game_lobby/4, through the worker of its group."""
        for h in lob:
            mode_name = self.mode_names[h["mode"]]
            group_name = self.group_names[h["group"]]
            first, n = int(h["first_member"]), int(h["n_members"])
            members = [self.players.pop(int(x)) for x in mem[first:first + n]]
            if self.window:  # kept aside until remove_user: requeue() puts it back
                for x in mem[first:first + n]:
                    at = self.enqueued_at.pop(int(x), None)
                    if at is not None:
                        self.matched_at[int(x)] = at
            size = n // self._teams_of(h["mode"])
            teams = {f"team {t + 1}": members[t * size:(t + 1) * size] for t in range(n // size)}
            payload = json.dumps({"teams": teams, "game-mode": mode_name})      # worker.ex:315-318
            worker = self.workers.get(group_name) or next(iter(self.workers.values()))
            worker.prepare_game_lobby(worker.channel_name, EXCHANGE_FORWARD, QUEUE_FORWARD, payload)

    # -- lobby budget ------------------------------------------------------------------------
    def _queues(self, group_names, mode_names):
        modes = range(len(self.mode_names)) if mode_names is None else [self.mode_names.index(m) for m in mode_names]
        return {m * len(self.group_names) + self.group_names.index(g) for g in group_names for m in modes}

    def _budget_arrays(self, per_mode=None):
        """-> (per-queue budgets: 0 for a paused queue, else unlimited; per-mode budgets from {mode name: lobbies}, or
        None)."""
        from .abi import MM_BUDGET_UNLIMITED
        queue = np.full(len(self.mode_names) * len(self.group_names), MM_BUDGET_UNLIMITED, np.uint32)
        queue[sorted(self.paused)] = 0
        mode = None
        if per_mode is not None:
            mode = np.array([min(max(int(per_mode.get(m, MM_BUDGET_UNLIMITED)), 0), MM_BUDGET_UNLIMITED)
                             for m in self.mode_names], np.uint32)
        return queue, mode

    def _budget_less(self, left, lobbies):
        """budget_offtick: the per-mode budgets of `left` less the lobbies just published, per mode (an unlimited mode
        stays unlimited)."""
        from .abi import MM_BUDGET_UNLIMITED
        if left is None or left[1] is None:
            return left
        used = np.bincount(np.asarray(lobbies["mode"], np.int64), minlength=len(self.mode_names))[:len(self.mode_names)]
        mode = left[1].astype(np.int64)
        return left[0], np.where(mode == MM_BUDGET_UNLIMITED, mode, np.maximum(mode - used, 0)).astype(np.uint32)

    def _set_budget(self, per_mode=None):
        queue, mode = self._budget_arrays(per_mode)
        self.engine.set_lobby_budget(per_queue=queue, per_mode=mode)
        if self.budget_offtick:  # the off-tick calls the pool runs, under the same budgets
            for _name, src in self._offtick_sources():
                self.engine.set_offtick_budget(src, per_queue=queue, per_mode=mode)

    def _offtick_sources(self):
        return ([("party_match", abi.MM_OFFTICK_PARTY_MATCH)] if self.party_rules else []) + \
            ([("widen", abi.MM_OFFTICK_WIDEN)] if self.widen else [])

    def pause(self, group_names, mode_names=None):
        """The queues of these groups (all modes, or only `mode_names`) emit no lobby from the next tick on; their
        players stay queued in order, waits and the search timeout running.  Undone by resume_queues()."""
        self.paused |= self._queues(group_names, mode_names)
        if self.lobby_budget is None:  # (with a budget callable the next tick sets both together)
            self._set_budget()

    def resume_queues(self, group_names, mode_names=None):
        self.paused -= self._queues(group_names, mode_names)
        if self.lobby_budget is None:
            self._set_budget()

    def held_back(self, group_name):
        """{mode name: lobbies the last tick could have emitted from the group's queue and did not} (candidates minus
        emitted, Engine.lobby_budget_report); {} for an unknown group.  With budget_offtick: {mode name: {source:
        lobbies}}, source "tick" and each off-tick call the pool runs ("party_match", "widen";
        Engine.offtick_budget_report)."""
        if group_name not in self.group_names:
            return {}
        g, G = self.group_names.index(group_name), len(self.group_names)
        reports = [("tick", self.engine.lobby_budget_report())]
        if self.budget_offtick:
            reports += [(name, self.engine.offtick_budget_report(src)) for name, src in self._offtick_sources()]
        held = {name: {m: int(cand[m * G + g]) - int(emitted[m * G + g]) for m in range(len(self.mode_names))}
                for name, (cand, emitted) in reports}
        if not self.budget_offtick:
            return {mode: held["tick"][m] for m, mode in enumerate(self.mode_names)}
        return {mode: {name: held[name][m] for name in held} for m, mode in enumerate(self.mode_names)}

    def _expire(self, now):
        expired, _seq = self.engine.expire(now, self.timeout_ms, want_seq=False)
        for h in expired.tolist():
            self.party_of.pop(h, None)
            self.party_book.pop(h, None)
            player = self.players.pop(h)
            self.enqueued_at.pop(h, None)
            self.queued.pop(h, None)
            self.handles.release(self.handles.id_of[h])
            if player.get("response-queue") is not None:
                worker = next(iter(self.workers.values()))
                worker.send_response(worker.channel_name, player["response-queue"], prepare_timeout_response(player))
        self.stats["timed_out"] += len(expired)

    # -- hand-over to a new process ------------------------------------------------------------
    CHECKPOINT_MAGIC = b"MMPOOL01"

    def checkpoint(self):
        """-> bytes: everything a new process needs to go on serving the queued players (resume()).  The staged
        deliveries are ingested first, so every acked player is in the image, and pending async results are waited
        for.  Layout: CHECKPOINT_MAGIC, u64 length of a JSON document (the host state: handle table, player documents,
        enqueue times, mode / group names, the pool clock and the wall time), the JSON, then the engine image
        (Engine.export_state, opaque here).  A pool with party_capacity releases its queued parties around the export
        (Engine.export_parties) and merges them back with their numbers, so it goes on unchanged; its JSON gains
        "party_of" (the queued parties' handles) and "party_image" (the party image's length in bytes), and the party
        image goes between the JSON and the engine image.  A pool without party capacity writes neither.  Stop
        consuming before the call: a delivery staged after it is not in the checkpoint, and it stays unacked, so the
        broker redelivers it."""
        self.flush()
        if hasattr(self.engine, "results_wait"):
            self.engine.results_wait()
        parties = None
        if self.party_capacity:  # released around the image and merged back with their numbers: the engine goes on
            parties = np.ascontiguousarray(self.engine.export_parties(), np.uint8)
            try:
                image = self.engine.export_state()
            finally:
                self.engine.merge_parties(parties, keep_seq=True)
        else:
            image = self.engine.export_state()
        image = image.tobytes() if isinstance(image, np.ndarray) else bytes(image)
        t = self.clock()
        state = {
            "mode_names": self.mode_names, "group_names": self.group_names,
            "id_of": self.handles.id_of, "free": self.handles.free,
            "players": [[h, doc] for h, doc in self.players.items()],
            "enqueued_at": [[h, t - at] for h, at in self.enqueued_at.items()],  # age at the checkpoint, in order
            "matched_at": [[h, t - at] for h, at in self.matched_at.items()],
            "queued": [[h, rec] for h, rec in self.queued.items()],  # queued, or matched and not yet removed
            "moved_out": sorted(self.moved_out),
            "now_ms": self.now_ms(), "wall": self.wall_clock(),
        }
        if parties is not None:  # the party image goes between the JSON and the engine image
            state["party_of"] = sorted({tuple(p) for p in self.party_of.values()})
            if self.requeue_parties:  # the matched players stay in the engine image: their parties' book goes too
                state["party_book"] = self._book_records(self.party_book)
                state["matched_parties"] = self._book_records(self.matched_parties)
            state["party_image"] = len(parties)
            image = parties.tobytes() + image
        doc = json.dumps(state).encode()
        return self.CHECKPOINT_MAGIC + len(doc).to_bytes(8, "little") + doc + image

    @classmethod
    def resume(cls, engine, blob, mode_names, group_names, regroup=False, **opts):
        """A pool on a FRESH engine that goes on where checkpoint() stopped: the engine imports the image
        (Engine.import_state), the handle table, player documents and enqueue times come back, and now_ms() goes on
        from the checkpoint's value plus the wall time the pool was down — the enqueue stamps in the engine stay
        valid, and waits (timeout_ms, queue_status) include the downtime.  opts: those of SearchPool().

        regroup=True deploys a new config (rating groups, default group, modes, order) without dropping the queue:
        the engine, created with the new config, re-files the checkpoint's players (Engine.import_regroup), each
        keeping its place.  Group names may differ freely; a mode keeps its index, so one mode list must be a prefix
        of the other.  Players whose rating or mode has no queue under the new config are not queued: their handles
        and records are dropped and their documents are in the returned pool's `regroup_dropped` — answer them with
        the error response timeout_ms uses (prepare_timeout_response) once the workers are up.  A checkpoint of a pool
        with queues moved out (move_out) is refused: those queues live in another pool under the old groups."""
        head = len(cls.CHECKPOINT_MAGIC)
        if blob[:head] != cls.CHECKPOINT_MAGIC:
            raise ValueError("not a SearchPool checkpoint")
        n = int.from_bytes(blob[head:head + 8], "little")
        state = json.loads(bytes(blob[head + 8:head + 8 + n]))
        if regroup:
            old, new = state["mode_names"], list(mode_names)
            if old[:len(new)] != new[:len(old)]:
                raise ValueError("regroup keeps each mode's index: one mode list must be a prefix of the other")
            if state.get("moved_out"):
                raise ValueError("the checkpoint's pool has queues moved out to another pool under the old groups")
        elif state["mode_names"] != list(mode_names) or state["group_names"] != list(group_names):
            raise ValueError("the checkpoint was taken with other mode or group names")
        pool = cls(engine, mode_names, group_names, **opts)
        image = bytes(blob[head + 8 + n:])
        k = int(state.get("party_image", 0))
        parties, image = image[:k], image[k:]
        if k and not pool.party_capacity:
            raise ValueError("the checkpoint holds parties: resume it with a party_capacity")
        rejected = []
        if regroup:
            from .engine import read_image
            idx = engine.import_regroup(image)
            rejected = read_image(image)[1]["id"][idx].tolist()
        else:
            engine.import_state(image)
        if k:  # the parties keep their numbers; a party with no queue under this config leaves like a rejected solo
            from .engine import read_party_image
            codes = engine.merge_parties(parties, keep_seq=True)
            _h, pc = read_party_image(parties)
            for c, hs in zip(codes.tolist(), np.split(pc["id"], np.cumsum(pc["size"].astype(np.int64))[:-1])):
                if c != 1:
                    rejected += hs.tolist()
        down = max(0.0, pool.wall_clock() - state["wall"])
        pool._t0 = pool.clock() - down - state["now_ms"] / 1000.0
        pool.handles.id_of = list(state["id_of"])
        pool.handles.free = list(state["free"])
        pool.handles.handle_of = {pid: h for h, pid in enumerate(pool.handles.id_of) if pid is not None}
        pool.players = {int(h): doc for h, doc in state["players"]}
        at = pool.clock() - down
        pool.enqueued_at = {int(h): at - age for h, age in state["enqueued_at"]}
        pool.matched_at = {int(h): at - age for h, age in state.get("matched_at", [])}
        pool.queued = {int(h): rec for h, rec in state.get("queued", [])}  # the image keeps every sequence number
        pool.moved_out = set(state.get("moved_out", []))
        pool.party_of = {int(h): tuple(int(x) for x in hs) for hs in state.get("party_of", []) for h in hs}
        if pool.requeue_parties:
            pool.party_book = cls._book_of(state.get("party_book", []))
            pool.matched_parties = cls._book_of(state.get("matched_parties", []))
        pool.regroup_dropped = []
        for h in rejected:  # not queued under the new config: they left
            pool.party_of.pop(h, None)
            pool.party_book.pop(h, None)
            pool.regroup_dropped.append(pool.players.pop(h))
            for d in (pool.queued, pool.enqueued_at, pool.matched_at):
                d.pop(h, None)
            pool.handles.release(pool.handles.id_of[h])
        return pool

    @staticmethod
    def _book_records(book):
        """The distinct party records of a book, as JSON."""
        recs = {id(r): r for r in book.values()}
        return [dict(r, members=list(r["members"]), rating=list(r["rating"])) for r in recs.values()]

    @staticmethod
    def _book_of(records):
        """_book_records -> handle -> record (one dict shared by the members)."""
        book = {}
        for r in records:
            rec = dict(r, members=tuple(int(x) for x in r["members"]), rating=tuple(int(x) for x in r["rating"]))
            book.update((h, rec) for h in rec["members"])
        return book

    def _book_parties(self, image, seq0, codes=None, handles=None):
        """requeue_parties: the parties of a party image merged without their numbers get seq0 + their index.  With
        handles (a moved-in image, in image member order), the merged ones (code 1) get a record."""
        from .engine import read_party_image
        _h, pc = read_party_image(image)
        cut = np.cumsum(pc["size"].astype(np.int64))
        for j, (lo, hi) in enumerate(zip(np.concatenate([[0], cut[:-1]]).tolist(), cut.tolist())):
            seq = (seq0 + j) & 0xFFFFFFFF
            if handles is None:
                rec = self.party_book.get(int(pc["id"][lo]))
                if rec is not None:
                    rec["seq"] = seq
            elif codes[j] == 1:
                rec = dict(members=tuple(handles[lo:hi]), rating=tuple(pc["rating"][lo:hi].tolist()),
                           mode=int(pc["mode"][j]), ts=int(pc["enq_ts"][j]), seq=seq)
                self.party_book.update((h, rec) for h in rec["members"])

    # -- moving queues to another running pool -----------------------------------------------------
    MOVE_MAGIC = b"MMMOVE01"

    def move_out(self, group_names, mode_names=None):
        """Release the queues of these groups (all modes, or only `mode_names`) to another running pool: -> bytes for
        move_in().  The staged deliveries are ingested first.  The engine releases the players in the same call that
        writes their image (Engine.export_queues), and this pool forgets their handles and documents.  Layout:
        MOVE_MAGIC, u64 length of a JSON document (mode / group names, the pool clock and the wall time, and per moved
        player in image order its id, document and age), the JSON, then the queue image.  A pool with party_capacity
        also releases the moved queues' parties into a party image (Engine.export_parties; its other parties step aside
        around the export and come back with their numbers): the JSON gains "party_players" (per member in image order
        its id and document) and "party_image" (the party image's length in bytes), and the party image goes between the
        JSON and the queue image.  Reroute the groups' deliveries to the new owner before the call: a delivery staged
        after it stays here."""
        self.flush()
        if hasattr(self.engine, "results_wait"):
            self.engine.results_wait()
        G, M = len(self.group_names), len(self.mode_names)
        mask = np.zeros((M, G), bool)
        modes = range(M) if mode_names is None else [self.mode_names.index(m) for m in mode_names]
        for g in group_names:
            for m in modes:
                mask[m, self.group_names.index(g)] = True
        from .engine import read_image, read_party_image
        pimage = None
        if self.party_capacity:  # mm_export_queues refuses while a party is queued: the others go back with their numbers
            pimage = np.ascontiguousarray(self.engine.export_parties(mask), np.uint8)
            rest = np.ascontiguousarray(self.engine.export_parties(~mask), np.uint8)
            try:
                image = np.ascontiguousarray(self.engine.export_queues(mask), np.uint8)
            except Exception:
                self.engine.merge_parties(rest, keep_seq=True)
                self.engine.merge_parties(pimage)
                raise
            self.engine.merge_parties(rest, keep_seq=True)
        else:
            image = np.ascontiguousarray(self.engine.export_queues(mask), np.uint8)
        _h, cols = read_image(image)
        t = self.clock()
        moved = []
        self.moved_out |= set(np.flatnonzero(mask.reshape(-1)).tolist())
        for h in cols["id"].tolist():
            pid = self.handles.id_of[h]
            self.queued.pop(h, None)
            at = self.enqueued_at.pop(h, None)
            moved.append([pid, self.players.pop(h), None if at is None else t - at])
            self.handles.release(pid)
        state = {"mode_names": self.mode_names, "group_names": self.group_names, "players": moved,
                 "now_ms": self.now_ms(), "wall": self.wall_clock()}
        if pimage is not None:  # per party member in image order its id and document; the party image before the queue's
            members = []
            for h in read_party_image(pimage)[1]["id"].tolist():
                pid = self.handles.id_of[h]
                self.party_of.pop(h, None)
                self.party_book.pop(h, None)
                members.append([pid, self.players.pop(h)])
                self.handles.release(pid)
            state["party_players"] = members
            state["party_image"] = len(pimage)
            image = np.concatenate([pimage, image])
        doc = json.dumps(state).encode()
        return self.MOVE_MAGIC + len(doc).to_bytes(8, "little") + doc + image.tobytes()

    def move_in(self, blob):
        """Load what move_out() released into this pool: every moved player gets a handle of this pool (the image's id
        column is rewritten), its enqueue stamp is shifted into this pool's clock (bridged by the wall time, as in
        resume(), so waits and the timeout count the time in the old pool), the engine merges the image
        (Engine.merge_queues), and the documents of players it rejects (already queued here) are dropped.  Staged
        deliveries are ingested first.  Moved parties merge after the solos (Engine.merge_parties, new numbers here);
        this pool's own parties step aside around the queue merge and come back, renumbered in their order when the
        queue image took numbers.  -> players merged (solos).  ValueError, before anything changes, if the mode or
        group names differ, if this pool's handle range cannot hold the players, or if the move carries parties and
        this pool's party table or hashed active set cannot hold them."""
        head = len(self.MOVE_MAGIC)
        if bytes(blob[:head]) != self.MOVE_MAGIC:
            raise ValueError("not a SearchPool queue move")
        n = int.from_bytes(blob[head:head + 8], "little")
        state = json.loads(bytes(blob[head + 8:head + 8 + n]))
        if state["mode_names"] != self.mode_names or state["group_names"] != self.group_names:
            raise ValueError("the queues were moved out of a pool with other mode or group names")
        k = int(state.get("party_image", 0))
        if k and not self.party_capacity:
            raise ValueError("the move carries parties: this pool has no party_capacity")
        self.flush()
        from .engine import read_image, read_party_image
        image = np.frombuffer(bytes(blob[head + 8 + n:]), np.uint8).copy()
        pimage, image = image[:k], image[k:]
        _h, cols = read_image(image)
        players = state["players"]
        party_players = state.get("party_players", [])
        if k:  # the parties merge after the solos: their room is checked before anything changes
            from .engine import active_set_limit
            queued = int(self.engine.party_read()["size"].sum(dtype=np.int64))
            if queued + len(party_players) > self.party_capacity:
                raise ValueError(f"this pool's party table holds {self.party_capacity} members: {queued} queued, "
                                 f"{len(party_players)} moved")
            limit = active_set_limit(self.engine.cfg)
            if limit is not None and self.engine.active_size() + len(players) + len(party_players) > limit:
                raise ValueError("this pool's active set cannot hold the moved players and parties")
        handles, fresh = [], []
        for pid, *_rest in players + party_players:
            h, is_new = self.handles.acquire(pid)
            if h is None:
                for p in fresh:
                    if p is not None:
                        self.handles.release(p)
                raise ValueError("this pool's handle range cannot hold the moved players")
            handles.append(h)
            fresh.append(pid if is_new else None)
        fresh_ids = [p for p in fresh if p is not None]
        handles, phandles = handles[:len(players)], handles[len(players):]
        fresh, pfresh = fresh[:len(players)], fresh[len(players):]
        cols["id"][:] = np.asarray(handles, cols["id"].dtype)
        down = max(0.0, self.wall_clock() - state["wall"])
        shift = (self.now_ms() - int(round(down * 1000.0)) - int(state["now_ms"])) & 0xFFFFFFFF
        cols["enq_ts"][:] = (cols["enq_ts"].astype(np.uint64) + np.uint64(shift)).astype(np.uint32)
        if k:  # the party columns get the same handles and clock
            _ph, pcols = read_party_image(pimage)
            pcols["id"][:] = np.asarray(phandles, pcols["id"].dtype)
            pcols["enq_ts"][:] = (pcols["enq_ts"].astype(np.uint64) + np.uint64(shift)).astype(np.uint32)
        own = None
        if self.party_capacity:  # mm_merge refuses while a party is queued here: ours step aside and come back
            own = np.ascontiguousarray(self.engine.export_parties(), np.uint8)
        seq0 = self.engine.seq_next() if hasattr(self.engine, "seq_next") else None
        try:
            rejected = set(self.engine.merge_queues(image).tolist())
        except Exception:
            for p in fresh_ids:
                self.handles.release(p)
            if own is not None:
                self.engine.merge_parties(own, keep_seq=True)
            raise
        t = self.clock() - down
        hdr = _h.config
        grp = np.full(len(handles), hdr.default_group, np.int64)
        for g in reversed(range(hdr.n_groups)):  # the first group that holds the rating
            grp[(cols["rating"] >= hdr.group_lo[g]) & (cols["rating"] <= hdr.group_hi[g])] = g
        queue = cols["mode"].astype(np.int64) * hdr.n_groups + grp
        self.moved_out -= set(queue.tolist())
        if seq0 is not None:  # mm_merge numbers its batch queue by queue, in the source's enqueue order in a queue
            order = np.lexsort(((cols["seq"] - np.uint32(_h.seq_next)).astype(np.uint32), queue))
            new_seq = np.empty(len(handles), np.int64)
            new_seq[order] = (seq0 + np.arange(len(handles))) & 0xFFFFFFFF
        merged = 0
        for i, ((pid, doc, age), h, new) in enumerate(zip(players, handles, fresh)):
            if i in rejected:  # already queued here: keep this pool's player, drop the moved document
                if new is not None:
                    self.handles.release(pid)
                continue
            self.players[h] = doc
            if seq0 is not None:
                self.queued[h] = [int(cols["rating"][i]), int(cols["mode"][i]), int(cols["enq_ts"][i]), int(new_seq[i])]
            if self.window and age is not None:
                self.enqueued_at[h] = t - age
            merged += 1
        if self.window:  # oldest first: the window reads the first entry
            self.enqueued_at = dict(sorted(self.enqueued_at.items(), key=lambda kv: kv[1]))
        # the solos are recorded: ours come back (with their numbers when the queue image took none, else renumbered in
        # their order), then the moved parties, whose room was checked above
        if own is not None:
            s_own = self.engine.seq_next()
            self.engine.merge_parties(own, keep_seq=s_own == seq0)
            if s_own != seq0 and self.requeue_parties:  # renumbered in their order
                self._book_parties(own, s_own)
        if k:
            s_moved = self.engine.seq_next()
            try:
                codes = self.engine.merge_parties(pimage)
                if self.requeue_parties:
                    self._book_parties(pimage, s_moved, codes.tolist(), phandles)
            except Exception:
                codes = np.zeros(len(pcols["size"]), np.uint8)
                raise
            finally:
                at = 0
                for c, size in zip(codes.tolist(), pcols["size"].tolist()):
                    hs = phandles[at:at + size]
                    for i in range(at, at + size):
                        if c == 1:
                            self.players[phandles[i]] = party_players[i][1]
                            self.party_of[phandles[i]] = tuple(hs)
                        elif pfresh[i] is not None and phandles[i] not in self.players:
                            self.handles.release(pfresh[i])
                    at += size
        return merged

    def _teams_of(self, mode):
        return self.engine.cfg.modes[int(mode)].teams

    def queue_status(self, group_name):
        """The engine's view of one rating group's queues (Engine.queue_stats at now_ms()), per mode name: players
        waiting, oldest / p50 / p99 wait, and the last tick's matched players and p99 wait at match, in ms.  Quantiles
        are the upper bounds of histogram buckets (at most 25 % high).  {} for a group the pool does not know."""
        from .engine import wait_quantile
        if group_name not in self.group_names:
            return {}
        g = self.group_names.index(group_name)
        out = {}
        for r in self.engine.queue_stats(self.now_ms()):
            if int(r["group"]) != g or int(r["mode"]) >= len(self.mode_names):
                continue
            out[self.mode_names[int(r["mode"])]] = {
                "waiting": int(r["n_waiting"]),
                "oldest_wait_ms": int(r["max_wait"]),
                "p50_wait_ms": wait_quantile(r["wait_hist"], 0.50),
                "p99_wait_ms": wait_quantile(r["wait_hist"], 0.99),
                "last_tick_matched": int(r["n_matched"]),
                "last_tick_p99_match_wait_ms": wait_quantile(r["match_wait_hist"], 0.99),
            }
        return out

    def match_quality(self, group_name):
        """How even the last tick's lobbies of one rating group are (Engine.match_quality), per mode name: lobbies, the
        mean / p50 / p99 / max rating spread and the mean / p99 / max team imbalance, in rating points.  Quantiles are
        the upper bounds of histogram buckets (at most 25 % high).  {} for a group the pool does not know, and while
        the report is void (before the first tick, after a failed one, after a restore or an import)."""
        from .engine import wait_quantile
        if group_name not in self.group_names:
            return {}
        g = self.group_names.index(group_name)
        out = {}
        for r in self.engine.match_quality()[0]:
            if int(r["group"]) != g or int(r["mode"]) >= len(self.mode_names):
                continue
            n = int(r["n_lobbies"])
            out[self.mode_names[int(r["mode"])]] = {
                "lobbies": n,
                "mean_spread": int(r["sum_spread"]) / n if n else 0.0,
                "p50_spread": wait_quantile(r["spread_hist"], 0.50),
                "p99_spread": wait_quantile(r["spread_hist"], 0.99),
                "max_spread": int(r["max_spread"]),
                "mean_imbalance": int(r["sum_imbalance"]) / n if n else 0.0,
                "p99_imbalance": wait_quantile(r["imbalance_hist"], 0.99),
                "max_imbalance": int(r["max_imbalance"]),
            }
        return out

    def offtick_status(self, group_name):
        """Waits and rating quality of the lobbies the last step formed outside the tick, in one rating group
        (Engine.offtick_report), per mode name and per source ("party_match" for party lobbies, "widen" for widened
        ones, each only when the pool runs it): lobbies, matched players, the p50 / p99 / max wait at match in ms, and
        the mean / p99 / max rating spread and team imbalance in rating points.  Quantiles are the upper bounds of
        histogram buckets (at most 25 % high).  A source whose report is void (no call yet, or a failed one) is left
        out; {} for a group the pool does not know."""
        from .engine import wait_quantile
        if group_name not in self.group_names:
            return {}
        g = self.group_names.index(group_name)
        out = {}
        for name, src in self._offtick_sources():
            waits, quality, _ = self.engine.offtick_report(src)
            held = self.engine.offtick_budget_report(src) if self.budget_offtick else None
            for w, r in zip(waits, quality):
                if int(w["group"]) != g or int(w["mode"]) >= len(self.mode_names):
                    continue
                n = int(r["n_lobbies"])
                out.setdefault(self.mode_names[int(w["mode"])], {})[name] = {
                    "lobbies": n,
                    "matched": int(w["n_matched"]),
                    "p50_match_wait_ms": wait_quantile(w["match_wait_hist"], 0.50),
                    "p99_match_wait_ms": wait_quantile(w["match_wait_hist"], 0.99),
                    "max_match_wait_ms": int(w["max_match_wait"]),
                    "mean_spread": int(r["sum_spread"]) / n if n else 0.0,
                    "p99_spread": wait_quantile(r["spread_hist"], 0.99),
                    "max_spread": int(r["max_spread"]),
                    "mean_imbalance": int(r["sum_imbalance"]) / n if n else 0.0,
                    "p99_imbalance": wait_quantile(r["imbalance_hist"], 0.99),
                    "max_imbalance": int(r["max_imbalance"]),
                }
                if held is not None:  # budget_offtick: lobbies the source's budget held back
                    q = int(w["mode"]) * len(self.group_names) + g
                    out[self.mode_names[int(w["mode"])]][name]["held_back"] = int(held[0][q]) - int(held[1][q])
        return out


class SearchWorker:
    """Matchmaking.Search.Worker — one consumer of `matchmaking.queues.<group>`."""

    CHANNEL_NAME = "Matchmaking.Search.Worker.Channel"  # worker.ex:20

    def __init__(self, connection, pool, config, opts):
        self.connection, self.pool = connection, pool
        self.config = config
        self.channel_name = opts.get("channel_name", self.CHANNEL_NAME)
        self.group_name = opts["group_name"]
        self.channel = None
        self.meta = None

    # worker.ex:68-71 + init/1 :220-237
    @classmethod
    def start_link(cls, connection, pool, opts):
        config = prepare_config(dict(opts, prefetch_count=opts.get("prefetch_count") or pool.max_batch))
        if connection is None:
            return ("error", "noconn")  # worker.ex:225-228
        w = cls(connection, pool, config, opts)
        w.channel = connection.spawn_channel(w.channel_name)
        connection.configure_channel(w.channel, config)  # exchange + queue + bind + qos (worker.ex:27-29)
        ok, w.meta = w.configure(w.channel_name, config)
        pool.workers[w.group_name] = w
        return ("ok", w)

    def configure(self, channel_name, opts):  # worker.ex:73-76
        consumer = self.create_consumer(channel_name, opts["queue"]["name"])
        return ("ok", {"consumer": consumer})

    def create_consumer(self, channel_name, queue_name):  # worker.ex:95-103
        return self.channel.basic_consume(queue_name, self)

    def ack(self, channel_name, tag):  # worker.ex:81-83
        return self.channel.basic_ack(tag)

    def nack(self, channel_name, tag):  # worker.ex:88-90
        return self.channel.basic_nack(tag)

    def status(self):  # worker.ex:115-117, 326-334
        st = dict(self.channel.queue_status(self.config["queue"]["name"]))
        st["pool"] = self.pool.engine.status() if hasattr(self.pool.engine, "status") else {}
        if hasattr(self.pool.engine, "queue_stats"):  # this worker's own group, per mode (the reference's queue depth)
            st["waiting"] = self.pool.queue_status(self.group_name)
        if hasattr(self.pool.engine, "match_quality"):  # how even this group's lobbies of the last tick are, per mode
            st["quality"] = self.pool.match_quality(self.group_name)
        if hasattr(self.pool.engine, "lobby_budget_report"):  # lobbies the last tick's budget held back, per mode
            st["held_back"] = self.pool.held_back(self.group_name)
        if self.pool.party_rules and hasattr(self.pool.engine, "party_read"):  # this group's queued parties, per mode
            st["parties"] = self.pool.party_status(self.group_name)
        if self.pool.party_rules and hasattr(self.pool.engine, "party_queue_stats"):  # their waits and sizes, per mode
            st["party_waiting"] = self.pool.party_queue_status(self.group_name)
        if (self.pool.party_rules or self.pool.widen) and hasattr(self.pool.engine, "offtick_report"):
            st["offtick"] = self.pool.offtick_status(self.group_name)  # party and widen lobbies of the last step
        return ("ok", st)

    def prepare_game_lobby(self, channel_name, exchange_forward, queue_forward, payload):  # worker.ex:250-261
        return self.channel.basic_publish(exchange_forward, queue_forward, payload, persistent=True,
                                          content_type="application/json")

    def send_response(self, channel_name, queue_name, payload):  # game-lobby/worker.ex:105-116
        return self.channel.basic_publish(EXCHANGE_RESPONSE, queue_name, payload, persistent=True,
                                          content_type="application/json")

    # worker.ex:291-324 — one delivery
    def consume(self, channel_name, group_name, tag, headers, payload):
        try:
            player_data = json.loads(payload)                     # :292
        except (ValueError, TypeError):
            return self.nack(channel_name, tag)
        if not isinstance(player_data, dict):                     # "[1, 2]" decodes, but is not a request
            return self.nack(channel_name, tag)
        game_mode = player_data.pop("game-mode", None)           # :294
        if "party" in player_data:  # extension: several players queued together, one delivery
            return self._consume_party(channel_name, tag, player_data["party"], game_mode)
        rating = player_data.get("rating")                        # generic/worker.ex:57 reads it top-level
        if rating is None and isinstance(player_data.get("detail"), dict):
            rating = player_data["detail"].get("rating")
        if ("id" not in player_data or not isinstance(player_data["id"], (str, int)) or not isinstance(game_mode, str)
                or isinstance(rating, bool) or not isinstance(rating, (int, float))
                or (isinstance(rating, float) and not math.isfinite(rating))):  # json.loads accepts NaN / Infinity
            return self.nack(channel_name, tag)
        if isinstance(rating, float) and rating != int(rating):
            rating = 2 ** 31 - 1  # falls between the integer ranges -> default group (generic/worker.ex:46-53)
        rating = max(-(2 ** 31), min(2 ** 31 - 1, int(rating)))
        self.pool.stage(self, tag, player_data, game_mode, rating)

    def _consume_party(self, channel_name, tag, party, game_mode):
        """{"party": [player documents], "game-mode": ...}: each document needs an "id" and a numeric "rating"."""
        docs = []
        for doc in party if isinstance(party, list) else [None]:
            rating = doc.get("rating") if isinstance(doc, dict) else None
            if (not isinstance(doc, dict) or "id" not in doc or not isinstance(doc["id"], (str, int))
                    or isinstance(rating, bool) or not isinstance(rating, (int, float))
                    or (isinstance(rating, float) and not math.isfinite(rating))):
                return self.nack(channel_name, tag)
            docs.append(dict(doc, rating=max(-(2 ** 31), min(2 ** 31 - 1, int(rating)))))
        if not isinstance(game_mode, str) or not docs:
            return self.nack(channel_name, tag)
        self.pool.stage_party(self, tag, docs, game_mode)

    # worker.ex:337-368
    def handle_info(self, msg):
        kind = msg[0]
        if kind in ("basic_consume_ok", "basic_cancel_ok"):
            return ("noreply", self)
        if kind == "basic_cancel":
            return ("stop", "normal", self)
        if kind == "basic_deliver":
            _, payload, headers = msg
            tag = headers.get("delivery_tag")
            try:  # in the reference a bad payload only kills the process spawned for this delivery (worker.ex:356)
                self.consume(self.channel_name, self.group_name, tag, headers, payload)
            except Exception:
                try:
                    self.nack(self.channel_name, tag)
                except Exception:
                    pass
            return ("noreply", self)
        if kind == "DOWN":  # re-register the consumer (worker.ex:361-368)
            self.meta = {"consumer": self.create_consumer(self.channel_name, self.config["queue"]["name"])}
            return ("noreply", self)
        return ("noreply", self)
