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
import json
import math

import numpy as np

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
    it has left.  One window per tick for the whole pool: the per-player form needs the
    sorted order on the device first and is future work."""

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

    Every ingest batch is stamped with now_ms(), the clock in milliseconds since the pool was created (u32, wraps
    after 49 days), and every tick passes the same clock as its `now`: the engine's per-queue waits
    (Engine.queue_stats, SearchWorker.status) are in milliseconds.
    """

    def __init__(self, engine, mode_names, group_names, max_batch=65536, window=None, clock=None, flush_every_s=0.005,
                 handle_capacity=None):
        import time
        self.window = window
        self.clock = clock or time.monotonic
        self._t0 = self.clock()
        self.enqueued_at = {}  # handle -> clock() when the player became resident (insertion = enqueue order)
        self.last_spread = None
        self.engine = engine
        self.mode_names = list(mode_names)
        self.mode_index = {m: i for i, m in enumerate(self.mode_names)}
        self.group_names = list(group_names)
        self.max_batch = max_batch
        self.flush_every_s = flush_every_s
        self.handles = HandleTable(handle_capacity)
        self.players = {}   # handle -> decoded player document (without "game-mode")
        self.workers = {}   # group name -> worker that publishes the group's lobbies
        self._staged = []   # (player id, rating, mode, player, worker, tag)
        self._staged_since = None
        self.stats = {"enqueued": 0, "duplicates": 0, "invalid": 0, "lobbies": 0, "failed_batches": 0}

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
            self.engine.remove([h])
            self.handles.release(player_id)
            self.players.pop(h, None)
            self.enqueued_at.pop(h, None)
        return ("ok", "removed")

    # -- ingest -----------------------------------------------------------------------------
    def stage(self, worker, tag, player, game_mode, rating):
        if not self._staged:
            self._staged_since = self.clock()
        self._staged.append((player["id"], int(rating), game_mode, player, worker, tag))
        if len(self._staged) >= self.max_batch or self.clock() - self._staged_since >= self.flush_every_s:
            self.flush()

    def flush(self):
        """mm_enqueue the staged deliveries; ack each one once its player is resident.  Never raises: a batch the
        engine refuses (active set full, CUDA error) is nacked as a whole — the broker redelivers it."""
        staged, self._staged = self._staged, []
        if not staged:
            return 0
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
        try:
            acc = self.engine.enqueue(ids, rating, mode, np.full(len(staged), self.now_ms(), np.uint32))
        except Exception:                       # nothing was enqueued (mm_enqueue refuses a batch as a whole)
            for pid in fresh:
                self.handles.release(pid)
            for (_pid, _r, _m, _player, worker, tag) in staged:
                worker.nack(worker.channel_name, tag)
            self.stats["failed_batches"] += 1
            return 0
        t_resident = self.clock() if self.window else None
        fresh = set(fresh)
        for code, h, (pid, _r, _m, player, worker, tag) in zip(acc, ids.tolist(), staged):
            if code == 1:
                self.players[h] = player
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
        lob, mem, _seq, _st = self.engine.tick(now)
        for h in lob:
            mode_name = self.mode_names[h["mode"]]
            group_name = self.group_names[h["group"]]
            first, n = int(h["first_member"]), int(h["n_members"])
            members = [self.players.pop(int(x)) for x in mem[first:first + n]]
            if self.window:
                for x in mem[first:first + n]:
                    self.enqueued_at.pop(int(x), None)
            size = n // self._teams_of(h["mode"])
            teams = {f"team {t + 1}": members[t * size:(t + 1) * size] for t in range(n // size)}
            payload = json.dumps({"teams": teams, "game-mode": mode_name})      # worker.ex:315-318
            worker = self.workers.get(group_name) or next(iter(self.workers.values()))
            worker.prepare_game_lobby(worker.channel_name, EXCHANGE_FORWARD, QUEUE_FORWARD, payload)
        self.stats["lobbies"] += len(lob)
        return len(lob)

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
        return ("ok", st)

    def prepare_game_lobby(self, channel_name, exchange_forward, queue_forward, payload):  # worker.ex:250-261
        return self.channel.basic_publish(exchange_forward, queue_forward, payload, persistent=True,
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
