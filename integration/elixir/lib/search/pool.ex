defmodule Matchmaking.Search.Pool do
  @moduledoc """
  Owner of the GPU-resident player pool shared by every Matchmaking.Search.Worker of this node.
  New process, no logic beyond batching: it is the Elixir twin of `SearchPool` in
  microservice-matchmaking_b200/search_worker.py (which the repository's tests run, CPU and GPU).

      stage/4        a search worker hands over one decoded delivery (patched consume/5, worker_patch.ex)
      :flush         Engine.enqueue_packed -> ack (codes 1, 0) / nack (codes 2, 3) per delivery; a delivery is acked
                     only once its player is resident (manual ack after processing, search/worker.ex:323)
      :tick          Engine.tick_packed -> one AMQP message per lobby with the payload and the publish options of
                     search/worker.ex:250-261,315-319
      in_queue?/1, remove_user/1    replace Matchmaking.Model.ActiveUser (models/active_user.ex:33-66)
      queue_status/1 one rating group's queues (Engine.queue_stats): waiting players, oldest / p50 / p99 wait, the
                     last tick's matched players and p99 wait at match, in ms — Search.Worker.status/0's queue depth;
                     with Engine.match_quality also the last tick's lobbies, mean / p50 / p99 / max rating spread and
                     mean / p99 / max team imbalance, in rating points (zero lobbies while the report is void)
                     and, with the parties / widen options, Engine.offtick_report's party_match / widen maps: the
                     last step's party or widened lobbies, matched players, p50 / p99 / max wait at match in ms and
                     mean / p99 / max rating spread and team imbalance (absent while that report is void)
      search_timeout_ms   option (extension, default nil = off): after each tick's lobbies are published, the players
                     still queued who have waited at least this long leave the pool (Engine.expire_packed) and get the
                     error response of game-lobby/worker.ex:63-71,105-116 on their "response-queue"
      widen          option (extension, default nil = off, needs a rating-order engine): %{mode name => {min_wait_ms,
                     w0, step_ms, inc, w_max}}.  After each tick's lobbies are published, and before the search timeout,
                     every player of the mode who has waited at least min_wait_ms anchors a lobby in a rating window of
                     w0 points either side, plus inc per whole step_ms past min_wait_ms, at most w_max (Engine.widen);
                     its lobbies are published like the tick's
      parties        option (extension, default nil = off, needs a rating-order engine): %{mode name => {min_wait_ms,
                     w0, step_ms, inc, w_max}}, the party window of the mode.  Before each tick, every party of the
                     mode that has waited at least min_wait_ms anchors a lobby (Engine.party_match): the other parties
                     of its window go to the first team with room, the nearest solos fill the rest; a party plays on
                     one team.  Parties arrive through stage_party/3, one delivery per party, acked or nacked as one
      party_capacity option (extension, default 0): how many party members the engine holds (Engine.set_party_capacity)
      requeue_parties option (extension, default false): requeue/1 puts matched parties back as parties at their age
                     position (Engine.requeue_party).  The pool keeps a book of every queued party (members, ratings,
                     mode, stamp, seq) and moves it aside when party_match places the party; two or more members of one
                     matched party go back as one party, a lone member as a solo with the party's seq.  The parties
                     go first; if the engine refuses them (the party table is full) they answer :gone and the solos go
                     on.  A lone member whose co-member went back the same way and is still queued in the same queue
                     answers :gone (one player of a party number per partition).  Off, requeue/1 answers a matched
                     party member :gone
      balance_teams  option (extension, default nil = off): a list of mode names.  Every lobby of those modes, from the
                     tick and from widen, is split into the two teams with the least rating difference
                     (Engine.set_team_balance); the lobby's players are the same, only who plays with whom changes
      balance_parties option (extension, default nil = off): a list of mode names.  Every party lobby of those modes
                     is split into its most even teams that keep every party whole (Engine.set_party_balance); the
                     published teams follow that order.  Independent of balance_teams
      lobby_budget   option (extension, default nil = no limit): a zero-arity function -> %{mode name => lobbies}, asked
                     before every tick — the free game-server slots (game-lobby/worker.ex:118-141).  The tick emits at
                     most that many lobbies of the mode, shared over the rating groups in proportion to what each could
                     emit (Engine.set_lobby_budget); the rest stay queued in order.  pause/1, resume_queues/1 stop and
                     restart the queues of rating groups; a checkpoint carries neither
      budget_offtick option (extension, default false): with lobby_budget, one tick's budget covers every lobby it
                     publishes (Engine.set_offtick_budget): party_match runs under the callback's per-mode budget F,
                     the tick under F minus its party lobbies per mode, widen under what is left; paused groups emit
                     nothing from any of the three
      checkpoint/0   hand-over: flushes the staged deliveries (so every acked player is in it), then returns
                     :erlang.term_to_binary of the engine image (Engine.export_image), the handle table, the player
                     documents, the pool clock and the wall time.  resume: <checkpoint> as an option of start_link/1
                     starts a pool on a fresh engine from it; the clock goes on from the checkpoint plus the time the
                     pool was down (INTEGRATION.md §3 has the order: stop consuming, checkpoint, start with resume:,
                     consume again).  regroup: true with resume: deploys another config (RatingGroups, modes)
                     without dropping the queue (Engine.import_regroup): players the new config has no queue for
                     leave the pool and get the search-timeout error response once a search worker has attached
      move_out/1, move_in/1   queue move between running pools: the queues of some rating groups leave this pool
                     with the players' documents and are merged into another pool (INTEGRATION.md §5)
      attach/1       a search worker hands over its open channel (patched init); the pool ticks only once it has a
                     channel to publish lobbies and timeout responses on — a staged delivery sets it too

  Every batch is stamped with the pool's clock (ms since the pool started, modulo 2^32) and every tick passes the same
  clock as its `now`, so the engine's waits are in milliseconds.

  Player ids are UUID strings (models/active_user.ex:7); the device stores a dense 32-bit handle
  (MM_F_DENSE_IDS).  The id <-> handle table lives here, handles are recycled when a player leaves — no hashing, so
  two players can never collide into "You are already in the queue.".
  QoS: the search workers must consume with prefetch_count >= @max_batch (not the reference's 10,
  search/worker.ex:29) — the broker stops delivering at `prefetch` unacknowledged messages.
  NOT COMPILED HERE (no BEAM toolchain in the build environment); see INTEGRATION.md.
  """
  use GenServer
  alias Matchmaking.Search.Engine

  @exchange_forward "open-matchmaking.matchmaking.game-lobby.direct"   # search/worker.ex:31
  @queue_forward "matchmaking.queues.lobbies"                          # search/worker.ex:32
  @exchange_response "open-matchmaking.responses.direct"               # game-lobby/worker.ex:27
  @timeout_details "No opponents were found within the search time limit."
  @max_batch 65_536
  @flush_ms 2
  @tick_ms 5

  def start_link(opts \\ []), do: GenServer.start_link(__MODULE__, opts, name: __MODULE__)
  def stage(player, game_mode, rating, ack_ref), do: GenServer.cast(__MODULE__, {:stage, player, game_mode, rating, ack_ref})
  @doc "Parties (extension): players = [{player, rating}] queued together; the delivery is acked or nacked as one."
  def stage_party(players, game_mode, ack_ref), do: GenServer.cast(__MODULE__, {:stage_party, players, game_mode, ack_ref})
  @doc "A search worker whose channel is open hands its channel name over (patched init, worker_patch.ex)."
  def attach(channel_name), do: GenServer.cast(__MODULE__, {:attach, channel_name})
  def in_queue?(player_id), do: GenServer.call(__MODULE__, {:in_queue?, player_id})
  def remove_user(player_id), do: GenServer.call(__MODULE__, {:remove_user, player_id})
  def queue_status(group_index), do: GenServer.call(__MODULE__, {:queue_status, group_index})
  def checkpoint, do: GenServer.call(__MODULE__, :checkpoint, :infinity)
  @doc """
  Queue move, old owner: the staged deliveries are ingested, then the queues of these rating groups (indices, all
  modes) leave the engine (Engine.export_queues) with the players' documents -> {:ok, blob} for move_in/1 on the new
  owner.  Reroute the groups' deliveries to the new owner first (INTEGRATION.md §5).
  """
  def move_out(groups), do: GenServer.call(__MODULE__, {:move_out, groups}, :infinity)
  @doc """
  Queue move, new owner: the moved players get handles of this pool, their enqueue stamps are shifted into its clock
  (bridged by the wall time), the engine merges the image (Engine.merge_image) and the documents of players already
  queued here are dropped -> {:ok, merged} | {:error, reason}; a refusal changes nothing (merge the blob back into the
  old owner, or keep it and retry).
  """
  def move_in(blob), do: GenServer.call(__MODULE__, {:move_in, blob}, :infinity)
  @doc """
  Requeue (extension): the members of a lobby that did not start (a declined ready check, no game server) go back into
  their queue at their enqueue position (Engine.requeue); players = the lobby's player documents.  -> one outcome per
  player: :requeued (queued again: its wait and the search timeout go on from its first enqueue), :queued (still
  queued) or :gone (removed, timed out, never queued, or its queue has moved to another pool: answer it as today).
  """
  def requeue(players), do: GenServer.call(__MODULE__, {:requeue, players}, :infinity)
  @doc """
  Backfill (extension): a running lobby that lost members asks for players instead of being disbanded.  requests:
  [{mode_name, group_index, target_rating, count}] or [{..., count, window}], served in order (Engine.backfill) -> one
  list of player documents per request (shorter than count when the queue runs short).  Backfilled players leave the
  pool as matched players do: requeue/1 puts them back, remove_user forgets them.
  """
  def backfill(requests), do: GenServer.call(__MODULE__, {:backfill, requests}, :infinity)
  @doc """
  Party backfill (extension; needs party_capacity): a running lobby's open team slots filled with whole queued parties
  first, then the nearest solos (Engine.backfill_party).  requests: [{mode_name, group_index, target_rating,
  open_slots}] or [{..., open_slots, window}], open_slots = one count per team of the mode, served in order -> {:ok,
  per request one list of player documents per team} (a team's parties, each party's members together, then its solos;
  shorter than its open slots when the queue runs short).  A placed party's book entry moves aside as after
  party_match, so requeue/1 with requeue_parties puts it back whole.
  """
  def backfill_teams(requests), do: GenServer.call(__MODULE__, {:backfill_teams, requests}, :infinity)
  @doc """
  Search status (extension): one map per player id, without ingesting the staged deliveries (Engine.locate):
  %{state: :searching | :matched | :staged | :unknown, game_mode, group, wait_ms, position, queue_size,
  next_tick: %{lobby: ordinal among the queue's lobbies, team: index} | nil}.  The prediction is for the engine as it
  is set now: a pool whose spread or budgets change before each tick predicts under the current ones.
  """
  def search_status(player_ids), do: GenServer.call(__MODULE__, {:search_status, player_ids})
  @doc """
  Party search status (extension): one map per player id, without ingesting the staged deliveries
  (Engine.party_locate under the pool's party rules): %{state: :searching (queued in a party) | :matched | :staged |
  :unknown, game_mode, group, party_size, wait_ms, position (parties of the queue ahead of its party), queue_size
  (parties of the queue), anchor, window, next_match: %{lobby: ordinal among the queue's lobbies of the next
  party_match, team: index} | nil}.  A queued solo is :unknown here (search_status/1 answers it).
  """
  def party_search_status(player_ids), do: GenServer.call(__MODULE__, {:party_search_status, player_ids})
  @doc "The queues of these rating groups (indices, all modes) emit no lobby until resume_queues/1; players stay queued."
  def pause(groups), do: GenServer.call(__MODULE__, {:pause, groups, true})
  def resume_queues(groups), do: GenServer.call(__MODULE__, {:pause, groups, false})

  @impl true
  def init(opts) do
    capacity = Keyword.get(opts, :capacity, 16_000_000)
    {:ok, ref} = Engine.new(Engine.pack_config(capacity: capacity, active_capacity: 2 * capacity, dense_ids: true))
    case Keyword.get(opts, :balance_teams) do
      nil -> :ok
      modes -> :ok = Engine.set_team_balance(ref, Enum.reduce(modes, 0, &Bitwise.bor(&2, Bitwise.bsl(1, Engine.mode_index(&1)))))
    end
    case Keyword.get(opts, :balance_parties) do
      nil -> :ok
      modes -> :ok = Engine.set_party_balance(ref, Enum.reduce(modes, 0, &Bitwise.bor(&2, Bitwise.bsl(1, Engine.mode_index(&1)))))
    end
    case Keyword.get(opts, :party_capacity) do
      nil -> :ok
      members -> :ok = Engine.set_party_capacity(ref, members)
    end
    # queued: handle -> {rating, mode, enq_ts, seq} at its enqueue, what requeue/1 hands back (kept until remove_user)
    st = %{ref: ref, staged: [], n_staged: 0, handle_of: %{}, players: %{}, free: [], next: 0, channel: nil,
           queued: %{}, moved_out: MapSet.new(),
           t0: System.monotonic_time(:millisecond), timeout: Keyword.get(opts, :search_timeout_ms),
           lobby_budget: Keyword.get(opts, :lobby_budget), paused: MapSet.new(), regroup_dropped: [],
           budget_offtick: Keyword.get(opts, :budget_offtick, false), step_budget: nil,
           widen: Keyword.get(opts, :widen), parties: Keyword.get(opts, :parties), staged_parties: [], party_of: %{},
           party_capacity: Keyword.get(opts, :party_capacity), stranded_parties: [],
           # requeue_parties: handle -> {members, ratings, mode, enq_ts, seq} of its queued (party_book) or matched party
           requeue_parties: Keyword.get(opts, :requeue_parties, false), party_book: %{}, matched_parties: %{}}
    case resume(st, Keyword.get(opts, :resume), Keyword.get(opts, :regroup, false)) do
      {:ok, st} ->
        Process.send_after(self(), :flush, @flush_ms)
        Process.send_after(self(), :tick, @tick_ms)
        {:ok, st}
      {:error, reason} -> {:stop, {:resume_failed, reason}}
    end
  end

  # -- hand-over: the engine image plus the host state ------------------------------------------------------------
  # The channel name is not carried: a name from the old process does not say that the new process has that channel
  # open.  Until a search worker attaches its channel (attach/1) or stages a delivery, :tick neither ticks nor
  # expires, so the players of the image are not matched into lobbies that could not be published.
  # regroup: the engine was created with another config than the checkpoint's (a new RatingGroups table or mode list;
  # a mode keeps its index).  A checkpoint with queues moved out is refused: those queues live in another pool under
  # the old groups.  The players the new config has no queue for are dropped here and answered by the first tick.
  defp resume(st, nil, _regroup), do: {:ok, st}
  defp resume(st, blob, regroup) do
    ck = :erlang.binary_to_term(blob, [:safe])
    loaded = cond do
      not regroup -> with :ok <- Engine.import_image(st.ref, ck.image), do: {:ok, <<>>}
      MapSet.size(Map.get(ck, :moved_out, MapSet.new())) > 0 -> {:error, :moved_out}
      true -> Engine.import_regroup(st.ref, ck.image)
    end
    case loaded do
      {:ok, rejected} ->
        down = max(0, System.os_time(:millisecond) - ck.wall_ms)
        # now_ms/1 goes on from the checkpoint's value plus the downtime: the engine's enqueue stamps stay valid
        st = %{st | handle_of: ck.handle_of, players: ck.players, free: ck.free, next: ck.next,
                    queued: Map.get(ck, :queued, %{}), moved_out: Map.get(ck, :moved_out, MapSet.new()),
                    party_of: Map.get(ck, :party_of, %{}), party_book: Map.get(ck, :party_book, %{}),
                    matched_parties: Map.get(ck, :matched_parties, %{}),
                    t0: System.monotonic_time(:millisecond) - ck.now_ms - down}
        st = drop_rejected(st, ck.image, rejected)
        case Map.get(ck, :party_image) do
          nil -> {:ok, st}
          parties ->  # with their numbers; a party with no queue under this config leaves like a rejected solo
            with {:ok, codes} <- Engine.merge_parties(st.ref, parties, true) do
              gone = for {hs, c} <- party_list(parties, codes), c != 1, h <- hs, do: h
              {:ok, Enum.reduce(gone, st, fn h, acc ->
                 {player, players} = Map.pop(acc.players, h)
                 %{acc | players: players, handle_of: Map.delete(acc.handle_of, player["id"]), free: [h | acc.free],
                         party_of: Map.delete(acc.party_of, h), party_book: Map.delete(acc.party_book, h),
                         regroup_dropped: [player | acc.regroup_dropped]}
               end)}
            end
        end
      {:error, _} = e -> e
    end
  end

  # every party of a party image as {[member handles], its code or nil}, in image order (include/mm_engine.h: sizes at
  # 624, then seq, enq_ts, mode, the u32 handles)
  defp party_list(image, codes) do
    <<_::binary-size(24), p::little-32, _::binary>> = image
    a8 = fn x -> Bitwise.band(x + 7, Bitwise.bnot(7)) end
    id_off = a8.(a8.(a8.(a8.(624 + p) + 4 * p) + 4 * p) + p)
    sizes = for <<s <- binary_part(image, 624, p)>>, do: s
    handles = for <<h::little-32 <- binary_part(image, id_off, 4 * Enum.sum(sizes))>>, do: h
    {parties, _} = Enum.map_reduce(sizes, handles, &Enum.split(&2, &1))
    Enum.zip(parties, Stream.concat(for(<<c <- codes>>, do: c), Stream.repeatedly(fn -> nil end)))
  end

  # mm_export, mm_export_queues and mm_merge refuse while a party is queued: with party capacity, every queued party
  # steps aside (Engine.export_parties) around `fun` and comes back, with its number when the sequence did not move.
  # -> {result of fun, the party image or nil, st}.  A refused export is fun's error and changes nothing; a party
  # image that cannot come back is kept in st.stranded_parties (merge it with Engine.merge_parties/3).
  # requeue_parties: the parties of a party image merged without their numbers got s1 + their index (mm_merge_parties);
  # the merged ones (code 1) get their book entry with that number, from the image's columns
  defp book_parties(%{requeue_parties: false} = st, _image, _codes, _s1), do: st
  defp book_parties(st, image, codes, s1) do
    <<_::binary-size(24), p::little-32, m::little-32, _::binary>> = image
    a8 = fn x -> Bitwise.band(x + 7, Bitwise.bnot(7)) end
    ts_off = a8.(a8.(624 + p) + 4 * p)
    mode_off = a8.(ts_off + 4 * p)
    rating_off = a8.(a8.(mode_off + p) + 4 * m)
    ts = for <<t::little-32 <- binary_part(image, ts_off, 4 * p)>>, do: t
    modes = :binary.bin_to_list(binary_part(image, mode_off, p))
    ratings = for <<r::little-signed-32 <- binary_part(image, rating_off, 4 * m)>>, do: r
    {st, _} =
      party_list(image, codes)
      |> Enum.zip(Enum.zip([ts, modes, 0..max(p - 1, 0)]))
      |> Enum.reduce({st, ratings}, fn {{hs, c}, {t, mode, j}}, {acc, left} ->
        {rat, left} = Enum.split(left, length(hs))
        rec = {hs, rat, mode, t, Bitwise.band(s1 + j, 0xFFFFFFFF)}
        acc = if c == 1, do: %{acc | party_book: Enum.reduce(hs, acc.party_book, &Map.put(&2, &1, rec))}, else: acc
        {acc, left}
      end)
    st
  end

  defp around_parties(%{party_capacity: nil} = st, fun), do: {fun.(), nil, st}
  defp around_parties(st, fun) do
    with {:ok, own} <- Engine.export_parties(st.ref, nil),
         {:ok, s0} <- Engine.seq_next(st.ref) do
      res = fun.()
      {:ok, s1} = Engine.seq_next(st.ref)
      keep = s1 == s0
      case Engine.merge_parties(st.ref, own, keep) do
        {:ok, codes} -> {res, own, if(keep, do: st, else: book_parties(st, own, codes, s1))}
        {:error, _} -> {res, own, %{st | stranded_parties: [own | st.stranded_parties]}}
      end
    else
      {:error, _} = e -> {e, nil, st}
    end
  end

  # the image's handle (section 2: u32, after the header and the partition counts) of each rejected index
  defp drop_rejected(st, _image, <<>>), do: st
  defp drop_rejected(st, image, rejected) do
    <<_::binary-size(24), n_parts::little-32, _::binary>> = image
    ids_at = div(624 + 4 * n_parts + 7, 8) * 8
    for <<i::little-32 <- rejected>>, reduce: st do
      acc ->
        <<_::binary-size(ids_at + 4 * i), h::little-32, _::binary>> = image
        {player, players} = Map.pop(acc.players, h)
        %{acc | players: players, handle_of: Map.delete(acc.handle_of, player["id"]), free: [h | acc.free],
                queued: Map.delete(acc.queued, h), regroup_dropped: [player | acc.regroup_dropped]}
    end
  end

  @impl true
  def handle_cast({:stage, player, game_mode, rating, ack_ref}, st) do
    st = %{st | staged: [{player, game_mode, rating, ack_ref} | st.staged], n_staged: st.n_staged + 1,
               channel: elem(ack_ref, 0)}   # lobbies go out on a search worker's channel, like prepare_game_lobby/4
    {:noreply, if(st.n_staged >= @max_batch, do: flush(st), else: st)}
  end

  def handle_cast({:stage_party, players, game_mode, ack_ref}, st) do
    {:noreply, %{st | staged_parties: [{players, game_mode, ack_ref} | st.staged_parties], channel: elem(ack_ref, 0)}}
  end

  def handle_cast({:attach, channel_name}, st), do: {:noreply, %{st | channel: channel_name}}

  @impl true
  def handle_call({:in_queue?, id}, _from, st) do
    reply = case st.handle_of do
      %{^id => h} -> Engine.in_queue?(st.ref, h)
      _ -> false
    end
    {:reply, reply, st}
  end

  def handle_call({:queue_status, group}, _from, st) do
    reply = with {:ok, recs} <- Engine.queue_stats(st.ref, now_ms(st)),
                 {:ok, qrecs} <- Engine.match_quality(st.ref) do
      quality = quality_of(qrecs, group)
      for <<mode, g, _::16, waiting::little-32, _removed::little-32, oldest::little-32, hist::binary-size(480),
            _lobbies::little-32, matched::little-32, _max_match::little-32, mhist::binary-size(480) <- recs>>,
          g == group, into: %{} do
        {Engine.mode_name(mode),
         Map.merge(%{waiting: waiting, oldest_wait_ms: oldest, p50_wait_ms: quantile(hist, 0.5),
                     p99_wait_ms: quantile(hist, 0.99), last_tick_matched: matched,
                     last_tick_p99_match_wait_ms: quantile(mhist, 0.99)},
                   Map.get(quality, mode, %{last_tick_lobbies: 0}))
         |> Map.merge(Map.get(offtick_of(st, group), mode, %{}))}
      end
    end
    {:reply, reply, st}
  end

  # the party_match (source 0) and widen (source 1) reports of one group -> %{mode => %{party_match: .., widen: ..}},
  # for the sources the pool runs; a void report adds nothing
  defp offtick_of(st, group) do
    for {key, src, on} <- [{:party_match, 0, st.parties}, {:widen, 1, st.widen}], on != nil,
        {:ok, wrecs, qrecs} <- [Engine.offtick_report(st.ref, src)],
        {mode, fields} <- offtick_fields(wrecs, qrecs, group),
        reduce: %{} do
      acc -> Map.update(acc, mode, %{key => fields}, &Map.put(&1, key, fields))
    end
  end

  defp offtick_fields(wrecs, qrecs, group) do
    quality = quality_of(qrecs, group)
    for <<mode, g, _::16, lobbies::little-32, matched::little-32, max_wait::little-32, whist::binary-size(480) <- wrecs>>,
        g == group do
      q = Map.fetch!(quality, mode)
      {mode, %{lobbies: lobbies, matched: matched, p50_match_wait_ms: quantile(whist, 0.5),
               p99_match_wait_ms: quantile(whist, 0.99), max_match_wait_ms: max_wait, mean_spread: q.mean_spread,
               p99_spread: q.p99_spread, max_spread: q.max_spread, mean_imbalance: q.mean_imbalance,
               p99_imbalance: q.p99_imbalance, max_imbalance: q.max_imbalance}}
    end
  end

  # mm_queue_quality records of one group -> %{mode => quality fields}; quantiles are bucket upper bounds as for waits
  defp quality_of(qrecs, group) do
    for <<mode, g, _::16, n::little-32, max_spread::little-32, max_imb::little-32, sum_spread::little-64,
          sum_imb::little-64, shist::binary-size(480), ihist::binary-size(480) <- qrecs>>,
        g == group, into: %{} do
      mean = fn s -> if n > 0, do: s / n, else: 0.0 end
      {mode, %{last_tick_lobbies: n, mean_spread: mean.(sum_spread), p50_spread: quantile(shist, 0.5),
               p99_spread: quantile(shist, 0.99), max_spread: max_spread, mean_imbalance: mean.(sum_imb),
               p99_imbalance: quantile(ihist, 0.99), max_imbalance: max_imb}}
    end
  end

  def handle_call({:remove_user, id}, _from, st) do
    st = flush(st)
    case Map.pop(st.handle_of, id) do
      {nil, _} -> {:reply, {:ok, :removed}, st}                       # Mnesia.delete of a missing key is fine too
      {h, _rest} ->
        Engine.remove_packed(st.ref, <<h::little-32>>)   # a queued party member: the engine removes the whole party
        hs = Map.get(st.party_of, h, [h])
        st = Enum.reduce(hs, st, fn x, acc ->
          {player, players} = Map.pop(acc.players, x)
          pid = if x == h, do: id, else: player && player["id"]
          %{acc | handle_of: Map.delete(acc.handle_of, pid), players: players, free: [x | acc.free],
                  queued: Map.delete(acc.queued, x), party_of: Map.delete(acc.party_of, x),
                  party_book: Map.delete(acc.party_book, x), matched_parties: Map.delete(acc.matched_parties, x)}
        end)
        {:reply, {:ok, :removed}, st}
    end
  end

  def handle_call(:checkpoint, _from, st) do
    st = flush(st)
    case around_parties(st, fn -> Engine.export_image(st.ref) end) do
      {{:ok, image}, parties, st} ->
        ck = %{image: image, handle_of: st.handle_of, players: st.players, free: st.free, next: st.next,
               queued: st.queued, moved_out: st.moved_out, now_ms: now_ms(st), wall_ms: System.os_time(:millisecond)}
        ck = if parties, do: Map.merge(ck, %{party_image: parties, party_of: st.party_of}), else: ck
        # the matched players stay in the engine image: their parties' book goes with them
        ck = if st.requeue_parties,
               do: Map.merge(ck, %{party_book: st.party_book, matched_parties: st.matched_parties}), else: ck
        {:reply, {:ok, :erlang.term_to_binary(ck)}, st}
      {{:error, _} = e, _, st} -> {:reply, e, st}
    end
  end

  # -- queue move: part of this pool into another running pool (INTEGRATION.md §5) ---------------------------------
  def handle_call({:move_out, groups}, _from, st) do
    st = flush(st)
    n_groups = Engine.n_groups()
    queues = for _m <- 0..(Engine.n_modes() - 1), g <- 0..(n_groups - 1), into: <<>>,
               do: <<(if g in groups, do: 1, else: 0)>>
    # with parties: the moved queues' parties in a party image of their own, the others step aside around the export
    exported = if st.party_capacity, do: Engine.export_parties(st.ref, queues), else: {:ok, nil}
    case exported do
      {:error, _} = e -> {:reply, e, st}   # refused before anything changed
      {:ok, moved_parties} -> move_out_queues(st, groups, queues, n_groups, moved_parties)
    end
  end

  defp move_out_queues(st, groups, queues, n_groups, moved_parties) do
    case around_parties(st, fn -> Engine.export_queues(st.ref, queues) end) do
      {{:error, _} = e, _, st} ->  # the moved parties come back (new numbers)
        st = if moved_parties && match?({:error, _}, Engine.merge_parties(st.ref, moved_parties, false)),
               do: %{st | stranded_parties: [moved_parties | st.stranded_parties]}, else: st
        {:reply, e, st}
      {{:ok, image}, _, st} ->
        {n, id_off, _} = image_sections(image)
        handles = for <<h::little-32 <- binary_part(image, id_off, 4 * n)>>, do: h
        {moved, st} = Enum.map_reduce(handles, st, fn h, acc ->
          {player, players} = Map.pop(acc.players, h)
          {{player["id"], player}, release(%{acc | players: players, queued: Map.delete(acc.queued, h)}, player["id"], h)}
        end)
        moved_q = for m <- 0..(Engine.n_modes() - 1), g <- groups, do: m * n_groups + g
        st = %{st | moved_out: MapSet.union(st.moved_out, MapSet.new(moved_q))}
        blob = %{image: image, players: moved, n_modes: Engine.n_modes(), n_groups: n_groups,
                 now_ms: now_ms(st), wall_ms: System.os_time(:millisecond)}
        {blob, st} =
          if moved_parties do  # the members' ids and documents leave with the party image
            hs = for {party, _} <- party_list(moved_parties, <<>>), h <- party, do: h
            {members, st} = Enum.map_reduce(hs, st, fn h, acc ->
              {player, players} = Map.pop(acc.players, h)
              {{player["id"], player},
               release(%{acc | players: players, party_of: Map.delete(acc.party_of, h)}, player["id"], h)}
            end)
            {Map.merge(blob, %{party_image: moved_parties, party_players: members}), st}
          else
            {blob, st}
          end
        {:reply, {:ok, :erlang.term_to_binary(blob)}, st}
    end
  end

  def handle_call({:move_in, blob}, _from, st) do
    st = flush(st)
    mv = :erlang.binary_to_term(blob, [:safe])
    if mv.n_modes != Engine.n_modes() or mv.n_groups != Engine.n_groups() do
      {:reply, {:error, :other_queues}, st}
    else
      # handles of this pool for the moved ids; the image's id column is rewritten with them
      {rows, st} = Enum.map_reduce(mv.players, st, fn {id, player}, acc ->
        {h, fresh, acc} = acquire(acc, id)
        {{h, fresh, id, player}, acc}
      end)
      {n, id_off, ts_off} = image_sections(mv.image)
      moved_members = length(Map.get(mv, :party_players, []))
      cond do
        moved_members > 0 and map_size(st.party_of) + moved_members > (st.party_capacity || 0) ->
          # the party table cannot take the moved parties: refused before anything changes
          st = Enum.reduce(rows, st, fn {h, fresh, id, _}, acc -> if fresh, do: release(acc, id, h), else: acc end)
          {:reply, {:error, :capacity}, st}
        true -> move_in_image(st, mv, rows, n, id_off, ts_off)
      end
    end
  end

  defp move_in_image(st, mv, rows, n, id_off, ts_off) do
    # enqueue stamps into this pool's clock: the wait at move_out plus the wall time in between, as resume/2 does
    down = max(0, System.os_time(:millisecond) - mv.wall_ms)
    shift = Bitwise.band(now_ms(st) - down - mv.now_ms, 0xFFFFFFFF)
    ids = for {h, _, _, _} <- rows, into: <<>>, do: <<h::little-32>>
    ts = for <<t::little-32 <- binary_part(mv.image, ts_off, 4 * n)>>, into: <<>>,
           do: <<Bitwise.band(t + shift, 0xFFFFFFFF)::little-32>>
    image = binary_part(mv.image, 0, id_off) <> ids <>
            binary_part(mv.image, id_off + 4 * n, ts_off - id_off - 4 * n) <> ts <>
            binary_part(mv.image, ts_off + 4 * n, byte_size(mv.image) - ts_off - 4 * n)
    {:ok, seq0} = Engine.seq_next(st.ref)
    {merged, _, st} = around_parties(st, fn -> Engine.merge_image(st.ref, image) end)
    case merged do
      {:ok, rejected} ->
        rej = MapSet.new(for <<i::little-32 <- rejected>>, do: i)
        # mm_merge numbers its batch queue by queue, in the source's enqueue order inside a queue: sort the image
        # indices by (queue, age), number them, and put the numbers back in image order (n log n, lists walked once)
        {cols, src_next} = image_cols(mv.image)
        seqs = cols |> Enum.with_index()
               |> Enum.sort_by(fn {{r, m, _t, s}, _i} -> {Engine.queue_of(r, m), Bitwise.band(s - src_next, 0xFFFFFFFF)} end)
               |> Enum.with_index(fn {_, i}, k -> {i, Bitwise.band(seq0 + k, 0xFFFFFFFF)} end)
               |> Enum.sort() |> Enum.map(&elem(&1, 1))
        st = Enum.zip([rows, cols, seqs]) |> Enum.with_index() |> Enum.reduce(st, fn {{{h, _, _, _}, {r, m, t, _}, q}, i}, acc ->
          if MapSet.member?(rej, i) do
            acc
          else
            %{acc | queued: Map.put(acc.queued, h, {r, m, Bitwise.band(t + shift, 0xFFFFFFFF), q}),
                    moved_out: MapSet.delete(acc.moved_out, Engine.queue_of(r, m))}
          end
        end)
        st = rows |> Enum.with_index() |> Enum.reduce(st, fn {{h, fresh, id, _}, i}, acc ->
          # a rejected player is already queued here: keep this pool's player and document
          if MapSet.member?(rej, i) and fresh, do: release(acc, id, h), else: acc
        end)
        players = for {{h, _, _, player}, i} <- Enum.with_index(rows), not MapSet.member?(rej, i), into: st.players,
                    do: {h, player}
        case move_in_parties(%{st | players: players}, mv, shift) do
          {:ok, st} -> {:reply, {:ok, n - MapSet.size(rej)}, st}
          # the solos are in; the party image is kept in stranded_parties (with this pool's handles and clock)
          {{:error, reason}, st} -> {:reply, {:error, {:parties_not_merged, reason, n - MapSet.size(rej)}}, st}
        end
      {:error, _} = e ->
        st = Enum.reduce(rows, st, fn {h, fresh, id, _}, acc -> if fresh, do: release(acc, id, h), else: acc end)
        {:reply, e, st}
    end
  end

  # The party image of a move, after its solos: this pool's handles for the members, the stamps in this pool's clock,
  # one merge (new numbers here); the members of parties that did not merge give their fresh handles back.
  defp move_in_parties(st, %{party_image: pimg, party_players: members}, shift) do
    {rows, st} = Enum.map_reduce(members, st, fn {id, player}, acc ->
      {h, fresh, acc} = acquire(acc, id)
      {{h, fresh, id, player}, acc}
    end)
    <<_::binary-size(24), p::little-32, _::binary>> = pimg
    a8 = fn x -> Bitwise.band(x + 7, Bitwise.bnot(7)) end
    ts_off = a8.(a8.(624 + p) + 4 * p)
    id_off = a8.(a8.(ts_off + 4 * p) + p)
    ts = for <<t::little-32 <- binary_part(pimg, ts_off, 4 * p)>>, into: <<>>,
           do: <<Bitwise.band(t + shift, 0xFFFFFFFF)::little-32>>
    ids = for {h, _, _, _} <- rows, into: <<>>, do: <<h::little-32>>
    image = binary_part(pimg, 0, ts_off) <> ts <> binary_part(pimg, ts_off + 4 * p, id_off - ts_off - 4 * p) <> ids <>
            binary_part(pimg, id_off + byte_size(ids), byte_size(pimg) - id_off - byte_size(ids))
    {:ok, s1} = Engine.seq_next(st.ref)
    case Engine.merge_parties(st.ref, image, false) do
      {:ok, codes} ->
        st = book_parties(st, image, codes, s1)
        {st, _} = Enum.reduce(party_list(image, codes), {st, rows}, fn {hs, c}, {acc, left} ->
          {mine, left} = Enum.split(left, length(hs))
          acc = Enum.reduce(mine, acc, fn {h, fresh, id, player}, a ->
            cond do
              c == 1 -> %{a | players: Map.put(a.players, h, player), party_of: Map.put(a.party_of, h, hs)}
              fresh -> release(a, id, h)
              true -> a
            end
          end)
          {acc, left}
        end)
        {:ok, st}
      {:error, reason} ->  # the members keep their handles and documents until the kept image is merged
        players = for {h, _, _, player} <- rows, into: st.players, do: {h, player}
        {{:error, reason}, %{st | players: players, stranded_parties: [image | st.stranded_parties]}}
    end
  end
  defp move_in_parties(st, _mv, _shift), do: {:ok, st}

  # -- requeue (extension): a lobby that did not start ----------------------------------------------------------------
  def handle_call({:requeue, players}, _from, st) do
    st = flush(st)
    {party_rows, solo_rows} = if st.requeue_parties, do: party_requeue_rows(st, players), else: {[], []}
    # the parties first: a refused call (the party table is full) changes nothing, and its parties answer :gone
    pcodes =
      case (if party_rows == [], do: {:ok, <<>>}, else: requeue_parties(st, party_rows)) do
        {:ok, pcodes} -> pcodes
        {:error, _reason} -> :binary.copy(<<4>>, length(party_rows))
      end
    whole = for {{_, hs, _, _} = row, c} <- Enum.zip(party_rows, :binary.bin_to_list(pcodes)), {i, h} <- hs,
              do: {{i, h, row}, c}
    docs = List.to_tuple(players)
    # a party requeued whole is a queued party again
    st = Enum.reduce(Enum.zip(party_rows, :binary.bin_to_list(pcodes)), st, fn
      {{_, hs, rat, {_, _, mode, ts, seq}}, 1}, acc ->
        members = for {_, h} <- hs, do: h
        rec = {members, rat, mode, ts, seq}
        acc = %{acc | players: Enum.reduce(hs, acc.players, fn {i, h}, a -> Map.put(a, h, elem(docs, i)) end)}
        Enum.reduce(members, acc, fn h, a ->
          %{a | matched_parties: Map.delete(a.matched_parties, h), party_of: Map.put(a.party_of, h, members),
                party_book: Map.put(a.party_book, h, rec)}
        end)
      _, acc -> acc
    end)
    rows = for {p, i} <- Enum.with_index(players), h = Map.get(st.handle_of, p["id"]), h != nil,
               rec = Map.get(st.queued, h), rec != nil, not MapSet.member?(st.moved_out, Engine.queue_of(elem(rec, 0), elem(rec, 1))),
               do: {i, h, rec}
    rows = Enum.uniq_by(rows ++ solo_rows, fn {_, h, _} -> h end)
    bin = fn f -> for {_, _, rec} <- rows, into: <<>>, do: f.(rec) end
    result =
      if rows == [] do
        {:ok, <<>>}
      else
        Engine.requeue(st.ref, (for {_, h, _} <- rows, into: <<>>, do: <<h::little-32>>),
                       bin.(fn {r, _, _, _} -> <<r::little-signed-32>> end), bin.(fn {_, m, _, _} -> <<m>> end),
                       bin.(fn {_, _, t, _} -> <<t::little-32>> end), bin.(fn {_, _, _, s} -> <<s::little-32>> end))
      end
    case result do
      {:ok, codes} ->
        solo = Enum.zip(rows, :binary.bin_to_list(codes))
        queued_members = for {p, i} <- Enum.with_index(players), h = Map.get(st.handle_of, p["id"]), h != nil,
                           Map.has_key?(st.party_book, h), not Enum.any?(whole, &match?({{_, ^h, _}, _}, &1)),
                           do: {{i, h, nil}, 0}
        by_h = Map.new(solo ++ whole ++ queued_members, fn {{_, h, _}, c} -> {h, c} end)
        outcome = Enum.map(players, fn p ->
          case by_h[Map.get(st.handle_of, p["id"])] do
            1 -> :requeued
            0 -> :queued
            _ -> :gone
          end
        end)
        back = for {{i, h, _}, 1} <- solo, into: st.players, do: {h, elem(docs, i)}
        st = %{st | players: back}
        # a lone member requeued as a solo is a solo from now on
        st = Enum.reduce(solo, st, fn
          {{_, h, rec}, 1}, acc when is_map_key(acc.matched_parties, h) ->
            %{acc | queued: Map.put(acc.queued, h, rec), matched_parties: Map.delete(acc.matched_parties, h)}
          _, acc -> acc
        end)
        {:reply, outcome, st}
      {:error, _} = e -> {:reply, e, st}
    end
  end

  # requeue_parties: the matched party members among `players`, by party -> {parties (two or more members: {index of
  # the first, [{index, handle}], ratings, record}), lone members as solo rows {index, handle, {rating, mode, ts, seq}}}
  defp party_requeue_rows(st, players) do
    asked = for {p, i} <- Enum.with_index(players), h = Map.get(st.handle_of, p["id"]), h != nil,
                Map.has_key?(st.matched_parties, h), do: {i, h}
    asked = Enum.uniq_by(asked, fn {_, h} -> h end)
    asked
    |> Enum.group_by(fn {_, h} -> elem(st.matched_parties[h], 4) end)
    |> Enum.reduce({[], []}, fn {_seq, hs}, {parties, solos} ->
      {members, ratings, mode, ts, seq} = rec = st.matched_parties[elem(hd(hs), 1)]
      at = Map.new(hs, fn {i, h} -> {h, i} end)
      mine = for {h, r} <- Enum.zip(members, ratings), Map.has_key?(at, h), do: {at[h], h, r}
      rat = for {_, _, r} <- mine, do: r
      q = Engine.queue_of(if(length(rat) == 1, do: hd(rat), else: Integer.floor_div(Enum.sum(rat), length(rat))), mode)
      cond do
        MapSet.member?(st.moved_out, q) -> {parties, solos}
        # a lone member goes back as a solo with the party's number, unless a co-member sent back the same way holds
        # it, still queued, in the same queue (mm_requeue would refuse the whole call): then it answers :gone
        length(mine) == 1 and Enum.any?(members, fn x ->
          x != elem(hd(mine), 1) and Map.has_key?(st.queued, x) and Map.has_key?(st.players, x) and
            Engine.queue_of(elem(st.queued[x], 0), elem(st.queued[x], 1)) == q
        end) -> {parties, solos}
        length(mine) == 1 -> {parties, [{elem(hd(mine), 0), elem(hd(mine), 1), {hd(rat), mode, ts, seq}} | solos]}
        true -> {[{elem(hd(mine), 0), for({i, h, _} <- mine, do: {i, h}), rat, rec} | parties], solos}
      end
    end)
  end

  defp requeue_parties(st, rows) do
    Engine.requeue_party(st.ref, (for {_, hs, _, _} <- rows, into: <<>>, do: <<length(hs)>>),
                         (for {_, hs, _, _} <- rows, {_, h} <- hs, into: <<>>, do: <<h::little-32>>),
                         (for {_, _, rat, _} <- rows, r <- rat, into: <<>>, do: <<r::little-signed-32>>),
                         (for {_, _, _, {_, _, m, _, _}} <- rows, into: <<>>, do: <<m>>),
                         (for {_, _, _, {_, _, _, t, _}} <- rows, into: <<>>, do: <<t::little-32>>),
                         (for {_, _, _, {_, _, _, _, s}} <- rows, into: <<>>, do: <<s::little-32>>))
  end

  def handle_call({:search_status, ids}, _from, st) do
    known = for id <- ids, h = Map.get(st.handle_of, id), do: {id, h}
    recs =
      case known do
        [] -> %{}
        _ ->
          {:ok, bin} = Engine.locate(st.ref, now_ms(st), for({_, h} <- known, into: <<>>, do: <<h::little-32>>))
          parts = for <<rec::binary-size(36) <- bin>>, do: rec
          Map.new(Enum.zip(Enum.map(known, &elem(&1, 0)), parts))
      end
    # st.staged is newest first: Map.new keeps the last entry of a key, the player's first delivery
    staged = Map.new(st.staged, fn {player, mode, _rating, _ack} -> {player["id"], mode} end)
    reply =
      Enum.map(ids, fn id ->
        base = %{state: :unknown, game_mode: nil, group: nil, wait_ms: nil, position: nil, queue_size: nil, next_tick: nil}
        case Map.get(recs, id) do
          <<1, m, g, 0, _r::little-signed-32, _ts::little-32, _seq::little-32, w::little-32, ahead::little-32,
            depth::little-32, lob::little-32, mem::little-16, _::16>> ->
            nt = if lob == 0xFFFFFFFF, do: nil, else: %{lobby: lob, team: div(mem, Engine.team_size(m))}
            %{base | state: :searching, game_mode: Engine.mode_name(m), group: g, wait_ms: w, position: ahead,
              queue_size: depth, next_tick: nt}
          <<2, _::binary>> -> %{base | state: :matched}
          _ ->
            case Map.get(staged, id) do
              nil -> base
              mode -> %{base | state: :staged, game_mode: mode}
            end
        end
      end)
    {:reply, reply, st}
  end

  def handle_call({:party_search_status, ids}, _from, st) do
    known = for id <- ids, h = Map.get(st.handle_of, id), do: {id, h}
    recs =
      case {known, st.parties, st.party_capacity} do
        {[], _, _} -> %{}
        {_, nil, _} -> %{}
        {_, _, nil} -> %{}
        _ ->
          {:ok, bin} = Engine.party_locate(st.ref, now_ms(st), party_rules(st),
                                           for({_, h} <- known, into: <<>>, do: <<h::little-32>>))
          parts = for <<rec::binary-size(48) <- bin>>, do: rec
          Map.new(Enum.zip(Enum.map(known, &elem(&1, 0)), parts))
      end
    # staged_parties is newest first: Map.new keeps the last entry of a key, the player's first delivery
    staged = Map.new(for {players, mode, _ack} <- st.staged_parties, p <- players, do: {p["id"], {mode, length(players)}})
    reply =
      Enum.map(ids, fn id ->
        base = %{state: :unknown, game_mode: nil, group: nil, party_size: nil, wait_ms: nil, position: nil,
                 queue_size: nil, anchor: nil, window: nil, next_match: nil}
        case Map.get(recs, id) do
          <<3, m, g, size, _index, anchor, 0::16, _r::little-signed-32, _pr::little-signed-32, _ts::little-32,
            _seq::little-32, w::little-32, win::little-signed-32, ahead::little-32, depth::little-32, lob::little-32,
            mem::little-16, _::16>> ->
            nm = if lob == 0xFFFFFFFF, do: nil, else: %{lobby: lob, team: div(mem, Engine.team_size(m))}
            %{base | state: :searching, game_mode: Engine.mode_name(m), group: g, party_size: size, wait_ms: w,
              position: ahead, queue_size: depth, anchor: anchor == 1, window: (if anchor == 1, do: win),
              next_match: nm}
          <<2, _::binary>> -> %{base | state: :matched}
          _ ->
            case Map.get(staged, id) do
              nil -> base
              {mode, n} -> %{base | state: :staged, game_mode: mode, party_size: n}
            end
        end
      end)
    {:reply, reply, st}
  end

  def handle_call({:backfill, requests}, _from, st) do
    st = flush(st)
    req = for r <- requests, into: <<>> do
      {mode, group, target, count, window} =
        case r do
          {m, g, t, c} -> {m, g, t, c, -1}
          {m, g, t, c, w} -> {m, g, t, c, w}
        end
      <<(Engine.mode_index(mode) || 255), group, 0::16, count::little-32, target::little-signed-32,
        window::little-signed-32>>
    end
    case Engine.backfill(st.ref, req) do
      {:ok, n_taken, handles} ->
        hs = for <<h::little-32 <- handles>>, do: h
        {out, _} = Enum.map_reduce(for(<<k::little-32 <- n_taken>>, do: k), hs, &Enum.split(&2, &1))
        docs = Enum.map(out, fn part -> Enum.map(part, &Map.fetch!(st.players, &1)) end)
        {:reply, {:ok, docs}, %{st | players: Map.drop(st.players, hs)}}
      {:error, _} = e -> {:reply, e, st}
    end
  end

  def handle_call({:backfill_teams, requests}, _from, st) do
    st = flush(st)
    reqs = for r <- requests do
      case r do
        {m, g, t, slots} -> {m, g, t, slots, -1}
        {m, g, t, slots, w} -> {m, g, t, slots, w}
      end
    end
    req = for {mode, group, target, slots, window} <- reqs, into: <<>> do
      <<(Engine.mode_index(mode) || 255), group, 0::16, Enum.sum(slots)::little-32, target::little-signed-32,
        window::little-signed-32>>
    end
    room = for {_, _, _, slots, _} <- reqs, s <- slots, into: <<>>, do: <<s::little-16>>
    # the engine reads teams_of(mode) room entries per request: a list of another length is refused here
    laid_out = Enum.all?(reqs, fn {mode, _, _, slots, _} ->
      m = Engine.mode_index(mode)
      m != nil and length(slots) == Engine.teams_of(m)
    end)
    result = if laid_out, do: Engine.backfill_party(st.ref, req, room), else: {:error, :badarg}
    case result do
      {:ok, filled, handles} ->
        hs = for <<h::little-32 <- handles>>, do: h
        counts = for <<f::little-16 <- filled>>, do: f
        {teams, _} = Enum.map_reduce(counts, hs, &Enum.split(&2, &1))
        {out, _} = Enum.map_reduce(reqs, teams, fn {_, _, _, slots, _}, rest -> Enum.split(rest, length(slots)) end)
        docs = Enum.map(out, fn per_team -> Enum.map(per_team, fn t -> Enum.map(t, &Map.fetch!(st.players, &1)) end) end)
        # a placed party's book entry moves aside, as after party_match, so requeue/1 can put the party back whole
        matched = for h <- hs, rec = Map.get(st.party_book, h), rec != nil, into: st.matched_parties, do: {h, rec}
        {:reply, {:ok, docs}, %{st | players: Map.drop(st.players, hs), party_of: Map.drop(st.party_of, hs),
                                     party_book: Map.drop(st.party_book, hs), matched_parties: matched}}
      {:error, _} = e -> {:reply, e, st}
    end
  end

  # The image's player columns (include/mm_engine.h): the 624-byte header, part_count u32[n_parts], then id (u32
  # handles on this MM_F_DENSE_IDS engine), rating, enq_ts, seq, mode, each section starting at a multiple of 8.
  defp image_sections(image) do
    <<_::binary-size(24), n_parts::little-32, n::little-32, _::binary>> = image
    a8 = fn x -> Bitwise.band(x + 7, Bitwise.bnot(7)) end
    id_off = a8.(624 + 4 * n_parts)
    rating_off = a8.(id_off + 4 * n)
    ts_off = a8.(rating_off + 4 * n)
    {n, id_off, ts_off}
  end


  # {rating, mode, enq_ts, seq} of every player of an image, and the header's seq_next
  defp image_cols(image) do
    <<_::binary-size(24), n_parts::little-32, n::little-32, _::binary-size(4), src_next::little-32, _::binary>> = image
    a8 = fn x -> Bitwise.band(x + 7, Bitwise.bnot(7)) end
    id_off = a8.(624 + 4 * n_parts)
    rt_off = a8.(id_off + 4 * n)
    ts_off = a8.(rt_off + 4 * n)
    sq_off = a8.(ts_off + 4 * n)
    md_off = a8.(sq_off + 4 * n)
    col = fn off, w -> for <<v::little-size(w) <- binary_part(image, off, div(w, 8) * n)>>, do: v end
    rts = for <<v::little-signed-32 <- binary_part(image, rt_off, 4 * n)>>, do: v
    {Enum.zip([rts, col.(md_off, 8), col.(ts_off, 32), col.(sq_off, 32)]), src_next}
  end

  @impl true
  def handle_info(:flush, st) do
    Process.send_after(self(), :flush, @flush_ms)
    {:noreply, flush(st)}
  end

  # no channel to publish on yet (a resumed pool before any search worker attached): hold the tick and the timeout
  def handle_info(:tick, %{channel: nil} = st) do
    Process.send_after(self(), :tick, @tick_ms)
    {:noreply, st}
  end

  def handle_info(:tick, st) do
    Process.send_after(self(), :tick, @tick_ms)
    for player <- st.regroup_dropped, do: send_timeout(st.channel, player)   # resume with regroup: true
    st = flush(%{st | regroup_dropped: []})
    now = now_ms(st)
    # budget_offtick: the step's budgets, less what the step has published so far (step_budget)
    st = %{st | step_budget: nil}
    st =
      cond do
        st.lobby_budget == nil -> st
        st.budget_offtick -> %{st | step_budget: budget_binaries(st, st.lobby_budget.())}
        true ->
          set_budget(st, st.lobby_budget.())
          st
      end
    st = party_match(st, now)   # before the tick: parties get the first pick of the solos
    if st.step_budget, do: :ok = Engine.set_lobby_budget(st.ref, elem(st.step_budget, 0), elem(st.step_budget, 1))
    case Engine.tick_packed(st.ref, now) do
      {:ok, lobbies, members, _stats} ->
        {:noreply, expire(widen(publish(lobbies, members, spend(st, lobbies)), now), now)}
      {:error, _reason} -> {:noreply, st}                              # nothing was consumed; the next tick retries
    end
  end

  # -- lobby budget (extension): per-mode budgets from the callback, paused groups as per-queue budget 0 --------------
  @unlimited 0xFFFFFFFF
  defp budget_binaries(st, per_mode) do
    n_groups = Engine.n_groups()
    per_queue = for _m <- 0..(Engine.n_modes() - 1), g <- 0..(n_groups - 1), into: <<>>,
                    do: <<(if MapSet.member?(st.paused, g), do: 0, else: @unlimited)::little-32>>
    modes = if per_mode == nil, do: <<>>, else:
      (for m <- 0..(Engine.n_modes() - 1), into: <<>>,
           do: <<min(max(Map.get(per_mode, Engine.mode_name(m), @unlimited), 0), @unlimited)::little-32>>)
    {per_queue, modes}
  end

  defp set_budget(st, per_mode) do
    {per_queue, modes} = budget_binaries(st, per_mode)
    :ok = Engine.set_lobby_budget(st.ref, per_queue, modes)
    if st.budget_offtick do   # the off-tick calls the pool runs, under the same budgets
      if st.parties, do: :ok = Engine.set_offtick_budget(st.ref, 0, per_queue, modes)
      if st.widen, do: :ok = Engine.set_offtick_budget(st.ref, 1, per_queue, modes)
    end
  end

  # budget_offtick: the step's per-mode budgets less the lobbies (mm_lobby_hdr binaries) just published
  defp spend(%{step_budget: nil} = st, _lobbies), do: st
  defp spend(%{step_budget: {_q, <<>>}} = st, _lobbies), do: st
  defp spend(%{step_budget: {per_queue, modes}} = st, lobbies) do
    used = Enum.frequencies(for <<_first::little-32, _n::little-16, m::8, _g::8 <- lobbies>>, do: m)
    left = for {b, m} <- Enum.with_index(for <<b::little-32 <- modes>>, do: b), into: <<>>,
               do: <<(if b == @unlimited, do: b, else: max(b - Map.get(used, m, 0), 0))::little-32>>
    %{st | step_budget: {per_queue, left}}
  end

  def handle_call({:pause, groups, on}, _from, st) do
    paused = if on, do: MapSet.union(st.paused, MapSet.new(groups)), else: MapSet.difference(st.paused, MapSet.new(groups))
    st = %{st | paused: paused}
    if st.lobby_budget == nil, do: set_budget(st, nil)   # with a callback the next tick sets both together
    {:reply, :ok, st}
  end

  # -- widening search (extension): before the timeout, so a player who waited long gets its widest window first ----
  defp widen(%{widen: nil} = st, _now), do: st
  defp widen(st, now) do
    rules = for m <- 0..(Engine.n_modes() - 1), _g <- 0..(Engine.n_groups() - 1), into: <<>> do
      case Map.get(st.widen, Engine.mode_name(m)) do
        {min_wait, w0, step, inc, w_max} ->
          <<min_wait::little-32, step::little-32, w0::little-signed-32, inc::little-signed-32, w_max::little-signed-32,
            0::32>>
        nil -> <<0xFFFFFFFF::little-32, 1::little-32, 0::32, 0::32, 0::32, 0::32>>
      end
    end
    if st.step_budget, do: :ok = Engine.set_offtick_budget(st.ref, 1, elem(st.step_budget, 0), elem(st.step_budget, 1))
    case Engine.widen(st.ref, now, rules) do
      {:ok, lobbies, members} -> publish(lobbies, members, st)
      {:error, _reason} -> st                                          # nothing was taken
    end
  end

  # -- parties (extension): one rule per queue, as widen; a party's members stay in the active set until remove_user --
  defp party_match(%{parties: nil} = st, _now), do: st
  defp party_match(st, now) do
    rules = party_rules(st)
    if st.step_budget, do: :ok = Engine.set_offtick_budget(st.ref, 0, elem(st.step_budget, 0), elem(st.step_budget, 1))
    case Engine.party_match(st.ref, now, rules) do
      {:ok, lobbies, members} ->
        st = publish(lobbies, members, spend(st, lobbies))
        placed = for <<h::little-32 <- members>>, do: h
        # requeue_parties: a placed party's book entry moves aside, so requeue/1 can put the party back whole
        matched = for h <- placed, rec = Map.get(st.party_book, h), rec != nil, into: st.matched_parties, do: {h, rec}
        %{st | party_of: Map.drop(st.party_of, placed), party_book: Map.drop(st.party_book, placed),
               matched_parties: matched}
      {:error, _reason} -> st                                          # nothing was taken
    end
  end

  # one mm_enqueue_party per flush; each party's delivery is acked (1 queued, 0 a member already queued) or nacked
  # one mm_widen_rule per (mode, group) queue: the party window of the queue's mode, MM_WIDEN_OFF for a mode without one
  defp party_rules(st) do
    for m <- 0..(Engine.n_modes() - 1), _g <- 0..(Engine.n_groups() - 1), into: <<>> do
      case Map.get(st.parties, Engine.mode_name(m)) do
        {min_wait, w0, step, inc, w_max} ->
          <<min_wait::little-32, step::little-32, w0::little-signed-32, inc::little-signed-32, w_max::little-signed-32,
            0::32>>
        nil -> <<0xFFFFFFFF::little-32, 1::little-32, 0::32, 0::32, 0::32, 0::32>>
      end
    end
  end

  defp flush_parties(%{staged_parties: []} = st), do: st
  defp flush_parties(st) do
    batch = Enum.reverse(st.staged_parties)
    {rows, st} = Enum.map_reduce(batch, %{st | staged_parties: []}, fn {players, mode, ack_ref}, acc ->
      {members, acc} = Enum.map_reduce(players, acc, fn {player, rating}, a ->
        {h, fresh, a} = acquire(a, player["id"])
        {{h, fresh, player, clamp(rating)}, a}
      end)
      {{members, Engine.mode_index(mode) || 255, ack_ref}, acc}
    end)
    sizes = for {ms, _, _} <- rows, into: <<>>, do: <<min(length(ms), 255)>>
    handles = for {ms, _, _} <- rows, {h, _, _, _} <- ms, into: <<>>, do: <<h::little-32>>
    ratings = for {ms, _, _} <- rows, {_, _, _, r} <- ms, into: <<>>, do: <<r::little-signed-32>>
    modes = for {_, m, _} <- rows, into: <<>>, do: <<m>>
    stamp = now_ms(st)
    ts = for _ <- rows, into: <<>>, do: <<stamp::little-32>>
    {:ok, seq0} = Engine.seq_next(st.ref)   # party j of the batch gets seq0 + j
    drop = fn acc, ms -> Enum.reduce(ms, acc, fn {h, fresh, p, _}, a -> if(fresh, do: release(a, p["id"], h), else: a) end) end
    case (if Enum.all?(rows, fn {ms, _, _} -> length(ms) <= 255 end),
            do: Engine.enqueue_party(st.ref, sizes, handles, ratings, modes, ts), else: {:error, :party_too_large}) do
      {:ok, codes} ->
        Enum.zip([:binary.bin_to_list(codes), rows, 0..(length(rows) - 1)])
        |> Enum.reduce(st, fn
          {1, {ms, mode, ack_ref}, j}, acc ->
            ack(ack_ref)
            hs = for {h, _, _, _} <- ms, do: h
            rec = {hs, (for {_, _, _, r} <- ms, do: r), mode, stamp, Bitwise.band(seq0 + j, 0xFFFFFFFF)}
            Enum.reduce(ms, acc, fn {h, _, p, _}, a ->
              a = %{a | players: Map.put(a.players, h, p), party_of: Map.put(a.party_of, h, hs)}
              if a.requeue_parties, do: %{a | party_book: Map.put(a.party_book, h, rec)}, else: a
            end)
          {0, {_, _, ack_ref}, _}, acc -> ack(ack_ref); acc                 # a member is already in the queue
          {_, {ms, _, ack_ref}, _}, acc -> nack(ack_ref); drop.(acc, ms)     # invalid, or the party table is full
        end)
      {:error, _reason} -> Enum.reduce(rows, st, fn {ms, _, ack_ref}, acc -> nack(ack_ref); drop.(acc, ms) end)
    end
  end

  # -- search timeout (extension): after the lobbies, so a player the tick matched is never timed out ---------------
  defp expire(%{timeout: nil} = st, _now), do: st
  defp expire(st, now) do
    case Engine.expire_packed(st.ref, now, st.timeout) do
      {:ok, handles} ->
        for <<h::little-32 <- handles>>, reduce: st do
          acc ->
            {player, players} = Map.pop(acc.players, h)
            send_timeout(acc.channel, player)
            %{acc | players: players, handle_of: Map.delete(acc.handle_of, player["id"]), free: [h | acc.free],
                    queued: Map.delete(acc.queued, h), party_of: Map.delete(acc.party_of, h),
                    party_book: Map.delete(acc.party_book, h)}
        end
      {:error, _reason} -> st                                          # nothing changed; the next tick retries
    end
  end

  defp send_timeout(channel, player) do
    case player["response-queue"] do
      nil -> :ok
      queue ->
        payload = Poison.encode!(%{"error" => %{"type" => "MatchmakingError", "details" => @timeout_details},
                                   "event-name" => player["event-name"]})
        Matchmaking.Search.Worker.safe_run(channel, fn channel ->
          AMQP.Basic.publish(channel, @exchange_response, queue, payload,
            persistent: true, content_type: "application/json")
        end)
    end
  end

  # -- ingest: one mm_enqueue_packed per batch -----------------------------------------------------------------------
  defp flush(st), do: st |> flush_solos() |> flush_parties()
  defp flush_solos(%{staged: []} = st), do: st
  defp flush_solos(st) do
    batch = Enum.reverse(st.staged)
    {rows, st} = Enum.map_reduce(batch, st, fn {player, mode, rating, ack_ref}, acc ->
      {h, fresh, acc} = acquire(acc, player["id"])
      {{h, fresh, player, Engine.mode_index(mode) || 7, clamp(rating), ack_ref}, acc}
    end)
    handles = for {h, _, _, _, _, _} <- rows, into: <<>>, do: <<h::little-32>>
    keys = for {_, _, _, m, r, _} <- rows, into: <<>>, do: <<(m * 8192 + r)::little-16>>   # mode << 13 | rating
    st = %{st | staged: [], n_staged: 0}
    stamp = now_ms(st)
    {:ok, seq0} = Engine.seq_next(st.ref)   # every offered entry of an accepted batch takes one sequence number
    ts = for _ <- rows, into: <<>>, do: <<stamp::little-32>>
    case Engine.enqueue_packed(st.ref, handles, keys, ts) do
      {:ok, codes} ->
        Enum.zip([:binary.bin_to_list(codes), rows, 0..(length(rows) - 1)])
        |> Enum.reduce(st, fn
          {1, {h, _, player, m, r, ack_ref}, i}, acc ->
            ack(ack_ref)
            %{acc | players: Map.put(acc.players, h, player),
                    queued: Map.put(acc.queued, h, {r, m, stamp, Bitwise.band(seq0 + i, 0xFFFFFFFF)})}
          {0, {_, _, _, _, _, ack_ref}, _}, acc -> ack(ack_ref); acc    # "You are already in the queue."
          {_, {h, fresh, player, _, _, ack_ref}, _}, acc -> nack(ack_ref); if(fresh, do: release(acc, player["id"], h), else: acc)
        end)
      {:error, _reason} ->                                              # the engine refused the whole batch
        Enum.reduce(rows, st, fn {h, fresh, player, _, _, ack_ref}, acc ->
          nack(ack_ref); if(fresh, do: release(acc, player["id"], h), else: acc)
        end)
    end
  end

  defp acquire(st, id) do
    case st do
      %{handle_of: %{^id => h}} -> {h, false, st}
      %{free: [h | rest]} -> {h, true, %{st | free: rest, handle_of: Map.put(st.handle_of, id, h)}}
      _ -> {st.next, true, %{st | next: st.next + 1, handle_of: Map.put(st.handle_of, id, st.next)}}
    end
  end
  defp release(st, id, h), do: %{st | handle_of: Map.delete(st.handle_of, id), free: [h | st.free]}
  defp now_ms(st), do: Bitwise.band(System.monotonic_time(:millisecond) - st.t0, 0xFFFFFFFF)

  # upper bound (largest wait) of the bucket holding the q-quantile of a wait histogram (bounds: include/mm_engine.h)
  defp quantile(hist, q) do
    counts = for <<c::little-32 <- hist>>, do: c
    case Enum.sum(counts) do
      0 -> 0
      total ->
        rank = max(1, ceil(q * total))
        b = counts |> Enum.scan(&+/2) |> Enum.find_index(&(&1 >= rank))
        if b < 8, do: b, else: Bitwise.bsl(5 + rem(b - 8, 4), div(b - 8, 4) + 1) - 1
    end
  end

  defp clamp(r) when is_integer(r), do: min(max(r, 0), 8191)
  defp clamp(_), do: 8191                                               # no integer group matches -> default group

  # -- emission: the payload of search/worker.ex:315-318, published with the options of :250-261 ----------------------
  defp publish(lobbies, members, st) do
    for <<first::little-32, n::little-16, mode, _group <- lobbies>>, reduce: st do
      acc ->
        hs = for <<h::little-32 <- binary_part(members, first * 4, n * 4)>>, do: h
        size = div(n, Engine.teams_of(mode))
        teams = hs |> Enum.map(&Map.fetch!(acc.players, &1)) |> Enum.chunk_every(size) |> Enum.with_index(1)
                |> Map.new(fn {team, i} -> {"team #{i}", team} end)
        payload = Poison.encode!(%{"teams" => teams, "game-mode" => Engine.mode_name(mode)})
        Matchmaking.Search.Worker.safe_run(acc.channel, fn channel ->
          AMQP.Basic.publish(channel, @exchange_forward, @queue_forward, payload,
            persistent: true, content_type: "application/json")
        end)
        %{acc | players: Map.drop(acc.players, hs)}     # the handles stay taken until remove_user (game-lobby/worker.ex:80)
    end
  end

  defp ack({channel_name, tag}), do: Matchmaking.Search.Worker.ack(channel_name, tag)     # search/worker.ex:81-83
  defp nack({channel_name, tag}), do: Matchmaking.Search.Worker.nack(channel_name, tag)   # search/worker.ex:88-90
end
