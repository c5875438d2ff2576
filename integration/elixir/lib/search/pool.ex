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
                     last tick's matched players and p99 wait at match, in ms — Search.Worker.status/0's queue depth

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
  @max_batch 65_536
  @flush_ms 2
  @tick_ms 5

  def start_link(opts \\ []), do: GenServer.start_link(__MODULE__, opts, name: __MODULE__)
  def stage(player, game_mode, rating, ack_ref), do: GenServer.cast(__MODULE__, {:stage, player, game_mode, rating, ack_ref})
  def in_queue?(player_id), do: GenServer.call(__MODULE__, {:in_queue?, player_id})
  def remove_user(player_id), do: GenServer.call(__MODULE__, {:remove_user, player_id})
  def queue_status(group_index), do: GenServer.call(__MODULE__, {:queue_status, group_index})

  @impl true
  def init(opts) do
    capacity = Keyword.get(opts, :capacity, 16_000_000)
    {:ok, ref} = Engine.new(Engine.pack_config(capacity: capacity, active_capacity: 2 * capacity, dense_ids: true))
    Process.send_after(self(), :flush, @flush_ms)
    Process.send_after(self(), :tick, @tick_ms)
    {:ok, %{ref: ref, staged: [], n_staged: 0, handle_of: %{}, players: %{}, free: [], next: 0, channel: nil,
            t0: System.monotonic_time(:millisecond)}}
  end

  @impl true
  def handle_cast({:stage, player, game_mode, rating, ack_ref}, st) do
    st = %{st | staged: [{player, game_mode, rating, ack_ref} | st.staged], n_staged: st.n_staged + 1,
               channel: elem(ack_ref, 0)}   # lobbies go out on a search worker's channel, like prepare_game_lobby/4
    {:noreply, if(st.n_staged >= @max_batch, do: flush(st), else: st)}
  end

  @impl true
  def handle_call({:in_queue?, id}, _from, st) do
    reply = case st.handle_of do
      %{^id => h} -> Engine.in_queue?(st.ref, h)
      _ -> false
    end
    {:reply, reply, st}
  end

  def handle_call({:queue_status, group}, _from, st) do
    reply = case Engine.queue_stats(st.ref, now_ms(st)) do
      {:ok, recs} ->
        for <<mode, g, _::16, waiting::little-32, _removed::little-32, oldest::little-32, hist::binary-size(480),
              _lobbies::little-32, matched::little-32, _max_match::little-32, mhist::binary-size(480) <- recs>>,
            g == group, into: %{} do
          {Engine.mode_name(mode), %{waiting: waiting, oldest_wait_ms: oldest, p50_wait_ms: quantile(hist, 0.5),
                                     p99_wait_ms: quantile(hist, 0.99), last_tick_matched: matched,
                                     last_tick_p99_match_wait_ms: quantile(mhist, 0.99)}}
        end
      {:error, _} = e -> e
    end
    {:reply, reply, st}
  end

  def handle_call({:remove_user, id}, _from, st) do
    st = flush(st)
    case Map.pop(st.handle_of, id) do
      {nil, _} -> {:reply, {:ok, :removed}, st}                       # Mnesia.delete of a missing key is fine too
      {h, rest} ->
        Engine.remove_packed(st.ref, <<h::little-32>>)
        {:reply, {:ok, :removed}, %{st | handle_of: rest, players: Map.delete(st.players, h), free: [h | st.free]}}
    end
  end

  @impl true
  def handle_info(:flush, st) do
    Process.send_after(self(), :flush, @flush_ms)
    {:noreply, flush(st)}
  end

  def handle_info(:tick, st) do
    Process.send_after(self(), :tick, @tick_ms)
    st = flush(st)
    case Engine.tick_packed(st.ref, now_ms(st)) do
      {:ok, lobbies, members, _stats} -> {:noreply, publish(lobbies, members, st)}
      {:error, _reason} -> {:noreply, st}                              # nothing was consumed; the next tick retries
    end
  end

  # -- ingest: one mm_enqueue_packed per batch -----------------------------------------------------------------------
  defp flush(%{staged: []} = st), do: st
  defp flush(st) do
    batch = Enum.reverse(st.staged)
    {rows, st} = Enum.map_reduce(batch, st, fn {player, mode, rating, ack_ref}, acc ->
      {h, fresh, acc} = acquire(acc, player["id"])
      {{h, fresh, player, Engine.mode_index(mode) || 7, clamp(rating), ack_ref}, acc}
    end)
    handles = for {h, _, _, _, _, _} <- rows, into: <<>>, do: <<h::little-32>>
    keys = for {_, _, _, m, r, _} <- rows, into: <<>>, do: <<(m * 8192 + r)::little-16>>   # mode << 13 | rating
    st = %{st | staged: [], n_staged: 0}
    stamp = now_ms(st)
    ts = for _ <- rows, into: <<>>, do: <<stamp::little-32>>
    case Engine.enqueue_packed(st.ref, handles, keys, ts) do
      {:ok, codes} ->
        Enum.zip(:binary.bin_to_list(codes), rows)
        |> Enum.reduce(st, fn
          {1, {h, _, player, _, _, ack_ref}}, acc -> ack(ack_ref); %{acc | players: Map.put(acc.players, h, player)}
          {0, {_, _, _, _, _, ack_ref}}, acc -> ack(ack_ref); acc       # "You are already in the queue."
          {_, {h, fresh, player, _, _, ack_ref}}, acc -> nack(ack_ref); if(fresh, do: release(acc, player["id"], h), else: acc)
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
