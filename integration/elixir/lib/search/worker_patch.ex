# worker_patch.ex — what changes inside matchmaking/lib/search/worker.ex (everything else stays: queue / exchange
# names :23-40, start_link/1 opts, configure/2, ack/nack, handle_info clauses :337-368, prepare_game_lobby/4).
# NOT COMPILED HERE; a fragment for the maintainer, mirrored 1:1 by SearchWorker.consume in search_worker.py.

  # :29 — the worker acks a delivery only once its player is resident in the pool, so the broker must be allowed a
  # whole ingest batch of unacknowledged messages (a prefetch of 10 would cap the ingest at 10 players per flush)
  @qos_options [prefetch_count: 65_536]

  # :291-324 — consume/5: no LobbyState pop, no strategist RPC, no per-player Mnesia lookups; the ack moves to the pool
  defp consume(channel_name, _group_name, tag, _headers, payload) do
    with {:ok, %{"id" => _} = player_data} <- Poison.decode(payload),
         {game_mode, player} when is_binary(game_mode) <- Map.pop(player_data, "game-mode"),
         rating when is_number(rating) <- player_data["rating"] || get_in(player_data, ["detail", "rating"]) do
      # generic/worker.ex:46-53: a float between the integer ranges matches no group -> the default group
      rating = if is_float(rating) and rating != trunc(rating), do: :no_group, else: trunc(rating)
      Matchmaking.Search.Pool.stage(player, game_mode, rating, {channel_name, tag})
    else
      _ -> nack(channel_name, tag)                      # malformed request: the reference would crash the spawned process
    end
  end

  # :115-117, 326-334 — status/0: the broker's queue is nearly always empty (deliveries are acked once resident), so the
  # group's waiting players come from the engine:  Map.put(status, :waiting, Matchmaking.Search.Pool.queue_status(group))

  # application.ex:42-60 — one more child, before the search workers:   {Matchmaking.Search.Pool, []}
  # middleware/worker.ex:65-70 — ActiveUser.in_queue?(id) -> Matchmaking.Search.Pool.in_queue?(id); add_user/1 goes away
  #                             (the enqueue itself answers "already in the queue", code 0)
  # game-lobby/worker.ex:80,96 — ActiveUser.remove_user(id) -> Matchmaking.Search.Pool.remove_user(id)
