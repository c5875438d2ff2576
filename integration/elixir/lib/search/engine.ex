defmodule Matchmaking.Search.Engine do
  @moduledoc """
  NIF façade of libmm_engine.so (include/mm_engine.h) — the GPU-resident player pool that
  replaces Matchmaking.Model.ActiveUser, Matchmaking.Model.LobbyState and the per-request
  body of Matchmaking.Search.Worker.consume/5.  Columns cross the boundary as binaries;
  every call returns a tagged tuple and never raises (same convention as the models).

  NOT COMPILED HERE (no BEAM toolchain in the build environment); see INTEGRATION.md.
  """
  @on_load :load_nif
  def load_nif, do: :erlang.load_nif(:filename.join(:code.priv_dir(:matchmaking), 'mm_nif'), 0)

  @rating_groups Confex.fetch_env!(:matchmaking, RatingGroups)
  @modes [{"1v1", 2, 1}, {"5v5", 2, 5}]
  @max_groups 64
  @max_modes 8

  @doc "Packs RatingGroups (config.exs:27-36) and the mode table into an mm_config binary."
  def pack_config(opts \\ []) do
    groups = @rating_groups
    n = length(groups)
    pad = fn list, len -> list ++ List.duplicate(0, len - length(list)) end
    los = pad.(Enum.map(groups, &elem(&1, 0)), @max_groups)
    his = pad.(Enum.map(groups, &elem(&1, 1)), @max_groups)
    default = if div(n, 2) + 1 < n, do: div(n, 2) + 1, else: -1   # generic/worker.ex:27
    modes = pad.(Enum.flat_map(@modes, fn {_, t, s} -> [t, s] end), 2 * @max_modes)
    <<2::little-32, n::little-32>> <>                                   # MM_ABI_VERSION
      for(v <- los, into: <<>>, do: <<v::little-signed-32>>) <>
      for(v <- his, into: <<>>, do: <<v::little-signed-32>>) <>
      <<default::little-signed-32, length(@modes)::little-32>> <>
      for(v <- modes, into: <<>>, do: <<v::little-16>>) <>
      <<Keyword.get(opts, :order_mode, 0)::little-32, Keyword.get(opts, :capacity, 1_048_576)::little-32,
        Keyword.get(opts, :active_capacity, 0)::little-32, Keyword.get(opts, :device, 0)::little-signed-32,
        (if Keyword.get(opts, :dense_ids, false), do: 2, else: 0)::little-32>>   # MM_F_DENSE_IDS
  end

  @doc "(mode, group) queue index (mode * n_groups + group) of a rating: first group that holds it, else the default."
  def queue_of(rating, mode) do
    n = length(@rating_groups)
    g = Enum.find_index(@rating_groups, fn {lo, hi} -> rating >= lo and rating <= hi end) ||
          (if div(n, 2) + 1 < n, do: div(n, 2) + 1, else: -1)
    if g < 0, do: -1, else: mode * n + g
  end

  def mode_index(name), do: Enum.find_index(@modes, fn {n, _, _} -> n == name end)
  def mode_name(index), do: elem(Enum.at(@modes, index), 0)
  def teams_of(index), do: elem(Enum.at(@modes, index), 1)
  def team_size(index), do: elem(Enum.at(@modes, index), 2)

  # Player ids (UUID strings) are mapped to dense device handles by a table in Matchmaking.Search.Pool — not by a
  # hash: no collisions, no hash function the Elixir and Python hosts would have to agree on.

  def new(_config), do: :erlang.nif_error(:nif_not_loaded)
  def enqueue(_ref, _ids, _ratings, _modes), do: :erlang.nif_error(:nif_not_loaded)
  def remove(_ref, _ids), do: :erlang.nif_error(:nif_not_loaded)
  @doc "Dense-handle engines: handles :: binary(u32[]), keys :: binary(u16[] = mode <<< 13 ||| rating) -> {:ok, codes}"
  def enqueue_packed(_ref, _handles, _keys), do: :erlang.nif_error(:nif_not_loaded)
  @doc "Same, with enq_ts :: binary(u32[]): the enqueue stamps queue_stats/2 measures waits from (the pool's clock)"
  def enqueue_packed(_ref, _handles, _keys, _enq_ts), do: :erlang.nif_error(:nif_not_loaded)
  def remove_packed(_ref, _handles), do: :erlang.nif_error(:nif_not_loaded)
  @doc "-> {:ok, lobbies :: binary(mm_lobby_hdr[]), member_handles :: binary(u32[]), stats}"
  def tick_packed(_ref, _now_ms), do: :erlang.nif_error(:nif_not_loaded)
  def in_queue?(_ref, _id), do: :erlang.nif_error(:nif_not_loaded)
  def tick(_ref, _now_ms), do: :erlang.nif_error(:nif_not_loaded)
  def status(_ref), do: :erlang.nif_error(:nif_not_loaded)
  @doc "-> {:ok, binary(mm_queue_stat[])}: per (mode, group) queue, waiting players and wait histograms (include/mm_engine.h)"
  def queue_stats(_ref, _now_ms), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Extension (match quality): the rating spread and team imbalance of the last tick's lobbies per (mode, group) queue
  (mm_match_quality) -> {:ok, binary(mm_queue_quality[])}, in queue_stats/2 record order; an empty binary while the
  report is void (no tick yet, a failed tick, a restore or an import since).
  """
  def match_quality(_ref), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Extension (off-tick report): the waits and the rating quality of the lobbies the last party_match (source 0) or
  widen (source 1) formed, per (mode, group) queue (mm_offtick_report) -> {:ok, binary(mm_match_waits[]),
  binary(mm_queue_quality[])}, in queue_stats/2 record order; empty binaries while the report is void (no such call
  yet, or its last one failed).
  """
  def offtick_report(_ref, _source), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Extension (search timeout): the queued players who have waited >= max_wait_ms at now_ms leave the pool and the
  active set, as if removed -> {:ok, handles :: binary(u32[])}; the caller answers each one.
  """
  def expire_packed(_ref, _now_ms, _max_wait_ms), do: :erlang.nif_error(:nif_not_loaded)

  @doc """
  Hand-over: the queued players and the active set as one binary (the image of include/mm_engine.h) -> {:ok, image}.
  The engine is not changed.
  """
  def export_image(_ref), do: :erlang.nif_error(:nif_not_loaded)
  @doc "Loads an export_image/1 image into a fresh engine of the same config -> :ok | {:error, :badarg | :capacity | :state}"
  def import_image(_ref, _image), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Regroup on import (extension): loads an export_image/1 image written under ANOTHER config (rating groups, default
  group, modes, order) into this fresh engine (mm_import_regroup); every player keeps its place -> {:ok, rejected ::
  binary(u32[])}, the image indices (ascending) of the players this config has no queue for, or {:error, :badarg |
  :capacity | :state}; after a refusal the engine is still fresh.
  """
  def import_regroup(_ref, _image), do: :erlang.nif_error(:nif_not_loaded)

  @doc """
  Re-cut of a sharded deployment (extension): loads the export_image/1 images of the old ranks (one config, possibly
  another than this engine's) into this fresh engine (mm_import_regroup_many).  keep :: binary | nil selects this
  rank's queues (one byte per queue in queue_stats/2 record order); active_image :: integer | nil is the image whose
  active section this engine takes -> {:ok, rejected :: binary((u32 image, u32 index)[]), n_elsewhere} or
  {:error, :badarg | :capacity | :state}; after a refusal the engine is still fresh.
  """
  def import_regroup_many(_ref, _images, _keep, _active_image), do: :erlang.nif_error(:nif_not_loaded)

  @doc """
  Re-cut with parties queued (extension): import_regroup_many/4 with, beside images[k], the export_parties/2 image
  party_images[k] that rank k took just before it (nil or <<>> = none); solos and parties are numbered in one order
  (mm_import_regroup_many_parties) -> {:ok, rejected, n_elsewhere, party_rejected :: binary((u32 image, u32 index)[]),
  party_elsewhere} or {:error, :badarg | :capacity | :state}; after a refusal the engine is still fresh.
  """
  def import_regroup_many_parties(_ref, _images, _party_images, _keep, _active_image),
    do: :erlang.nif_error(:nif_not_loaded)

  @doc """
  Queue move: the selected (mode, group) queues (queues :: binary, one byte per queue in queue_stats/2 record order,
  mode * n_groups + group, non-zero = selected) leave the engine in a queue image -> {:ok, image}.  The players are
  released as if removed, in the same call; matched players not yet removed stay here.
  """
  def export_queues(_ref, _queues), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Loads an export_queues/2 image into this running engine -> {:ok, rejected :: binary(u32[] image indices)} |
  {:error, :badarg | :capacity | :state}; a refusal changes nothing.
  """
  def merge_image(_ref, _image), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Party hand-over: the queued parties of the selected queues (queues as export_queues/2 takes them, or nil for every
  queue) leave the engine in a party image -> {:ok, image}, released as if one member of each were removed.
  """
  def export_parties(_ref, _queues), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Merges a party image -> {:ok, codes :: binary(u8[] per party)}: 1 merged, 0 a member already active, 2 no queue here.
  keep_seq = true after import_image / import_regroup of the image taken at the same stop: every party keeps its number.
  All or nothing on room: {:error, :capacity} changes nothing.
  """
  def merge_parties(_ref, _image, _keep_seq), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Requeue (extension): the members of a lobby that did not start go back into their queue at their enqueue position
  (mm_requeue).  handles: binary(u32[]); ratings: binary(i32[]); modes: binary(u8[]); enq_ts, seq: binary(u32[]) — the
  columns each player had when it was queued -> {:ok, codes :: binary(u8[])}: 1 requeued, 0 still queued, 4 gone.
  """
  def requeue(_ref, _handles, _ratings, _modes, _enq_ts, _seq), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Backfill (extension): the open slots of running lobbies filled from their queues, nearest rating first (mm_backfill).
  requests: binary of 16-byte records <<mode, group, 0::16, count::little-32, target::little-signed-32,
  window::little-signed-32>> (window < 0: no limit) -> {:ok, n_taken :: binary(u32[]), handles :: binary(u32[])}:
  request 0's players, then request 1's, ...; they leave the pool and stay in the active set until remove_user.
  """
  def backfill(_ref, _requests), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Party backfill (extension): the open team slots of running lobbies filled with whole queued parties first, then the
  nearest solos (mm_backfill_party).  requests: the 16-byte records of backfill/2, count = the sum of the request's room
  entries; room: binary of u16 open slots, teams_of(mode) entries per request, in request order -> {:ok, filled ::
  binary(u16[]) (members per team, parallel to room), handles :: binary(u32[])}: request 0's members team by team (a
  team's parties, then its solos), then request 1's, ...  Placed parties leave the party table, taken solos the pool;
  all stay in the active set until remove_user.
  """
  def backfill_party(_ref, _requests, _room), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Widening search (extension): lobbies formed around the players who waited longest, each in a rating window that
  grows with its wait (mm_widen).  rules: binary of n_modes * n_groups 24-byte records <<min_wait::little-32,
  step::little-32, w0::little-signed-32, inc::little-signed-32, w_max::little-signed-32, 0::32>>, queue
  mode * n_groups + group, min_wait 0xFFFFFFFF = off -> {:ok, lobbies :: binary(mm_lobby_hdr[]), handles ::
  binary(u32[])}; the members leave the pool and stay in the active set until remove_user.
  """
  def widen(_ref, _now, _rules), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Parties (extension): queue players together (mm_enqueue_party).  sizes: binary(u8[]) per party; handles
  binary(u32[]) and ratings binary(little-signed-32[]) of the members, party after party; modes binary(u8[]) and enq_ts
  binary(little-32[]) per party -> {:ok, codes :: binary(u8[])}: 1 queued, 0 a member already queued, 2 invalid, 3 the
  party table is full.
  """
  def enqueue_party(_ref, _sizes, _handles, _ratings, _modes, _enq_ts), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Parties (extension): lobbies around the parties that waited longest, each party whole on one team (mm_party_match);
  rules as widen/3 takes them -> {:ok, lobbies, handles}.  Run it before the tick: parties get the first pick of the
  solos.  The solos leave the pool and every member stays in the active set until remove_user.
  """
  def party_match(_ref, _now, _rules), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Parties (extension): the parties of a lobby that did not start go back into the party table as parties, at their age
  position (mm_requeue_party).  Party j's members are the next sizes[j] handles and ratings; modes, enq_ts and seq per
  party, what it had when it was queued -> {:ok, codes :: binary(u8[])}: 1 requeued, 0 a member still queued, 4 a
  member gone.
  """
  def requeue_party(_ref, _sizes, _handles, _ratings, _modes, _enq_ts, _seq), do: :erlang.nif_error(:nif_not_loaded)
  @doc "Parties (extension): how many party members the engine holds (mm_set_option(\"party_capacity\"))."
  def set_party_capacity(_ref, _members), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Search status (extension): where each player's search stands (mm_locate).  handles: binary(u32[]) -> {:ok, records}:
  36-byte records <<state, mode, group, 0, rating::little-signed-32, enq_ts::little-32, seq::little-32,
  wait::little-32, ahead::little-32, depth::little-32, lobby::little-32, member::little-16, 0::16>>; state 0 gone,
  1 queued, 2 matched or taken and not yet removed; lobby 0xFFFFFFFF: the next tick leaves the player queued.
  """
  def locate(_ref, _now, _handles), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Party search status (extension, mm_party_queue_stats): the queued parties per (mode, group) queue ->
  {:ok, binary(mm_party_queue_stat[])} in queue_stats/2 record order; 560-byte records <<mode, group, 0::16,
  n_parties::little-32, n_members::little-32, max_wait::little-32, wait_hist::binary-480, size_hist::binary-64>>
  (one wait count per party in queue_stats/2's buckets; size_hist[k] parties of k members, [15] of 15 or more).
  """
  def party_queue_stats(_ref, _now_ms), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Party search status (extension, mm_party_locate): where each party member's search stands and the lobby the next
  party_match/3 with the same now and rules gives it.  handles: binary(u32[]) -> {:ok, records}: 48-byte records
  <<state, mode, group, size, index, anchor, 0::16, rating::little-signed-32, party_rating::little-signed-32,
  enq_ts::little-32, seq::little-32, wait::little-32, window::little-signed-32, ahead::little-32, depth::little-32,
  lobby::little-32, member::little-16, 0::16>>; state 3 queued in a party (0 gone, 1 queued solo, 2 matched);
  ahead / depth count parties; lobby 0xFFFFFFFF: the party stays queued.
  """
  def party_locate(_ref, _now, _rules, _handles), do: :erlang.nif_error(:nif_not_loaded)
  @doc "The enqueue sequence number the next offered player will get (mm_seq_next) -> {:ok, seq}."
  def seq_next(_ref), do: :erlang.nif_error(:nif_not_loaded)
  def n_modes, do: length(@modes)
  def n_groups, do: length(@rating_groups)

  @doc """
  Extension (flow control, mm_set_lobby_budget): lobbies every (mode, group) queue / every mode may emit per tick, from
  the next tick until set again.  per_queue: binary(u32[n_modes * n_groups]), queue mode * n_groups + group; per_mode:
  binary(u32[n_modes]); <<>> = no limit, 0xFFFFFFFF in an entry = no limit for it, 0 = emits nothing.  A mode's budget
  is shared over its groups by largest remainder; a queue emits its first lobbies, everyone else stays queued.
  """
  def set_lobby_budget(_ref, _per_queue, _per_mode), do: :erlang.nif_error(:nif_not_loaded)
  @doc "-> {:ok, candidates, emitted} (binary(u32[]) per queue) of the last tick: what it could have emitted and did."
  def lobby_budget_report(_ref), do: :erlang.nif_error(:nif_not_loaded)
  @doc "-> {:ok, binary(u32[])}: the lobbies a tick without a budget would emit from every queue now; changes nothing."
  def lobby_candidates(_ref), do: :erlang.nif_error(:nif_not_loaded)
  @doc """
  Extension (flow control, mm_set_offtick_budget): the lobby budget of party_match (source 0) or widen (source 1) from
  its next call until set again; binaries as in set_lobby_budget.  Each source's budget is its own, apart from the
  tick's.  The call emits every queue's first lobbies, as if the queue's plan had stopped there.
  """
  def set_offtick_budget(_ref, _source, _per_queue, _per_mode), do: :erlang.nif_error(:nif_not_loaded)
  @doc "-> {:ok, candidates, emitted} (binary(u32[]) per queue) of the source's last call (or dry run)."
  def offtick_budget_report(_ref, _source), do: :erlang.nif_error(:nif_not_loaded)

  @doc "Extension (not reference behaviour): maximum rating spread of a lobby for the following ticks; < 0 = off."
  def set_max_spread(_ref, _w), do: :erlang.nif_error(:nif_not_loaded)

  @doc """
  Extension (not reference behaviour): bit m of mask splits every lobby of mode m into the two teams with the least
  rating difference (two-team modes of at most 8 players a team); 0 = off.  Team t is still members [t S, (t + 1) S).
  """
  def set_team_balance(_ref, _mask), do: :erlang.nif_error(:nif_not_loaded)

  @doc """
  Extension (not reference behaviour): bit m of mask splits every party_match lobby of mode m into its most even teams
  that keep every party whole (two-team modes of at most 8 players a team); 0 = off.  Independent of
  set_team_balance/2, which never splits party lobbies.
  """
  def set_party_balance(_ref, _mask), do: :erlang.nif_error(:nif_not_loaded)
end
