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

  def mode_index(name), do: Enum.find_index(@modes, fn {n, _, _} -> n == name end)
  def mode_name(index), do: elem(Enum.at(@modes, index), 0)
  def teams_of(index), do: elem(Enum.at(@modes, index), 1)

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

  @doc "Extension (not reference behaviour): maximum rating spread of a lobby for the following ticks; < 0 = off."
  def set_max_spread(_ref, _w), do: :erlang.nif_error(:nif_not_loaded)
end
