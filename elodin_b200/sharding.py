"""World-axis sharding for multi-GPU runs (SURVEY §8e).

Worlds are independent units — the reference runs one OS process per Monte-Carlo world
(libs/monte-carlo/src/lib.rs:2083) — so ranks own contiguous world ranges and the data path
needs no collective.  `torch.distributed` is used for the end-of-run gather and counters
only; on GPUs that is NCCL over NVLink, in the CPU tests gloo.
"""

from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np


def shard_worlds(n_worlds: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Contiguous, balanced world range [w0, w1) of `rank` (sizes differ by at most 1)."""
    if world_size < 1 or not (0 <= rank < world_size):
        raise ValueError(f"bad rank {rank} / world_size {world_size}")
    base, rem = divmod(int(n_worlds), world_size)
    w0 = rank * base + min(rank, rem)
    return w0, w0 + base + (1 if rank < rem else 0)


def shard_sizes(n_worlds: int, world_size: int) -> List[int]:
    return [shard_worlds(n_worlds, r, world_size)[1] - shard_worlds(n_worlds, r, world_size)[0] for r in range(world_size)]


def shard_groups(sizes: Sequence[int], rank: int, world_size: int) -> List[int]:
    """The world groups of `rank` in a world-sharded grouped campaign: the global group sizes cut to the rank's world
    range (shard_worlds), zeros kept, so every rank has the same number of groups and group g of every rank's grouped
    tables is part of global group g.  gather_ensemble / gather_histograms then merge the grouped tables as they merge
    the ungrouped ones (a count-0 part is the identity of the merge)."""
    w0, w1 = shard_worlds(sum(int(s) for s in sizes), rank, world_size)
    out, g0 = [], 0
    for s in sizes:
        g1 = g0 + int(s)
        out.append(max(0, min(g1, w1) - max(g0, w0)))
        g0 = g1
    return out


def shard_retained(retain: Sequence[int], n_worlds: int, rank: int, world_size: int) -> List[int]:
    """The entries of a global `retain` list (World.build(..., ensemble=True, retain=...)) that fall in `rank`'s world
    range (shard_worlds), as indices local to that range, in the given order: every rank of a world-sharded campaign
    retains the global runs it holds.  A rank may get none (then it builds without `retain`)."""
    w0, w1 = shard_worlds(n_worlds, rank, world_size)
    return [int(w) - w0 for w in retain if w0 <= int(w) < w1]


def gather_worlds(local, n_worlds: int, group=None):
    """End-of-run gather of a per-world tensor [w_local, ...] from every rank into the global
    world order [n_worlds, ...] (all ranks get the result).  Ragged shards are padded to the
    largest shard for the fixed-size all_gather and trimmed afterwards."""
    import torch
    import torch.distributed as dist

    ws = dist.get_world_size(group)
    sizes = shard_sizes(n_worlds, ws)
    mx = max(sizes)
    if min(sizes) == mx and local.shape[0] == mx:
        # equal shards: one flat all-gather straight into the result (no per-rank staging tensors)
        out = torch.empty((ws * mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out = [torch.empty_like(pad) for _ in range(ws)]
    dist.all_gather(out, pad, group=group)
    return torch.cat([o[:s] for o, s in zip(out, sizes)], 0)


def _all_gather_tables(table, group) -> List[np.ndarray]:
    """Every rank's host table, in rank order: a CUDA copy for NCCL groups, host memory for gloo."""
    import torch
    import torch.distributed as dist

    local = table.detach().to("cpu", torch.float64) if isinstance(table, torch.Tensor) else torch.from_numpy(
        np.ascontiguousarray(table, dtype=np.float64))
    dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    local = local.to(dev).contiguous()
    parts = [torch.empty_like(local) for _ in range(dist.get_world_size(group))]
    dist.all_gather(parts, local, group=group)
    return [p.cpu().numpy() for p in parts]


def gather_ensemble(table, group=None) -> np.ndarray:
    """Ensemble statistics of a world-sharded campaign: every rank passes the table of its own worlds ([..., 5] from
    `B200Exec.trajectory_stats` / `state_stats`, numpy or torch), the tables are all-gathered and merged in rank order
    with `merge_stats` (b200_stats_merge) on the host.  Every rank gets the same bits.  The tables are small (5 f64
    per group)."""
    from .executor import merge_stats

    return merge_stats(_all_gather_tables(table, group))


def gather_covariance(table, group=None) -> np.ndarray:
    """Ensemble covariance of a world-sharded campaign: every rank passes the table of its own worlds ([..., 1 + p + p*p]
    from `B200Exec.trajectory_covariance` / `state_covariance`, numpy or torch, the same selection on every rank), the
    tables are all-gathered and merged in rank order with `merge_covariance` (b200_covariance_merge) on the host.  Every
    rank gets the same bits."""
    from .executor import merge_covariance

    return merge_covariance(_all_gather_tables(table, group))


def gather_histograms(table, group=None) -> np.ndarray:
    """Ensemble histograms of a world-sharded campaign: every rank passes the table of its own worlds (from
    `B200Exec.trajectory_histograms` / `state_histograms`, numpy or torch, the same specs on every rank), the tables are
    all-gathered and summed with `merge_histograms`.  The counts are integers, so every rank gets the same bits: exactly
    the histogram of the union of the worlds."""
    from .executor import merge_histograms

    return merge_histograms(_all_gather_tables(table, group))


def all_reduce_min(value: int, group=None) -> int:
    """The least of every rank's integer `value` (on a CUDA tensor for NCCL groups, host memory for gloo)."""
    import torch
    import torch.distributed as dist

    t = torch.tensor([int(value)], dtype=torch.int64, device="cuda" if dist.get_backend(group) == "nccl" else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
    return int(t.item())


_ARGUMENT_ERROR = -1  # the status a rank sends for a source or levels it cannot use


def _quantile_descriptor(ex, levels: np.ndarray, source: str, groups: bool, status: int) -> List[int]:
    """What every rank of a sharded quantile call must agree on, as int64 words: source, grouping, the table's shape
    (groups, entities, width, samples, outcomes, levels), the levels' bits; then the rank's worlds and begin's status."""
    from . import _lib

    try:
        shape = list(ex.sharded_quantiles_shape(levels, source, groups))
    except Exception:  # noqa: BLE001 - a rank that cannot even describe its table differs from the others
        shape = []
    shape = (shape + [-1] * 6)[:6]
    bits = np.zeros(_lib.MAX_QUANTILES, dtype=np.float64)
    bits[: min(levels.size, _lib.MAX_QUANTILES)] = levels[: _lib.MAX_QUANTILES]
    return ([(_lib.QUANTILE_SOURCES.get(source, -1) if isinstance(source, str) else -1), int(bool(groups)), int(levels.size)] + shape
            + [int(b) for b in bits.view(np.int64)] + [int(ex.n_worlds), int(status)])


def _sharded_call(what: str, args: str, fields: str, begin, descriptor, round_, end, arg_err, group,
                  world_cap: Optional[int] = None):
    """The lockstep protocol of a sharded call (b200_sixdof_sharded_quantiles_* / _ranks_*), on every rank: `begin()`
    (returning the largest round in bytes; None when `arg_err`, an argument this rank cannot use, is set), then an
    all-gather of `descriptor(status)` (int words, ending with the rank's worlds and its begin's status), then the
    rounds of `round_(reduced, reduced_bytes, partial)` with their u32 words summed by one all-reduce each (on a CUDA
    buffer for NCCL groups, host memory for gloo), then `end()`.  A disagreement in the descriptors, a global world
    count of `world_cap` or more, or any rank's failure (at begin or in a later round) raises the same error on every
    rank instead of leaving the others waiting.  `what` names the call, `args` its arguments and `fields` its descriptor in
    the messages."""
    import torch.distributed as dist

    from . import _lib

    if not (dist.is_available() and dist.is_initialized()):
        if arg_err is not None:
            raise arg_err
        raise RuntimeError(f"{what} needs an initialized torch.distributed process group")
    import torch

    cuda = dist.get_backend(group) == "nccl"
    dev = "cuda" if cuda else "cpu"
    status, err, max_round = (_ARGUMENT_ERROR, arg_err, 0) if arg_err is not None else (0, None, 0)
    if arg_err is None:
        try:
            max_round = begin()
        except _lib.B200Error as e:
            status, err = int(e.code), e
    mine = torch.tensor(descriptor(status), dtype=torch.int64, device=dev)
    every = [torch.empty_like(mine) for _ in range(dist.get_world_size(group))]
    dist.all_gather(every, mine, group=group)
    every = [d.cpu().numpy() for d in every]
    failed = [r for r, d in enumerate(every) if d[-1] != 0]
    if failed:
        if err is not None:
            raise err
        r, code = failed[0], int(every[failed[0]][-1])
        if code == _ARGUMENT_ERROR:
            raise ValueError(f"{what}: rank {r} passed {args} it cannot use")
        raise _lib.B200Error(code, f"{what}: rank {r} could not begin (code {code})")
    differ = [r for r, d in enumerate(every) if not np.array_equal(d[:-2], every[0][:-2])]
    if differ:
        raise ValueError(f"{what}: rank {differ[0]} differs from rank 0 in {fields} (descriptors {every[0][:9].tolist()} "
                         f"and {every[differ[0]][:9].tolist()})")
    n_worlds = sum(int(d[-2]) for d in every)
    if world_cap is not None and n_worlds >= world_cap:
        raise ValueError(f"{what}: {n_worlds} worlds in all, at most {world_cap - 1}")

    def settle():
        # NCCL works on its own stream and only orders torch's current stream after it; the library reads and writes
        # the buffer on the handle's stream, so the host waits for the buffer before every round call
        if cuda:
            torch.cuda.current_stream().synchronize()

    # int32 words: a two's-complement sum wraps exactly as the u32 sum the rounds are defined by
    partial = torch.zeros(max(max_round // 4, 1), dtype=torch.int32, device=dev)
    settle()
    nbytes = 0
    while True:
        ok = 1
        try:
            nbytes = round_(partial if nbytes else None, nbytes, partial)
        except _lib.B200Error as e:
            ok, err = 0, e
        # status and round size in one collective: a failure, or ranks whose rounds differ, raise on every rank
        word = torch.tensor([ok, nbytes, -nbytes], dtype=torch.int64, device=dev)
        dist.all_reduce(word, op=dist.ReduceOp.MIN, group=group)
        ok_all, least, most = int(word[0].item()), int(word[1].item()), -int(word[2].item())
        if not ok_all:
            raise err if err is not None else _lib.B200Error(_lib.ERR_INVALID_ARGUMENT,
                                                             f"{what}: a round failed on another rank")
        if least != most:
            raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT, f"{what}: the ranks' rounds differ ({least} to "
                                 f"{most} bytes): their rows or arguments are not those of one campaign")
        if nbytes == 0:
            break
        dist.all_reduce(partial[: nbytes // 4], op=dist.ReduceOp.SUM, group=group)
        settle()
    # the end's status too, so that a rank whose end fails (out of memory, say) raises on every rank before a caller's
    # next collective
    ok, out = 1, None
    try:
        out = end()
    except _lib.B200Error as e:
        ok, err = 0, e
    word = torch.tensor([ok], dtype=torch.int64, device=dev)
    dist.all_reduce(word, op=dist.ReduceOp.MIN, group=group)
    if not int(word[0].item()):
        raise err if not ok else _lib.B200Error(_lib.ERR_INVALID_ARGUMENT, f"{what}: the end failed on another rank")
    return out


def gather_quantiles(ex, q, source: str = "ring", groups: bool = False, group=None) -> np.ndarray:
    """Quantile tables of a world-sharded campaign, exact over every rank's worlds: every rank passes its executor (its
    own worlds; with `groups`, the global groups cut to them by shard_groups), the same levels `q` and the same source
    ("ring", "state" or "outcomes"); the ranks run b200_sixdof_sharded_quantiles_* in lockstep, summing each round's
    u32 words with one all-reduce (on a CUDA buffer for NCCL groups, host memory for gloo).  Every rank returns the table
    of trajectory_ / state_ / outcome_[group_]quantiles(q) on one executor holding every rank's worlds in rank order,
    bit for bit.  Before the first round the ranks all-gather a descriptor of their calls; a disagreement, a global
    world count of 2^32 or more, or any rank's failure (then or in a later round) raises the same error on every
    rank."""
    from . import _lib

    # An argument this rank cannot use still goes through the descriptor exchange as a failed status, so that a rank
    # whose arguments differ from the others' raises with them instead of leaving them waiting.
    arg_err, levels = None, np.zeros(0)
    try:
        if source not in _lib.QUANTILE_SOURCES:
            raise ValueError(f"quantile source {source!r}: 'ring', 'state' or 'outcomes'")
        levels = np.ascontiguousarray(np.atleast_1d(np.asarray(q, dtype=np.float64)).ravel())
    except (TypeError, ValueError) as e:
        arg_err = e
    return _sharded_call("sharded quantiles", "a source or levels", "source, grouping, levels or table shape",
                         lambda: ex.sharded_quantiles_begin(levels, source, groups),
                         lambda status: _quantile_descriptor(ex, levels, source, groups, status),
                         lambda *a: ex.sharded_quantiles_round(*a), lambda: ex.sharded_quantiles_end(), arg_err, group,
                         world_cap=1 << 32)


def _rank_descriptor(ex, sel: List[int], groups: bool, status: int) -> List[int]:
    """What every rank of a sharded rank call must agree on, as int64 words: the planes (padded with -1), their count,
    grouping, the group and outcome counts; then the rank's worlds and begin's status."""
    from . import _lib

    sel = sel[: _lib.MAX_OUTCOMES]
    try:
        shape = [int(ex.world_groups) if groups else 1, int(ex.n_outcomes)]
    except Exception:  # noqa: BLE001 - a rank that cannot even describe its call differs from the others
        shape = [-1, -1]
    return sel + [-1] * (_lib.MAX_OUTCOMES - len(sel)) + [len(sel), int(bool(groups))] + shape + [int(ex.n_worlds), int(status)]


def _rank_planes(planes, least: int = 1) -> List[int]:
    sel = [int(p) for p in np.atleast_1d(np.asarray(planes)).ravel()]
    if len(sel) < least or len(set(sel)) != len(sel) or min(sel, default=0) < 0:
        raise ValueError(f"sharded ranks: planes {sel!r}, {least} or more distinct outcome planes")
    return sel


def _gather_rank_call(ex, planes, groups: bool, group, ranks: bool, covariance: bool):
    """The sharded rank call (b200_sixdof_sharded_ranks_*) over every rank of `group`, with the checks of
    gather_quantiles: this rank's (ranks, covariance records) of B200Exec.sharded_ranks_end."""
    import torch.distributed as dist

    arg_err, sel = None, []
    try:
        sel = _rank_planes(planes, 2 if covariance else 1)  # a correlation needs two planes, as the unsharded call
    except (TypeError, ValueError) as e:
        arg_err = e
    rank = dist.get_rank(group) if dist.is_available() and dist.is_initialized() else 0
    n_ranks = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    return _sharded_call("sharded ranks", "planes", "planes, grouping, group or outcome count",
                         lambda: ex.sharded_ranks_begin(sel, groups, rank, n_ranks),
                         lambda status: _rank_descriptor(ex, sel, groups, status), lambda *a: ex.sharded_ranks_round(*a),
                         lambda: ex.sharded_ranks_end(ranks, covariance), arg_err, group)


def gather_ranks(ex, planes, groups: bool = False, group=None) -> np.ndarray:
    """Midranks of a world-sharded campaign: every rank passes its executor (its own worlds; with `groups`, the global
    groups cut to them by shard_groups) and the same outcome `planes`; the ranks run b200_sixdof_sharded_ranks_* in
    lockstep, as gather_quantiles does.  Every rank returns [its n_worlds, p]: the rows of its own worlds in
    outcome_[group_]ranks(planes) on one executor holding every rank's worlds in rank order, bit for bit."""
    return _gather_rank_call(ex, planes, groups, group, True, False)[0]


def gather_rank_correlation(ex, planes, groups: bool = False, group=None) -> np.ndarray:
    """Rank correlation of a world-sharded campaign: the sharded rank call of gather_ranks, then every rank's covariance
    records of its rank planes, all-gathered and merged in rank order (merge_covariance), turned into
    [1 + p*p] (or [G, 1 + p*p] with `groups`) records by executor.rank_correlation.  Every rank gets the same bits;
    with one rank those of outcome_[group_]rank_correlation(planes)."""
    from .executor import merge_covariance, rank_correlation

    cov = _gather_rank_call(ex, planes, groups, group, False, True)[1]
    merged = merge_covariance(_all_gather_tables(cov, group))
    out = rank_correlation(merged, len(_rank_planes(planes, 2)))
    return out if groups else out[0]


def outcome_ranks(exec_, names=None, groups: bool = False) -> dict:
    """Exec.outcome_ranks over every rank of a world-sharded campaign (World.build(..., process_group=pg)): a
    collective, every rank passing the same names.  Returns this rank's dict, {name: [its n_worlds]} of campaign
    midranks."""
    from .world import _ranks_dict

    names, planes = exec_._rank_names("outcome_ranks", names, groups, 1, sharded=True, one=True)
    return _ranks_dict(names, gather_ranks(exec_.backend, planes, groups, exec_._pg))


def outcome_rank_correlation(exec_, names=None, groups: bool = False) -> dict:
    """Exec.outcome_rank_correlation over every rank of a world-sharded campaign: a collective; every rank gets the
    same dict."""
    from .world import _rank_correlation_dict

    names, planes = exec_._rank_names("outcome_rank_correlation", names, groups, 2, sharded=True)
    return _rank_correlation_dict(names, gather_rank_correlation(exec_.backend, planes, groups, exec_._pg))


def outcome_sensitivity(exec_, inputs, outputs, groups: bool = False) -> dict:
    """Exec.outcome_sensitivity over every rank of a world-sharded campaign: a collective; every rank gets the same
    dict (rho and PRCC from the merged rank correlation)."""
    from .world import _sensitivity_dict

    inputs, outputs, planes = exec_._sensitivity_names(inputs, outputs, groups, sharded=True)
    return _sensitivity_dict(inputs, outputs, gather_rank_correlation(exec_.backend, planes, groups, exec_._pg))


def _top_worlds_descriptor(planes, k, largest, groups, shape, n_worlds: int, status: int) -> List[int]:
    """What every rank of a sharded worst-worlds call must agree on, as int64 words: the planes (padded with -1), their
    count, k, largest, grouping and the table's shape; then the rank's worlds and its local call's status."""
    from . import _lib

    sel = [int(p) for p in planes][: _lib.MAX_OUTCOMES] if planes is not None else []
    shape = (list(shape) + [-1] * 3)[:3]
    return (sel + [-1] * (_lib.MAX_OUTCOMES - len(sel)) + [len(sel), int(k), int(bool(largest)), int(bool(groups))] + shape
            + [int(n_worlds), int(status)])


def gather_top_worlds(ex, planes, k: int, largest: bool, groups: bool = False, group=None) -> np.ndarray:
    """Worst worlds of a world-sharded campaign, exact over every rank's worlds: every rank passes its executor (its
    own worlds; with `groups`, the global groups cut to them by shard_groups) and the same planes, k and direction.
    Each rank computes its own records (B200Exec.outcome_[group_]top_worlds), the ranks all-gather a descriptor of
    their calls and then the records (1 + 2k f64 per task), and merge them with merge_top_worlds, offsetting each
    rank's worlds by the worlds of the ranks before it.  Every rank returns the table of the same call on one executor
    holding every rank's worlds in rank order, with campaign world indices.  A disagreement in the arguments or the
    table shape, or any rank's failure, raises on every rank."""
    import torch
    import torch.distributed as dist

    from . import _lib
    from .executor import merge_top_worlds

    if not (dist.is_available() and dist.is_initialized()):
        raise RuntimeError("sharding.gather_top_worlds needs an initialized torch.distributed process group")
    dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    status, err, table, sel = 0, None, None, None
    try:
        sel = [int(p) for p in np.atleast_1d(np.asarray(planes)).ravel()]
        table = ex.outcome_group_top_worlds(sel, k, largest) if groups else ex.outcome_top_worlds(sel, k, largest)
    except _lib.B200Error as e:
        status, err = int(e.code), e
    except (TypeError, ValueError) as e:
        status, err = _ARGUMENT_ERROR, e
    shape = table.shape if table is not None else ()
    try:
        words = _top_worlds_descriptor(sel, k, largest, groups, shape if groups else (1,) + tuple(shape), ex.n_worlds, status)
    except (TypeError, ValueError) as e:  # a k or flag that is not a number: this rank differs from the others
        status, err = _ARGUMENT_ERROR, err or e
        words = _top_worlds_descriptor(None, -1, False, groups, (), ex.n_worlds, status)
    mine = torch.tensor(words, dtype=torch.int64, device=dev)
    every = [torch.empty_like(mine) for _ in range(dist.get_world_size(group))]
    dist.all_gather(every, mine, group=group)
    every = [d.cpu().numpy() for d in every]
    failed = [r for r, d in enumerate(every) if d[-1] != 0]
    if failed:
        if err is not None:
            raise err
        r, code = failed[0], int(every[failed[0]][-1])
        if code == _ARGUMENT_ERROR:
            raise ValueError(f"sharded top worlds: rank {r} passed planes, k or largest it cannot use")
        raise _lib.B200Error(code, f"sharded top worlds: rank {r} failed (code {code})")
    differ = [r for r, d in enumerate(every) if not np.array_equal(d[:-2], every[0][:-2])]
    if differ:
        raise ValueError(f"sharded top worlds: rank {differ[0]} differs from rank 0 in planes, k, largest, grouping or "
                         f"table shape")
    offsets = np.concatenate([[0], np.cumsum([int(d[-2]) for d in every])[:-1]])
    return merge_top_worlds(_all_gather_tables(table, group), offsets, largest)


def total_entity_steps(local_entity_steps: int, group=None) -> int:
    import torch
    import torch.distributed as dist

    dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    t = torch.tensor([int(local_entity_steps)], dtype=torch.int64, device=dev)
    dist.all_reduce(t, group=group)
    return int(t.item())


class Comm:
    """One rank of the library's own NCCL communicator (include/b200_sixdof.h `b200_comm`): the C-ABI route of
    the end-of-run trajectory gather, usable by a host without torch.  Rank 0 creates the 128-byte id with
    `Comm.unique_id()` and hands it to every rank over whatever channel the host has (here: a
    `torch.distributed` broadcast; the reference's Monte-Carlo driver would write it into context.json)."""

    def __init__(self, unique_id: bytes, n_ranks: int, rank: int, device: int = -1):
        from . import _lib

        self._L = _lib.lib()
        buf = (C.c_uint8 * _lib.COMM_ID_BYTES).from_buffer_copy(bytes(unique_id))
        h = C.c_void_p()
        _lib.check(self._L.b200_comm_create(buf, int(n_ranks), int(rank), int(device), C.byref(h)))
        self._h = h
        self.n_ranks, self.rank = int(n_ranks), int(rank)

    @staticmethod
    def available() -> bool:
        from . import _lib

        return bool(_lib.lib().b200_comm_available())

    @staticmethod
    def unique_id() -> bytes:
        from . import _lib

        buf = (C.c_uint8 * _lib.COMM_ID_BYTES)()
        _lib.check(_lib.lib().b200_comm_unique_id(buf, _lib.COMM_ID_BYTES))
        return bytes(buf)

    @property
    def last_ms(self) -> float:
        return float(self._L.b200_comm_last_ms(self._h))

    def trajectory_allgather(self, exec_, worlds_per_rank: Sequence[int], out: Optional[np.ndarray] = None,
                             out_ptr: Optional[int] = None):
        """World-sharded all-gather of `exec_`'s device trajectory ring: [sum(worlds), samples, n_entities, width]
        on every rank, in rank order.  `out_ptr` may be a device pointer (e.g. a torch CUDA tensor's data_ptr())."""
        from . import _lib

        wpr = (C.c_uint64 * self.n_ranks)(*[int(w) for w in worlds_per_rank])
        nbytes = int(self._L.b200_sixdof_trajectory_gather_bytes(exec_._h, wpr, self.n_ranks))
        if out_ptr is None:
            if out is None:
                out = np.empty((int(sum(worlds_per_rank)), exec_.trajectory_len(), exec_.n_entities, exec_.trajectory_width()))
            if out.nbytes != nbytes:
                raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH, f"gathered trajectory is {nbytes} bytes, buffer has {out.nbytes}")
            out_ptr = out.ctypes.data
        _lib.check(self._L.b200_sixdof_trajectory_allgather(exec_._h, self._h, wpr, C.c_void_p(out_ptr), nbytes))
        return out

    def step_row_sharded(self, exec_, n_ticks: int) -> None:
        """ONE world, source rows split over the ranks (b200_sixdof_step_row_sharded): every rank holds the whole
        world and integrates rows [rank * N / R, (rank + 1) * N / R); the rows' new position / velocity planes are
        all-gathered over NCCL after every tick."""
        from . import _lib

        _lib.check(self._L.b200_sixdof_step_row_sharded(exec_._h, self._h, int(n_ticks)))

    def peer_attach(self, exec_) -> None:
        """Map every rank's peer window (b200_comm_peer_attach; collective): step_row_sharded then exchanges the rows
        with direct NVLink stores and counter releases instead of a collective per tick.  Raises B200Error
        (ERR_UNSUPPORTED) on every rank when the processes cannot share memory over CUDA IPC."""
        from . import _lib

        _lib.check(self._L.b200_comm_peer_attach(self._h, exec_._h))

    @property
    def peer_attached(self) -> bool:
        return bool(self._L.b200_comm_peer_attached(self._h))

    def peer_detach(self) -> None:
        """Collective: unmap the peers' windows, then free the own one.  Call before closing the attached executor."""
        self._L.b200_comm_peer_detach(self._h)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._L.b200_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RowShardedWorld:
    """bench.py helper for SURVEY §8e's second case ("report both"): one n-body world on N GPUs as replicas vs row
    shards.  Not a product class: the product entry is Comm.step_row_sharded / b200_sixdof_step_row_sharded."""

    @staticmethod
    def _comm(torch, dist, world_size, rank, local):
        uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            uid = torch.tensor(list(Comm.unique_id()), dtype=torch.uint8, device="cuda")
        dist.broadcast(uid, 0)
        return Comm(bytes(uid.cpu().tolist()), world_size, rank, local)

    @staticmethod
    def _timed(torch, el, stream, local, comm, barrier, max_over_ranks, world, grav, warm, ticks, peer, math="fast"):
        """One route of the row-sharded world: `peer` = NVLink stores into the peers' windows, else ncclAllGather per tick."""
        from . import _lib
        from .executor import WORLD_POS

        p, v, I = world
        N = p.shape[1]
        ex = el.B200Exec(N, 1, 3600.0, None, [grav(N)], "rk4", math, device=local)
        ex.set_stream(stream.cuda_stream)
        ex.set_state(p, v, I)
        why = None
        if peer:
            try:
                comm.peer_attach(ex)
            except _lib.B200Error as e:  # every rank gets the same answer (the attach is agreed across ranks)
                why = str(e)[:200]
        if peer and why:
            ex.close()
            return None, None, why
        ev = lambda: torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            comm.step_row_sharded(ex, warm)
            barrier()
            a, b = ev(), ev()
            a.record(stream)
            comm.step_row_sharded(ex, ticks)
            b.record(stream)
            barrier()
        ms = max_over_ranks(a.elapsed_time(b))
        pos = ex.download(WORLD_POS)
        if peer:
            comm.peer_detach()
        ex.close()
        return ms, pos, None

    @staticmethod
    def _both(torch, dist, el, stream, local, rank, world_size, barrier, max_over_ranks, world, grav, ref_pos, warm, ticks):
        comm = RowShardedWorld._comm(torch, dist, world_size, rank, local)
        N = world[0].shape[1]
        scale = float(np.max(np.abs(ref_pos[..., 4:])))
        out = {"ranks": world_size, "rows_per_gpu": N // world_size, "unit": "entity-steps/s"}
        for name, peer in (("nccl", False), ("peer", True)):
            ms, pos, why = RowShardedWorld._timed(torch, el, stream, local, comm, barrier, max_over_ranks, world, grav, warm, ticks, peer)
            if why:
                out[name] = {"unavailable": why}
                continue
            out[name] = {"us_per_tick": ms * 1e3 / ticks, "value": N * ticks / (ms * 1e-3),
                         "max_rel_diff_vs_replica": float(np.max(np.abs(pos[..., 4:] - ref_pos[..., 4:])) / scale)}
        out["nccl"]["exchange"] = "6 planes x N/R f64 per rank, in-place ncclAllGather per plane, one NCCL group per tick (inside libb200_sixdof.so)"
        out["peer"]["exchange"] = ("rows stored straight into every rank's CUDA-IPC window over NVLink + one counter release per peer; "
                                   "the next tick's gravity waits on the counters (no collective in the tick loop)")
        best = min((o for o in (out["nccl"], out["peer"]) if "us_per_tick" in o), key=lambda o: o["us_per_tick"])
        out["us_per_tick"], out["value"] = best["us_per_tick"], best["value"]
        out["max_rel_diff_vs_replica"] = best["max_rel_diff_vs_replica"]
        comm.close()
        return out

    @staticmethod
    def bench(args, torch, dist, el, stream, local, rank, world_size, barrier, max_over_ranks, world, grav, ref_pos):
        """ref_pos: the replica's positions after 420 ticks."""
        return RowShardedWorld._both(torch, dist, el, stream, local, rank, world_size, barrier, max_over_ranks, world, grav, ref_pos, 20, 400)

    @staticmethod
    def bench_large(torch, dist, el, stream, local, rank, world_size, barrier, max_over_ranks, world, grav, ref_pos, warm, ticks):
        return RowShardedWorld._both(torch, dist, el, stream, local, rank, world_size, barrier, max_over_ranks, world, grav, ref_pos, warm, ticks)
