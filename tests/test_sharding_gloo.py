"""The N>1 host logic on CPU: 2 ranks over gloo (127.0.0.1), no GPU needed."""

import numpy as np
import pytest
import torch

from elodin_b200.sharding import gather_worlds, shard_sizes, shard_worlds, total_entity_steps
from tests.ensemble_util import run_gloo


def test_shard_ranges_cover_exactly():
    for n in (0, 1, 7, 8, 9, 100000, 100003):
        for ws in (1, 2, 3, 8):
            spans = [shard_worlds(n, r, ws) for r in range(ws)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = shard_sizes(n, ws)
            assert max(sizes) - min(sizes) <= 1 and sum(sizes) == n
    with pytest.raises(ValueError):
        shard_worlds(10, 2, 2)


def _worker(rank, ws, n_worlds):
    w0, w1 = shard_worlds(n_worlds, rank, ws)
    # each rank "integrates" its own worlds: the global world id is recoverable from the data
    local = torch.arange(w0, w1, dtype=torch.float64).reshape(-1, 1, 1).repeat(1, 2, 13)
    full = gather_worlds(local, n_worlds)
    steps = total_entity_steps((w1 - w0) * 2 * 10)
    return full.numpy(), steps


@pytest.mark.parametrize("n_worlds", [11, 12])  # ragged (6 + 5) and equal shards (flat all-gather path)
def test_two_rank_gather_and_counters(n_worlds):
    ws = 2
    got = run_gloo(_worker, ws, n_worlds)
    want = np.arange(n_worlds, dtype=np.float64).reshape(-1, 1, 1).repeat(2, 1).repeat(13, 2)
    for rank, (full, steps) in enumerate(got):
        assert full.shape == (n_worlds, 2, 13)
        assert np.array_equal(full, want), rank  # global world order, no holes, no duplicates
        assert steps == n_worlds * 2 * 10
