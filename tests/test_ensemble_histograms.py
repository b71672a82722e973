"""Ensemble histograms over the world axis (b200_sixdof_trajectory_histograms / _state_histograms, el.Histogram,
Exec.histogram, merge_histograms, gather_histograms) against numpy, bit for bit: every 1D record is
[nonfinite, below, above] + np.histogram(x[finite], bins, range)[0], every 2D record [nonfinite, outside] +
np.histogram2d(x[m], y[m], bins, range)[0].ravel() with m = both finite, and every record conserves the worlds.

The data catalogue puts values on every edge and one ulp to each side of it, on lo and hi, on signed zeros at a zero
edge, subnormals, NaN, +-inf and +-1e300, and in bins one to two ulps wide at a 1e6 offset, where an index computed
from (x - lo) / w alone disagrees with the edges.  It goes in through set_state, which writes it bit for bit, and is
read through the state entries and through rings of width 13 and 25."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from tests.ensemble_util import (ROCKET, handle, need_gpu, no_device, rocket_world, run_gloo,  # noqa: F401
                                 split, two_body_world)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("exact", "fast")
NAN, INF = float("nan"), float("inf")
K_CHUNK_TASKS, K_MIN_WORLDS = 2 * 132, 256 * 4  # hist_kernels.cu: kChunkTasks, kMinWorlds


def ulps(x, k):
    """x moved k ulps up."""
    for _ in range(k):
        x = np.nextafter(x, INF)
    return float(x)


ORBIT = 1.0e6
NARROW = ulps(ORBIT, 300)  # 300 ulps in 200 bins: bins one or two ulps wide

# (entity, planes, bins, lo, hi): the B200Exec spec form.  Planes of the 25-plane sample layout; all below 13, so the
# same specs run on a ring of width 13.
SPECS = [
    (1, 4, 7, -3.0, 5.0),                                       # edges that are not representable steps
    (0, 5, 4096, -1.0, 1.0),                                    # the most bins, a zero edge in the middle
    (2, 6, 200, ORBIT, NARROW),                                 # bins 1-2 ulps wide at a 1e6 offset
    (1, 4, 1, -2.5, 0.0),                                       # one bin, hi at zero
    (1, (4, 5), (64, 64), (-3.0, -1.0), (5.0, 1.0)),
    (2, (6, 4), (1, 4096), (ORBIT, -3.0), (NARROW, 5.0)),
    (0, 10, 16, -1e300, 1e300),                                 # values on the range edges at 1e300
    (2, (5, 9), (3, 5), (-1.0, -0.5), (1.0, 0.75)),
]


def axes(spec):
    """[(plane, bins, lo, hi)] of a spec."""
    entity, planes, bins, lo, hi = spec
    return list(zip(*(np.atleast_1d(v).tolist() for v in (planes, bins, lo, hi))))


def record_len(spec):
    a = axes(spec)
    return 3 + a[0][1] if len(a) == 1 else 2 + a[0][1] * a[1][1]


def ref_record(x, spec):
    """x [worlds, entities, W] -> the spec's record, from numpy."""
    e = spec[0]
    a = axes(spec)
    if len(a) == 1:
        (p, n, lo, hi), = a
        v = x[:, e, p]
        f = np.isfinite(v)
        c = np.histogram(v[f], bins=n, range=(lo, hi))[0]
        return np.concatenate([[np.sum(~f), np.sum(v[f] < lo), np.sum(v[f] > hi)], c]).astype(np.float64)
    (pa, na, la, ha), (pb, nb, lb, hb) = a
    u, v = x[:, e, pa], x[:, e, pb]
    m = np.isfinite(u) & np.isfinite(v)
    inside = m & (u >= la) & (u <= ha) & (v >= lb) & (v <= hb)
    c = np.histogram2d(u[m], v[m], bins=(na, nb), range=((la, ha), (lb, hb)))[0]
    return np.concatenate([[np.sum(~m), np.sum(m & ~inside)], c.ravel()]).astype(np.float64)


def ref_row(x, specs):
    return np.concatenate([ref_record(x, s) for s in specs])


def check_conservation(row, specs, n_worlds):
    off = 0
    for s in specs:
        r = row[..., off:off + record_len(s)]
        assert np.all(r.sum(-1) == n_worlds), s
        off += record_len(s)
    assert off == row.shape[-1]


def axis_catalogue(lo, hi, n, rng):
    e = np.linspace(lo, hi, n + 1)
    w = hi - lo
    special = [lo, hi, -0.0, 0.0, 5e-324, -5e-324, 2.2250738585072014e-308, -1e-310, NAN, INF, -INF, 1e300, -1e300,
               np.nextafter(lo, -INF), np.nextafter(hi, INF), ulps(lo, 1), np.nextafter(hi, -INF)]
    return np.concatenate([special, e, np.nextafter(e, -INF), np.nextafter(e, INF),
                           rng.uniform(lo - 0.1 * w, hi + 0.1 * w, 2000)])


def catalogue(specs, M, E, seed=0):
    """x [M, E, 25]: every plane a spec reads holds, in random world order and for every entity, the catalogue of every
    axis on it (padded with draws from it, or cut to M worlds: 21 000 hold all of SPECS'); the other planes are normal
    draws with a few NaN."""
    rng = np.random.default_rng(seed)
    per_plane = {}
    for s in specs:
        for p, n, lo, hi in axes(s):
            per_plane.setdefault(p, []).append(axis_catalogue(lo, hi, n, rng))
    x = rng.normal(size=(M, E, 25))
    x[rng.random((M, E, 25)) < 0.01] = NAN
    for p, vals in per_plane.items():
        v = np.concatenate(vals)
        for e in range(E):
            col = v if len(v) >= M else np.concatenate([v, rng.choice(v, M - len(v))])
            x[:, e, p] = rng.permutation(col)[:M]
    return x


def state_handle(x, mode, **kw):
    M, E, _ = x.shape
    ine = np.broadcast_to(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 7))
    ex = el.B200Exec(E, M, 0.01, None, [], "rk4", mode, **kw)
    ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
    return ex


def launches_of(ex, call):
    n0 = ex.timings()["kernel_launches"]
    got = call()
    return got, ex.timings()["kernel_launches"] - n0


def hist_chunks(n_worlds, n_groups):
    """hist_kernels.cu hist_chunks, restated: (worlds per chunk, chunks)."""
    want = max(1, -(-K_CHUNK_TASKS // max(n_groups, 1)))
    C = max(1, min(want, n_worlds // K_MIN_WORLDS))
    Wc = -(-n_worlds // C)
    return Wc, -(-n_worlds // Wc)


# --------------------------------------------------------------------------- CPU: el.Histogram and World.build


def test_histogram_spec_and_edges():
    h = el.Histogram("rocket.world_pos", 4, range=(-500.0, 500.0), bins=100)
    assert h.planes == (4,) and h.bins == (100,) and h.record_len == 103 and h.entity == "rocket"
    assert h.edges.tobytes() == np.linspace(-500.0, 500.0, 101).tobytes()
    h2 = el.Histogram("rocket.world_vel", (3, 4), range=((-500, 500), (-200, 200)), bins=(64, 32))
    assert h2.planes == (10, 11) and h2.record_len == 2 + 64 * 32
    ea, eb = h2.edges
    assert ea.tobytes() == np.linspace(-500.0, 500.0, 65).tobytes() and eb.tobytes() == np.linspace(-200.0, 200.0, 33).tobytes()
    assert el.Histogram("b.force", (0, 5), range=((0, 1), (0, 1)), bins=8).bins == (8, 8)  # an int is every axis's
    assert h2._spec(3) == (3, (10, 11), (64, 32), (-500.0, -200.0), (500.0, 200.0))


@pytest.mark.parametrize("lo, k, n", [(6.4e6, 2, 2), (6.4e6, 300, 200), (-6.4e6, 5, 4), (ORBIT, 4096, 4096),
                                      (4.2e7, 7, 3), (-1.0, 1, 1), (1e-300, 9, 8), (-3e5, 4097, 4096)])
def test_edges_equal_linspace_near_degenerate(lo, k, n):
    """Ranges a few ulps wide at orbital offsets that still have strictly increasing edges: accepted, with numpy's edges
    bit for bit (the same edges the library computes and counts with)."""
    hi = ulps(lo, k)
    e = np.linspace(lo, hi, n + 1)
    assert np.all(e[:-1] < e[1:])
    h = el.Histogram("r.world_pos", 6, range=(lo, hi), bins=n)
    assert h.edges.tobytes() == e.tobytes()
    assert h.edges[0] == lo and h.edges[-1] == hi


@pytest.mark.parametrize("args, kw", [
    (("r.world_pos", 7), {"range": (0.0, 1.0)}),                      # index out of the component
    (("r.world_pos", 1.0), {"range": (0.0, 1.0)}),
    (("r.world_pos", True), {"range": (0.0, 1.0)}),
    (("r.world_pos", (1, 2, 3)), {"range": ((0, 1),) * 3}),            # 3 axes
    (("r.world_pos", (4, 4)), {"range": ((0, 1), (0, 1))}),           # one plane twice
    (("r.world_pos", 4), {"range": (0.0, 1.0), "bins": 0}),
    (("r.world_pos", 4), {"range": (0.0, 1.0), "bins": -3}),
    (("r.world_pos", 4), {"range": (0.0, 1.0), "bins": 4097}),        # more than 4096 cells
    (("r.world_pos", (4, 5)), {"range": ((0, 1), (0, 1)), "bins": (65, 64)}),
    (("r.world_pos", (4, 5)), {"range": ((0, 1), (0, 1)), "bins": (4, 5, 6)}),
    (("r.world_pos", 4), {"range": (0.0, 1.0), "bins": 2.0}),
    (("r.world_pos", 4), {"range": (1.0, 1.0)}),                      # lo >= hi
    (("r.world_pos", 4), {"range": (2.0, 1.0)}),
    (("r.world_pos", 4), {"range": (NAN, 1.0)}),
    (("r.world_pos", 4), {"range": (0.0, INF)}),
    (("r.world_pos", 4), {"range": (-1.7e308, 1.7e308)}),             # hi - lo overflows
    (("r.world_pos", 4), {"range": (0.0, 5e-324), "bins": 4}),        # step = 0
    (("r.world_pos", 4), {"range": (ORBIT, ulps(ORBIT, 3)), "bins": 4}),  # edges not strictly increasing
    (("r.world_pos", 4), {"range": (6.4e6, ulps(6.4e6, 1)), "bins": 2}),
    (("r.world_pos", 4), {"range": (0.0, 1.0, 2.0)}),
    (("r.world_pos", (4, 5)), {"range": (0.0, 1.0)}),                 # a 2D spec needs a range per axis
    (("r.world_pos", 4), {"range": ("0", 1.0)}),
])
def test_histogram_refusals(args, kw):
    with pytest.raises(ValueError):
        el.Histogram(*args, **kw)


def test_histogram_refuses_unsampled_components():
    for pair in ("r.inertia", "world_pos", "r.thrust"):
        with pytest.raises(_lib.B200ValueError, match="component not found"):
            el.Histogram(pair, 0, range=(0.0, 1.0))


def test_build_validates_histograms_before_the_device(no_device):
    w, sys_ = two_body_world(), el.six_dof()
    ok = el.Histogram("rocket.world_pos", 6, range=(0.0, 2.0), bins=4)
    for bad in ([ok], [], ["x"]):                                      # the mode is checked before the specs
        with pytest.raises(_lib.B200Error, match="ensemble=True") as e:
            w.build(sys_, histograms=bad)
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    with pytest.raises(ValueError, match="1 to 8"):
        w.build(sys_, ensemble=True, histograms=[])
    with pytest.raises(ValueError, match="1 to 8"):
        w.build(sys_, ensemble=True, histograms=[ok] * 9)
    for bad in ("rocket.world_pos", [("rocket.world_pos", 6)], [ok, None]):
        with pytest.raises(TypeError):
            w.build(sys_, ensemble=True, histograms=bad)
    for pair in ("nobody.world_pos", "Globals.world_pos"):
        with pytest.raises(_lib.B200ValueError, match="component not found"):
            w.build(sys_, ensemble=True, histograms=[ok, el.Histogram(pair, 0, range=(0.0, 1.0))])


# --------------------------------------------------------------------------- CPU: merge, gather, layout


def test_merge_histograms_sums_exactly():
    rng = np.random.default_rng(5)
    x = catalogue(SPECS[:2], 20_000, 3, seed=1)
    parts = split(rng, 20_000, 4)
    tables = [ref_row(x[idx], SPECS[:2]) for idx in parts]
    got = el.merge_histograms(tables)
    assert got.tobytes() == ref_row(x, SPECS[:2]).tobytes()
    check_conservation(got, SPECS[:2], 20_000)
    two = el.merge_histograms([np.stack([t, t]) for t in tables])     # any leading shape, e.g. [rows, record]
    assert two.shape == (2, got.size) and two[1].tobytes() == got.tobytes()


def test_merge_histograms_refusals():
    with pytest.raises(_lib.B200ValueError):
        el.merge_histograms([np.zeros((3, 7)), np.zeros((4, 7))])     # shapes differ
    with pytest.raises(_lib.B200ValueError):
        el.merge_histograms([])
    with pytest.raises(_lib.B200ValueError):
        el.merge_histograms([np.zeros(2)])                            # shorter than any record
    with pytest.raises(_lib.B200ValueError):
        el.merge_histograms([np.float64(3.0)])
    for bad in (-1.0, 0.5, NAN, INF):
        t = np.zeros(7)
        t[3] = bad
        with pytest.raises(_lib.B200Error, match="not a count|2\\^53") as e:
            el.merge_histograms([np.zeros(7), t])
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    big = np.zeros(4)
    big[3] = 2.0 ** 52 + 1
    with pytest.raises(_lib.B200Error, match="2\\^53"):
        el.merge_histograms([big, big])
    assert el.merge_histograms([np.zeros(3)]).shape == (3,)


def _rank_table(rank):
    x = catalogue(SPECS[4:6], 3000 + 17 * rank, 3, seed=20 + rank)
    return ref_row(x, SPECS[4:6])


def _gather_worker(rank, ws):
    from elodin_b200.sharding import gather_histograms

    return gather_histograms(_rank_table(rank))


def test_gather_histograms_two_gloo_ranks():
    got = run_gloo(_gather_worker, 2)
    want = _rank_table(0) + _rank_table(1)
    assert got[0].tobytes() == want.tobytes() and got[1].tobytes() == want.tobytes()
    check_conservation(got[0], SPECS[4:6], 3000 + 3017)


def test_histogram_struct_layout_matches_header(tmp_path):
    st = _lib.Histogram
    assert ctypes.sizeof(st) == 64
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200_sixdof.h"', 'int main(void) {',
           'printf("size %zu\\n", sizeof(b200_histogram));',
           'printf("max %u %u\\n", B200_MAX_HISTOGRAMS, B200_MAX_HISTOGRAM_CELLS);']
    for fname, _ in st._fields_:
        src.append(f'printf("{fname} %zu\\n", offsetof(b200_histogram, {fname}));')
    src += ["return 0; }"]
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", str(c), "-I", os.path.join(ROOT, "include"), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    got = {line.split()[0]: line.split()[1:] for line in out}
    assert int(got["size"][0]) == ctypes.sizeof(st)
    assert [int(v) for v in got["max"]] == [_lib.MAX_HISTOGRAMS, _lib.MAX_HISTOGRAM_CELLS]
    for fname, _ in st._fields_:
        assert int(got[fname][0]) == getattr(st, fname).offset, fname


def test_hist_chunks_restatement_boundaries():
    """The shapes the GPU sweep runs are the boundaries of the restated chunking."""
    assert hist_chunks(1, 1) == (1, 1) and hist_chunks(K_MIN_WORLDS - 1, 1) == (K_MIN_WORLDS - 1, 1)
    assert hist_chunks(2 * K_MIN_WORLDS, 1) == (K_MIN_WORLDS, 2)
    assert hist_chunks(K_CHUNK_TASKS * K_MIN_WORLDS, 1) == (K_MIN_WORLDS, K_CHUNK_TASKS)
    Wc, C = hist_chunks(K_CHUNK_TASKS * K_MIN_WORLDS + 1, 1)
    assert C == K_CHUNK_TASKS and Wc == K_MIN_WORLDS + 1           # a short last chunk
    assert hist_chunks(1 << 20, 8)[1] == K_CHUNK_TASKS // 8


# --------------------------------------------------------------------------- GPU: against numpy


@pytest.mark.gpu
def test_catalogue_state_entries_match_numpy():
    need_gpu()
    x = catalogue(SPECS, 21_000, 3)
    want = ref_row(x, SPECS)
    check_conservation(want, SPECS, 21_000)
    got = {}
    for mode in MODES:
        with state_handle(x, mode) as ex:
            got[mode], n = launches_of(ex, lambda: ex.state_histograms(SPECS))
            assert n == 1
            for k, s in enumerate(SPECS):                              # one spec alone: its record of the 8-spec call
                off = sum(record_len(t) for t in SPECS[:k])
                assert ex.state_histograms([s]).tobytes() == got[mode][off:off + record_len(s)].tobytes(), s
    for mode in MODES:
        assert got[mode].tobytes() == want.tobytes(), mode
    check_conservation(got["exact"], SPECS, 21_000)


@pytest.mark.gpu
@pytest.mark.parametrize("width", (13, 25))
@pytest.mark.parametrize("mode", MODES)
def test_catalogue_ring_matches_numpy(width, mode):
    need_gpu()
    M, E = 21_000, 3
    x = catalogue(SPECS, M, E, seed=3)
    x[..., 7:13] = 0.0                                                 # at rest: the catalogue stays in world_pos
    with state_handle(x, mode, trajectory_every=1, trajectory_capacity=3, trajectory_full=width == 25) as ex:
        ex.step(3)
        traj = ex.trajectory()                                         # [3, M, E, width]
        got, n = launches_of(ex, lambda: ex.trajectory_histograms(SPECS))
        assert n == 1 and got.shape == (3, sum(record_len(s) for s in SPECS))
        for k in range(3):
            assert got[k].tobytes() == ref_row(traj[k], SPECS).tobytes(), k
        check_conservation(got, SPECS, M)
        wide = [(0, 13, 4, -1.0, 1.0)]
        if width == 13:
            with pytest.raises(_lib.B200Error) as e:
                ex.trajectory_histograms(wide)
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        else:
            assert ex.trajectory_histograms(wide)[1].tobytes() == ref_row(traj[1], wide).tobytes()
        assert ex.trajectory_histograms(SPECS).tobytes() == got.tobytes()    # the same call twice: the same bytes


def shape_specs(E):
    """8 specs mixing 1D and 2D on the first, a middle and the last entity."""
    first, mid, last = 0, E // 2, E - 1
    return [(first, 4, 64, -2.0, 2.0), (mid, (4, 5), (64, 64), (-2.0, -2.0), (2.0, 2.0)), (last, 6, 4096, -3.0, 3.0),
            (last, (5, 6), (1, 4096), (-1.0, -3.0), (1.0, 3.0)), (mid, 12, 1, -1.0, 1.0), (first, 24, 33, -0.5, 0.5),
            (mid, (7, 19), (8, 3), (-1.0, -1.0), (1.0, 1.0)), (first, 5, 100, 0.0, 0.1)]


def shape_data(M, E, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(M, E, 25))
    x[rng.random(x.shape) < 0.02] = NAN
    x[rng.random(x.shape) < 0.01] = -INF
    if M > 40:
        x[: M // 3, :, 4] = 0.25                                        # a third of the worlds in one bin
    return x


SHAPES = [(1, 1), (31, 1), (32, 1), (33, 1), (K_MIN_WORLDS - 1, 1), (K_MIN_WORLDS, 1), (K_MIN_WORLDS + 1, 1),
          (2 * K_MIN_WORLDS - 1, 1), (2 * K_MIN_WORLDS, 1), (K_CHUNK_TASKS * K_MIN_WORLDS - 1, 1),
          (K_CHUNK_TASKS * K_MIN_WORLDS + 1, 1), ((1 << 20) + 5, 1), (33, 3), (K_MIN_WORLDS + 1, 3), (5000, 3),
          (1024, 1024), (3, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("M, E", SHAPES)
def test_launch_shapes_match_numpy(M, E):
    need_gpu()
    x = shape_data(M, E, seed=M + E)
    specs = shape_specs(E)
    want = ref_row(x, specs)
    for mode in MODES:
        with state_handle(x, mode) as ex:
            got, n = launches_of(ex, lambda: ex.state_histograms(specs))
            assert n == 1
            assert got.tobytes() == want.tobytes(), mode
            assert ex.state_histograms(specs[:1]).tobytes() == want[:record_len(specs[0])].tobytes()
    check_conservation(want, specs, M)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_ring_of_16_equals_ring_of_1(mode):
    """A sample has the same bits whatever else the ring holds."""
    need_gpu()
    M, N = 3000, 2
    specs = [(0, 6, 50, 0.0, 2.0), (1, (4, 5), (16, 16), (-1.0, -1.0), (1.0, 1.0)), (0, 10, 8, -10.0, 10.0)]
    big, st = handle(ROCKET, M, N, mode, capacity=16, seed=9)
    one, _ = handle(ROCKET, M, N, mode, capacity=1, state=st)
    with big, one:
        big.step(16)
        all16 = big.trajectory_histograms(specs)
        traj = big.trajectory()
        for k in range(16):
            one.trajectory_reset()
            one.step(1)
            row = one.trajectory_histograms(specs)[0]
            assert row.tobytes() == ref_row(one.trajectory()[0], specs).tobytes(), k
            assert all16[k].tobytes() == ref_row(traj[k], specs).tobytes(), k
            if one.trajectory()[0].tobytes() == traj[k].tobytes():     # the same sample: the same bits
                assert row.tobytes() == all16[k].tobytes(), k


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_split_handles_sum_to_one(seed):
    need_gpu()
    rng = np.random.default_rng(seed)
    M, E = 40_000, 2
    x = shape_data(M, E, seed=100 + seed)
    specs = shape_specs(E)[:5]
    want = ref_row(x, specs)
    k = int(rng.integers(2, 5))
    parts = [idx for idx in split(rng, M, k) if len(idx)]
    tables = []
    for idx in parts:
        with state_handle(x[idx], "fast") as ex:
            tables.append(ex.state_histograms(specs))
    assert el.merge_histograms(tables).tobytes() == want.tobytes()
    with state_handle(x, "exact") as ex:
        assert ex.state_histograms(specs).tobytes() == want.tobytes()


@pytest.mark.gpu
def test_refusals_and_plumbing():
    need_gpu()
    import torch

    L = _lib.lib()
    M, N = 700, 3
    ex, _ = handle(ROCKET, M, N, "exact", capacity=4)
    with ex:
        ex.step(2)
        good = ex.trajectory_histograms(SPECS[:3])
        args, row = ex._hist_specs(SPECS[:3])
        assert good.shape == (2, row)
        buf = np.empty(good.size + 1)
        for wrong in (good.nbytes - 8, good.nbytes + 8, 0):
            assert L.b200_sixdof_trajectory_histograms(ex._h, *args, buf.ctypes.data, wrong) == _lib.ERR_VALUE_SIZE_MISMATCH
        assert L.b200_sixdof_trajectory_histograms(None, *args, buf.ctypes.data, good.nbytes) == _lib.ERR_INVALID_ARGUMENT
        bad = [
            [],                                                         # zero specs
            [SPECS[0]] * 9,                                             # more than 8
            [(3, 4, 8, 0.0, 1.0)],                                      # entity >= n_entities
            [(0, 25, 8, 0.0, 1.0)],                                     # plane >= 25
            [(0, (4, 4), (8, 8), (0.0, 0.0), (1.0, 1.0))],              # one plane twice
            [(0, 4, 0, 0.0, 1.0)],
            [(0, 4, 4097, 0.0, 1.0)],
            [(0, (4, 5), (64, 65), (0.0, 0.0), (1.0, 1.0))],
            [(0, 4, 8, 1.0, 1.0)], [(0, 4, 8, 1.0, 0.0)], [(0, 4, 8, NAN, 1.0)], [(0, 4, 8, 0.0, INF)],
            [(0, 4, 8, -1.7e308, 1.7e308)], [(0, 4, 4, 0.0, 5e-324)], [(0, 4, 4, ORBIT, ulps(ORBIT, 3))],
            [(0, (4, 5, 6), (2, 2, 2), (0.0,) * 3, (1.0,) * 3)],         # 3 axes
        ]
        for specs in bad:                                               # the specs are checked before `bytes`
            a, _ = ex._hist_specs(specs)
            for fn in (L.b200_sixdof_trajectory_histograms, L.b200_sixdof_state_histograms):
                assert fn(ex._h, *a, buf.ctypes.data, 0) == _lib.ERR_INVALID_ARGUMENT, specs
        a, _ = ex._hist_specs(SPECS[:1])
        a[0][0].reserved = 1
        assert L.b200_sixdof_state_histograms(ex._h, *a, buf.ctypes.data, 0) == _lib.ERR_INVALID_ARGUMENT
        assert L.b200_sixdof_state_histograms(ex._h, None, 1, buf.ctypes.data, 0) == _lib.ERR_INVALID_ARGUMENT
        assert L.b200_sixdof_status(ex._h) == 0
        assert ex.trajectory_histograms(SPECS[:3]).tobytes() == good.tobytes()
        dev = torch.empty(good.shape, dtype=torch.float64, device="cuda")    # a device destination
        ex.trajectory_histograms(SPECS[:3], out_ptr=dev.data_ptr())
        assert dev.cpu().numpy().tobytes() == good.tobytes()
        ex.trajectory_reset()                                           # an empty ring: bytes = 0, no launch
        got, n = launches_of(ex, lambda: ex.trajectory_histograms(SPECS[:3]))
        assert got.shape == (0, row) and n == 0
    thin = el.B200Exec(N, M, 0.01, None, [], "rk4", "exact")              # no ring: every plane refused
    with thin:
        a, _ = thin._hist_specs([(0, 0, 4, 0.0, 1.0)])
        assert L.b200_sixdof_trajectory_histograms(thin._h, *a, buf.ctypes.data, 0) == _lib.ERR_INVALID_ARGUMENT


# --------------------------------------------------------------------------- GPU: Exec end to end

HISTS = lambda: [el.Histogram("rocket.world_pos", 6, range=(0.0, 3.0), bins=30),
                 el.Histogram("rocket.world_pos", (4, 5), range=((-4.0, 4.0), (-1.0, 1.0)), bins=(16, 8)),
                 el.Histogram("rocket.world_vel", 3, range=(-20.0, 20.0), bins=40),
                 el.Histogram("ball.world_vel", (3, 4), range=((0.0, 2.0), (1.0, 3.0)), bins=4)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_exec_routes_match_default_mode(mode):
    need_gpu()
    M, ticks = 2500, 47
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=12.0, math=mode, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ref.run(ticks)
    with pytest.raises(_lib.B200Error, match="histograms="):            # refused outside ensemble mode
        ref.histogram(0)
    hist = {p: ref.history_worlds(p) for p in ("rocket.world_pos", "rocket.world_vel", "ball.world_vel")}
    runs = {}
    for route, extra, run_kw in (("resident", {}, {}), ("ring1", {"ensemble_ring": 1}, {}),
                                 ("ring3", {"ensemble_ring": 3}, {}),
                                 ("callback", {}, {"post_step": lambda tick, ctx: None})):
        ex = w.build(sys_, ensemble=True, histograms=HISTS(), **extra, **kw)
        ex.run(ticks, **run_kw)
        runs[route] = [ex.histogram(i) for i in range(4)]
        with pytest.raises(IndexError):
            ex.histogram(4)
        ex.backend.close()
    rows = hist["rocket.world_pos"].shape[0]
    assert rows == 1 + ticks // 10 + (ticks % 10 > 0)
    for i, h in enumerate(HISTS()):
        x = hist[h.pair]                                               # [rows, M, width]
        for route, got in runs.items():
            g = got[i]
            assert g["counts"].dtype == np.int64 and g["counts"].shape[0] == rows
            for r in range(rows):
                if len(h.bins) == 1:
                    v = x[r, :, h.index]
                    f = np.isfinite(v)
                    want = np.histogram(v[f], bins=h.bins[0], range=h.range[0])[0]
                    assert np.array_equal(g["counts"][r], want), (route, i, r)
                    assert g["below"][r] == np.sum(v[f] < h.range[0][0]) and g["above"][r] == np.sum(v[f] > h.range[0][1])
                    total = g["below"][r] + g["above"][r]
                else:
                    u, v = x[r, :, h.index[0]], x[r, :, h.index[1]]
                    m = np.isfinite(u) & np.isfinite(v)
                    want = np.histogram2d(u[m], v[m], bins=h.bins, range=h.range)[0]
                    assert np.array_equal(g["counts"][r], want), (route, i, r)
                    total = g["outside"][r]
                assert g["nonfinite"][r] + total + g["counts"][r].sum() == M
            e = g["edges"]
            assert all(a.tobytes() == b.tobytes() for a, b in zip(e if isinstance(e, tuple) else (e,),
                                                                  h.edges if isinstance(h.edges, tuple) else (h.edges,)))
        for route in runs:
            assert all(np.array_equal(runs[route][i][k], runs["resident"][i][k]) for k in runs[route][i] if k != "edges")
    ref.backend.close()
