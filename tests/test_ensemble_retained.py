"""Retained worlds in ensemble mode: the full rows of chosen worlds, gathered on the device
(b200_sixdof_{trajectory,state}_download_worlds, gather_worlds_kernel) and recorded by World.build(..., ensemble=True,
retain=[...]).  The GPU tests hold every retained row to the full download and to a default-mode Exec of the same build,
bit for bit, and every ensemble table to the same build without `retain`; the CPU tests check the option's validation,
the refusals and the campaign helpers with a call-recording fake backend."""

import ctypes
import os

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200 import db_sink as D
from elodin_b200 import monte_carlo as mc
from elodin_b200.executor import FORCE, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from elodin_b200.export import export_csv
from elodin_b200.sharding import shard_retained, shard_worlds
from tests.ensemble_util import FREE, ROCKET, SAMPLED, handle, need_gpu, rocket_world
from tests.test_host_logic import _FakeBackend, _two_body_world

PAIRS = [f"{e}.{c}" for e in ("rocket", "ball") for c in SAMPLED]
PASS_THROUGH = ("rocket.inertia", "ball.inertia", "rocket.thrust", "rocket.wind")


def _files(root):
    """relative path -> content; AppendLogs (sparse files of the reference's fixed map size) by header + committed bytes"""
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(d, f)
            out[os.path.relpath(p, root)] = D._read_log(p) if f in ("index", "data") else open(p, "rb").read()
    return out


# ---------------------------------------------------------------------------------------------------------------- CPU


class _EnsembleFake(_FakeBackend):
    """_FakeBackend with what ensemble mode calls: all-zero tables and the rows of chosen worlds of its own state."""

    created = 0

    def __init__(self, *a, **kw):
        _EnsembleFake.created += 1
        super().__init__(*a, **kw)

    def _state25(self):
        z = np.zeros(self.state[el.component_id("world_pos")].shape[:-1] + (6,))
        return np.concatenate([self.state[el.component_id("world_pos")], self.state[el.component_id("world_vel")],
                               self.state.get(el.component_id("world_accel"), z), self.state.get(el.component_id("force"), z)], -1)

    def state_stats(self):
        return np.zeros((self.n_entities, 25, 5))

    def trajectory_stats(self):
        return np.zeros((len(self.samples), self.n_entities, 25, 5))

    def state_worlds(self, worlds):
        return self._state25()[list(worlds)]

    def trajectory_worlds(self, worlds):
        return np.stack(self.samples)[:, list(worlds)]

    def download(self, cid, out):
        out[...] = self.state[cid]

    def invoke_batch_ptrs(self, in_ptrs, out_ptrs, n):
        """The invoke_batch route on the fake: the inputs read from the host buffers, n ticks, the outputs written."""
        _FakeBackend.calls.append(("invoke", n))

        def view(ptr, cid):
            nb = self.column_bytes(cid)
            a = np.frombuffer((ctypes.c_char * nb).from_address(ptr), np.uint64 if cid == el.component_id("tick") else np.float64)
            return a if nb == 8 else a.reshape(self.n_worlds, self.n_entities, -1)

        for cid, p in zip(self.input_ids, in_ptrs):
            if p:
                self.state[cid] = view(p, cid).copy()
        self.step(n)
        for cid, p in zip(self.output_ids, out_ptrs):
            if p:
                view(p, cid)[...] = self.state[cid]


@pytest.fixture
def fake(monkeypatch):
    from elodin_b200 import world as W

    monkeypatch.setattr(W, "B200Exec", _EnsembleFake)
    _EnsembleFake.created = 0
    return _EnsembleFake


@pytest.mark.parametrize("retain, exc, match", [
    ("0", TypeError, "sequence"), (3, TypeError, "sequence"), ([0, 1.0], TypeError, "1.0"), ([True], TypeError, "True"),
    ([np.bool_(False)], TypeError, "False"), ([0, 4], ValueError, r"\[0, 4\)"), ([-1], ValueError, "-1"),
    ([], ValueError, "at least one"), ([2, 0, 2], ValueError, "2 is listed twice"),
])
def test_retain_is_validated_before_any_handle(fake, retain, exc, match):
    with pytest.raises(exc, match=match):
        _two_body_world().build(el.six_dof(), n_worlds=4, ensemble=True, retain=retain)
    assert fake.created == 0


def test_retain_needs_ensemble_and_bounds_the_bodies(fake):
    with pytest.raises(_lib.B200Error, match="ensemble=True") as e:
        _two_body_world().build(el.six_dof(), n_worlds=4, retain=[0])
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    assert _lib.MAX_RETAINED_BODIES == 65536
    n = _lib.MAX_RETAINED_BODIES // 2 + 1                                      # two entities per world
    with pytest.raises(ValueError, match="65538 bodies"):
        _two_body_world().build(el.six_dof(), n_worlds=n, ensemble=True, retain=np.arange(n))
    assert fake.created == 0
    ex = _two_body_world().build(el.six_dof(), n_worlds=n, ensemble=True, retain=np.arange(n - 1)[::-1])
    assert ex.retained == tuple(range(n - 2, -1, -1)) and all(type(w) is int for w in ex.retained[:3])
    ex = _two_body_world().build(el.six_dof(), n_worlds=4, ensemble=True, retain=[np.int64(3), 1])
    assert ex.retained == (3, 1)
    assert _two_body_world().build(el.six_dof(), n_worlds=4, ensemble=True).retained is None


def test_retained_rows_follow_the_default_mode_bookkeeping(fake):
    """On the fake, the retained rows are the default mode's rows of those worlds, in `retain` order."""
    kw = dict(simulation_rate=120.0, telemetry_rate=40.0, n_worlds=5,
              world_params={"world_vel": np.arange(5 * 2 * 6, dtype=float).reshape(5, 2, 6)})
    ref = _two_body_world().build(el.six_dof(), **kw)
    ref._ring_cap = ref.backend.cap = 4
    ref.run(30)                                                   # 10 whole cycles in ring-fulls of 4, 4, 2
    ex = _two_body_world().build(el.six_dof(), ensemble=True, ensemble_ring=4, retain=[4, 0, 2], **kw)
    ex.run(30)
    assert ex.tick == ref.tick == 30
    for pair in ("a.world_pos", "b.world_vel", "a.world_accel", "b.force", "a.inertia"):
        got, want = ex.history_worlds(pair), ref.history_worlds(pair)[:, [4, 0, 2]]
        assert got.shape == want.shape == (11, 3, got.shape[-1])
        assert np.array_equal(got, want), pair
    assert ex._globals_hist == ref._globals_hist
    h = ex.history(["a.world_pos", "globals.tick"])
    assert np.array_equal(h["a.world_pos"], ref.history("a.world_pos")["a.world_pos"])
    assert list(h["globals.tick"]) == list(ref.history("globals.tick")["globals.tick"])


def test_unretained_worlds_are_refused(fake, tmp_path):
    ex = _two_body_world().build(el.six_dof(), n_worlds=4, ensemble=True, retain=[3, 1])
    ex.run(3)
    assert ex.history_worlds("a.world_pos").shape == (4, 2, 7)
    with pytest.raises(_lib.B200Error, match=r"retain=\[3, 1\]"):
        ex.history("a.world_pos")
    for call in (lambda: ex.write_db(str(tmp_path / "db"), world=0), lambda: ex.attach_db(str(tmp_path / "db"), world=2),
                 lambda: export_csv(ex, str(tmp_path / "csv"), world=0)):
        with pytest.raises(_lib.B200Error, match=r"retain=\[3, 1\]") as e:
            call()
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    assert not os.path.exists(tmp_path / "db") and not os.path.exists(tmp_path / "csv")
    ex.write_db(str(tmp_path / "w1"), world=1)
    export_csv(ex, str(tmp_path / "c3"), world=3)
    # without retain every per-world accessor refuses as before, the sinks included
    plain = _two_body_world().build(el.six_dof(), n_worlds=4, ensemble=True)
    for call in (lambda: plain.history("a.world_pos"), lambda: plain.history_worlds("a.world_pos"),
                 lambda: plain.write_db(str(tmp_path / "p")), lambda: plain.attach_db(str(tmp_path / "p")),
                 lambda: export_csv(plain, str(tmp_path / "p")),
                 lambda: mc.write_run_databases(plain, [{}] * 4, str(tmp_path / "p"), keep=[0])):
        with pytest.raises(_lib.B200Error, match="ensemble"):
            call()
    assert not os.path.exists(tmp_path / "p")


def test_write_run_databases_keeps_the_retained_runs(fake, tmp_path):
    ex = _two_body_world().build(el.six_dof(), n_worlds=4, ensemble=True, retain=[3, 1])
    ex.run(2)
    rows = [{"run_id": f"run_{k}"} for k in range(4)]
    with pytest.raises(ValueError, match=r"\[2\] are not retained"):
        mc.write_run_databases(ex, rows, str(tmp_path / "c"), keep=[1, 2])
    assert not os.path.exists(tmp_path / "c")
    paths = mc.write_run_databases(ex, rows, str(tmp_path / "c"))
    assert [os.path.relpath(p, tmp_path) for p in paths] == ["c/runs/run_3/db", "c/runs/run_1/db"]
    assert sorted(os.listdir(tmp_path / "c" / "runs")) == ["run_1", "run_3"]


def test_host_systems_writes_to_sampled_components_are_in_the_retained_rows(fake):
    """The host-callback route: a host system after six_dof() halves world_vel; the retained rows hold the halved
    values, as the default mode's rows do (they are taken after the callbacks, not from the ring)."""
    def damp(ctx):
        ctx.column("world_vel")[...] *= 0.5

    kw = dict(simulation_rate=120.0, telemetry_rate=40.0, n_worlds=3,
              world_params={"world_vel": np.arange(3 * 2 * 6, dtype=float).reshape(3, 2, 6) + 1.0})
    sys_ = el.six_dof() | el.host_system(damp)
    ref = _two_body_world().build(sys_, **kw)
    ref.run(8)                                                    # 2 whole cycles and a partial one
    ex = _two_body_world().build(sys_, ensemble=True, ensemble_ring=2, retain=[2, 0], **kw)
    ex.run(8)
    assert ("invoke", 1) in _FakeBackend.calls
    for pair in ("a.world_pos", "a.world_vel", "b.world_vel", "b.inertia"):
        got, want = ex.history_worlds(pair), ref.history_worlds(pair)[:, [2, 0]]
        assert got.shape == want.shape == (4, 2, got.shape[-1]) and np.array_equal(got, want), pair
    assert ex._globals_hist == ref._globals_hist


def test_write_run_databases_takes_keep_as_any_iterable(fake, tmp_path):
    rows = [{"run_id": f"run_{k}"} for k in range(4)]
    ref = _two_body_world().build(el.six_dof(), n_worlds=4)
    paths = mc.write_run_databases(ref, rows, str(tmp_path / "d"), keep=(k for k in (0, 2)))
    assert sorted(os.listdir(tmp_path / "d" / "runs")) == ["run_0", "run_2"] and len(paths) == 2
    ex = _two_body_world().build(el.six_dof(), n_worlds=4, ensemble=True, retain=[3, 1])
    paths = mc.write_run_databases(ex, rows, str(tmp_path / "e"), keep=iter([1]))
    assert os.listdir(tmp_path / "e" / "runs") == ["run_1"] and len(paths) == 1


@pytest.mark.parametrize("retain", [[0, 3, 4, 9, 10], [10, 4, 0, 9, 3, 5]])
def test_shard_retained_keeps_each_ranks_runs_in_order(retain):
    n_worlds, size = 11, 3                                        # uneven shards: 4, 4, 3 worlds
    got = [shard_retained(retain, n_worlds, r, size) for r in range(size)]
    back = []
    for r, local in enumerate(got):
        w0, w1 = shard_worlds(n_worlds, r, size)
        assert all(0 <= w < w1 - w0 for w in local)
        back += [w0 + w for w in local]
    assert sorted(back) == sorted(retain)
    for r, local in enumerate(got):                               # order within a rank is the global order
        w0 = shard_worlds(n_worlds, r, size)[0]
        assert [w0 + w for w in local] == [w for w in retain if w in [w0 + x for x in local]]
    assert shard_retained([0], 11, 2, 3) == []


# ---------------------------------------------------------------------------------------------------------------- GPU


def _sampled(ex, ws):
    return np.concatenate([ex.download(c) for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)], -1)[ws]


@pytest.mark.gpu
@pytest.mark.parametrize("kind, M, N, width", [(ROCKET, 300, 1, 25), (ROCKET, 77, 3, 13), (FREE, 1, 1, 25),
                                               (FREE, 129, 2, 13)])
def test_download_worlds_equals_the_full_download(kind, M, N, width):
    need_gpu()
    import torch

    ex, _ = handle(kind, M, N, "exact", width=width, every=2, capacity=5)
    ex.step(9)                                                    # 4 samples
    traj = ex.trajectory()
    assert traj.shape[0] == 4
    for ws in ([0], [M - 1], [0, M - 1, M // 2, 1 % M, M // 2], [M - 1, 0, M - 1, 0]):
        t0 = ex.timings()["kernel_launches"]
        got = ex.trajectory_worlds(ws)
        assert ex.timings()["kernel_launches"] == t0 + 1
        assert got.shape == (4, len(ws), N, width) and got.tobytes() == np.ascontiguousarray(traj[:, ws]).tobytes()
        st = ex.state_worlds(ws)
        assert st.shape == (len(ws), N, 25) and st.tobytes() == np.ascontiguousarray(_sampled(ex, ws)).tobytes()
        dev = torch.empty((4, len(ws), N, width), dtype=torch.float64, device="cuda")
        assert ex.trajectory_worlds(ws, dev.data_ptr(), dev.numel() * 8) is None
        assert dev.cpu().numpy().tobytes() == got.tobytes()
        dev.zero_()
        assert ex.trajectory_worlds(ws, dev.data_ptr()) is None                  # bytes default to the rows' size
        assert dev.cpu().numpy().tobytes() == got.tobytes()
        dev = torch.empty((len(ws), N, 25), dtype=torch.float64, device="cuda")
        ex.state_worlds(ws, dev.data_ptr(), dev.numel() * 8)
        assert dev.cpu().numpy().tobytes() == st.tobytes()
        dev.zero_()
        ex.state_worlds(ws, dev.data_ptr())
        assert dev.cpu().numpy().tobytes() == st.tobytes()
    ex.close()


@pytest.mark.gpu
def test_download_worlds_in_two_staging_slices():
    """65 536 retained bodies x 25 planes are 13.1 MB a sample: 24 samples take two 256 MiB slices (20 + 4)."""
    need_gpu()
    import torch

    M = 1024
    ex, _ = handle(ROCKET, M, 1, "fast", width=25, every=1, capacity=24)
    ex.step(24)
    ws = np.random.default_rng(1).integers(0, M, 65536)
    ws[0], ws[-1] = 0, M - 1
    want = ex.trajectory()[:, ws]
    assert 65536 * 25 * 8 * 24 > (256 << 20)
    t0 = ex.timings()["kernel_launches"]
    got = ex.trajectory_worlds(ws)
    assert ex.timings()["kernel_launches"] == t0 + 2
    assert got.tobytes() == want.tobytes()
    dev = torch.empty(want.shape, dtype=torch.float64, device="cuda")
    ex.trajectory_worlds(ws, dev.data_ptr(), dev.numel() * 8)
    assert dev.cpu().numpy().tobytes() == want.tobytes()
    ex.close()


@pytest.mark.gpu
def test_download_worlds_refusals():
    need_gpu()
    ex, _ = handle(FREE, 10, 2, "exact", width=25, every=1, capacity=4)
    ex.step(2)
    L, out = ex._L, np.empty((2, 1, 2, 25))
    u64p = ctypes.POINTER(ctypes.c_uint64)
    ws = np.array([3], dtype=np.uint64)
    for fn in (L.b200_sixdof_trajectory_download_worlds, L.b200_sixdof_state_download_worlds):
        bad = np.array([1, 10], dtype=np.uint64)
        assert fn(ex._h, bad.ctypes.data_as(u64p), 2, out.ctypes.data, out.nbytes) == _lib.ERR_INVALID_ARGUMENT
        assert "world index 10 (entry 1)" in L.b200_last_error().decode()
        assert fn(ex._h, ws.ctypes.data_as(u64p), 0, out.ctypes.data, out.nbytes) == _lib.ERR_INVALID_ARGUMENT
        assert fn(ex._h, None, 1, out.ctypes.data, out.nbytes) == _lib.ERR_INVALID_ARGUMENT
        assert fn(None, ws.ctypes.data_as(u64p), 1, out.ctypes.data, out.nbytes) == _lib.ERR_INVALID_ARGUMENT
        assert fn(ex._h, ws.ctypes.data_as(u64p), 1, out.ctypes.data, out.nbytes + 8) == _lib.ERR_VALUE_SIZE_MISMATCH
    with pytest.raises(_lib.B200ValueError):
        ex.state_worlds([3], out.ctypes.data, 8)
    ex.trajectory_reset()
    t0 = ex.timings()["kernel_launches"]
    assert ex.trajectory_worlds([0, 9]).shape == (0, 2, 2, 25)
    assert L.b200_sixdof_trajectory_download_worlds(ex._h, ws.ctypes.data_as(u64p), 1, None, 0) == _lib.OK
    assert ex.timings()["kernel_launches"] == t0
    ex.close()


def _routes():
    return [("ring1", 1, None, 23), ("ring3", 3, None, 25), ("default_ring", None, None, 23), ("host", 3, "thrust", 23),
            ("host_sampled", 3, "world_vel", 23)]


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("route, ring, host, ticks", _routes())
def test_retained_rows_equal_the_default_mode(math_mode, route, ring, host, ticks):
    """Rocket worlds (two entities, a thrust column on the rocket only): the retained rows of every sampled and
    pass-through column equal a default-mode Exec's rows of those worlds bit for bit, on every run route; 23 ticks of
    5-tick cycles end with a partial cycle.  On the host-callback route a host system after six_dof() scales the column
    `host`: the pass-through thrust column, or world_vel, a sampled component whose written value the rows must hold."""
    need_gpu()
    M = 40
    retain = [0, 7, M - 1, 3]
    w, sys_, params = rocket_world(M)
    if host:
        def scale(ctx):
            ctx.column(host)[..., -1] *= 0.999
        sys_ = sys_ | el.host_system(scale)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, math=math_mode, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ref.run(ticks)
    ex = w.build(sys_, ensemble=True, ensemble_ring=ring, retain=retain, **kw)
    ex.run(ticks)
    for pair in PAIRS + list(PASS_THROUGH):
        got, want = ex.history_worlds(pair), ref.history_worlds(pair)[:, retain]
        assert got.shape == want.shape and got.dtype == want.dtype, pair
        assert got.tobytes() == want.tobytes(), f"{route}: {pair}"
    h, r = ex.history(PAIRS + ["globals.tick"]), ref.history(PAIRS + ["globals.tick"])
    assert all(h[p].tobytes() == r[p].tobytes() for p in r)


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
def test_retained_rows_of_a_graph_world(math_mode):
    """Three bodies under edge gravity in 12 worlds: multi-entity rows and the edge entities' u64 columns."""
    need_gpu()
    G, M = 6.6743e-11, 12
    w = el.World()
    ids = {}
    for k, x in zip("abc", (0.89, -0.66, -0.23)):
        ids[k] = w.spawn(el.Body(world_pos=el.SpatialTransform(linear=[x, 0.0, 0.0]),
                                 world_vel=el.SpatialMotion(linear=[0.0, x, 0.0]), inertia=el.SpatialInertia(1.0 / G)),
                         name=k.upper())
    Edge = el.Annotated[el.Edge, el.Component("gravity_edge", el.ComponentType.Edge)]

    @el.dataclass
    class Constraint(el.Archetype):
        a: Edge

    for s, d in ("ab", "ba", "ac", "bc", "ca", "cb"):
        w.spawn(Constraint(el.Edge(ids[s], ids[d])), name=f"{s} -> {d}")
    pos = np.tile(np.array([0, 0, 0, 1, 0, 0, 0.0]), (M, 3, 1))
    pos[:, :, 4] = np.array([0.89, -0.66, -0.23]) * np.linspace(0.9, 1.1, M)[:, None]
    kw = dict(simulation_rate=120.0, telemetry_rate=40.0, math=math_mode, n_worlds=M, world_params={"world_pos": pos})
    sys_ = el.six_dof(sys=el.GravityEdges("newton", G=G))
    ref = w.build(sys_, **kw)
    ref.run(20)
    ex = w.build(sys_, ensemble=True, ensemble_ring=2, retain=[11, 0, 5], **kw)
    ex.run(20)
    for pair in [f"{e}.{c}" for e in "ABC" for c in SAMPLED] + ["A.inertia", "a -> b.gravity_edge"]:
        got, want = ex.history_worlds(pair), ref.history_worlds(pair)[:, [11, 0, 5]]
        assert got.dtype == want.dtype and got.tobytes() == want.tobytes(), pair


@pytest.mark.gpu
def test_tables_are_unchanged_by_retain():
    need_gpu()
    M = 96
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, n_worlds=M, world_params=params, ensemble=True, ensemble_ring=3,
              extrema=True, thresholds=[el.Threshold("rocket.world_pos", 6, below=0.5)], quantiles=[0.1, 0.5, 0.9],
              covariance=["world_pos"], histograms=[el.Histogram("rocket.world_pos", 6, (-5.0, 5.0), 16)],
              groups=[30, 0, 66])
    runs = []
    for retain in (None, [5, 95, 0]):
        ex = w.build(sys_, retain=retain, **kw)
        ex.run(23)
        runs.append(ex)
    a, b = runs
    assert a._ens_rows.keys() == b._ens_rows.keys() and len(a._ens_rows) == 8
    for kind in a._ens_rows:
        assert np.concatenate(a._ens_rows[kind]).tobytes() == np.concatenate(b._ens_rows[kind]).tobytes(), kind
    assert a.backend.extrema().tobytes() == b.backend.extrema().tobytes()
    assert a.backend.thresholds().tobytes() == b.backend.thresholds().tobytes()
    assert a._globals_hist == b._globals_hist


@pytest.mark.gpu
def test_sinks_of_a_retained_world_equal_the_default_mode(tmp_path):
    need_gpu()
    M, t0 = 24, 1_700_000_000_000_000
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ex = w.build(sys_, ensemble=True, ensemble_ring=2, retain=[9, 2], **kw)
    live = {"ref": ref.attach_db(str(tmp_path / "ref_live"), t0, world=9),
            "ens": ex.attach_db(str(tmp_path / "ens_live"), t0, world=9)}
    for e in (ref, ex):
        e.run(23)
        e.close_db()
    assert live["ref"].rows_written == live["ens"].rows_written == 6
    a, b = _files(tmp_path / "ref_live"), _files(tmp_path / "ens_live")
    assert a.keys() == b.keys() and all(a[k] == b[k] for k in a)
    for world in (9, 2):
        ref.write_db(str(tmp_path / f"ref_{world}"), t0, world=world)
        ex.write_db(str(tmp_path / f"ens_{world}"), t0, world=world)
        a, b = _files(tmp_path / f"ref_{world}"), _files(tmp_path / f"ens_{world}")
        assert a.keys() == b.keys() and all(a[k] == b[k] for k in a)
        fa = export_csv(ref, str(tmp_path / f"ref_csv_{world}"), world=world)
        fb = export_csv(ex, str(tmp_path / f"ens_csv_{world}"), world=world)
        assert [os.path.basename(p) for p in fa] == [os.path.basename(p) for p in fb]
        assert all(open(p, "rb").read() == open(q, "rb").read() for p, q in zip(fa, fb))
    rows = [{"run_id": f"run_{k:03}"} for k in range(M)]
    paths = mc.write_run_databases(ex, rows, str(tmp_path / "campaign"), start_timestamp_us=t0)
    assert sorted(os.listdir(tmp_path / "campaign" / "runs")) == ["run_002", "run_009"]
    a, b = _files(paths[0]), _files(tmp_path / "ref_9")
    assert a.keys() == b.keys() and all(a[k] == b[k] for k in a)
