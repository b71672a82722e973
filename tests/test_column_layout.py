"""The column layout kernels against numpy indexing of the caller's array, bit for bit.

Every input and output crosses between the caller's [body][width] rows and the device's SoA planes (plane k of a
column at plane_stride * k doubles, bodies [0, n_bodies), padding up to the stride): aos_to_soa_kernel /
soa_to_aos_kernel (upload, download, pipelined invoke_batch), multi_transpose_kernel (every column of a small
invoke_batch in one launch), the trajectory download (launches of at most 32768 samples, staging chunks of at most
256 MB) and traj_world_major_kernel (the world-major layout of the trajectory gather).

Layout is a pure copy, so every comparison is on uint64 views, and the data carries NaNs with distinct payloads
(quiet and signalling), +-0, subnormals, +-inf and +-DBL_MAX beside random bit patterns: any arithmetic or
canonicalisation on the way through shows up.  The device planes are read and written directly (through
b200_sixdof_device_plane), so an upload is checked on its own, a download on its own, and the padding past the last
body must keep a sentinel.

A column of 24 doubles (an 8-wheel torque column) needs more than 48 KB of dynamic shared memory per tile: the cases
that carry one run in a fresh child process, so that they cannot pass because an earlier test raised a kernel's
limit in the same process.
"""

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200.executor import FORCE, INERTIA, SIMULATION_TIME_STEP, TICK, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests.util import random_world, run_child

SENTINEL = 0x7FF4DEADBEEF0001  # a signalling NaN: no kernel writes it
DT = 0.01

_SPECIALS = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF0000000000001,  # NaNs (payload added)
             0x0000000000000000, 0x8000000000000000, 0x0000000000000001, 0x800FFFFFFFFFFFFF,  # +-0, subnormals
             0x7FF0000000000000, 0xFFF0000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF]  # +-inf, +-DBL_MAX


def special_bits(shape, seed):
    """float64 data of random bit patterns with, at every fifth element, one of _SPECIALS; each NaN gets a payload
    from its position, so no two NaNs share their bits."""
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, np.iinfo(np.uint64).max, size=shape, dtype=np.uint64, endpoint=True)
    flat = bits.reshape(-1)
    pos = np.arange(0, flat.size, 5)
    sp = np.array(_SPECIALS, dtype=np.uint64)[(pos // 5) % len(_SPECIALS)]
    nan = (sp & np.uint64(0x7FF0000000000000)) == np.uint64(0x7FF0000000000000)
    nan &= (sp & np.uint64(0x000FFFFFFFFFFFFF)) != 0
    sp[nan] |= (pos[nan].astype(np.uint64) << np.uint64(4)) & np.uint64(0x0007FFFFFFFFFFF0)
    flat[pos] = sp
    return bits.view(np.float64)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


# --------------------------------------------------------------------------- the device planes through torch


def _plane(ex, cid, k):
    """Plane k of column cid, the whole stride (padding included), as an int64 torch tensor on the device."""
    import torch

    ptr = ex.device_plane(cid, k)
    assert ptr, f"no plane {k} of column {cid}"

    class Plane:
        __cuda_array_interface__ = {"shape": (ex.plane_stride,), "typestr": "<i8", "data": (ptr, False), "version": 3}

    return torch.as_tensor(Plane(), device="cuda")


def _fill_padding(ex, cid, width):
    """Write the sentinel into every plane's padding [n_bodies, stride)."""
    import torch

    n = ex.n_worlds * ex.n_entities
    for k in range(width):
        _plane(ex, cid, k)[n:] = SENTINEL
    torch.cuda.synchronize()


def _write_planes(ex, cid, a):
    """Bodies [0, n_bodies) of every plane of column cid := a[..., k], written through the device pointers."""
    import torch

    rows = np.ascontiguousarray(a).reshape(-1, a.shape[-1]).view(np.int64)
    for k in range(a.shape[-1]):
        _plane(ex, cid, k)[:rows.shape[0]].copy_(torch.from_numpy(np.ascontiguousarray(rows[:, k])))
    torch.cuda.synchronize()


def _assert_planes(ex, cid, a, what, padding=True):
    """Plane k of column cid holds a[..., k] body for body, and (padding=True) the sentinel past the last body."""
    import torch

    torch.cuda.synchronize()
    width = a.shape[-1]
    want = _bits(a).reshape(-1, width)
    n = want.shape[0]
    for k in range(width):
        got = _plane(ex, cid, k).cpu().numpy().view(np.uint64)
        bad = np.flatnonzero(got[:n] != want[:, k])
        assert bad.size == 0, (f"{what}: plane {k} of {width}, {bad.size} of {n} bodies differ; first body {bad[0]}: "
                               f"{int(got[bad[0]]):#018x}, want {int(want[bad[0], k]):#018x}")
        if padding:
            pad = np.flatnonzero(got[n:] != SENTINEL)
            assert pad.size == 0, f"{what}: plane {k} of {width}: padding body {n + pad[0]} overwritten ({int(got[n + pad[0]]):#018x})"


# --------------------------------------------------------------------------- every width the ABI creates

# name: (width, effector owning column "col", or None for the Inertia column)
COLUMNS = {
    "thrust": (1, lambda: el.ThrustBody((1.0, 0.0, 0.0), "col")),
    "drag": (3, lambda: el.DragQuadratic(column="col")),
    "drag_per_body": (5, lambda: el.DragQuadratic(column="col", per_body_params=True)),
    "wrench": (6, lambda: el.WrenchBody("col")),
    "inertia": (7, None),
    **{f"wheels{k}": (3 * k, (lambda k=k: el.TorqueBodyFold("col", k))) for k in range(1, 9)},
}

# (worlds, entities): one world at the 256-body tile edges, and many worlds of a few bodies
SHAPES = [(1, 1), (1, 127), (1, 128), (1, 129), (1, 255), (1, 256), (1, 257), (1, 1024), (1, 1025), (1, 4097),
          (129, 1), (43, 3), (257, 4), (1366, 3)]


def _upload_download_case(name):
    """Download: planes written directly come back as the caller's rows (first, so that in a fresh process no upload
    has run before it).  Upload: the planes hold the caller's columns and the padding keeps the sentinel."""
    width, make = COLUMNS[name]
    cid = INERTIA if make is None else "col"
    for i, (M, N) in enumerate(SHAPES):
        what = f"{name} (width {width}), {M} x {N}"
        with el.B200Exec(N, M, DT, None, [] if make is None else [make()], "rk4", "exact") as ex:
            _fill_padding(ex, cid, width)
            b = special_bits((M, N, width), 5000 * width + i)
            _write_planes(ex, cid, b)
            got = ex.download(cid)
            bad = np.flatnonzero(np.any(_bits(got) != _bits(b), axis=-1).reshape(-1))
            assert bad.size == 0, f"download {what}: {bad.size} rows differ, first body {bad[0]}"
            a = special_bits((M, N, width), 1000 * width + i)
            ex.upload(cid, a)
            _assert_planes(ex, cid, a, f"upload {what}")


def _child(out, args):
    """Child-process entry: run one case function of this module (its assertions fail the child)."""
    globals()[args["fn"]](*args["args"])
    np.savez(out, ok=1)


def _in_child(tmp_path, fn, *args):
    run_child("tests.test_column_layout:_child", str(tmp_path / "child.npz"), {"fn": fn, "args": list(args)})


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(COLUMNS))
def test_upload_and_download_every_width(name, tmp_path):
    if COLUMNS[name][0] > 21:
        _in_child(tmp_path, "_upload_download_case", name)
    else:
        _upload_download_case(name)


# --------------------------------------------------------------------------- invoke_batch and tick_fn


def _invoke_effectors(N):
    """Eight effectors, every column width of the ABI among them (24 = eight wheels), each on no entity: the ticks
    never read the special bits of the columns and integrate free bodies."""
    effs = [el.ThrustBody((1.0, 0.0, 0.0), "t1"), el.DragQuadratic(column="d3"), el.TorqueBodyFold("w24", 8),
            el.DragQuadratic(column="d5", per_body_params=True), el.WrenchBody("wb6"), el.WrenchWorld("ww6"),
            el.TorqueBodyFold("w15", 5), el.ThrustBody((0.0, 1.0, 0.0), "t1b")]
    return [e.with_mask(np.zeros(N, dtype=np.uint8)) for e in effs]


_STATE = (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)


def _invoke_case(path, shapes):
    """invoke_batch (or tick_fn) of one EXACT RK4 tick with 12 live input columns (Force is dead on input) against
    the planes it left and against a second handle given the same columns through upload() and step(1)."""
    for i, (M, N, chunk) in enumerate(shapes):
        what = f"{path} {M} x {N}" + (f", ranges of {chunk} bodies" if chunk else "")
        pos, vel, ine = random_world(300 + i, M, N)
        acc = np.random.default_rng(400 + i).normal(size=(M, N, 6))
        ex = el.B200Exec(N, M, DT, None, _invoke_effectors(N), "rk4", "exact", invoke_chunk_bodies=chunk)
        ref = el.B200Exec(N, M, DT, None, _invoke_effectors(N), "rk4", "exact")
        try:
            values = {WORLD_POS: pos, WORLD_VEL: vel, INERTIA: ine, WORLD_ACCEL: acc, FORCE: np.zeros((M, N, 6)),
                      TICK: np.array([0], dtype=np.uint64), SIMULATION_TIME_STEP: np.array([DT])}
            for k, name in enumerate(("t1", "d3", "w24", "d5", "wb6", "ww6", "w15", "t1b")):
                values[el.component_id(name)] = special_bits(ex.column_shape(name), 7000 + 31 * i + k)
            live = [c for c in ex.input_ids if c not in (TICK, SIMULATION_TIME_STEP, FORCE)]
            assert len(live) == 12 and max(ex.column_shape(c)[-1] for c in live) == 24
            for c in live + [FORCE]:
                _fill_padding(ex, c, ex.column_shape(c)[-1])
            ins = [values[c] for c in ex.input_ids]
            n0 = ex.timings()["kernel_launches"]
            if path == "tick_fn":
                outs = [np.empty(ex.column_shape(c), dtype=np.uint64 if c == TICK else np.float64) for c in ex.output_ids]
                ex.tick_fn(ins, outs)
            else:
                outs = ex.invoke_batch(ins, 1)
            launches = ex.timings()["kernel_launches"] - n0
            if chunk:  # every range: one layout launch per live input and per state output
                ranges = -(-M // max(1, chunk // N))
                assert launches >= ranges * (12 + 4), f"{what}: {launches} launches for {ranges} ranges"
            else:  # one layout launch in, the tick, one layout launch out
                assert launches <= 4, f"{what}: {launches} launches, expected the one-launch layout of a small batch"
            # the inputs the tick does not write, on the device; their padding untouched
            for c in live:
                if c not in _STATE:
                    _assert_planes(ex, c, values[c], f"{what}: input column {c:#x}")
            got = dict(zip(ex.output_ids, outs))
            for c in _STATE:  # the outputs are the planes the tick left
                _assert_planes(ex, c, got[c], f"{what}: output column {c:#x}", padding=False)
            for c in live:  # pass-through outputs are the inputs
                if c not in _STATE:
                    assert np.array_equal(_bits(got[c]), _bits(values[c])), f"{what}: pass-through column {c:#x}"
            # the same columns through upload() and step(): the state inputs landed where the tick reads them
            for c in live:
                ref.upload(c, values[c])
            ref.step(1, sync=True)
            for c in _STATE:
                want = ref.download(c)
                bad = np.flatnonzero(np.any(_bits(got[c]) != _bits(want), axis=-1).reshape(-1))
                assert bad.size == 0, f"{what}: column {c:#x} differs from upload + step in {bad.size} bodies, first {bad[0]}"
            assert np.all(np.isfinite(got[WORLD_POS])), f"{what}: the masked effectors reached the state"
        finally:
            ex.close()
            ref.close()


SMALL_SHAPES = [(1, 1, 0), (1, 127, 0), (1, 128, 0), (1, 129, 0), (1, 255, 0), (1, 256, 0), (1, 257, 0), (1, 1024, 0),
                (341, 3, 0), (4, 255, 0)]
# ranges of 77 worlds of 3 bodies start at odd bodies off the 256-body tiles; 128-world ranges of single bodies;
# one world of 4097 bodies in one range
PIPE_SHAPES = [(1366, 3, 231), (5, 257, 514), (1025, 1, 200), (1, 4097, 1000)]


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["small", "tick_fn", "pipelined"])
def test_invoke_batch_columns(path, tmp_path):
    _in_child(tmp_path, "_invoke_case", path, PIPE_SHAPES if path == "pipelined" else SMALL_SHAPES)


# --------------------------------------------------------------------------- the trajectory ring


def _traj_handle(M, N, W, S, **kw):
    return el.B200Exec(N, M, DT, None, [el.GravityConst()], "rk4", "exact", trajectory_every=1, trajectory_capacity=S,
                       trajectory_full=W == 25, **kw)


def _sample(ex, W):
    return np.concatenate([ex.download(c) for c in _STATE[:2 if W == 13 else 4]], -1)


def _assert_traj(got, want, what):
    g, w = _bits(got), _bits(want)
    assert g.shape == w.shape, f"{what}: shape {g.shape}, want {w.shape}"
    bad = np.argwhere(np.any(g != w, axis=-1))
    assert bad.size == 0, f"{what}: {len(bad)} rows differ, first (sample, world, entity) {tuple(bad[0])}"


@pytest.mark.gpu
@pytest.mark.parametrize("W", [13, 25])
@pytest.mark.parametrize("M,N", [(1, 1), (1, 129), (43, 3), (1, 4097)])
def test_trajectory_matches_the_state_after_each_tick(M, N, W):
    """trajectory() and trajectory_to_ptr into a device buffer: sample s is the state downloaded after tick s + 1."""
    import torch

    S = 4
    pos, vel, ine = random_world(11 + N, M, N)
    with _traj_handle(M, N, W, S) as ex:
        ex.set_state(pos, vel, ine)
        want = []
        for _ in range(S):
            ex.step(1, sync=True)
            want.append(_sample(ex, W))
        want = np.stack(want)
        _assert_traj(ex.trajectory(), want, f"trajectory() {M} x {N}, {W} planes")
        dev = torch.full((S, M, N, W), float("nan"), dtype=torch.float64, device="cuda")
        ex.trajectory_to_ptr(dev.data_ptr(), dev.numel() * 8)
        torch.cuda.synchronize()
        _assert_traj(dev.cpu().numpy(), want, f"trajectory_to_ptr {M} x {N}, {W} planes")


@pytest.mark.gpu
def test_trajectory_past_32768_samples(oracle):
    """40 000 samples of one body: the download splits at 32768 samples (the grid's y limit).  The reference is the
    oracle stepped tick by tick, which EXACT math matches bit for bit; every sample differs from its neighbours."""
    O = oracle
    S = 40000
    pos, vel, ine = random_world(21, 1, 1)
    w = O.World(pos, vel, ine)
    eff = [O.Effector(O.EFF_GRAVITY_CONST, p=(0.0, 0.0, -9.81))]
    want = np.empty((S, 1, 1, 25))
    for s in range(S):
        w.rk4(DT, 1, eff, threads=1)
        want[s] = np.concatenate([w.pos, w.vel, w.accel, w.force], -1)
    assert np.all(np.any(want[1:] != want[:-1], axis=-1)), "neighbouring samples must differ"
    for W in (13, 25):
        with _traj_handle(1, 1, W, S) as ex:
            ex.set_state(pos, vel, ine)
            ex.step(S, sync=True)
            _assert_traj(ex.trajectory(), want[..., :W], f"{S} samples, {W} planes")


@pytest.mark.gpu
def test_trajectory_download_in_staging_chunks():
    """2^17 bodies x 13 planes is 13.6 MB a sample: 45 samples download through the 256 MB staging buffer in chunks
    of 19, 19 and 7 samples.  Sample s is the state downloaded after tick s + 1."""
    M, N, W, S = 1, 1 << 17, 13, 45
    per_sample = M * N * W * 8
    assert [min(19, S - s0) for s0 in range(0, S, (256 << 20) // per_sample)] == [19, 19, 7]
    pos, vel, ine = random_world(31, M, N)
    with _traj_handle(M, N, W, S) as ex:
        ex.set_state(pos, vel, ine)
        want = np.empty((S, M, N, W))
        for s in range(S):
            ex.step(1, sync=True)
            want[s] = _sample(ex, W)
        _assert_traj(ex.trajectory(), want, f"{S} samples of {N} bodies")


# --------------------------------------------------------------------------- the world-major gather layout

# (worlds, entities, planes, samples): rows of a world split across 128-body tiles, and past 32768 samples
GATHER_CASES = [(130, 1, 13, 5), (130, 1, 25, 5), (45, 3, 13, 5), (45, 3, 25, 5), (3, 129, 13, 5), (3, 129, 25, 5),
                (2, 1, 13, 32768 + 37)]


def _gather_case():
    """One-rank communicator: trajectory_allgather into host and device buffers is trajectory() world-major."""
    import torch

    from elodin_b200.sharding import Comm

    comm = Comm(Comm.unique_id(), 1, 0, 0)
    try:
        for i, (M, N, W, S) in enumerate(GATHER_CASES):
            what = f"gather {M} x {N}, {W} planes, {S} samples"
            pos, vel, ine = random_world(50 + i, M, N)
            with _traj_handle(M, N, W, S, device=0) as ex:
                ex.set_state(pos, vel, ine)
                ex.step(S, sync=True)
                want = np.ascontiguousarray(ex.trajectory().transpose(1, 0, 2, 3))
                assert np.all(np.any(want[:, 1:] != want[:, :-1], axis=-1)), f"{what}: neighbouring samples must differ"
                _assert_traj(comm.trajectory_allgather(ex, [M]), want, f"{what}, host")
                dev = torch.full(want.shape, float("nan"), dtype=torch.float64, device="cuda:0")
                comm.trajectory_allgather(ex, [M], out_ptr=dev.data_ptr())
                torch.cuda.synchronize()
                _assert_traj(dev.cpu().numpy(), want, f"{what}, device")
    finally:
        comm.close()


@pytest.mark.gpu
def test_trajectory_gather_is_world_major(tmp_path):
    from elodin_b200.sharding import Comm

    if not Comm.available():
        pytest.skip("libnccl.so.2 is not loadable")
    _in_child(tmp_path, "_gather_case")


# --------------------------------------------------------------------------- CPU: the test data


def test_special_bits_cover_the_encodings():
    a = _bits(special_bits((1, 257, 24), 3)).reshape(-1)
    for v in _SPECIALS[4:]:
        assert np.any(a == np.uint64(v)), f"{v:#018x} missing"
    nan = a[np.isnan(a.view(np.float64))]
    assert nan.size >= 2 * len(_SPECIALS) and np.unique(nan).size == nan.size, "NaNs need distinct payloads"
    assert np.any((nan & np.uint64(0x0008000000000000)) == 0), "signalling NaNs missing"
    assert np.unique(a).size > 0.85 * a.size
    assert not np.any(a == np.uint64(SENTINEL))
