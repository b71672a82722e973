"""Outcome tables (b200_sixdof_set_outcomes and the outcome_* entries) on one GPU, against the host route.

    python scripts/outcome_perf.py [--calls 20] [--out r.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query) and the device copy probe;
  2. for 2^20 and 2^22 worlds of one entity and 2^18 worlds of 4, each with P = 8 and P = 25 outcomes of every kind
     (extrema fields and ticks, threshold ticks and planes, moment rms / std, dwell ticks, input columns, host values):
     the value pass's kernel time (torch.profiler, median over the calls) and the bytes it must move (8 B written per
     world and outcome; 8 B read per extrema, threshold, dwell and column outcome, 16 B for count / mean, 24 B for
     std and 32 B for rms) over that time, against the copy probe;
  3. the wall time of each outcome entry (stats, quantiles at 5 levels, covariance of all P, one 64-bin histogram), for
     G = 1 (ungrouped), 12 and 256 groups; each entry synchronises, so a host clock measures it;
  4. the host route for the same answers: the per-world downloads (extrema, thresholds, moments, dwells and the input
     columns) into pinned memory, then numpy; the two routes' values must be equal bit for bit, the counts, minima,
     maxima, quantiles and histograms equal, the means within 1e-9 relative and m2 within 1e-9 of count * (mean^2 + 1)
     (numpy's two-pass sums round differently from the device's chunked merge), each co-moment within 1e-9 of
     sqrt(M_aa * M_bb).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np

KERNEL = "outcome_kernel"
LEVELS = [0.01, 0.25, 0.5, 0.75, 0.99]
CASES = [(1 << 20, 1, 8), (1 << 20, 1, 25), (1 << 22, 1, 8), (1 << 22, 1, 25), (1 << 18, 4, 8), (1 << 18, 4, 25)]


def campaign(M, E, P):
    """A handle of M worlds x E entities with extrema, 2 thresholds, 2 moment planes and 2 dwells folded over 8 rows,
    and P outcomes of every kind on entity E - 1."""
    import elodin_b200 as el
    from elodin_b200 import _lib

    rng = np.random.default_rng(7)
    ex = el.B200Exec(E, M, 1e-3, None, [el.GravityConst((0.0, 0.0, -9.81)), el.ThrustBody((-1.0, 0.0, 0.0), "thrust")],
                     "rk4", "fast")
    pos = np.zeros((M, E, 7))
    pos[..., 3] = 1.0
    pos[..., 4:] = rng.normal(0.0, 10.0, (M, E, 3))
    vel = rng.normal(0.0, 5.0, (M, E, 6))
    ine = np.tile(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 1))
    ine[..., 6] = rng.uniform(0.5, 1.5, (M, E))
    ex.set_state(pos, vel, ine, thrust=rng.uniform(5.0, 15.0, (M, E, 1)))
    e = E - 1
    conds = [(e, 6, False, -1.0), (e, 4, True, 5.0)]
    ex.summary_begin(True, conds, moments=[6, 12], dwells=conds)
    for _ in range(8):
        ex.step(4)
        ex.summary_add_state()
    gain = rng.uniform(0.8, 1.2, M)
    X, T, MO, D, C, V = (_lib.OUTCOME_EXTREMA, _lib.OUTCOME_THRESHOLD, _lib.OUTCOME_MOMENT, _lib.OUTCOME_DWELL,
                         _lib.OUTCOME_COLUMN, _lib.OUTCOME_VALUES)
    outs = [(X, 1, 6, e), (X, 3, 6, e), (T, 0, 0), (T, 5, 0), (MO, 3, 0, e), (D, 2, 1), (C, 6, 0, e, "inertia"),
            (V, 0, 0, 0, 0, gain)]
    more = [(X, 0, 4, e), (X, 1, 4, e), (X, 0, 5, e), (X, 1, 5, e), (X, 2, 6, e), (X, 4, 6, e), (T, 0, 1), (T, 6, 1),
            (T, 7, 0), (MO, 2, 0, e), (MO, 1, 1, e), (MO, 0, 1, e), (D, 0, 0), (D, 1, 0), (D, 0, 1), (C, 0, 0, e, "thrust"),
            (X, 1, 12, e)]
    outs = (outs + more)[:P]
    ex.set_outcomes(outs)
    return ex, outs, gain


def host_values(ex, outs, gain, M, E):
    """The same values from the per-world downloads into pinned memory, then numpy: (values [M, P], download s)."""
    import elodin_b200 as el
    from elodin_b200 import _lib

    L, h = _lib.lib(), ex._h
    t0 = time.perf_counter()
    tables = {}
    for name, shape in (("extrema", (M, E, 25, 5)), ("thresholds", (M, 2, 26)), ("moments", (M, E, 2, 3)),
                        ("dwells", (M, 2, 3))):
        buf = el.pinned_empty(shape)
        _lib.check(getattr(L, f"b200_sixdof_{name}_download")(h, buf.ctypes.data, buf.nbytes))
        tables[name] = buf
    cols = {}
    for c, w in (("inertia", 7), ("thrust", 1)):
        buf = el.pinned_empty((M, E, w))
        ex.download_ptr(c, buf.ctypes.data, buf.nbytes)
        cols[c] = buf
    dl = time.perf_counter() - t0
    v = np.empty((M, len(outs)))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for k, o in enumerate(outs):
            kind, field, index = o[:3]
            if kind == _lib.OUTCOME_EXTREMA:
                x, tick = tables["extrema"][:, o[3], index, field], field >= 2
            elif kind == _lib.OUTCOME_THRESHOLD:
                x, tick = tables["thresholds"][:, index, field], field == 0
            elif kind == _lib.OUTCOME_DWELL:
                x, tick = tables["dwells"][:, index, field], field > 0
            elif kind == _lib.OUTCOME_MOMENT:
                n, mean, m2 = (tables["moments"][:, o[3], index, f] for f in range(3))
                x, tick = (n, mean, np.sqrt(m2 / n), np.sqrt(mean * mean + m2 / n))[field], False
            elif kind == _lib.OUTCOME_COLUMN:
                x, tick = cols[o[4]][:, o[3], field], False
            else:
                x, tick = gain, False
            v[:, k] = np.where(x == -1.0, np.nan, x) if tick else x
    for b in list(tables.values()) + list(cols.values()):
        el.pinned_free(b)
    return v, dl


def host_tables(v, sizes, spec):
    """numpy: per group stats [G, P, 5], quantiles [G, P, n_q], covariance [G, 1 + P + P^2], 1D histogram [G, 3 + n]."""
    P = v.shape[1]
    st, qs, cv, hs = [], [], [], []
    w0 = 0
    lo, hi, n = spec
    for s in sizes:
        g = v[w0:w0 + s]
        w0 += s
        fin = np.isfinite(g)
        cnt = fin.sum(0)
        with np.errstate(invalid="ignore", divide="ignore"):
            mean = np.where(fin, g, 0.0).sum(0) / cnt
            m2 = np.where(cnt > 0, np.where(fin, (g - mean) ** 2, 0.0).sum(0), np.nan)
        mn = np.array([g[fin[:, k], k].min() if cnt[k] else np.nan for k in range(P)])
        mx = np.array([g[fin[:, k], k].max() if cnt[k] else np.nan for k in range(P)])
        st.append(np.stack([cnt, mean, m2, mn, mx], -1))
        qs.append(np.stack([np.quantile(g[fin[:, k], k], LEVELS) if cnt[k] else np.full(len(LEVELS), np.nan)
                            for k in range(P)]))
        ok = fin.all(1)
        y = g[ok]
        c = np.full(1 + P + P * P, np.nan)
        c[0] = len(y)
        if len(y):
            c[1:1 + P] = y.mean(0)
            d = y - y.mean(0)
            c[1 + P:] = (d.T @ d).ravel()
        cv.append(c)
        x = g[:, 0]
        f = x[np.isfinite(x)]
        hs.append(np.concatenate([[np.sum(~np.isfinite(x)), np.sum(f < lo), np.sum(f > hi)], np.histogram(f, n, (lo, hi))[0]]))
    return np.array(st), np.array(qs), np.array(cv), np.array(hs, dtype=np.float64)


def kernel_ms(ex, calls):
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ex.outcome_stats()
        torch.cuda.synchronize()
    ms = [(e.end_ns() - e.start_ns()) / 1e6 for e in prof.profiler.kineto_results.events()
          if e.device_type() == DeviceType.CUDA and KERNEL in e.name()]
    return float(np.median(ms)) if ms else float("nan")


def pass_bytes(outs, M):
    from elodin_b200 import _lib

    per = 0
    for o in outs:
        if o[0] == _lib.OUTCOME_VALUES:
            continue
        per += 8 + ({0: 8, 1: 16, 2: 24, 3: 32}[o[1]] if o[0] == _lib.OUTCOME_MOMENT else 8)
    return per * M


def wall_ms(call, calls):
    call()
    t0 = time.perf_counter()
    for _ in range(calls):
        call()
    return (time.perf_counter() - t0) / calls * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    import elodin_b200 as el
    from elodin_b200 import _lib
    from ensemble_perf import card

    if el.device_count() < 1:
        raise SystemExit("outcome_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["cases"] = []
    spec = (-50.0, 50.0, 64)
    for M, E, P in CASES:
        ex, outs, gain = campaign(M, E, P)
        ms = kernel_ms(ex, a.calls)
        b = pass_bytes(outs, M)
        row = {"worlds": M, "entities": E, "P": P, "pass_ms": ms, "pass_bytes": b,
               "pass_of_probe": b / (ms * 1e-3) / 1e9 / probe}
        print(f"M={M} E={E} P={P}: value pass {ms * 1e3:.1f} us, {b / 1e6:.1f} MB, {row['pass_of_probe']:.2f} of the probe")
        t0 = time.perf_counter()
        hv, dl = host_values(ex, outs, gain, M, E)
        dv = ex.outcome_values()
        assert np.array_equal(np.where(np.isnan(hv), 0, hv).view(np.uint64), np.where(np.isnan(dv), 0, dv).view(np.uint64))
        assert np.array_equal(np.isnan(hv), np.isnan(dv))
        for G in (1, 12, 256):
            sizes = [M] if G == 1 else [M // G + (g < M % G) for g in range(G)]
            if G > 1:
                ex.set_world_groups(sizes)
            pre = "outcome_group_" if G > 1 else "outcome_"
            calls = {"stats": (), "quantiles": (LEVELS,), "covariance": (list(range(P)),),
                     "histograms": ([(0, (0,), (spec[2],), (spec[0],), (spec[1],))],)}
            times = {k: wall_ms(lambda k=k: getattr(ex, pre + k)(*arg), a.calls) for k, arg in calls.items()}
            dev = [getattr(ex, pre + k)(*arg) for k, arg in calls.items()]
            if G == 1:
                dev = [d[None] for d in dev]
            t0 = time.perf_counter()
            host = host_tables(hv, sizes, spec)
            host_ms = (time.perf_counter() - t0) * 1e3 + dl * 1e3
            st, qs, cv, hs = dev
            assert np.array_equal(st[..., [0, 3, 4]], host[0][..., [0, 3, 4]], equal_nan=True)
            scale = host[0][..., 0] * (host[0][..., 1] ** 2 + 1.0)  # the m2 of values of that size: where rounding lives
            with np.errstate(invalid="ignore", divide="ignore"):
                err = np.nanmax(np.abs(st[..., 1:3] - host[0][..., 1:3]) / np.stack([np.abs(host[0][..., 1]) + 1e-300, scale], -1))
            assert np.array_equal(np.isnan(st[..., 1:3]), np.isnan(host[0][..., 1:3])) and err < 1e-9, err
            assert np.array_equal(np.abs(qs), np.abs(host[1]), equal_nan=True)
            assert cv[:, 0].tolist() == host[2][:, 0].tolist()
            Md, Mh = cv[:, 1 + P:].reshape(-1, P, P), host[2][:, 1 + P:].reshape(-1, P, P)
            d = np.sqrt(np.abs(np.einsum("gii->gi", Mh)))
            with np.errstate(invalid="ignore", divide="ignore"):
                err = np.nanmax(np.abs(Md - Mh) / (d[:, :, None] * d[:, None, :] + 1e-300))
            assert np.array_equal(np.isnan(Md), np.isnan(Mh)) and not err > 1e-9, err
            assert np.array_equal(hs, host[3])
            row[f"G{G}_entry_ms"] = times
            row[f"G{G}_host_ms"] = host_ms
            print(f"  G={G}: entries " + ", ".join(f"{k} {t:.3f} ms" for k, t in times.items())
                  + f"; host route (downloads {dl * 1e3:.1f} ms + numpy) {host_ms:.1f} ms; same answers")
        res["cases"].append(row)
        del ex
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
