"""Arrival-rate matrices for wva_solve_loads, and what the per-scenario loop gives for them.

`forecast(img, n_l)` is a planner's matrix: multipliers 0.2 ... 2.0 of the uploaded load and one zero column.  `mixed(img)`
adds the rates with a meaning of their own: the uploaded rates, +0, -0, negative rates and positive rates whose rpm / 60
is 0.  `binding(...)` sets capacities to a fraction of the median scenario's unlimited demand, so that they bind in most
scenarios.  `oracle_columns(...)` sizes every column with oracle.analyze_pairs once, and `expected(...)` solves each column
with oracle.solve(limited) and oracle.allocate_by_type -- the loop wva_solve_loads stands for -- in the call's output
layout.  Shared by tests/test_solve_loads_cpu.py (the matrices reach what they are built for) and
tests/test_solve_loads_gpu.py (the call against the oracle and against the library's own loop).
"""
import numpy as np

import solve_capacities_cases as sc
import solve_inject_tables as st
from test_pairs_loads_cpu import with_rates

abi = st.abi
F = np.float32
TINY = np.array([1.4e-45, 4.2e-44], dtype=F)        # positive, but rpm / 60 is 0 in float32


def forecast(img, n_l, lo=0.2, hi=2.0):
    """[S, n_l]: n_l - 1 multipliers from lo to hi of the uploaded rates, then a zero column"""
    base = img.srv_arrival_rpm.astype(F)
    fac = np.linspace(lo, hi, n_l - 1).astype(F)
    cols = [(base * f).astype(F) for f in fac] + [np.zeros(img.S, dtype=F)]
    return np.stack(cols, axis=1).astype(F)


def mixed(img, seed=11):
    """[S, 10]: the uploaded rates (column 0), multipliers, +0 and -0 columns, and columns mixing negative, zero, tiny
    positive and scaled rates server by server.  Tiny rates go only to servers with MinNumReplicas > 0 or a TPS target
    (elsewhere the reference's Analyze never returns on them)."""
    base = img.srv_arrival_rpm.astype(F)
    rng = np.random.default_rng(seed)
    cols = [base, F(0.5) * base, F(1.7) * base, np.zeros(img.S, dtype=F), np.full(img.S, -0.0, dtype=F)]
    tiny_ok = (img.srv_min_replicas > 0) | (img.srv_slo_tps > 0)
    for _ in range(5):
        pick = rng.integers(0, 5, img.S)
        c = (base * rng.uniform(0.1, 3.0, img.S).astype(F)).astype(F)
        c[pick == 0] = -1.0
        c[pick == 1] = 0.0
        c[pick == 2] = -0.0
        c[(pick == 3) & tiny_ok] = rng.choice(TINY, int(((pick == 3) & tiny_ok).sum()))
        cols.append(c)
    return np.stack(cols, axis=1).astype(F)


def oracle_columns(oracle, img, rpm):
    """per column j: (image with rates rpm[:, j], pairs, feasible) as oracle.analyze_pairs gives them"""
    out = []
    for j in range(rpm.shape[1]):
        im = with_rates(img, rpm[:, j])
        pairs, feasible, _ = oracle.analyze_pairs(im, threads=oracle.hardware_threads())
        out.append((im, pairs, feasible))
    return out


def binding(img, oracle, cols, fraction=0.6, round_robin=False):
    """capacities per type: `fraction` of the median over the columns of the unlimited solve's demand (at least 1)"""
    dem = np.array([sc.demand(im, p, f, oracle) for im, p, f in cols], dtype=np.int64)
    cap = np.maximum(np.ceil(fraction * np.median(dem, axis=0)), 1).astype(np.int64)
    return np.minimum(cap, st.ROUND_ROBIN_ROUNDS) if round_robin else cap


def expected(oracle, cols, capacity, delayed, policy):
    """(acc [n_l, S], recs [n_l, S], count [n_l, T], cost [n_l, T]) of one limited oracle solve per column under
    `capacity`"""
    n = len(cols)
    S, T = cols[0][0].S, cols[0][0].T
    acc = np.zeros((n, S), dtype=np.int32)
    recs = np.zeros((n, S), dtype=abi.PAIR_REC_DTYPE)
    count = np.zeros((n, T), dtype=np.int64)
    cost = np.zeros((n, T), dtype=np.float32)
    for j, (im, pairs, feasible) in enumerate(cols):
        saved = im.type_capacity.copy()
        im.type_capacity[:] = capacity
        try:
            a, ch = oracle.solve(im, pairs, feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
            acc[j], recs[j] = a, sc.to_recs(a, ch)
            count[j], cost[j] = oracle.allocate_by_type(im, a, ch)
        finally:
            im.type_capacity[:] = saved
    return acc, recs, count, cost


def shared_group_servers(im, pairs, feasible):
    """servers with a run in a shared group of the static order (tools/greedy_static_model.py): equal keys held by runs
    of more than one server"""
    import greedy_static_model as gm
    servers, _, _ = st.Table(im, pairs, feasible, "generated").to_model()
    members = {}
    for key, s, _, _ in gm.static_order(servers):
        members.setdefault(key, set()).add(s)
    return set().union(*[m for m in members.values() if len(m) > 1] or [set()])
