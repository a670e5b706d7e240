"""Capacity lists for wva_solve_capacities, and what the one-vector loop gives for them.

`ladder(img, pairs, feasible, oracle)` builds the 64 vectors a generated image is solved under: nothing, fractions 0.05 ...
1.2 of the unlimited demand per type, exactly the first candidates' demand and one unit either side, a negative capacity,
2^62, and each type starved in turn while the others have plenty.  Under the round-robin policies every entry is capped
at ROUND_ROBIN_ROUNDS (the oracle hands out one replica per round).  `expected(...)` solves the image once per vector with
oracle.solve / oracle.allocate_by_type -- the loop wva_solve_capacities stands for -- in the call's output layout.
Shared by tests/test_solve_capacities_cpu.py (the vectors reach the branches they are built for) and
tests/test_solve_capacities_gpu.py (the call against the oracle and against the library's own loop).
"""
import numpy as np

import solve_inject_tables as st

abi = st.abi

FRACTIONS = [0.05, 0.1, 0.15, 0.2, 0.25, 0.3, 0.35, 0.4, 0.45, 0.5, 0.55, 0.6, 0.65, 0.7, 0.75, 0.8, 0.85, 0.9, 0.95, 1.0,
             1.05, 1.1, 1.15, 1.2]
N_LADDER = 64
PLENTY = 1 << 40


def demand(img, pairs, feasible, oracle):
    """units per type that the unlimited solve places"""
    acc, chosen = oracle.solve(img, pairs, feasible, unlimited=True)
    return oracle.allocate_by_type(img, acc, chosen)[0]


def ladder(img, pairs, feasible, oracle, round_robin=False, n=N_LADDER, seed=5):
    T = img.T
    dem = demand(img, pairs, feasible, oracle).astype(np.int64)
    first, _ = st.first_counts(st.Table(img, pairs, feasible, "generated"))
    first = np.array(first, dtype=np.int64)
    rows = [np.zeros(T, dtype=np.int64)]
    rows += [np.ceil(f * dem).astype(np.int64) for f in FRACTIONS]
    rows += [first, first - 1, first + 1]
    rows += [np.full(T, -5, dtype=np.int64), np.full(T, 1 << 62, dtype=np.int64)]
    for t in range(T):
        r = np.full(T, PLENTY, dtype=np.int64)
        r[t] = 0
        rows.append(r)
    rng = np.random.default_rng(seed)
    while len(rows) < n:                      # mixed fractions per type
        rows.append(np.ceil(rng.choice(FRACTIONS, T) * dem).astype(np.int64))
    out = np.array(rows[:n], dtype=np.int64)
    if round_robin:
        out = np.minimum(out, st.ROUND_ROBIN_ROUNDS)
    return out


def to_recs(acc, chosen):
    """an oracle / wva_solve decision in wva_pair_rec form: feasible = 1 where a candidate was chosen"""
    n = len(acc)
    r = np.zeros(n, dtype=abi.PAIR_REC_DTYPE)
    for name, _ in abi.ALLOC_FIELDS:
        r[name] = getattr(chosen, name)
    r["feasible"] = (np.asarray(acc) >= 0).astype(np.uint8)
    return r


def expected(oracle, img, pairs, feasible, caps, delayed, policy):
    """(acc [n, S], recs [n, S], count [n, T], cost [n, T]) of one oracle solve per capacity vector"""
    saved = img.type_capacity.copy()
    n, S, T = len(caps), img.S, img.T
    acc = np.zeros((n, S), dtype=np.int32)
    recs = np.zeros((n, S), dtype=abi.PAIR_REC_DTYPE)
    count = np.zeros((n, T), dtype=np.int64)
    cost = np.zeros((n, T), dtype=np.float32)
    try:
        for j, cap in enumerate(caps):
            img.type_capacity[:] = cap
            a, ch = oracle.solve(img, pairs, feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
            acc[j], recs[j] = a, to_recs(a, ch)
            count[j], cost[j] = oracle.allocate_by_type(img, a, ch)
    finally:
        img.type_capacity[:] = saved
    return acc, recs, count, cost


def same_floats(a, b):
    """bit for bit, two NaNs equal whatever their payload"""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    both = np.isnan(a) & np.isnan(b)
    return np.array_equal(np.where(both, np.uint32(0), a.view(np.uint32)), np.where(both, np.uint32(0), b.view(np.uint32)))


def same_recs(a, b):
    """-> the first differing field of two wva_pair_rec arrays, or None"""
    for name in abi.PAIR_REC_DTYPE.names:
        x, y = a[name], b[name]
        if x.dtype == np.float32:
            if not same_floats(x, y):
                return name
        elif not np.array_equal(x, y):
            return name
    return None


def check(got, want, what):
    acc, recs, count, cost = got
    w_acc, w_recs, w_count, w_cost = want
    assert np.array_equal(acc, w_acc), (what, np.argwhere(acc != w_acc)[:8])
    field = same_recs(recs, w_recs)
    assert field is None, (what, field)
    assert np.array_equal(count, w_count), what
    assert same_floats(cost, w_cost), what


def stacks_per_vector(t, caps):
    """per capacity vector, the runs that went onto each shared group's stack in tools/greedy_static_model.py's pass
    (what k_greedy_scan_multi keeps per vector)"""
    import greedy_static_model as gm
    servers, _, _ = t.to_model()
    out = []
    for cap in caps:
        pushes = []
        gm.static_allocate(servers, [int(c) for c in cap], pushes)
        out.append(tuple(pushes))
    return out
