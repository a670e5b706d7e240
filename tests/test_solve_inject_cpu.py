"""CPU: the reference side of tests/test_solve_inject_gpu.py, run end to end without a device.

The candidate tables of tests/solve_inject_tables.py are built for the limited-capacity solver's branches (accelerator
counts, types, priorities, capacities, wrapped counts, special float values, dropped entries).  Here: the generator is
deterministic, every family's table has the property its GPU test relies on, the oracle's `allocate` agrees with a second,
independent restatement of the reference's sorted slice (tools/greedy_static_model.py: `queue_allocate`, and the static-order
form `static_allocate` that k_greedy_scan runs) on keys with NaN, infinities and signed zeros, the oracle finishes on every
table under every policy it is asked to solve, and the closed-form round-robin jump equals the oracle's round-by-round
allocateEqually.
"""
import os
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import greedy_static_model as gm
import solve_inject_tables as st

IDS = [c[0] for c in st.CASES]


def _solve_all(oracle, t):
    """oracle decisions of every (policy, schedule) the table is solved with on the GPU -> {(policy, delayed): (acc, chosen)}"""
    out = {}
    for policy in t.policies():
        for delayed in (False, True):
            out[(policy, delayed)] = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
    return out


def _check_second_witness(oracle, t):
    """policy None: the sorted slice restated in Python, and its static-order form, place the same servers at the same
    candidates as the oracle"""
    servers, avail, orders = t.to_model()
    placed_q, unalloc_q, avail_q = gm.queue_allocate(servers, avail)
    assert (placed_q, sorted(unalloc_q), avail_q) == (lambda r: (r[0], sorted(r[1]), r[2]))(gm.static_allocate(servers, avail))
    assert all(st.I64_MIN <= x <= st.I64_MAX for x in avail_q)
    want = np.full(t.img.S, -1, dtype=np.int32)
    for s, j in placed_q.items():
        want[s] = orders[s][j]
    for delayed in (False, True):
        acc, chosen = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, delayed_best_effort=delayed, policy=st.abi.POLICY_NONE)
        assert np.array_equal(acc, want), (t.kind, delayed, np.nonzero(acc != want)[0][:10])
        placed = acc >= 0
        i = np.arange(t.img.S)[placed] * t.img.A + acc[placed]
        assert np.array_equal(chosen.num_replicas[placed], t.pairs.num_replicas[i])
        assert chosen.value[placed].tobytes() == t.pairs.value[i].tobytes()
    return placed_q, unalloc_q


def test_generator_is_deterministic():
    for case in st.CASES[::5]:
        a, b = st.case_table(case), st.case_table(case)
        assert a.feasible.tobytes() == b.feasible.tobytes()
        assert all(getattr(a.pairs, n).tobytes() == getattr(b.pairs, n).tobytes() for n, _ in st.abi.ALLOC_FIELDS)
        assert all(getattr(a.img, n).tobytes() == getattr(b.img, n).tobytes() for n, _ in a.img.ALL_FIELDS)


@pytest.mark.parametrize("case", st.CASES, ids=IDS)
def test_tables_stay_inside_what_the_kernels_index(case):
    t = st.case_table(case)
    img, A = t.img, t.img.A
    own = np.tile(np.arange(A, dtype=np.int32), img.S)
    assert ((t.pairs.acc == -1) | (t.pairs.acc == own)).all()
    assert set(np.unique(t.feasible)) <= {0, 1}
    assert (img.acc_type >= 0).all() and (img.acc_type < img.T).all() and img.T <= 256
    assert (img.srv_priority >= 1).all() and (img.srv_priority <= 100).all()
    assert (img.srv_model >= -1).all() and (img.srv_model < img.M).all()
    assert (img.srv_arrival_rpm == 0).all()
    cnt, _ = st.counts_array(t)
    assert (cnt != st.I64_MIN).all() and (cnt[cnt < 0] > -(1 << 40)).all() and (img.type_capacity <= (1 << 62)).all()
    if not t.huge:                                   # the round-robin bound: one oracle round per replica
        assert img.type_capacity.max() <= st.ROUND_ROBIN_ROUNDS


@pytest.mark.parametrize("case", st.CASES, ids=IDS)
def test_oracle_against_second_witness(oracle, case):
    t = st.case_table(case)
    t0 = time.perf_counter()
    sol = _solve_all(oracle, t)
    dt = time.perf_counter() - t0
    print("%s: oracle %.3f s for %d solves" % (case[0], dt, len(sol)))
    assert dt < 60.0
    _check_second_witness(oracle, t)


def family_reach(oracle, kind):
    """sums over the family's tables, policies and schedules of what the reference side went through, plus the tables'
    static-order structure; the GPU file asserts the same sums before it compares"""
    tot = {}
    for case in st.CASES:
        if case[1] != kind:
            continue
        t = st.case_table(case)
        servers, avail, orders = t.to_model()
        placed, unalloc, _ = gm.queue_allocate(servers, avail)
        add = dict(t.structure())
        add["longest_run"] = 0
        add["placed"], add["unallocated"] = len(placed), len(unalloc)
        add["unallocated_priorities"] = len({int(t.img.srv_priority[s]) for s in unalloc})
        add["deep16"] = 0
        for k, (acc, chosen) in _solve_all(oracle, t).items():
            r = st.reach(t, acc, chosen)
            add["deep16"] += r["deepest"] >= 16
            for f in ("negative_placed", "best_effort", "unplaced"):
                add[f] = add.get(f, 0) + r[f]
            if k[0] == st.abi.POLICY_PRIORITY_EXHAUSTIVE:          # best effort went past a candidate without accelerator
                add["skipped_then_served"] = add.get("skipped_then_served", 0) + sum(
                    1 for s in unalloc if acc[s] >= 0 and
                    any(t.pairs.acc[s * t.img.A + b] < 0 for b in t.order(s)[:t.order(s).index(int(acc[s]))]))
        for f, v in add.items():
            tot[f] = tot.get(f, 0) + int(v)
    return tot


REACH = {
    "accels": ("shared_keys", "stacked_runs", "smaller_later", "larger_later", "deep16", "unallocated", "best_effort"),
    "types": ("placed", "unallocated", "best_effort", "stacked_runs"),
    "priorities": ("unallocated", "best_effort"),
    "capacities": ("placed", "unallocated"),
    "wrap": ("negative_placed", "best_effort", "unplaced"),
    "wrap_huge": ("negative_placed",),
    "values": ("shared_keys", "stacked_runs", "smaller_later", "larger_later", "unallocated"),
    "dropped": ("placed", "unallocated", "best_effort"),
}


@pytest.mark.parametrize("kind", sorted(REACH))
def test_family_reaches_its_branches(oracle, kind):
    tot = family_reach(oracle, kind)
    print(kind, tot)
    for f in REACH[kind]:
        assert tot[f] > 0, (kind, f, tot)
    if kind == "priorities":
        assert tot["unallocated_priorities"] > 10                      # best effort runs at many priority changes


@pytest.mark.parametrize("case", st.CASES, ids=IDS)
def test_table_has_its_family_property(case):
    t = st.case_table(case)
    name, kind, A = case[0], case[1], t.img.A
    if kind == "accels":
        assert (t.feasible == 1).all() and t.structure()["longest_run"] >= max(A - 1, 1)
    elif kind == "types":
        used = np.unique(t.img.acc_type)
        if "high" in name:
            assert used.max() == t.img.T - 1 and used.min() >= t.img.T - 32
        if name in ("types-A256-T256", "types-A64-T256"):
            assert max(len({int(t.img.acc_type[a]) for a in t.order(s)}) for s in range(t.img.S)) > 32
        if t.img.T < A or "low" in name:
            assert len(used) < A                                        # some types are shared by several accelerators
    elif kind == "priorities":
        pr = np.unique(t.img.srv_priority, return_counts=True)
        assert pr[0].min() == 1 and pr[0].max() == 100 and 85 <= len(pr[0]) < 100 and (pr[1] == 1).any() and (pr[1] > 3).any()
    elif kind == "capacities":
        cap = t.img.type_capacity
        assert not np.isin(np.arange(t.img.T), t.img.acc_type).all()                # a type nobody maps to
        if name == "capacities-zero":
            assert (cap == 0).all()
        elif name == "capacities-first-type-empty":
            assert all(t.order(s)[0] == 0 for s in range(t.img.S)) and cap[t.img.acc_type[0]] == 0 and cap.max() > 0
    elif kind in ("wrap", "wrap_huge"):
        cnt, units = st.counts_array(t)
        reps = t.pairs.num_replicas
        assert ((cnt < 0) & (reps > 0)).any() and ((cnt == 0) & (reps != 0) & (units > 0)).any()       # products that wrap
        assert (reps == st.I64_MIN).any() and (reps == 0).any() and (t.img.type_capacity < 0).any()
    elif kind == "values":
        v = t.pairs.value
        assert np.isnan(v).any() and np.isinf(v).any() and (v.view(np.uint32) == 0x80000000).any()
        assert any(K[0] == (1, 0.0) for s in range(t.img.S) for K in t.keys(s))     # a NaN delta
    elif kind == "dropped":
        assert (t.img.srv_model < 0).any() and (t.feasible.reshape(t.img.S, A).sum(axis=1) == 0).any()
        where = set()
        for s in range(t.img.S):
            o = t.order(s)
            for k, a in enumerate(o):
                if t.pairs.acc[s * A + a] < 0 and len(o) >= 3:
                    where.add("first" if k == 0 else "last" if k == len(o) - 1 else "middle")
        assert where == {"first", "middle", "last"}


def test_ample_and_zero_capacities(oracle):
    by = {c[0]: c for c in st.CASES}
    t = st.case_table(by["capacities-ample"])
    for k, (acc, chosen) in _solve_all(oracle, t).items():          # every server at its first candidate, nothing scaled
        has = [s for s in range(t.img.S) if t.order(s)]
        assert len(has) > 100 and all(acc[s] == t.order(s)[0] for s in has) and st.reach(t, acc, chosen)["best_effort"] == 0
    t = st.case_table(by["capacities-zero"])
    for k, (acc, chosen) in _solve_all(oracle, t).items():
        assert (acc == -1).all()
    t = st.case_table(by["capacities-first-type-empty"])
    acc, _ = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, policy=0)
    assert (acc > 0).any() and not (acc == 0).any()


def test_fuzz_tables_oracle_and_second_witness(oracle):
    t0 = time.perf_counter()
    n = 0
    seen = dict(negative_placed=0, best_effort=0, unplaced=0, deep=0)
    for seed, count, a_max in st.FUZZ:
        for t in st.fuzz_tables(seed, count, a_max):
            assert t.huge or t.img.type_capacity.max() <= st.ROUND_ROBIN_ROUNDS
            sol = _solve_all(oracle, t)
            _check_second_witness(oracle, t)
            for k in sol:
                r = st.reach(t, *sol[k])
                seen["negative_placed"] += r["negative_placed"]; seen["best_effort"] += r["best_effort"]
                seen["unplaced"] += r["unplaced"]; seen["deep"] += r["deepest"] >= 16
            n += 1
    print("fuzz: %d tables, oracle and both restatements in %.1f s, %s" % (n, time.perf_counter() - t0, seen))
    assert all(v > 0 for v in seen.values()), seen


def test_round_robin_closed_form_equals_round_by_round(oracle):
    """greedy_allocate_equally applies k whole rounds at once; the oracle hands out one replica per round"""
    t = st.round_robin_case()
    A = t.img.A
    first = [t.order(s)[0] for s in range(t.img.S)]
    assert all(t.count(s, first[s]) > int(t.img.type_capacity[t.img.acc_type[first[s]]]) for s in range(t.img.S))   # everyone fails
    # one candidate each: delta MaxFloat32 for all, so the unallocated list is in descending value
    servers = sorted(range(t.img.S), key=lambda s: -float(t.pairs.value[s * A + first[s]]))
    got, left = st.equally_closed_form(t, servers)
    assert max(got.values()) >= 10_000 and len(set(got.values())) >= 3 and all(0 <= x < 5 for x in left)
    for policy in st.ROUND_ROBIN:
        for delayed in (False, True):
            acc, chosen = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
            for s in range(t.img.S):
                if got[s] == 0:
                    assert acc[s] == -1
                    continue
                assert acc[s] == first[s] and chosen.num_replicas[s] == got[s]
                cost, value = st.scaled(t, s, first[s], got[s])
                assert chosen.cost[s].tobytes() == cost.tobytes() and chosen.value[s].tobytes() == value.tobytes()
    count, _ = oracle.allocate_by_type(t.img, acc, chosen)
    assert np.array_equal(count, t.img.type_capacity - np.array(left))


def test_large_tables_oracle_time(oracle):
    """the two large tables of the automatic fallbacks: the oracle's slice erases from the front, so its time is checked
    here, and the state counts lie on the intended sides of the ranked queue's reach"""
    bitmap = lambda n: (-(-n // 64) + -(-n // 4096) + -(-n // 262144) + 1) * 8       # greedy_bitmap_bytes
    for case in st.LARGE:
        t = st.case_table(case)
        assert bitmap(t.img.S * t.img.A) + 4096 > 220 * 1024 and t.img.S * t.img.A < (1 << 24)
        for policy, delayed in ((st.abi.POLICY_PRIORITY_EXHAUSTIVE, False), (st.abi.POLICY_ROUND_ROBIN, True)):
            t0 = time.perf_counter()
            acc, chosen = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
            dt = time.perf_counter() - t0
            print("%s policy %d delayed %d: oracle %.2f s, %d unplaced" % (case[0], policy, delayed, dt, int((acc < 0).sum())))
            assert dt < 60.0
            r = st.reach(t, acc, chosen)
            assert r["unplaced"] > 0 and r["deepest"] >= 1
