"""GPU: the limited-capacity solve on injected candidate tables, every solver path against the oracle.

The tables of tests/solve_inject_tables.py are written over the resident pair arrays (wva_pairs_device + wva_pairs_commit,
the door the host-driven multi-GPU flow uses), so the solver is tested apart from pair sizing, at accelerator, type,
priority, capacity and replica counts the synthetic generator never produces.  Decisions, scaled records and per-type
totals are compared bit for bit with oracle.solve / oracle.allocate_by_type on the same arrays, for the static-order scan
(path 3), the ranked queue (2) and the heap (1), every saturation policy and both best-effort schedules.  That the tables
reach the branches they are built for is asserted on the CPU (tests/test_solve_inject_cpu.py); here each test asserts the
path that ran and what the scan's counters show.

Every table is a legal input: acc is -1 or the record's accelerator, feasible is 0 or 1, types lie below T, priorities in
[1, 100].  Under the round-robin policies available / units stays near 1e5 (the oracle hands out one replica per round);
tables with larger capacities are solved with the policies None and PriorityExhaustive only.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import solve_inject_tables as st

pytestmark = pytest.mark.gpu

IDS = [c[0] for c in st.CASES]


def _inject(ctx, t):
    """size the (zero-load) pairs so that the resident arrays are valid, then write the table over them"""
    import torch
    from inferno_autoscaler_b200 import distributed
    ctx.analyze_pairs(download=False)
    dev = torch.device("cuda", ctx.device)
    n = t.img.S * t.img.A
    ptrs = ctx.pairs_device()
    with torch.cuda.stream(torch.cuda.ExternalStream(ctx.stream(), device=dev)):
        for name, (ptr, dt) in ptrs.items():
            src = t.feasible if name == "feasible" else getattr(t.pairs, name)
            distributed.device_tensor(ptr, n, dt, dev).copy_(torch.from_numpy(src))
    ctx.pairs_commit()                                   # synchronises the device


def inject_and_solve(ctx, t, *, delayed, policy, ranked):
    """-> (acc, chosen, path, stats, count, cost) of one limited solve of table `t` on the chosen solver setting; the
    image must be uploaded.  A limited solve scales records in place, so every solve injects afresh."""
    _inject(ctx, t)
    ctx.solve_set_ranked(ranked)
    try:
        acc, chosen = ctx.solve(unlimited=False, delayed_best_effort=delayed, policy=policy)
        path, stats = ctx.solve_greedy_path(), ctx.solve_stats()
    finally:
        ctx.solve_set_ranked(2)
    f_acc, f_chosen = ctx.solution_fetch()
    assert np.array_equal(f_acc, acc) and f_chosen.equal_bits(chosen)[0]
    count, cost = ctx.allocate_by_type()
    return acc, chosen, path, stats, count, cost


def _same_floats(a, b):
    """bit for bit, except that two NaNs are equal whatever their payload (as AllocArrays.equal_bits has it: an invalid
    operation yields 0xFFC00000 on amd64 and 0x7FFFFFFF on the GPU)"""
    both = np.isnan(a) & np.isnan(b)
    return np.array_equal(np.where(both, np.uint32(0), a.view(np.uint32)), np.where(both, np.uint32(0), b.view(np.uint32)))


def expected_path(t, ranked):
    """what wva_solve picks by itself: the scan up to 32 accelerators, the ranked queue while its bitmap fits, the heap"""
    n = t.img.S * t.img.A
    bitmap = (-(-n // 64) + -(-n // 4096) + -(-n // 262144) + 1) * 8
    if ranked >= 2 and t.img.A <= 32:
        return 3
    return 2 if ranked >= 1 and bitmap + 4096 <= 220 * 1024 else 1


def compare(ctx, oracle, t, *, policies=None, schedules=(False, True), settings=(2, 1, 0)):
    """all requested (policy, schedule, solver setting) of one table against the oracle; returns the paths that ran and
    the scan's counters"""
    ctx.upload(t.img)
    paths, scan_stats = set(), []
    for policy in (t.policies() if policies is None else policies):
        for delayed in schedules:
            w_acc, w_chosen = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
            w_count, w_cost = oracle.allocate_by_type(t.img, w_acc, w_chosen)
            for ranked in settings:
                acc, chosen, path, stats, count, cost = inject_and_solve(ctx, t, delayed=delayed, policy=policy, ranked=ranked)
                what = (t.kind, policy, delayed, ranked, path)
                assert path == expected_path(t, ranked), what
                assert np.array_equal(acc, w_acc), what + (np.nonzero(acc != w_acc)[0][:8],)
                ok, field = chosen.equal_bits(w_chosen)
                assert ok, what + (field,)
                assert np.array_equal(count, w_count) and _same_floats(cost, w_cost), what
                paths.add(path)
                if path == 3:
                    scan_stats.append(stats)
    return paths, scan_stats


@pytest.mark.parametrize("case", st.CASES, ids=IDS)
def test_injected_table_all_paths(oracle, ctx, case):
    """families 1 and 3-8: every policy, both schedules, the default setting and the two fallbacks.  Up to 32 accelerators
    that is scan / ranked queue / heap; above, the default falls back to the ranked queue by itself."""
    t = st.case_table(case)
    paths, scan_stats = compare(ctx, oracle, t)
    if t.img.A <= 32:
        assert paths == {3, 2, 1}
    else:
        assert paths == {2, 1}
    if case[1] == "accels" and 2 < t.img.A <= 32:
        # shared groups were met with runs waiting on their stacks, and those runs were popped
        assert any((s[0] >> 32) > 0 and (s[1] >> 32) > 0 for s in scan_stats), case[0]


@pytest.mark.parametrize("case", st.LARGE, ids=[c[0] for c in st.LARGE])
def test_automatic_fallback_large(oracle, ctx, case):
    """family 2: more states than the ranked queue's bitmap holds.  64 accelerators: the default setting goes to the heap
    by itself.  32 accelerators: the scan takes them, and asking for the ranked queue falls to the heap."""
    t = st.case_table(case)
    settings = (2,) if t.img.A > 32 else (2, 1)
    ctx.upload(t.img)
    seen = set()
    for policy, delayed in ((st.abi.POLICY_PRIORITY_EXHAUSTIVE, False), (st.abi.POLICY_ROUND_ROBIN, True)):
        w_acc, w_chosen = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
        w_count, w_cost = oracle.allocate_by_type(t.img, w_acc, w_chosen)
        for ranked in settings:
            acc, chosen, path, stats, count, cost = inject_and_solve(ctx, t, delayed=delayed, policy=policy, ranked=ranked)
            assert path == expected_path(t, ranked) == (3 if (t.img.A <= 32 and ranked == 2) else 1)
            assert np.array_equal(acc, w_acc), (policy, delayed, ranked)
            ok, field = chosen.equal_bits(w_chosen)
            assert ok, (policy, delayed, ranked, field)
            assert np.array_equal(count, w_count) and _same_floats(cost, w_cost)
            seen.add(path)
    assert seen == ({1} if t.img.A > 32 else {3, 1})


def test_round_robin_closed_form(oracle, ctx):
    """family 6's round-robin case: more than 10^4 rounds on two types, tickets of unequal units dropping out between the
    closed-form jumps, a partial last round"""
    t = st.round_robin_case()
    compare(ctx, oracle, t, policies=st.ROUND_ROBIN)
    acc, chosen = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, policy=st.abi.POLICY_ROUND_ROBIN)
    assert chosen.num_replicas.max() >= 10_000 and len(set(chosen.num_replicas.tolist())) >= 4


def test_more_than_256_types_is_rejected(wva, oracle, ctx):
    """T = 257: the limited solve is refused, the context still solves unlimited and takes the next upload"""
    from inferno_autoscaler_b200 import binding
    rng = np.random.Generator(np.random.PCG64(42))
    t = st.make_table(rng, 30, 8, 257, "types", type_map="scatter")
    ctx.upload(t.img)
    _inject(ctx, t)
    with pytest.raises(binding.WvaError) as e:
        ctx.solve(unlimited=False)
    assert e.value.code == wva.abi.EINVAL
    acc, chosen = ctx.solve(unlimited=True)
    w_acc, w_chosen = oracle.solve(t.img, t.pairs, t.feasible, unlimited=True)
    assert np.array_equal(acc, w_acc) and chosen.equal_bits(w_chosen)[0]
    t2 = st.make_table(rng, 30, 8, 256, "types", type_map="scatter")
    assert compare(ctx, oracle, t2, policies=(st.abi.POLICY_PRIORITY_EXHAUSTIVE,))[0] == {3, 2, 1}


def test_fuzz_small_tables(oracle, ctx):
    """family 9: small tables drawing every dimension at once, all policies, both schedules, every path that takes them"""
    n, paths = 0, set()
    for seed, count, a_max in st.FUZZ:
        for t in st.fuzz_tables(seed, count, a_max):
            paths |= compare(ctx, oracle, t)[0]
            n += 1
    assert n == sum(f[1] for f in st.FUZZ) and paths == {3, 2, 1}
