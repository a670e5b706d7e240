"""CPU: the capacity lists of tests/solve_capacities_cases.py reach the branches they are built for (checked with the oracle
and tools/greedy_static_model.py), the static-order pass equals the reference's queue under every vector, and the C-ABI
of wva_solve_capacities compiles as C99, links and rejects bad arguments without a device."""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import greedy_static_model as gm  # noqa: E402
import solve_capacities_cases as sc  # noqa: E402
import solve_inject_tables as st  # noqa: E402

abi = st.abi


def _generated(wva, oracle, S=200, A=8, T=3, seed=3):
    img = wva.synth.make_system(S, A, seed=seed, n_types=T)
    pairs, feasible, _ = oracle.analyze_pairs(img)
    return img, pairs, feasible


def test_ladder_shape_and_branches(wva, oracle):
    """64 vectors; placements change along the fractions; some vectors exhaust a type, some place everyone; best effort
    hands out fewer replicas than asked somewhere"""
    img, pairs, feasible = _generated(wva, oracle)
    caps = sc.ladder(img, pairs, feasible, oracle)
    assert caps.shape == (sc.N_LADDER, img.T) and caps.dtype == np.int64
    assert (caps == 0).all(axis=1).any() and (caps < 0).all(axis=1).any() and (caps == 1 << 62).all(axis=1).any()
    acc, recs, count, _ = sc.expected(oracle, img, pairs, feasible, caps, False, abi.POLICY_PRIORITY_EXHAUSTIVE)
    ladder = acc[1:1 + len(sc.FRACTIONS)]
    assert len({a.tobytes() for a in ladder}) >= len(sc.FRACTIONS) // 2
    placed = (acc >= 0).sum(axis=1)
    assert placed.min() == 0 and placed.max() >= 0.9 * (oracle.solve(img, pairs, feasible, unlimited=True)[0] >= 0).sum()
    asked = pairs.num_replicas.reshape(img.S, img.A)
    short = 0
    for j in range(len(caps)):
        placed = acc[j] >= 0
        s = np.nonzero(placed)[0]
        short += int((recs[j]["num_replicas"][s] < asked[s, acc[j][s]]).sum())
    assert short > 0
    exhausted = 0
    for j in range(len(caps)):
        exhausted += int(((caps[j] > 0) & (count[j] == caps[j])).any())
    assert exhausted > 0
    # the starved vectors: nothing lands on the starved type
    for t in range(img.T):
        j = 1 + len(sc.FRACTIONS) + 5 + t
        assert caps[j][t] == 0 and count[j][t] == 0 and (caps[j] == sc.PLENTY).sum() == img.T - 1


def test_round_robin_ladder_is_capped(wva, oracle):
    img, pairs, feasible = _generated(wva, oracle, S=60, A=4, T=2, seed=4)
    caps = sc.ladder(img, pairs, feasible, oracle, round_robin=True)
    assert caps.max() <= st.ROUND_ROBIN_ROUNDS


def _table_vectors(t, n, seed):
    dem, one = st.first_counts(t)
    rng = np.random.default_rng(seed)
    rows = [t.img.type_capacity.astype(np.int64), np.zeros(t.img.T, dtype=np.int64)]
    while len(rows) < n:
        rows.append((rng.choice([0.0, 0.1, 0.3, 0.5, 0.8, 1.0, 1.5], t.img.T) * np.array(dem)).astype(np.int64))
    return np.minimum(np.array(rows, dtype=np.int64), st.ROUND_ROBIN_ROUNDS)


def test_stacks_differ_between_vectors():
    """the same shared groups receive different runs under different vectors: one stack per vector is needed"""
    for name in ("accels-A8", "accels-A16", "accels-A32"):
        t = st.case_table(next(c for c in st.CASES if c[0] == name))
        pushes = sc.stacks_per_vector(t, _table_vectors(t, 8, 1))
        assert any(pushes), name
        assert len(set(pushes)) >= 3, name


def test_static_order_equals_queue_for_every_vector():
    for name in ("accels-A8", "accels-A32", "wrap-500", "values-600", "dropped-700", "priorities"):
        t = st.case_table(next(c for c in st.CASES if c[0] == name))
        servers, _, _ = t.to_model()
        for cap in _table_vectors(t, 8, 2):
            avail = [int(c) for c in cap]
            assert gm.queue_allocate(servers, avail) == gm.static_allocate(servers, avail), (name, avail)


def test_oracle_loop_agrees_with_table_capacity(oracle):
    """the fixture's expected() at the table's own capacity is one plain oracle solve"""
    t = st.case_table(next(c for c in st.CASES if c[0] == "capacities-400"))
    caps = t.img.type_capacity[None, :].astype(np.int64)
    acc, recs, count, cost = sc.expected(oracle, t.img, t.pairs, t.feasible, caps, True, abi.POLICY_PRIORITY_ROUND_ROBIN)
    a, ch = oracle.solve(t.img, t.pairs, t.feasible, unlimited=False, delayed_best_effort=True, policy=abi.POLICY_PRIORITY_ROUND_ROBIN)
    assert np.array_equal(acc[0], a) and sc.same_recs(recs[0], sc.to_recs(a, ch)) is None
    w_count, w_cost = oracle.allocate_by_type(t.img, a, ch)
    assert np.array_equal(count[0], w_count) and sc.same_floats(cost[0], w_cost)


def test_record_dtype_and_header():
    assert abi.PAIR_REC_DTYPE.itemsize == 48 and abi.SOLVE_MAX_CAPACITIES == 8192
    hdr = open(os.path.join(ROOT, "include", "wva_b200.h")).read()
    assert "#define WVA_SOLVE_MAX_CAPACITIES 8192" in hdr
    for name in ("wva_solve_capacities(", "wva_solve_capacities_counters(", "wva_solve_capacities_set_budget(",
                 "wva_group_solve_capacities("):
        assert name in hdr, name


def test_c99_declarations_link_and_reject_null(wva):
    import __graft_entry__ as g
    g.build_cuda()
    host = os.path.join(ROOT, "inferno-autoscaler_b200", "host")
    libdir = os.path.dirname(g.LIB)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "solve_capacities_c99")
        subprocess.check_call([os.environ.get("CC", "cc"), "-std=c99", "-O1", "-Wall", "-Wextra", "-pedantic", "-Werror",
                               "-I" + os.path.join(ROOT, "include"), "-o", exe, os.path.join(host, "solve_capacities_c99.c"),
                               "-L" + libdir, "-lwva_b200", "-Wl,-rpath," + libdir])
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "solve_capacities c99: ok" in out.stdout, out.stdout + out.stderr

