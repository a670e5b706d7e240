"""Candidate tables for the limited-capacity solver, built for its branches rather than by pair sizing.

`make_table(rng, S, A, T, kind)` returns a `Table`: a SystemImage whose servers carry no load (pair sizing on it is instant
and only makes the resident pair arrays valid) plus the S*A candidate records and feasibility flags that a test writes
over those arrays before a limited solve.  Values, replica counts, units and capacities come from small discrete sets, so
equal keys, equal counts and exhausted types are the norm.  Shared by tests/test_solve_inject_cpu.py (properties of the
tables, the oracle against a second restatement) and tests/test_solve_inject_gpu.py (the three solver paths against
the oracle).

What every table keeps, because the kernels index with it and the oracle's arithmetic relies on it:
  * acc is -1 or the record's own accelerator index, feasible is 0 or 1, acc_type < T, priorities lie in [1, 100];
  * `available - count` never leaves int64: capacities are at most 2^62, negative counts are small, and no candidate's
    wrapped count is MinInt64 (the oracle subtracts with a plain signed `-=`);
  * under the two round-robin policies `available / units` stays near 1e5 at most, because the oracle's allocateEqually
    hands out one replica per round; tables with larger capacities say `huge=True` and are solved with the policies None
    and PriorityExhaustive only.
"""
import numpy as np

import wva_import

_wva = wva_import.load()
abi = _wva.abi
SystemImage = _wva.image.SystemImage

MAXF = np.float32(3.4028234663852886e38)
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
ROUND_ROBIN_ROUNDS = 100_000                     # bound on available / units where a round-robin policy is solved

ORDINARY = np.array([0.0, 1.0, 2.0, 2.5, 7.0, 40.0, 40.5, 100.0, 250.0], dtype=np.float32)
SPECIAL = np.array([-np.inf, -3e38, -1.0, -0.0, 0.0, 1e-45, 1.0, 1.0 + 2.0 ** -23, 3e38, MAXF, np.inf, np.nan, 2.0, 40.0],
                   dtype=np.float32)
TAME_REPS = [1, 1, 2, 3, 5, 40]
WRAP_REPS = [0, 1, (1 << 31) - 1, 1 << 31, 1 << 40, 1 << 62, I64_MIN, -1, I64_MAX, 2, 3]

POLICIES = (abi.POLICY_NONE, abi.POLICY_PRIORITY_EXHAUSTIVE, abi.POLICY_PRIORITY_ROUND_ROBIN, abi.POLICY_ROUND_ROBIN)
ROUND_ROBIN = (abi.POLICY_PRIORITY_ROUND_ROBIN, abi.POLICY_ROUND_ROBIN)


def wrap64(x):
    """Go's int64 arithmetic: the low 64 bits, signed"""
    return ((int(x) + (1 << 63)) % (1 << 64)) - (1 << 63)


class Table:
    def __init__(self, img, pairs, feasible, kind, huge=False):
        self.img, self.pairs, self.feasible, self.kind, self.huge = img, pairs, feasible, kind, huge

    def policies(self):
        return tuple(p for p in POLICIES if not (self.huge and p in ROUND_ROBIN))

    # ---- the quantities greedy.go computes from a record, in Python integers wrapped by hand --------------------------
    def units(self, s, a):
        """model.NumInstances(acc) * multiplicity of record (s, a); None where the entry is dropped (no model / no accelerator)"""
        img = self.img
        m, gi = int(img.srv_model[s]), int(self.pairs.acc[s * img.A + a])
        if m < 0 or gi < 0:
            return None
        n = int(img.perf_acc_count[m * img.A + gi])
        return wrap64((n if n > 0 else 1) * int(img.acc_multiplicity[gi]))

    def count(self, s, a):
        u = self.units(s, a)
        return None if u is None else wrap64(int(self.pairs.num_replicas[s * self.img.A + a]) * u)

    def order(self, s):
        """the server's feasible accelerators, stable-sorted by cmp.Compare(value): NaN first, -0 == +0"""
        A = self.img.A
        idx = [a for a in range(A) if self.feasible[s * A + a]]
        idx.sort(key=lambda a: _cmp_key(self.pairs.value[s * A + a]))
        return idx

    def keys(self, s, order=None):
        """K of each candidate in `order`, ascending = earlier in the reference's slice, without the priority: orderFunc
        compares the delta to the next candidate descending, then the value descending; cmp.Compare puts NaN lowest, and
        two NaN deltas compare equal whatever the values are"""
        A = self.img.A
        order = self.order(s) if order is None else order
        v = [np.float32(self.pairs.value[s * A + a]) for a in order]
        out = []
        with np.errstate(all="ignore"):
            for k in range(len(v)):
                d = np.float32(v[k + 1] - v[k]) if k + 1 < len(v) else MAXF
                if d != d:
                    out.append(((1, 0.0), (0, 0.0)))
                else:
                    out.append(((0, -float(d)), (1, 0.0) if v[k] != v[k] else (0, -float(v[k]))))
        return out

    def to_model(self):
        """(servers, avail) in the format of tools/greedy_static_model.py, and each server's candidate order"""
        img = self.img
        servers, orders = [], []
        for s in range(img.S):
            order = self.order(s)
            cands = []
            for a, K in zip(order, self.keys(s, order)):
                c = self.count(s, a)
                if c is None:
                    cands.append((K, 0, 0, True))
                else:
                    cands.append((K, int(img.acc_type[int(self.pairs.acc[s * img.A + a])]), c, False))
            servers.append((int(img.srv_priority[s]), cands))
            orders.append(order)
        return servers, [int(c) for c in img.type_capacity], orders

    def structure(self):
        """what the static order looks like: the longest run, the (priority, M) keys shared by several servers, the runs
        that wait on a shared key's stack (they do not start at candidate 0), and the servers with a later candidate
        whose key is smaller than an earlier one's (tried at once) or larger (re-inserted further back)"""
        groups, longest, smaller, larger = {}, 0, 0, 0
        runs = []
        for s in range(self.img.S):
            M, start, sm, lg = None, 0, False, False
            ks = self.keys(s)
            for j, K in enumerate(ks):
                if M is None or K > M:
                    if M is not None:
                        runs.append((s, start, j, M)); lg = True
                    M, start = K, j
                elif K < M:
                    sm = True
            if ks:
                runs.append((s, start, len(ks), M))
            smaller += sm; larger += lg
        for s, j0, j1, M in runs:
            longest = max(longest, j1 - j0)
            groups.setdefault((int(self.img.srv_priority[s]), M), set()).add(s)
        shared = {g for g, ss in groups.items() if len(ss) > 1}
        stacked = sum(1 for s, j0, j1, M in runs if j0 > 0 and (int(self.img.srv_priority[s]), M) in shared)
        return dict(longest_run=longest, shared_keys=len(shared), stacked_runs=stacked, smaller_later=smaller, larger_later=larger)


def _cmp_key(v):
    return (0, 0.0) if v != v else (1, float(v))


# ---- profiles: what each family draws from ----------------------------------------------------------------------------
_BASE = dict(values=ORDINARY, costs=ORDINARY[1:], reps=TAME_REPS, mults=[1, 1, 2, 4, 8], acc_counts=[0, 1, 1, 2, 4],
             p_feasible=1.0, p_noacc=0.0, p_nomodel=0.0, p_empty=0.0, prios=[1, 5, 10], type_map="low", protos=4, p_proto=0.6,
             capacity="fractions", fractions=[0.0, 0.2, 0.5, 0.8], long_runs=False, huge=False, deep_last=False, p_big=0.12)
PROFILES = {
    # every server holds all A candidates; prototype rows give equal keys on many servers, two of them built so that one run
    # spans (almost) every candidate.  The last accelerator has a type of its own that keeps some room, so the servers whose
    # order is the accelerator index are placed at their very last candidate once everything before it has failed
    "accels": dict(long_runs=True, deep_last=True, protos=5, p_proto=0.85, prios=[3, 4], fractions=[0.1, 0.3, 0.6], reps=[1, 1, 2, 3, 5, 9]),
    "types": dict(long_runs=True, p_feasible=0.9, fractions=[0.0, 0.3, 0.6, 1.0]),
    "priorities": dict(prios="all100", p_feasible=0.8, fractions=[0.02, 0.05, 0.1]),
    "capacities": dict(capacity="edges", p_feasible=0.9, prios=[1, 2]),
    "wrap": dict(reps=WRAP_REPS, capacity="wrap", prios=[1, 2], p_feasible=0.95, type_map="dense", protos=2, p_proto=0.3),
    "wrap_huge": dict(reps=WRAP_REPS, capacity="wrap_huge", prios=[1, 2], p_feasible=0.95, type_map="dense", protos=2, p_proto=0.3, huge=True),
    "values": dict(values=SPECIAL, costs=SPECIAL, protos=6, p_proto=0.7, prios=[7, 8], fractions=[0.1, 0.3, 0.5]),
    "dropped": dict(p_feasible=0.8, p_noacc=0.15, p_nomodel=0.15, p_empty=0.1, fractions=[0.1, 0.3, 0.6]),
    "fuzz": dict(values=SPECIAL, costs=SPECIAL, reps=TAME_REPS + WRAP_REPS, capacity="fuzz", prios="some", p_feasible=0.85,
                 p_noacc=0.04, p_nomodel=0.05, p_empty=0.05, type_map="scatter", long_runs=True),
    "fuzz_huge": dict(values=SPECIAL, costs=SPECIAL, reps=TAME_REPS + WRAP_REPS, capacity="wrap_huge", prios="some", p_feasible=0.85,
                      p_noacc=0.04, p_nomodel=0.05, p_empty=0.05, type_map="scatter", long_runs=True, huge=True),
    # many servers, few failures: the large tables of the automatic fallbacks (the oracle's slice erases from the front)
    "large": dict(p_feasible=0.5, fractions=[0.9, 0.97, 1.0], reps=[1, 1, 2, 3], prios=[1, 5, 10], protos=3, p_proto=0.3),
}


def _acc_types(rng, A, T, how):
    a = np.arange(A)
    if how == "low":                                  # the lowest indices, neighbours sharing a type now and then
        t = (a * 3 // 4) % T
    elif how == "high":                               # the top of the range: the high end of the record's 8-bit type field
        t = T - 1 - ((a * 3 // 4) % T)
    elif how == "dense":                              # few types, long stretches of one type
        t = (a // 4) % min(T, 2)
    elif how == "one_each":
        t = a % T
    else:                                             # scattered
        t = rng.integers(0, T, A)
    return t.astype(np.int32)


def _long_run_row(A, first_head):
    """a value row whose candidates from `first_head` on form one run: that candidate's delta is the smallest (its key the
    largest), everything after it has the large delta of 100 and is tried back to back"""
    v = np.zeros(A, dtype=np.float32)
    x = 0.0
    for k in range(A):
        v[k] = x
        x += 1.0 if k == first_head else (50.0 if k < first_head else 100.0)
    return v


def make_table(rng, S, A, T, kind, **over):
    p = dict(_BASE); p.update(PROFILES[kind]); p.update(over)
    M = 3
    img = SystemImage(S, A, M, T)
    img.acc_cost[:] = 1.0
    img.acc_multiplicity[:] = rng.choice(np.array(p["mults"], dtype=np.int32), A)
    deep = p["deep_last"] and A > 1 and T > 1
    if deep:
        img.acc_type[:A - 1] = _acc_types(rng, A - 1, T - 1, p["type_map"])
        img.acc_type[A - 1] = T - 1
        img.acc_multiplicity[A - 1] = 1
    else:
        img.acc_type[:] = _acc_types(rng, A, T, p["type_map"])
    img.perf_alpha[:] = 10.0; img.perf_beta[:] = 0.1; img.perf_gamma[:] = 10.0; img.perf_delta[:] = 0.01
    img.perf_max_batch[:] = 8; img.perf_at_tokens[:] = 128
    img.perf_acc_count[:] = rng.choice(np.array(p["acc_counts"], dtype=np.int32), M * A)
    img.perf_valid[:] = 1
    img.srv_model[:] = rng.integers(0, M, S)
    img.srv_model[rng.uniform(0, 1, S) < p["p_nomodel"]] = -1
    img.srv_target_valid[:] = 1
    img.srv_slo_itl[:] = 100.0; img.srv_slo_ttft[:] = 1000.0
    if isinstance(p["prios"], str) and p["prios"] == "all100":
        # every priority from 1 to 100 except a few left empty; 1 and 100 present; some hold one server
        empty = set(int(x) for x in rng.choice(np.arange(2, 100), 7, replace=False))
        present = np.array([q for q in range(1, 101) if q not in empty], dtype=np.int32)
        pr = np.concatenate([present, rng.choice(present[::3], max(S - len(present), 0))])[:S]
        img.srv_priority[:] = rng.permutation(pr)
    elif isinstance(p["prios"], str):
        img.srv_priority[:] = rng.choice(rng.integers(1, 101, int(rng.integers(1, 6))), S)
    else:
        img.srv_priority[:] = rng.choice(np.array(p["prios"], dtype=np.int32), S)

    n = S * A
    pairs = abi.AllocArrays(n)
    feasible = (rng.uniform(0, 1, n) < p["p_feasible"]).astype(np.uint8)
    feasible.reshape(S, A)[rng.uniform(0, 1, S) < p["p_empty"]] = 0
    acc = np.tile(np.arange(A, dtype=np.int32), S)
    acc[rng.uniform(0, 1, n) < p["p_noacc"]] = -1
    pairs.acc[:] = acc
    protos = [rng.choice(p["values"], A) for _ in range(p["protos"])]
    if p["long_runs"]:
        protos += [_long_run_row(A, 0), _long_run_row(A, min(1, A - 1))]
    val = rng.choice(p["values"], (S, A))
    pick = rng.integers(0, len(protos), S)
    use = rng.uniform(0, 1, S) < p["p_proto"]
    for s in np.nonzero(use)[0]:
        val[s] = protos[pick[s]]
    pairs.value[:] = val.reshape(-1)
    pairs.cost[:] = rng.choice(p["costs"], n)
    reps = np.array([wrap64(x) for x in p["reps"]], dtype=np.int64)[rng.integers(0, len(p["reps"]), n)].reshape(S, A)
    # some servers ask for 64 times as much everywhere: they fail on every candidate while room for single replicas is
    # left, which is what best effort then hands out
    big = rng.uniform(0, 1, S) < p["p_big"]
    if deep:
        big |= use & (pick >= p["protos"])
    small = (reps > 0) & (reps < (1 << 20))
    reps[big[:, None] & small] *= 64
    if deep:
        reps[:, A - 1] = 1
    pairs.num_replicas[:] = reps.reshape(-1)
    pairs.batch_size[:] = acc.astype(np.int64) + 1
    pairs.itl[:] = (np.arange(n) % 7).astype(np.float32) + 0.5
    pairs.ttft[:] = (np.arange(n) % 11).astype(np.float32) * 3.0
    pairs.rho[:] = (np.arange(n) % 5).astype(np.float32) / 8.0
    pairs.max_arrv_rate_per_replica[:] = (np.arange(n) % 13).astype(np.float32) / 4.0
    t = Table(img, pairs, feasible, kind, huge=p["huge"])
    # a wrapped count of MinInt64 cannot be subtracted inside int64 from a capacity >= 0: such records keep a wrapping
    # product (MaxInt64 replicas) but lose the one value that would leave the range
    cnt, units = counts_array(t)
    bad = cnt == I64_MIN
    pairs.num_replicas[bad & (units > 1)] = I64_MAX
    pairs.num_replicas[bad & (units <= 1)] = -1
    if p.get("first_zero"):                          # every server tries accelerator 0 first, and its type has nothing
        pairs.value.reshape(S, A)[:, 0] = -5.0
        feasible.reshape(S, A)[:, 0] = 1
        pairs.acc.reshape(S, A)[:, 0] = 0
    img.type_capacity[:] = _capacities(rng, t, p)
    if p.get("first_zero"):
        other = max(first_counts(t)[0]) // 3
        img.type_capacity[:] = np.maximum(img.type_capacity, other)
        img.type_capacity[img.acc_type[0]] = 0
    if p["capacity"] in ("wrap", "wrap_huge"):
        img.type_capacity[img.acc_type[0]] = -5
    if deep:
        img.type_capacity[T - 1] = max(S // 3, 1)
    return t


def counts_array(t):
    """(count, units) of every record as greedy.go computes them (int64 products that wrap); 0 where the entry is dropped"""
    img = t.img
    S, A = img.S, img.A
    m = np.repeat(img.srv_model.astype(np.int64), A)
    gi = t.pairs.acc.astype(np.int64)
    ok = (m >= 0) & (gi >= 0)
    n = img.perf_acc_count[np.where(ok, m * A + gi, 0)].astype(np.int64)
    units = np.where(ok, np.where(n > 0, n, 1) * img.acc_multiplicity[np.where(ok, gi, 0)].astype(np.int64), 0)
    with np.errstate(over="ignore"):
        cnt = (t.pairs.num_replicas.view(np.uint64) * units.view(np.uint64)).view(np.int64)
    return cnt, units


def first_counts(t):
    """per type: the units the servers' first candidates ask for (ordinary positive counts only), and one such count"""
    img = t.img
    S, A = img.S, img.A
    v = t.pairs.value.reshape(S, A)
    nan = np.isnan(v)
    first = np.lexsort((np.where(nan, 0, v), ~nan, t.feasible.reshape(S, A) == 0), axis=-1)[:, 0]     # cmp.Compare order
    i = np.arange(S) * A + first
    cnt, _ = counts_array(t)
    use = (t.feasible[i] == 1) & (t.pairs.acc[i] >= 0) & (cnt[i] > 0) & (cnt[i] < (1 << 40))
    dem, one = [0] * img.T, [1] * img.T
    for ty, c in zip(img.acc_type[first[use]], cnt[i][use]):
        dem[int(ty)] += int(c); one[int(ty)] = int(c)
    return dem, one


def _capacities(rng, t, p):
    T = t.img.T
    dem, one = first_counts(t)
    cap = np.zeros(T, dtype=np.int64)
    how = p["capacity"]
    for ty in range(T):
        if how == "fractions":
            cap[ty] = int(float(rng.choice(p["fractions"])) * dem[ty])
        elif how == "zero":
            cap[ty] = 0
        elif how == "ample":                         # exactly what the first candidates ask for: nothing fails
            cap[ty] = dem[ty]
        elif how == "edges":
            cap[ty] = int(rng.choice(np.array([0, 1, one[ty] - 1, one[ty], one[ty] + 1, sum(dem), dem[ty] // 2, dem[ty] // 3], dtype=object)))
        elif how == "wrap":                          # small, some negative: a count of 0 fails there until a negative count lifts it
            cap[ty] = int(rng.choice(np.array([-5, 0, 3, 40, 1000, ROUND_ROBIN_ROUNDS], dtype=object)))
        elif how == "wrap_huge":
            cap[ty] = int(rng.choice(np.array([-5, 0, 40, (1 << 31) + 5, (1 << 40) + (1 << 36), 1 << 62], dtype=object)))
        else:                                        # fuzz: everything above that a round-robin policy can follow
            cap[ty] = int(rng.choice(np.array([-5, 0, 1, one[ty], dem[ty] // 3, dem[ty] // 2, dem[ty], 1000, ROUND_ROBIN_ROUNDS], dtype=object)))
        if not p["huge"]:                            # the round-robin bound
            cap[ty] = min(int(cap[ty]), ROUND_ROBIN_ROUNDS)
    return cap


def round_robin_case():
    """Four servers of one priority whose only candidate fails and which then share two types round by round: units of
    1, 2, 3 and 5 per replica, capacities of 50 003 and 61 007, so more than 10^4 rounds are handed out, the tickets on the
    first type run dry before those on the second, and the last round is partial"""
    S, A, T = 6, 4, 2
    img = SystemImage(S, A, 1, T)
    img.acc_cost[:] = 1.0
    img.acc_multiplicity[:] = [1, 2, 3, 5]
    img.acc_type[:] = [0, 0, 1, 1]
    img.perf_alpha[:] = 10.0; img.perf_beta[:] = 0.1; img.perf_gamma[:] = 10.0; img.perf_delta[:] = 0.01
    img.perf_max_batch[:] = 8; img.perf_at_tokens[:] = 128; img.perf_acc_count[:] = 1; img.perf_valid[:] = 1
    img.srv_target_valid[:] = 1
    img.srv_priority[:] = 4
    img.type_capacity[:] = [50_003, 61_007]
    pairs = abi.AllocArrays(S * A)
    feasible = np.zeros(S * A, dtype=np.uint8)
    pairs.acc[:] = np.tile(np.arange(A, dtype=np.int32), S)
    want = [(0, 100_000), (1, 70_000), (2, 90_000), (3, 60_000), (1, 30_001), (3, 1 << 40)]
    for s, (a, reps) in enumerate(want):
        i = s * A + a
        feasible[i] = 1
        pairs.num_replicas[i] = reps
        pairs.cost[i] = np.float32(3.0 * reps)
        pairs.value[i] = np.float32(7.0 + s)
    return Table(img, pairs, feasible, "round_robin")


def equally_closed_form(t, servers):
    """numpy restatement of the jump greedy_allocate_equally makes: `servers` in list order, each with one candidate.
    Round 1 gives every ticket that fits one replica; then, as long as tickets are live, one ordinary round followed by
    k = min over types of available // (units of the live tickets) whole rounds at once.  Returns replicas per server."""
    img = t.img
    avail = [int(c) for c in img.type_capacity]
    tk = []
    for s in servers:
        a = t.order(s)[0]
        tk.append(dict(s=s, a=a, upr=t.units(s, a), ty=int(img.acc_type[a]), cur=int(t.pairs.num_replicas[s * img.A + a]), got=0))
    live = []
    for x in tk:
        if x["upr"] > 0 and avail[x["ty"]] >= x["upr"] and x["cur"] > 0:
            x["got"] = 1; avail[x["ty"]] -= x["upr"]; live.append(x)
    while live:
        nxt = []
        for x in live:
            if avail[x["ty"]] >= x["upr"]:
                x["got"] += 1; avail[x["ty"]] -= x["upr"]; nxt.append(x)
        live = nxt
        if not live:
            break
        usum = np.zeros(img.T, dtype=np.int64)
        for x in live:
            usum[x["ty"]] += x["upr"]
        k = min(avail[ty] // int(usum[ty]) for ty in range(img.T) if usum[ty] > 0)
        if k > 0:
            for ty in range(img.T):
                avail[ty] -= k * int(usum[ty])
            for x in live:
                x["got"] += k
    return {x["s"]: x["got"] for x in tk}, avail


def scaled(t, s, a, got):
    """the record of (s, a) after best effort gave it `got` of its replicas (greedy.go:208-212): cost and value times
    float32(got) / float32(cur)"""
    i = s * t.img.A + a
    f = np.float32(got) / np.float32(int(t.pairs.num_replicas[i]))
    return np.float32(t.pairs.cost[i] * f), np.float32(t.pairs.value[i] * f)


def reach(t, acc, chosen):
    """what a solve of `t` went through, from the reference side's decisions alone"""
    img = t.img
    A = img.A
    idx_max, neg_placed, short, unplaced = -1, 0, 0, 0
    for s in range(img.S):
        o = t.order(s)
        if not o:
            continue
        a = int(acc[s])
        if a < 0:
            unplaced += 1
            continue
        idx_max = max(idx_max, o.index(a))
        c = t.count(s, a)
        if c is not None and c < 0 and int(chosen.num_replicas[s]) == int(t.pairs.num_replicas[s * A + a]):
            neg_placed += 1
        if int(chosen.num_replicas[s]) != int(t.pairs.num_replicas[s * A + a]):
            short += 1
    return dict(deepest=idx_max, negative_placed=neg_placed, best_effort=short, unplaced=unplaced)


# ---- the families: (id, kind, seed, S, A, T, overrides) ------------------------------------------------------------------
def _cases():
    c = []
    for A in (1, 2, 7, 8, 9, 16, 17, 21, 31, 32):                                   # the scan's 8 / 16 / 32 lanes per popped run
        c.append(("accels-A%d" % A, "accels", 100 + A, 160, A, min(A, 4), {}))
    for A in (33, 64, 255, 256):                                                     # beyond the scan: ranked queue, heap
        c.append(("accels-A%d" % A, "accels", 100 + A, 40, A, 4, {}))
    for T, how in ((1, "low"), (31, "low"), (32, "one_each"), (33, "high"), (255, "scatter"), (256, "high"), (256, "scatter"), (256, "low")):
        c.append(("types-A32-T%d-%s" % (T, how), "types", 200 + T, 120, 32, T, dict(type_map=how)))
    c.append(("types-A256-T256", "types", 290, 40, 256, 256, dict(type_map="one_each", fractions=[0.0, 0.5, 1.0])))
    c.append(("types-A64-T256", "types", 291, 80, 64, 256, dict(type_map="scatter", fractions=[0.0, 0.5, 1.0])))
    c.append(("priorities", "priorities", 300, 300, 6, 3, {}))
    for seed in (400, 401, 402, 403):
        c.append(("capacities-%d" % seed, "capacities", seed, 200, 6, 6, {}))           # A = 6 maps to types 0..3: types 4 and 5 are used by nobody
    c.append(("capacities-zero", "capacities", 410, 120, 6, 6, dict(capacity="zero")))
    c.append(("capacities-ample", "capacities", 411, 120, 6, 6, dict(capacity="ample", p_feasible=1.0)))
    c.append(("capacities-first-type-empty", "capacities", 412, 120, 6, 6, dict(capacity="fractions", fractions=[0.5, 0.8], first_zero=True)))
    for seed in (500, 501, 502):
        c.append(("wrap-%d" % seed, "wrap", seed, 200, 8, 3, {}))
        c.append(("wrap-huge-%d" % seed, "wrap_huge", seed, 200, 8, 3, {}))
    c.append(("wrap-A32", "wrap", 510, 100, 32, 3, {}))
    for seed in (600, 601, 602):
        c.append(("values-%d" % seed, "values", seed, 200, 8, 3, {}))
    c.append(("values-A32", "values", 610, 120, 32, 4, {}))
    for seed in (700, 701):
        c.append(("dropped-%d" % seed, "dropped", seed, 200, 6, 3, {}))
    return c


CASES = _cases()
LARGE = [("large-A64-S30000", "large", 800, 30_000, 64, 8, {}), ("large-A32-S60000", "large", 801, 60_000, 32, 8, {})]


FUZZ = ((900, 120, 32), (901, 24, 256))            # (seed, tables, largest accelerator count)


def case_table(case):
    name, kind, seed, S, A, T, over = case
    return make_table(np.random.Generator(np.random.PCG64(seed)), S, A, T, kind, **over)


def fuzz_tables(seed, n, a_max):
    """n small tables drawing every dimension at once; a_max bounds the accelerator count"""
    rng = np.random.Generator(np.random.PCG64(seed))
    for i in range(n):
        S = int(rng.integers(1, 201)) if a_max <= 32 else int(rng.integers(1, 41))
        A = int(rng.choice([1, 2, 3, 5, 8, 9, 16, 17, 24, 32])) if a_max <= 32 else int(rng.choice([33, 40, 64, 100, 255, 256]))
        T = int(rng.choice([1, 2, 3, 7, 40, 256]))
        yield make_table(rng, S, A, T, "fuzz_huge" if i % 4 == 3 else "fuzz")
