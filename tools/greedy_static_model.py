"""Design check of the static-order form of `allocate` (greedy.go:107-166), CPU only.

The reference keeps a sorted slice of server entries; the head is tried on its current candidate, and on failure the server
moves to its next candidate and is re-inserted (leftmost position among equal keys).  `queue_allocate` below restates that
literally.  `static_allocate` is what k_greedy_scan does on the GPU: no queue.

  * Along one server the candidates are tried in order; candidate j is tried when the queue's head key has reached
    M(s,j) = max_{i<=j} K(s,i) (the running maximum of the server's keys), because the server's entry is only ever at the head
    when nothing smaller is queued.  So the order in which (server, candidate) pairs are *tried* is the order of M, whatever
    the capacities are -- a pair is skipped when its server has already been placed / dropped.
  * A maximal stretch of one server's candidates with the same M is a "run": once its first candidate is at the head the
    others follow immediately (each is re-inserted at the very front).
  * Runs of different servers with one M (a tie group) are taken most-recently-inserted first; a run is inserted when the
    server's previous run ends in failure, the first runs (candidate 0) count as inserted before everything, in descending
    server index.  That is one stack per tie group, pushed while scanning, popped when the scan reaches the group, followed
    by the group's first runs in ascending server index.

python tools/greedy_static_model.py [rounds]   -- random cases with heavy ties, both forms must agree."""
import sys
import random


def queue_allocate(servers, avail):
    """servers: list of (priority, [ (key_delta_value_tuple...) ]) -- here each candidate is (K, type, count, skip) with K any
    totally ordered key *without* the priority; returns (placed: {s: j}, unalloc: [s...], avail)."""
    avail = list(avail)
    entries = []
    for s, (pr, cands) in enumerate(servers):
        if cands:
            entries.append([s, 0])
    keyof = lambda e: (servers[e[0]][0], servers[e[0]][1][e[1]][0])
    entries.sort(key=keyof)                                  # stable: equal keys in ascending server index
    placed, unalloc = {}, []
    while entries:
        top = entries.pop(0)
        s, j = top
        K, t, count, skip = servers[s][1][j]
        if skip:
            continue
        if avail[t] >= count:
            avail[t] -= count
            placed[s] = j
            continue
        j += 1
        if j == len(servers[s][1]):
            unalloc.append(s)
            continue
        top[1] = j
        k = keyof(top)
        lo, hi = 0, len(entries)
        while lo < hi:                                       # leftmost i with entries[i] >= top
            mid = (lo + hi) // 2
            if keyof(entries[mid]) < k:
                lo = mid + 1
            else:
                hi = mid
        entries.insert(lo, top)
    return placed, unalloc, avail


def static_order(servers):
    """events sorted by (priority, M, server, j) plus the run / tie-group structure; nothing here depends on capacities"""
    ev = []
    for s, (pr, cands) in enumerate(servers):
        M = None
        run = -1
        for j, (K, t, count, skip) in enumerate(cands):
            if M is None or K > M:
                M = K
                run += 1
            ev.append(((pr, M), s, j, run))
    ev.sort(key=lambda e: (e[0], e[1], e[2]))
    return ev


def static_allocate(servers, avail, pushes=None):
    """pushes, when a list: receives (group key, run-head event index) of every run pushed onto a shared group's stack"""
    avail = list(avail)
    ev = static_order(servers)
    n = len(ev)
    # tie groups: ranges of equal (pr, M) that hold runs of more than one server
    placed, unalloc, done = {}, [], set()
    pos_of = {(e[1], e[2]): i for i, e in enumerate(ev)}

    def run_range(i):
        # events of the run that starts at ev[i]
        k = i
        while k + 1 < n and ev[k + 1][1] == ev[i][1] and ev[k + 1][3] == ev[i][3]:
            k += 1
        return i, k + 1

    stacks = {}                                              # group key -> list of run-head event indices

    def try_run(i0, i1):
        """walk one run; returns True when the server got through it without being placed / dropped / exhausted"""
        s = ev[i0][1]
        if s in done:
            return False
        for i in range(i0, i1):
            _, _, j, _ = ev[i]
            K, t, count, skip = servers[s][1][j]
            if skip:
                done.add(s)
                return False
            if avail[t] >= count:
                avail[t] -= count
                placed[s] = j
                done.add(s)
                return False
            if j + 1 == len(servers[s][1]):
                unalloc.append(s)
                done.add(s)
                return False
        return True

    def after_run(i1, s):
        # the server's next run starts at candidate j+1; if its group is shared, push it there
        j = ev[i1 - 1][2] + 1
        h = pos_of[(s, j)]
        g = ev[h][0]
        if multi[g]:
            stacks.setdefault(g, []).append(h)
            if pushes is not None:
                pushes.append((g, h))

    # which groups hold more than one server
    multi = {}
    cnt = {}
    for e in ev:
        cnt.setdefault(e[0], set()).add(e[1])
    for g, ss in cnt.items():
        multi[g] = len(ss) > 1
    i = 0
    while i < n:
        g = ev[i][0]
        if not multi[g]:
            i0, i1 = run_range(i)
            if try_run(i0, i1):
                after_run(i1, ev[i0][1])
            i = i1
            continue
        # a shared group: stack first (most recent first; runs that fail through may push onto *later* groups only)
        gend = i
        while gend < n and ev[gend][0] == g:
            gend += 1
        st = stacks.get(g, [])
        while st:
            h = st.pop()
            i0, i1 = run_range(h)
            if try_run(i0, i1):
                after_run(i1, ev[i0][1])
        k = i
        while k < gend:
            i0, i1 = run_range(k)
            if ev[i0][2] == 0:                               # first runs, ascending server index
                if try_run(i0, i1):
                    after_run(i1, ev[i0][1])
            k = i1
        i = gend
    return placed, unalloc, avail


def batch_resolve(events, avail, done):
    """greedy_scan_batch: up to 32 events in lane order, resolved the way the warp does it.  events: list of
    (server, type, count, skip, last); returns (placed [(server, lane)], unalloc [server...]); avail / done are updated.
    Every lane tests against a register copy of its type's capacity; the first lane that can stop (placement or drop)
    does; lanes of that type re-test, later lanes of that server die; repeat.  Equals one-by-one processing also when a
    negative count makes the capacity grow."""
    n = len(events)
    alive = [e[0] not in done for e in events]
    av = [avail[e[1]] for e in events]
    cand = [alive[i] and (events[i][3] or av[i] >= events[i][2]) for i in range(n)]
    won = [False] * n
    while any(cand):
        f = cand.index(True)
        sf, tf, cf, skf, _ = events[f]
        won[f] = True; cand[f] = False; alive[f] = False
        for i in range(n):
            s, t, c, sk, _ = events[i]
            if not skf and not sk and t == tf:
                av[i] -= cf
                if i > f and alive[i]:
                    cand[i] = av[i] >= c
            if i > f and alive[i] and s == sf:
                alive[i] = False; cand[i] = False
    placed, unalloc = [], []
    for i in range(n):
        s, t, c, sk, last = events[i]
        if won[i]:
            if not sk:
                avail[t] -= c
                placed.append((s, i))
            done.add(s)
        elif alive[i] and last:
            unalloc.append(s)
            done.add(s)
    return placed, unalloc


def sequential_resolve(events, avail, done):
    placed, unalloc = [], []
    for i, (s, t, c, sk, last) in enumerate(events):
        if s in done:
            continue
        if sk:
            done.add(s)
        elif avail[t] >= c:
            avail[t] -= c
            placed.append((s, i))
            done.add(s)
        elif last:
            unalloc.append(s)
            done.add(s)
    return placed, unalloc


def random_batch(rng):
    """up to 32 events as a batch of the pass holds them: a server's candidates in their own order (the last one flagged),
    interleaved with other servers'; some servers have stopped before the batch"""
    T = rng.randint(1, 3)
    seqs = []
    for s in range(rng.randint(1, 10)):
        nc = rng.randint(1, 5)
        first = rng.randint(0, nc - 1)                       # the batch may start in the middle of a server's candidates
        seqs.append([(s, rng.randrange(T), rng.randint(-3, 9), rng.random() < 0.05, k == nc - 1) for k in range(first, nc)])
    ev = []
    while any(seqs) and len(ev) < 32:
        q = rng.choice([x for x in seqs if x])
        ev.append(q.pop(0))
    avail = [rng.randint(-2, 20) for _ in range(T)]
    done = set(rng.sample(range(10), rng.randint(0, 3)))
    return ev, avail, done


def random_case(rng):
    S = rng.randint(1, 40)
    T = rng.randint(1, 3)
    nkeys = rng.choice([1, 2, 3, 5, 50])
    servers = []
    for s in range(S):
        pr = rng.randint(1, rng.choice([1, 1, 3]))
        nc = rng.randint(0, 5)
        cands = []
        for j in range(nc):
            cands.append((rng.randint(0, nkeys - 1), rng.randrange(T), rng.randint(0, 6), rng.random() < 0.05))
        servers.append((pr, cands))
    avail = [rng.randint(0, 25) for _ in range(T)]
    return servers, avail


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
    rng = random.Random(7)
    for r in range(rounds):
        servers, avail = random_case(rng)
        a = queue_allocate(servers, avail)
        b = static_allocate(servers, avail)
        if a != b:
            print("MISMATCH in case", r)
            print(servers, avail)
            print("queue ", a)
            print("static", b)
            return 1
    for r in range(rounds):
        ev, avail, done = random_batch(rng)
        a1, d1 = list(avail), set(done)
        a2, d2 = list(avail), set(done)
        if (batch_resolve(ev, a1, d1), a1, d1) != (sequential_resolve(ev, a2, d2), a2, d2):
            print("BATCH MISMATCH", ev, avail, done)
            return 1
    print("ok:", rounds, "cases")
    return 0


if __name__ == "__main__":
    sys.exit(main())


# ---- allocateMaximally (greedy.go:194-223), 32 servers at a time ---------------------------------------------------

def go_div(a, b):
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def maximally_sequential(servers, avail):
    """servers: list of candidate lists [(type or -1, upr, cur)]; returns {server: (k, replicas)}"""
    avail = list(avail)
    got = {}
    for s, cands in enumerate(servers):
        for k, (t, upr, cur) in enumerate(cands):
            if t < 0 or upr <= 0:
                continue
            m = min(go_div(avail[t], upr), cur)
            if m > 0:
                got[s] = (k, m)
                avail[t] -= m * upr
                break
    return got, avail


def maximally_batched(servers, avail):
    """greedy_allocate_maximally: lane = server with a forward-only cursor, winners served in list order, the lanes
    waiting on the served type look again (same candidate first)"""
    avail = list(avail)
    got = {}
    for i0 in range(0, len(servers), 32):
        lanes = list(range(i0, min(i0 + 32, len(servers))))
        cur_k = {s: 0 for s in lanes}

        def look(s):
            cands = servers[s]
            while cur_k[s] < len(cands):
                t, upr, cur = cands[cur_k[s]]
                if t >= 0 and upr > 0 and min(go_div(avail[t], upr), cur) > 0:
                    return True
                cur_k[s] += 1
            return False

        has = {s: look(s) for s in lanes}
        while any(has.values()):
            f = min(s for s in lanes if has[s])
            t, upr, cur = servers[f][cur_k[f]]
            m = min(go_div(avail[t], upr), cur)
            got[f] = (cur_k[f], m)
            avail[t] -= m * upr
            has[f] = False
            for s in lanes:
                if has[s] and servers[s][cur_k[s]][0] == t:
                    has[s] = look(s)
    return got, avail


def random_maximally(rng):
    T = rng.randint(1, 3)
    servers = []
    for s in range(rng.randint(1, 70)):
        servers.append([(rng.choice([-1] + list(range(T))), rng.randint(0, 4), rng.randint(0, 6)) for _ in range(rng.randint(0, 5))])
    return servers, [rng.randint(-3, 40) for _ in range(T)]


# ---- allocateEqually, round 1 (greedy.go:239-273): every ticket takes its first replica -------------------------------

def equally_round1_sequential(servers, avail):
    avail = list(avail)
    tickets, live = {}, []
    for s, cands in enumerate(servers):
        for k, (t, upr, cur) in enumerate(cands):
            if t >= 0 and upr > 0 and avail[t] >= upr:
                got = 0
                if cur > 0:
                    got = 1
                    avail[t] -= upr
                    live.append(s)
                tickets[s] = (k, got)
                break
    return tickets, live, avail


def equally_round1_batched(servers, avail):
    avail = list(avail)
    tickets, live = {}, []
    for i0 in range(0, len(servers), 32):
        lanes = list(range(i0, min(i0 + 32, len(servers))))
        cur_k = {s: 0 for s in lanes}

        def look(s):
            cands = servers[s]
            while cur_k[s] < len(cands):
                t, upr, cur = cands[cur_k[s]]
                if t >= 0 and upr > 0 and avail[t] >= upr:
                    return True
                cur_k[s] += 1
            return False

        has = {s: look(s) for s in lanes}
        batch_live = []
        while any(has.values()):
            f = min(s for s in lanes if has[s])
            t, upr, cur = servers[f][cur_k[f]]
            got = 0
            if cur > 0:
                got = 1
                avail[t] -= upr
                batch_live.append(f)
            tickets[f] = (cur_k[f], got)
            has[f] = False
            for s in lanes:
                if has[s] and servers[s][cur_k[s]][0] == t:
                    has[s] = look(s)
        live += batch_live
    return tickets, live, avail
