"""Write tests/golden/hard_rounding.json: sweep candidates whose reference float32 results sit on a rounding boundary.

A deterministic CPU search (no seeds beyond the fixed tables below).  For each batch size b of the coverage list and
two (profile, replicas) choices it steps through consecutive float32 ARRIVAL RATES downward from a load where the
certificates' preconditions hold (a row's lambda is f32(f32(f32(rpm / 60) / r) / 1000), so not every lambda is
reachable), restates the reference's float64 chain for all of them at once (tests/test_hard_rounding_cpu.chain) and keeps
the candidates of each class (the classes are defined in tests/test_hard_rounding_cpu.py).  Pair entries (Q) are sized
once by the oracle for their pair's rate per replica, then searched among the arrival rates that keep that replica
count.  The expected float32 results come from the oracle.  Running it again reproduces the file byte for byte.

    python tools/hard_rounding.py [--out PATH]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_hard_rounding_cpu as H  # noqa: E402

F = np.float32

# (alpha, beta, gamma, delta, in tokens, out tokens): tame profiles of make_system's ranges, one of them decode-only
PROFILES = [
    (22.619, 0.181, 226.19, 0.018, 128, 128),
    (8.5, 0.05, 12.0, 0.0007, 512, 64),
    (15.0, 0.6, 90.0, 0.004, 2048, 256),
    (27.0, 0.02, 3.5, 0.0001, 0, 1024),
]
PER_SEARCH = dict(P=3, Pf=1, C=3, Cf=1)
ELEMENT_STEPS = 1 << 25            # arrival rates per batch ~ ELEMENT_STEPS / K
MAX_BATCHES = 8
PAIR_N = (40, 64, 100, 256)
SLO_NONE = H.f32_hex(F(0))


def profile(i):
    a, b, g, d, inn, out = PROFILES[i]
    return F(a), F(b), F(g), F(d), inn, out


def table(i, n):
    return H.rate_table(*profile(i), n)


def arrivals_down(rpm0, start, n):
    """n consecutive float32 arrival rates, start .. start + n - 1 ulps below rpm0"""
    bits = np.asarray(rpm0, dtype=F).view(np.uint32).astype(np.int64) - np.arange(start, start + n, dtype=np.int64)
    return bits.astype(np.uint32).view(F)


def rpm_for(lam, r):
    """the float32 arrival rate whose row-r lambda is the last one at or below lam"""
    a = F(float(lam) * 1000.0 * 60.0 * r)
    while H.row_lambda(a, r) > lam:
        a = np.nextafter(a, F(0))
    return a


def entry(cls, pi, rpm, r, b, n_pair=0):
    a, be, g, d, inn, out = profile(pi)
    return dict(cls=cls, alpha=H.f32_hex(a), beta=H.f32_hex(be), gamma=H.f32_hex(g), delta=H.f32_hex(d), **{"in": inn},
                out=out, arrival=H.f32_hex(rpm), r=int(r), b=int(b), n_pair=int(n_pair), slo_itl=SLO_NONE,
                slo_ttft=SLO_NONE)


def analysed(tab, b, rpm, r):
    """Analyze accepts: 0 < rate <= RateRange.Max (queueanalyzer.go:135-150)"""
    rate = F(F(rpm) / F(60)) / F(r)
    return (rate > 0) & (rate <= (tab[b - 1] * (F(1) - F(0.001))) * F(1000))


def search(pi, b, r, t, want, seen):
    """consecutive arrival rates below 1 - lambda / s[b-1] = t: up to want[c] new entries of each class c"""
    tab = table(pi, b)
    lam0 = F(float(tab[b - 1]) * (1.0 - t))
    rpm0 = rpm_for(lam0, r)
    L = max(2048, ELEMENT_STEPS // (11 * b))
    got = {c: [] for c in want}
    for k in range(MAX_BATCHES):
        rpm = arrivals_down(rpm0, k * L, L)
        lam = H.row_lambda(rpm, r)
        _, first = np.unique(lam, return_index=True)          # one arrival rate per lambda
        keep = np.zeros(L, bool)
        keep[first] = True
        keep &= analysed(tab, b, rpm, r)
        rpm, lam = rpm[keep], lam[keep]
        st = H.chain(tab, b, lam)
        for c in want:
            if len(got[c]) >= want[c]:
                continue
            for j in np.flatnonzero(H.classify(c, st, lam, tab, b)):
                key = (pi, b, float(lam[j]))
                if key in seen:
                    continue
                seen.add(key)
                got[c].append(entry(c, pi, rpm[j], r, b))
                if len(got[c]) >= want[c]:
                    break
        if all(len(got[c]) >= want[c] for c in want):
            break
    return got


def _start(tab, b, t):
    lam = np.array([F(float(tab[b - 1]) * (1.0 - t))])
    return H.chain(tab, b, lam)


def plane_target(b, tab):
    """1 - r for the plane's search: the first of 0.0025 .. 0.00105 (RateRange.Max is at 0.001) at which p_block is a
    normal float32 well above the subnormals (log2 p[K] > -100), so that its rounding is relative"""
    for t in (0.0025, 0.0016, 0.0012, 0.00105):
        t = max(t, 0.45 / (10 * b))
        if np.log2(_start(tab, b, t)["pK"][0]) > -100:
            return t
    return t


def usable(pi, b):
    """the profile's ramp at b stays far inside the value window near RateRange.Max"""
    st = _start(table(pi, b), b, 0.00105)
    return st["pmax"][0] < 2.0 ** 900 and st["S"][0] < 2.0 ** 900


def search_main(out, seen):
    for bi, b in enumerate(H.B_VALUES):
        used = set()
        for k in range(2):
            pi = next(p for p in ((bi + k + j) % len(PROFILES) for j in range(len(PROFILES)))
                      if p not in used and usable(p, b))
            used.add(pi)
            r = 1 if k == 0 else 2 + bi % 3
            tab = table(pi, b)
            t0 = time.time()
            tc, tp = max(0.0025, 0.45 / (10 * b)), plane_target(b, tab)
            got = search(pi, b, r, tc, dict(C=PER_SEARCH["C"], Cf=PER_SEARCH["Cf"]), seen)
            got.update(search(pi, b, r, tp, dict(P=PER_SEARCH["P"], Pf=PER_SEARCH["Pf"]), seen))
            for c in PER_SEARCH:
                out.extend(got[c])
            print("b=%5d profile %d r=%d 1-r=%.5f/%.5f: %s  (%.1f s)" %
                  (b, pi, r, tc, tp, {c: len(v) for c, v in got.items()}, time.time() - t0), flush=True)


def _edge(tab, b, r, rpm, pred):
    """(last, first): the two consecutive float32 arrival rates between which pred(restated chain, lambda) turns from
    False to True; pred is monotone in the load and rpm is an ascending grid on which it turns"""
    ok = pred(H.chain(tab, b, H.row_lambda(rpm, r)), H.row_lambda(rpm, r))
    j = int(np.argmax(ok))
    if not (0 < j and ok[j]):
        return None                                   # the chain leaves the value window before the edge
    lo, hi = (int(x) for x in rpm[j - 1:j + 1].view(np.uint32))
    while hi - lo > 1:
        mid = np.unique(np.linspace(lo, hi, 66).astype(np.int64))[1:-1]
        a = mid.astype(np.uint32).view(F)
        lam = H.row_lambda(a, r)
        ok = pred(H.chain(tab, b, lam), lam)
        lo = int(mid[~ok][-1]) if (~ok).any() else lo
        hi = int(mid[ok][0]) if ok.any() else hi
    return np.uint32(lo).view(F), np.uint32(hi).view(F)


def search_zero_edge(out, seen):
    """Pz: on either side of the certified zero's threshold (the two consecutive arrival rates whose bound
    log2 p[N] + M log2 rho straddles -160), and the lightest load whose p_block is not 0 (a float32 subnormal, the
    nonzero result nearest to the threshold: a looser threshold turns it into 0)"""
    frac = np.concatenate([np.geomspace(2.0 ** -24, 0.5, 4096), 1.0 - np.geomspace(0.5, 2.0 ** -10, 4096)])
    nonzero = lambda st, lam: st["pK"].astype(F) > 0
    for bi, b in enumerate((1, 3, 8, 32, 100, 256, 512, 1024)):
        used = set()
        for k in range(2):
            r = 1 if k == 0 else 3
            for j in range(len(PROFILES)):                 # the first profile of the rotation whose chain reaches both edges
                pi = (bi + k + j) % len(PROFILES)
                if pi in used:
                    continue
                tab = table(pi, b)
                lam = np.unique((tab[b - 1].astype(np.float64) * frac).astype(F))
                lam = lam[lam.astype(np.float64) >= 2.0 ** -100]
                rpm = np.unique(np.array([rpm_for(x, r) for x in lam], dtype=F))
                st = H.chain(tab, b, H.row_lambda(rpm, r))
                rpm = rpm[(st["pmin"] >= H.WIN_LO) & (st["S"] < 2.0 ** 990)]      # the chain stays in the value window
                zero = lambda st, lam: H.block_terms(st, lam, tab, b)["zero"] >= -160.0
                e1, e2 = _edge(tab, b, r, rpm, zero), _edge(tab, b, r, rpm, nonzero)
                if e1 is not None and e2 is not None:
                    break
            used.add(pi)
            (below, above), (_, first) = e1, e2
            n = 0
            for a in (below, above, first):
                lam1 = H.row_lambda(np.array([a]), r)
                key = (pi, b, float(lam1[0]))
                if key in seen or not analysed(tab, b, np.array([a]), r)[0]:
                    continue
                assert H.classify("Pz", H.chain(tab, b, lam1), lam1, tab, b)[0]
                seen.add(key)
                out.append(entry("Pz", pi, a, r, b))
                n += 1
            print("Pz b=%d profile %d r=%d: %d" % (b, pi, r, n), flush=True)


def search_pairs(out, seen, wva, oracle):
    """Q: for each pair (profile, N) the oracle sizes the pair once; arrival rates just under r x its rate per
    replica keep r replicas, and those whose final Analyze at (r, N) is C-hard are kept"""
    for i, N in enumerate(PAIR_N):
        for pi in range(len(PROFILES)):
            if (i + pi) % 2:
                continue
            tab = table(pi, N)
            probe = entry("Q", pi, F(60.0), 1, N, n_pair=N)
            img = H.entries_image(wva, [probe])
            pairs, feas, _ = oracle.analyze_pairs(img)
            star = float(pairs.max_arrv_rate_per_replica[0])     # rateStar / 1000: lambda at the pair's sizing limit
            for r in (1, 2):
                lam0 = F(star * (1.0 - 2.0 ** -12))
                rpm0 = rpm_for(lam0, r)
                L = max(4096, ELEMENT_STEPS // (11 * N))
                n = 0
                for kb in range(MAX_BATCHES):
                    rpm = arrivals_down(rpm0, kb * L, L)
                    lam = H.row_lambda(rpm, r)
                    _, first = np.unique(lam, return_index=True)
                    sel = np.sort(first)
                    rpm, lam = rpm[sel], lam[sel]
                    st = H.chain(tab, N, lam)
                    hard = np.flatnonzero(H.classify("Q", st, lam, tab, N))
                    cand = [entry("Q", pi, rpm[j], r, N, n_pair=N) for j in hard[:8]]
                    if cand:
                        pimg = H.entries_image(wva, cand)
                        pr, _, _ = oracle.analyze_pairs(pimg)
                        for q, (j, e) in enumerate(zip(hard[:8], cand)):
                            key = (pi, N, float(lam[j]), "Q")
                            if key in seen or n >= 2:
                                continue
                            if pr.num_replicas[q] == r and pr.batch_size[q] == N and pr.acc[q] == 0:
                                seen.add(key)
                                out.append(e)
                                n += 1
                    if n >= 2:
                        break
                print("Q N=%d profile %d r=%d: %d" % (N, pi, r, n), flush=True)


def fill_expected(entries, wva, oracle, ob):
    img = H.entries_image(wva, entries)
    m, st, pb = H.oracle_candidates(oracle, ob, img, [e["r"] for e in entries], [e["b"] for e in entries])
    for i, e in enumerate(entries):
        e["status"] = int(st[i])
        e["metrics"] = [H.f32_hex(x) for x in m[i].tolist()]
        e["p_block"] = H.f32_hex(pb[i])
    # the distance each entry's class is about, from the restated chain
    for i, e in enumerate(entries):
        a, be, g, d = (H.hex_f32(e[k]) for k in ("alpha", "beta", "gamma", "delta"))
        tab = H.rate_table(a, be, g, d, e["in"], e["out"], e["b"])
        lam = np.array([H.row_lambda(H.hex_f32(e["arrival"]), e["r"])], dtype=F)
        dist = float(H.class_distance(e["cls"], H.chain(tab, e["b"], lam), lam, tab, e["b"])[0])
        e["dist"] = dist if np.isfinite(dist) else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=H.FIXTURE)
    args = ap.parse_args()
    import wva_import
    import oracle
    import oracle_blocking
    wva = wva_import.load()
    oracle.build()
    oracle_blocking.build()
    entries, seen = [], set()
    search_main(entries, seen)
    search_zero_edge(entries, seen)
    search_pairs(entries, seen, wva, oracle)
    fill_expected(entries, wva, oracle, oracle_blocking)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    keys = ["cls", "b", "r", "n_pair", "arrival", "alpha", "beta", "gamma", "delta", "in", "out", "slo_itl", "slo_ttft",
            "dist", "status", "p_block", "metrics"]
    with open(args.out, "w") as f:
        f.write('{"u": "2^-53", "entries": [\n')
        f.write(",\n".join(json.dumps({k: e[k] for k in keys}) for e in entries))
        f.write("\n]}\n")
    count = {c: sum(e["cls"] == c for e in entries) for c in H.CLASSES}
    print("wrote %s: %d entries %s" % (args.out, len(entries), count))


if __name__ == "__main__":
    main()
