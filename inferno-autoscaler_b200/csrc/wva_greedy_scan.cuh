// wva_greedy_scan.cuh — SolveGreedy's `allocate` (greedy.go:107-166) WITHOUT a queue: one static order, one linear scan.
//
// The reference keeps a sorted slice of server entries.  The head is tried on its current candidate; on failure the
// server moves to its next candidate and is re-inserted by binary search (leftmost among equal keys).  A server's entry is
// only ever at the head when nothing smaller is queued, so candidate j of server s is tried when the head key has reached
//
//     M(s,j) = max_{i<=j} K(s,i)            K = (priority, delta to the next candidate, value), see k_greedy_states
//
// -- the running maximum of the server's keys -- whatever the capacities are: a later candidate with a smaller key is
// re-inserted at the very front and tried at once.  Capacities only decide WHERE a server stops.  Hence:
//
//   * the order in which (server, candidate) pairs are tried is the order of (M, server, j), fixed once the candidates are
//     sized.  It is produced by the same bitonic sort the ranked queue uses, with M in place of K;
//   * `allocate` is a linear pass over that order; a pair is skipped when its server has stopped (placed, dropped, exhausted);
//   * a maximal stretch of one server's candidates with one M is a RUN (they are tried back to back);
//   * runs of DIFFERENT servers with one M (a shared group: equal keys, e.g. zero-load servers on one accelerator) are
//     taken most-recently-inserted first; a run is inserted when the server's previous run ends in failure, and the runs
//     that start at candidate 0 count as inserted before everything else in ascending server index.  That is one stack
//     per shared group: pushed while scanning, popped when the scan reaches the group, then the group's first runs
//     follow in the static order.  Runs that wait on a stack carry GREEDY_STACKED and are skipped by the linear pass.
//
// tools/greedy_static_model.py checks this restructuring against a literal restatement of the reference's slice on random
// cases with heavy ties; the GPU tests compare decisions with the oracle for all three solver paths.
//
// The pass itself is one warp, 32 consecutive events at a time, the next 32 records already in flight (addresses are
// static, nothing to chase).  Lanes test `available >= count` in parallel; the successes -- the only steps that change
// `available` -- are then applied one by one in lane order, every later lane of the same type re-testing after each one
// (exactly the sequential semantics, also when a wrapped negative count makes `available` grow).

#pragma once

namespace wva {

constexpr int GREEDY_RUNHEAD = 1 << 25, GREEDY_STACKED = 1 << 26, GREEDY_GSTART = 1 << 27, GREEDY_PUSH = 1 << 28;

struct GreedyScan {
    unsigned long long* ka;    // [N2] sort key of an event: priority << 32 | ~sortable(delta), running maximum along the server
    unsigned* kb;              // [N2]                        ~sortable(value)
    unsigned* kslot;           // [N2] state s*A+k, 0xffffffff for padding
    unsigned* posOf;           // [S*A] position of a state in the static order
    unsigned char* runHead;    // [S*A] 1 where the state's key exceeds every earlier key of its server (candidate 0 included)
    int4* ev;                  // [N2] per position: { count lo, count hi, type (8 bits) | candidate << 8 | GREEDY_* | priority << 18, server }
    int2* push;                // [N2] for GREEDY_PUSH events: { position of the next run's head, start of that run's shared group }
    int* gbeg;                 // [N2] start of the shared group a position belongs to, -1 elsewhere
    int* stackTop;             // [N2] per shared group (indexed by its start): runs waiting
    int* stackBuf;             // [N2] the stack of the group that starts at g0 occupies [g0, g0 + runs)
    int* nEv;                  // [1] number of events
    unsigned n2;
};

// key of state (s,k): k_greedy_states' encoding of orderFunc (greedy.go:76-85)
__device__ __forceinline__ void greedy_state_key(const GreedyCand* cand, int n, int k, unsigned prio, unsigned long long& a, unsigned& b) {
    const float v = cand[k].val;
    const float d = k + 1 < n ? cand[k + 1].val - v : 3.40282346638528859811704183484516925e+38f;
    a = ((unsigned long long)prio << 32) | (unsigned)~f32_sortable(d);
    b = d != d ? 0u : ~f32_sortable(v);           // NaN deltas compare equal without looking at the values (greedy.go:78-80)
}

// event keys: the running maximum of the server's state keys; runHead where it grows
__global__ void k_greedy_scan_keys(DevSystem sys, GreedyBufs g, GreedyScan gs) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= gs.n2) return;
    unsigned long long a = ~0ull; unsigned b = ~0u, slot = ~0u;
    if (i < (unsigned)sys.S * (unsigned)sys.A) {
        const int s = (int)(i / (unsigned)sys.A), k = (int)(i - (unsigned)s * (unsigned)sys.A);
        const int n = g.nCand[s];
        unsigned char head = 0;
        if (k < n) {
            const GreedyCand* cand = g.cand + (size_t)s * sys.A;
            const unsigned prio = (unsigned)sys.srv_priority[s];
            unsigned long long ma = 0; unsigned mb = 0;
            for (int q = 0; q < k; ++q) {
                unsigned long long qa; unsigned qb;
                greedy_state_key(cand, n, q, prio, qa, qb);
                if (q == 0 || qa > ma || (qa == ma && qb > mb)) { ma = qa; mb = qb; }
            }
            greedy_state_key(cand, n, k, prio, a, b);
            if (k == 0 || a > ma || (a == ma && b > mb)) head = 1;
            else { a = ma; b = mb; }
            slot = i;
        }
        gs.runHead[i] = head;
    }
    gs.ka[i] = a; gs.kb[i] = b; gs.kslot[i] = slot;
}

// shared groups: positions with one key that hold runs of more than one server (the last position of a group marks it)
__global__ void k_greedy_scan_groups(DevSystem sys, GreedyScan gs) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 || i >= gs.n2 || gs.kslot[i] == ~0u) return;
    const unsigned long long a = gs.ka[i]; const unsigned b = gs.kb[i];
    if (i + 1 < gs.n2 && gs.kslot[i + 1] != ~0u && gs.ka[i + 1] == a && gs.kb[i + 1] == b) return;     // not the last of its key
    if (!(gs.ka[i - 1] == a && gs.kb[i - 1] == b)) return;                                               // alone
    unsigned j = i - 1;
    while (j > 0 && gs.ka[j - 1] == a && gs.kb[j - 1] == b) --j;
    // equal keys are laid out in ascending state: one server <=> first and last state belong to the same server
    if (gs.kslot[j] / (unsigned)sys.A == gs.kslot[i] / (unsigned)sys.A) return;
    for (unsigned q = j; q <= i; ++q) gs.gbeg[q] = (int)j;
}

// the record the pass reads at every position, and where a run that ends in failure sends its server
__global__ void k_greedy_scan_records(DevSystem sys, GreedyBufs g, GreedyScan gs) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= gs.n2) return;
    const unsigned slot = gs.kslot[i];
    if (slot == ~0u) return;
    if (i + 1 == gs.n2 || gs.kslot[i + 1] == ~0u) *gs.nEv = (int)i + 1;
    const unsigned A = (unsigned)sys.A;
    const GreedyCand cd = g.cand[slot];
    int flags = cd.tf | ((int)(slot % A) << 8) | ((int)(gs.ka[i] >> 32) << 18);      // type <= 255 (wva_solve checks), candidate <= 31
    if (gs.runHead[slot]) flags |= GREEDY_RUNHEAD;
    const int gb = gs.gbeg[i];
    if (gb >= 0) {
        unsigned h = slot;
        while (!gs.runHead[h]) --h;                               // the run's first state (candidate 0 is always a head)
        if (h % A != 0) flags |= GREEDY_STACKED;
        if (gb == (int)i) flags |= GREEDY_GSTART;
    }
    if (!(cd.tf & GREEDY_LAST) && gs.runHead[slot + 1]) {
        const unsigned h = gs.posOf[slot + 1];
        const int g0 = gs.gbeg[h];
        if (g0 >= 0) { flags |= GREEDY_PUSH; gs.push[i] = make_int2((int)h, g0); }
    }
    int4 v;
    v.x = (int)(unsigned)((unsigned long long)cd.count & 0xffffffffull);
    v.y = (int)(unsigned)((unsigned long long)cd.count >> 32);
    v.z = flags;
    v.w = (int)(slot / A);
    gs.ev[i] = v;
}

// a push in flight: the leader lane of each group holds the counter's old value
struct GreedyPend { int old, leader, rank, h, g0; bool on; };

__device__ __forceinline__ void greedy_scan_flush(const GreedyScan& gs, GreedyPend& pd) {
    if (!__ballot_sync(0xffffffffu, pd.on)) return;
    const int base = __shfl_sync(0xffffffffu, pd.old, pd.on ? pd.leader : 0);
    if (pd.on) ((volatile int*)gs.stackBuf)[pd.g0 + base + pd.rank] = pd.h;
    pd.on = false;
    __syncwarp();
}

// One batch of the pass: the lanes' events in lane order.  `alive` = the event is tried (its server has not stopped).
// Every lane keeps the capacity of its own type in a register and follows the successes as they are broadcast, so one
// success costs a ballot and four shuffles; shared memory is brought up to date once per batch.
__device__ __forceinline__ void greedy_scan_batch(GreedyCtx& c, const GreedyScan& gs, unsigned* doneBits, bool alive, long long count, int flags,
                                                  int s, int2 pushInfo, GreedyPend& pd, int& nUn) {
    const unsigned FULL = 0xffffffffu;
    const unsigned lt = (1u << c.lane) - 1u;
    const bool skip = (flags & GREEDY_SKIP) != 0;                 // no model / GetAccelerator("") == nil: the entry is dropped
    const int t = flags & 0xff;
    const int key = (s << 9) | (skip ? 256 : 0) | t;              // server | dropped | type
    long long av = c.avail[t];
    bool cand = alive && (skip || av >= count);
    bool won = false;
    for (;;) {
        const unsigned m = __ballot_sync(FULL, cand);
        if (!m) break;
        const int f = __ffs(m) - 1;                               // every alive lane before f fails for good
        const int kf = __shfl_sync(FULL, key, f);
        const unsigned clo = __shfl_sync(FULL, (unsigned)((unsigned long long)count & 0xffffffffull), f);
        const unsigned chi = __shfl_sync(FULL, (unsigned)((unsigned long long)count >> 32), f);
        const bool later = c.lane > f && alive;
        if (c.lane == f) { won = true; cand = false; alive = false; }
        if (((key ^ kf) & 0x1ff) == 0 && !skip) {                 // same type, neither dropped: follow the capacity
            av -= (long long)(((unsigned long long)chi << 32) | clo);
            if (later) cand = av >= count;
        }
        if (later && (key >> 9) == (kf >> 9)) { alive = false; cand = false; }    // later candidates of the server that just stopped
    }
    // every lane of a type holds the type's capacity after the batch: no atomics (a 64-bit shared-memory add is a CAS loop)
    if (__ballot_sync(FULL, won) && !skip) c.avail[t] = av;
    if (won) {
        if (!skip) c.chosen[s] = s * c.sys.A + ((flags >> 8) & 31);
        atomicOr(&doneBits[s >> 5], 1u << (s & 31));
    }
    // what is still alive failed.  Last candidate: the server is unallocated (greedy.go:150-153) ...
    const bool failLast = alive && (flags & GREEDY_LAST);
    const unsigned mu = __ballot_sync(FULL, failLast);
    if (failLast) {
        c.g.unalloc[nUn + __popc(mu & lt)] = s;
        atomicOr(&doneBits[s >> 5], 1u << (s & 31));
    }
    nUn += __popc(mu);
    // ... end of a run whose successor waits in a shared group: push it there (lane order = insertion order).  The
    // group's counter is bumped by one atomic per group whose RESULT is not looked at here: the slot is written one
    // batch later (greedy_scan_flush), when the atomic has long returned.
    const bool pushes = alive && (flags & GREEDY_PUSH);
    if (__ballot_sync(FULL, pushes)) {
        greedy_scan_flush(gs, pd);
        const int g0 = pushes ? pushInfo.y : -1 - c.lane;
        const unsigned same = __match_any_sync(FULL, g0);
        pd.leader = __ffs(same) - 1;
        pd.rank = __popc(same & lt);
        pd.h = pushInfo.x; pd.g0 = g0; pd.on = pushes;
        if (pushes && c.lane == pd.leader) pd.old = atomicAdd(gs.stackTop + g0, __popc(same));
    }
    __syncwarp();
}

// The pass over the static order, one warp: k_greedy_scan runs it once on wva_solve's state, k_greedy_scan_multi once per
// capacity vector on state of the vector's own.  c holds the context without its pool; `capacity` the T starting capacities.
// groupSlot maps the position where a shared group starts to the index of its stack in gs.stackTop / gs.stackBuf, and
// gs.n2 bounds gs.stackBuf.  st = the four words of wva_solve_stats.
template <class Ctx, class GroupSlot>
__device__ __forceinline__ void greedy_scan_pass(Ctx& c, const GreedyScan& gs, const long long* capacity, unsigned char* greedy_pool,
                                                 int delayedBestEffort, int policy, GroupSlot groupSlot, unsigned long long st[4]) {
    const unsigned FULL = 0xffffffffu;
    const int lane = c.lane;
    const DevSystem& sys = c.sys;
    const unsigned A = (unsigned)sys.A;
    unsigned* doneBits = reinterpret_cast<unsigned*>(greedy_pool);
    const size_t doneWords = ((size_t)sys.S + 31) / 32;
    const size_t doneBytes = (doneWords * 4 + 15) & ~(size_t)15;
    c.pool = greedy_pool + doneBytes;
    c.g.smemBytes = c.g.smemBytes - (int)doneBytes;
    for (int t = lane; t < sys.T; t += 32) c.avail[t] = capacity[t];
    for (size_t i = lane; i < doneWords; i += 32) doneBits[i] = 0;
    __syncwarp();
    const int nEv = *gs.nEv;
    // runs popped from a stack: 32 / W at a time, W lanes each (a run has at most A events)
    const int W = A <= 8 ? 8 : (A <= 16 ? 16 : 32);
    const int perPop = 32 / W;
    const unsigned lt = (1u << lane) - 1u;
    int curPr = -1, nUn = 0;
    unsigned long long cycScan = 0, cycBest = 0, nBatches = 0, nPopped = 0, nGroups = 0;
    const int4 none = make_int4(0, 0, 0, 0);
    int4 nextRec = lane < nEv ? gs.ev[lane] : none;
    int2 nextPush = lane < nEv ? gs.push[lane] : make_int2(0, 0);
    GreedyPend pd; pd.old = 0; pd.leader = 0; pd.rank = 0; pd.h = 0; pd.g0 = 0; pd.on = false;
    long long t0 = clock64();
    for (int base = 0; base < nEv; base += 32) {
        const int4 rec = nextRec;
        const int2 pushInfo = nextPush;
        if (base + 32 + lane < nEv) { nextRec = gs.ev[base + 32 + lane]; nextPush = gs.push[base + 32 + lane]; }
        const bool valid = base + lane < nEv;
        const int flags = rec.z, s = rec.w;
        const long long count = (long long)(((unsigned long long)(unsigned)rec.y << 32) | (unsigned)rec.x);
        const int pr = (flags >> 18) & 0x7f;
        const unsigned mValid = __ballot_sync(FULL, valid);
        const unsigned mG = __ballot_sync(FULL, valid && (flags & GREEDY_GSTART));
        // where the block has to be cut: a shared group starts (its stack goes first) or the priority changes
        const int prPrev = __shfl_up_sync(FULL, pr, 1);
        const unsigned mCut = __ballot_sync(FULL, valid && ((flags & GREEDY_GSTART) || (lane > 0 && pr != prPrev)));
        int lo = 0;
        while (lo < 32 && (mValid >> lo)) {
            // a new priority: bestEffort for the group that ends here (greedy.go:96-103)
            const int prLo = __shfl_sync(FULL, pr, lo);
            if (prLo != curPr) {
                if (curPr >= 0 && !delayedBestEffort) {
                    const long long t1 = clock64();
                    greedy_best_effort(c, c.g.unalloc, nUn, policy);
                    nUn = 0;
                    const long long t2 = clock64();
                    cycScan += (unsigned long long)(t1 - t0); cycBest += (unsigned long long)(t2 - t1); t0 = t2;
                }
                curPr = prLo;
            }
            // a shared group starts at lo: the runs inserted so far go first, the most recent one on top
            if ((mG >> lo) & 1u) {
                const int g0 = groupSlot(base + lo);
                greedy_scan_flush(gs, pd);                         // pushes still in flight may belong to this group
                // the count and the first 32 entries travel together (one exposed latency), the runs' records are the second
                int top = *((volatile int*)gs.stackTop + g0);
                const int hMine = (unsigned)(g0 + lane) < gs.n2 ? ((volatile int*)gs.stackBuf)[g0 + lane] : -1;
                if (top > 0) ++nGroups;
                while (top > 0) {
                    const int q = lane / W, off = lane - q * W;
                    const int k = top < perPop ? top : perPop;
                    const int idx = top - 1 - q;                  // run q of this round: the stack's entry idx
                    const bool mine = q < k;
                    const int hv = __shfl_sync(FULL, hMine, mine && idx < 32 ? idx : 0);
                    int h = -1;
                    if (mine) h = idx < 32 ? hv : ((volatile int*)gs.stackBuf)[g0 + idx];
                    int4 r2 = none; int2 p2 = make_int2(0, 0); bool v2 = false;
                    if (h >= 0 && h + off < nEv) { r2 = gs.ev[h + off]; p2 = gs.push[h + off]; v2 = true; }
                    const int s2 = v2 ? r2.w : -1;
                    const int sHead = __shfl_sync(FULL, s2, q * W);
                    bool ok = v2 && s2 == sHead && (off == 0 || !(r2.z & GREEDY_RUNHEAD));
                    const unsigned seg = (W == 32 ? FULL : ((1u << W) - 1u) << (q * W));
                    const unsigned bad = __ballot_sync(FULL, !ok);
                    ok = ok && !(bad & seg & lt);                  // the run is the contiguous stretch after its head
                    const int s2c = s2 < 0 ? 0 : s2;
                    const bool alive2 = ok && !((doneBits[s2c >> 5] >> (s2c & 31)) & 1u);
                    const long long count2 = (long long)(((unsigned long long)(unsigned)r2.y << 32) | (unsigned)r2.x);
                    greedy_scan_batch(c, gs, doneBits, alive2, count2, r2.z, s2c, p2, pd, nUn);
                    top -= k; nPopped += (unsigned long long)k;
                }
            }
            // up to the next shared group or priority
            const unsigned stop = mCut & ~((2u << lo) - 1u);
            const int hi = stop ? __ffs(stop) - 1 : 32;
            const bool alive = valid && lane >= lo && lane < hi && !(flags & GREEDY_STACKED) && !((doneBits[s >> 5] >> (s & 31)) & 1u);
            greedy_scan_batch(c, gs, doneBits, alive, count, flags, s, pushInfo, pd, nUn);
            ++nBatches;
            lo = hi;
        }
    }
    const long long t1 = clock64();
    greedy_best_effort(c, c.g.unalloc, nUn, policy);
    cycScan += (unsigned long long)(t1 - t0); cycBest += (unsigned long long)(clock64() - t1);
    st[0] = (unsigned long long)nEv + (nGroups << 32); st[1] = nBatches + (nPopped << 32); st[2] = cycScan; st[3] = cycBest;
}

__global__ void __launch_bounds__(32) k_greedy_scan(DevSystem sys, DevAllocs pairs, GreedyBufs g, GreedyScan gs, int* chosen,
                                                      int delayedBestEffort, int policy) {
    extern __shared__ __align__(16) unsigned char greedy_pool[];
    __shared__ long long avail[256];
    __shared__ long long usum[256];
    if (blockIdx.x != 0) return;
    GreedyCtx c; c.sys = sys; c.pairs = pairs; c.g = g; c.chosen = chosen; c.avail = avail; c.usum = usum; c.lane = threadIdx.x;
    unsigned long long st[4];
    greedy_scan_pass(c, gs, sys.type_capacity, greedy_pool, delayedBestEffort, policy, [](int g0) { return g0; }, st);
    if (threadIdx.x == 0) { g.stats[0] = st[0]; g.stats[1] = st[1]; g.stats[2] = st[2]; g.stats[3] = st[3]; }
}

// ---- many capacity vectors over one static order (wva_solve_capacities) --------------------------------------------
// The order, the event records and the shared groups do not depend on the capacities; what the pass mutates does: the
// capacities, the stopped bits, the chosen slots, the unallocated list, the round-robin tickets and the shared-group
// stacks.  Each vector gets its own copy of those, one block of one warp per vector.  The stacks are indexed by a compact
// slot over the positions that lie in shared groups (a group starting at slot c0 keeps its stack in [c0, c0 + runs)),
// so a vector's stacks take as many words as there are such positions.

// per block of 256 positions: how many lie in shared groups
__global__ void k_greedy_group_count(GreedyScan gs, int* __restrict__ blockCnt) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = __syncthreads_count(i < gs.n2 && gs.gbeg[i] >= 0);
    if (threadIdx.x == 0) blockCnt[blockIdx.x] = n;
}

// exclusive prefix sum of the block counts in place (one block of 1024 threads); *total = positions in shared groups
__global__ void __launch_bounds__(1024) k_greedy_group_offsets(int* __restrict__ blockCnt, int nb, int* __restrict__ total) {
    __shared__ int part[1024];
    const int tid = threadIdx.x;
    const int per = (nb + 1023) / 1024, lo = min(nb, tid * per), hi = min(nb, lo + per);
    int sum = 0;
    for (int i = lo; i < hi; ++i) sum += blockCnt[i];
    part[tid] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int v = tid >= o ? part[tid - o] : 0;
        __syncthreads();
        part[tid] += v;
        __syncthreads();
    }
    int run = part[tid] - sum;
    for (int i = lo; i < hi; ++i) { const int c = blockCnt[i]; blockCnt[i] = run; run += c; }
    if (tid == 1023) *total = part[1023];
}

// slot[i] = compact index of position i (positions in shared groups, in order)
__global__ void k_greedy_group_slots(GreedyScan gs, const int* __restrict__ blockOff, int* __restrict__ slot) {
    __shared__ int warpCnt[8];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool in = i < gs.n2 && gs.gbeg[i] >= 0;
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if (lane == 0) warpCnt[warp] = __popc(m);
    __syncthreads();
    int off = blockOff[blockIdx.x];
    for (int w = 0; w < warp; ++w) off += warpCnt[w];
    if (in) slot[i] = off + __popc(m & ((1u << lane) - 1u));
}

// the push records with the target group's compact slot in place of its position
__global__ void k_greedy_group_push(GreedyScan gs, const int* __restrict__ slot, int2* __restrict__ pushSlot) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)*gs.nEv) return;
    const int2 p = gs.push[i];
    pushSlot[i] = (gs.ev[i].z & GREEDY_PUSH) ? make_int2(p.x, slot[p.y]) : make_int2(0, 0);
}

// what each vector's pass owns, vector j at offset j * S (j * P for the stacks)
struct GreedyScanVecs {
    const long long* capacity;   // [nv * T]
    int* chosen;                 // [nv * S] chosen slot, -1 before the pass
    int* unalloc;                // [nv * S]
    GreedyTicket* tickets;       // [nv * S] and
    int* liveIdx;                // [nv * S] round-robin ticket pool, nullptr when it fits shared memory
    long long* got;              // [nv * S] best-effort scaling, 0 before the pass
    long long* cur;              // [nv * S]
    int* stackTop;               // [nv * P] 0 before the pass
    int* stackBuf;               // [nv * P]
    unsigned P;                  // positions in shared groups
    unsigned long long* maxCycles;   // SM cycles of the slowest vector's pass
};

__global__ void __launch_bounds__(32) k_greedy_scan_multi(DevSystem sys, GreedyBufs g, GreedyScan gs, const int* __restrict__ groupSlot,
                                                            const int2* __restrict__ pushSlot, GreedyScanVecs v, int delayedBestEffort, int policy) {
    extern __shared__ __align__(16) unsigned char greedy_pool[];
    __shared__ long long avail[256];
    __shared__ long long usum[256];
    const size_t j = blockIdx.x, S = (size_t)sys.S;
    GreedyCtxMulti c; c.sys = sys; c.pairs = DevAllocs{}; c.g = g; c.avail = avail; c.usum = usum; c.lane = threadIdx.x;
    c.chosen = v.chosen + j * S; c.g.unalloc = v.unalloc + j * S;
    if (v.tickets) { c.g.tickets = v.tickets + j * S; c.g.liveIdx = v.liveIdx + j * S; }
    c.got = v.got + j * S; c.cur = v.cur + j * S;
    GreedyScan mine = gs;
    mine.push = const_cast<int2*>(pushSlot);
    mine.stackTop = v.stackTop + j * v.P; mine.stackBuf = v.stackBuf + j * v.P; mine.n2 = v.P;
    unsigned long long st[4];
    greedy_scan_pass(c, mine, v.capacity + j * (size_t)sys.T, greedy_pool, delayedBestEffort, policy, [&](int g0) { return groupSlot[g0]; }, st);
    if (threadIdx.x == 0) atomicMax(v.maxCycles, st[2] + st[3]);
}

// chosen_acc and the chosen record of (vector, server) i = j * S + s: the resident record scaled as greedy_scale does
// (got == nullptr: the records were scaled in place already)
__global__ void k_greedy_collect_multi(DevSystem sys, DevAllocs pairs, const int* __restrict__ order, const int* __restrict__ chosen_key,
                                       const long long* __restrict__ got, const long long* __restrict__ cur, size_t n,
                                       int* __restrict__ chosen_acc, wva_pair_rec* __restrict__ chosen) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = (int)(i % (size_t)sys.S);
    const int slot = chosen_key[i];
    const int key = slot >= 0 ? order[slot] : -1;
    chosen_acc[i] = key;
    AllocRec r = key >= 0 ? load_alloc(pairs, (size_t)s * sys.A + key) : empty_alloc();
    if (key >= 0 && got && got[i] > 0) {
        const float factor = (float)got[i] / (float)cur[i];
        r.cost = r.cost * factor;
        r.value = r.value * factor;
        r.numReplicas = got[i];
    }
    chosen[i] = to_pair_rec(r, key >= 0);
}

// the chosen records of one vector of wva_solve_capacities: chosen_acc[s] >= 0 marks a chosen server
struct TotalsPairRec {
    const int* __restrict__ chosen_acc; const wva_pair_rec* __restrict__ rec;
    __device__ bool chosen(int s) const { return chosen_acc[s] >= 0; }
    __device__ int acc(int s) const { return rec[s].acc; }
    __device__ long long replicas(int s) const { return rec[s].num_replicas; }
    __device__ float cost(int s) const { return rec[s].cost; }
};

// k_totals over every server for each vector of a chunk: block (t, j) sums type t of vector j in k_totals' order
__global__ void __launch_bounds__(1024) k_totals_multi(DevSystem sys, const int* __restrict__ chosen_acc, const wva_pair_rec* __restrict__ chosen,
                                                       long long* __restrict__ count, float* __restrict__ cost) {
    const size_t j = blockIdx.y;
    totals_block(sys, blockIdx.x, 0, sys.S, TotalsPairRec{chosen_acc + j * sys.S, chosen + j * sys.S}, count + j * sys.T, cost + j * sys.T);
}

// ---- many arrival-rate scenarios (wva_solve_loads) ---------------------------------------------------------------
// The candidate values depend on the load, so every scenario has records, a candidate order, a static order and greedy
// buffers of its own (one GreedyPlan each, built by the kernels above); only the image, its capacities included, is
// shared.  Each scenario's records are used once, so best effort scales them in place as in wva_solve.

// chunk records, scenario-major: plane item ((s * nL + j) * A + a) of k_pairs_loads -> (j * S + s) * A + a, so that
// scenario j's records are a DevAllocs at offset j * S * A
__global__ void k_loads_records(const wva_pair_rec* __restrict__ plane, int S, int A, int nL, DevAllocs out, unsigned char* __restrict__ feasible) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)S * nL * A) return;
    const size_t a = i % (size_t)A, sj = i / (size_t)A, j = sj % (size_t)nL, s = sj / (size_t)nL;
    const size_t o = (j * S + s) * A + a;
    const wva_pair_rec r = plane[i];
    out.acc[o] = r.acc; out.num_replicas[o] = r.num_replicas; out.batch_size[o] = r.batch_size;
    out.cost[o] = r.cost; out.value[o] = r.value; out.itl[o] = r.itl; out.ttft[o] = r.ttft; out.rho[o] = r.rho;
    out.max_arrv[o] = r.max_arrv_rate_per_replica;
    feasible[o] = r.feasible;
}

// what the pass of one scenario works on: its records, its greedy buffers, its static order and its chosen slots
struct GreedyLoadView {
    DevAllocs pairs; GreedyBufs g; GreedyScan gs; int* chosen;
};

// the static-order pass of k_greedy_scan once per scenario, one block of one warp each; maxCycles = SM cycles of the
// slowest scenario's pass
__global__ void __launch_bounds__(32) k_greedy_scan_loads(DevSystem sys, const GreedyLoadView* __restrict__ views, int delayedBestEffort,
                                                            int policy, unsigned long long* maxCycles) {
    extern __shared__ __align__(16) unsigned char greedy_pool[];
    __shared__ long long avail[256];
    __shared__ long long usum[256];
    const GreedyLoadView& v = views[blockIdx.x];
    GreedyCtx c; c.sys = sys; c.pairs = v.pairs; c.g = v.g; c.chosen = v.chosen; c.avail = avail; c.usum = usum; c.lane = threadIdx.x;
    unsigned long long st[4];
    greedy_scan_pass(c, v.gs, sys.type_capacity, greedy_pool, delayedBestEffort, policy, [](int g0) { return g0; }, st);
    if (threadIdx.x == 0) atomicMax(maxCycles, st[2] + st[3]);
}

}  // namespace wva
