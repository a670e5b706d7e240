// wva_block.cuh — blocking probability of the sweep's candidates (DESIGN.md 4.v).
//
// For a candidate (s, a, r, b) that Analyze accepts, p_block is float32(p[K]) of the reference's
// computeProbabilities (mm1modelstatedependent.go:70-112): the normalised probability that the K = 11 b
// places of the system are all taken, i.e. the share of requests turned away.  The sweep never needs it
// (its truncation rule and its certificate only decide 1 - float32(p[K])), so it is computed here, by
// kernels of its own, beside the sweep:
//
//   k_block_scan     one THREAD per row (s, a, r).  The row's ramp p[1..b_max] is the reference's own
//                    sequence (same operations, same order: bit-identical), and so is the running sum.
//                    Every candidate b of the row is then O(1): its tail is M = 10 b steps at the constant
//                    ratio lambda / s[b-1], and p_block is decided by a certificate (certified zero, or
//                    the closed form p[N] r^M / S with an error bound that covers the reference's own
//                    roundings) or the candidate is listed for an exact chain (non-tame table, a ramp that meets
//                    a rescale predicate, values outside the window the bounds assume, an ambiguous rounding).
//   k_block_exact    one thread per listed candidate: the reference's untruncated chain, streamed.  A
//                    chain that meets a rescale predicate is listed for the materialised path.
//   k_block_literal  one thread per candidate of that list: analyze_candidate on a p[] scratch row, i.e.
//                    solve_literal; p_block is the normalised p[K] it leaves there.
//
// Candidate ids are cube indices relative to the shard: ((sl*A + a)*r_max + (r-1))*b_max + (b-1).
#pragma once

namespace wva {

struct BlockParams {
    int r_max, b_max, s0, ns;
    float* plane;                                             // [ns*A*r_max*b_max]
    unsigned long long* exact_list; unsigned long long exact_cap;    // candidates for k_block_exact
    unsigned long long* lit_list; unsigned long long lit_cap;        // candidates for k_block_literal
    unsigned long long* list_count;                                  // [0] exact list, [1] literal list (64-bit: cannot wrap)
    unsigned long long* counts;                               // [0] certified zero, [1] certified closed form, [2] exact chain
};

#define WVA_BLOCK_NAN 0x7fc00000u
#define WVA_BLOCK_ZERO 0
#define WVA_BLOCK_CLOSED 1
#define WVA_BLOCK_EXACT 2

// Certificate of one candidate from the reference's own p[N] and sum_{i<=N} p[i] (DESIGN.md 4.v).
// lam = (double)lambda, s = (double)servRate[N-1] > 0, M = 10 N tail steps, K = 11 N.
__device__ __forceinline__ int block_certify(const double pN, const double sumRamp, const double lam, const double s,
                                             const int M, const int K, float& out) {
    // no reference value leaves [0, 2^1008) in the tail: p*lambda, every tail term and the sum stay finite
    if (!(pN < 0x1p990) || !(pN * lam < 0x1p1000) || !(sumRamp < 0x1p1000)) return WVA_BLOCK_EXACT;
    // rho >= r (1+u)^2 bounds one rounded tail step: p' <= rho p + 2^-1074 (1 + 1/s) <= rho p + 2^-924
    const double rho = __dmul_ru(__ddiv_ru(lam, s), 1.0 + 0x1p-50);
    if (!(rho <= 1.0 - 0x1p-11)) return WVA_BLOCK_EXACT;
    // certified zero: reference p[K] <= rho^M pN + 2^-913 < 2^-151, and p[K] / S <= p[K] since S >= 1
    if (pN < 0x1p-170) { out = 0.0f; return WVA_BLOCK_ZERO; }
    if (log2(pN) + (double)M * log2(rho) < -160.0) { out = 0.0f; return WVA_BLOCK_ZERO; }
    // certified closed form: v = pN r^M / (sumRamp + pN T0), T0 = sum_{j=1..M} r^j = r (1 - r^M) / (1 - r), with
    // 1 - r^M = -expm1(M ln r) and ln r from log1p(-(1 - r)) when r >= 1/2: no cancellation for any M (1 - r)
    const double r = lam / s;
    const double oneR = (s - lam) / s;                          // s - lam: exact when r >= 2^-29 (two float32 values)
    const double lr = oneR <= 0.5 ? log1p(-oneR) : log(r);
    const double T0 = r * -expm1((double)M * lr) / oneR;
    const double S = sumRamp + pN * T0;
    const double P = exp(log(pN) + (double)M * lr);
    if (!(S < 0x1p1000) || !(P >= 0x1p-200)) return WVA_BLOCK_EXACT;
    const double v = P / S;
    // reference: <= 2M roundings on p[K], <= M on S, one on the division; ours <= 5700 (DESIGN.md 4.v)
    const double E = (10.0 * (double)K + 16384.0) * 0x1p-53;
    return same_f32(v, E * v, out) ? WVA_BLOCK_CLOSED : WVA_BLOCK_EXACT;
}

__device__ __forceinline__ void block_append(unsigned long long* list, unsigned long long cap, unsigned long long* count,
                                             unsigned long long id) {
    const unsigned long long k = atomicAdd(count, 1ULL);
    if (k < cap) list[k] = id;
}

__global__ void __launch_bounds__(128)
k_block_scan(DevSystem sys, BlockParams bp) {
    const int A = sys.A, R = bp.r_max, B = bp.b_max;
    const long long nRows = (long long)bp.ns * A * R;
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long cnt[3] = {0, 0, 0};
    if (row < nRows) {
        const int r = (int)(row % R) + 1;
        const int a = (int)((row / R) % A);
        const int s = bp.s0 + (int)(row / ((long long)R * A));
        const size_t base = (size_t)row * B;
        float* out = bp.plane + base;
        const float qnan = __uint_as_float(WVA_BLOCK_NAN);
        GridServer gs;
        if (grid_pair_status(sys, s, a, gs) != WVA_CAND_OK) {
            for (int n = 0; n < B; ++n) out[n] = qnan;
        } else {
            ServFormula sf; sf.init(gs.sp, gs.inTok, gs.outTok);
            const bool tame = tame_parms(gs.sp, gs.inTok, gs.outTok);
            const float rate = gs.totalRate / (float)r;
            const float lambda = rate / 1000.0f;
            const double lam = (double)lambda;
            // the reference's ramp: p[n+1] = (p[n] * lambda) / s[n], sum = p[0] + ... + p[n+1]
            double p = 1.0, sum = 1.0;
            bool goodTable = true;                              // servRate[0..b-1] all positive and finite
            bool rampOk = true;                                 // no rescale predicate met by p[1..b] or their sum
            for (int n = 0; n < B; ++n) {
                const int b = n + 1;
                const float sF = sf.rate(b);
                if (!(sF > 0.0f) || !(sF < CUDART_INF_F)) goodTable = false;
                if (goodTable && rampOk) {
                    const double t = p * lam;
                    p = t / (double)sF;
                    sum += p;
                    if (!(p >= 0.0) || !(p < CUDART_INF) || !(sum < CUDART_INF)) rampOk = false;
                }
                float v = qnan;
                if (!goodTable) {                               // Analyze on this table: the literal path decides (status included)
                    block_append(bp.lit_list, bp.lit_cap, bp.list_count + 1, (unsigned long long)(base + n));
                    cnt[WVA_BLOCK_EXACT]++;
                } else if (rate > 0.0f && !(rate > (sF * (1.0f - WVA_EPSILON)) * 1000.0f) && !(lambda < 0.0f)) {
                    // analysed (queueanalyzer.go:135-150 with the sweep's predicates)
                    int how = WVA_BLOCK_EXACT;
                    if (rampOk && tame) how = block_certify(p, sum, lam, (double)sF, 10 * b, 11 * b, v);
                    if (how == WVA_BLOCK_ZERO) cnt[WVA_BLOCK_ZERO]++;
                    else if (how == WVA_BLOCK_CLOSED) cnt[WVA_BLOCK_CLOSED]++;
                    else {
                        block_append(bp.exact_list, bp.exact_cap, bp.list_count, (unsigned long long)(base + n));
                        cnt[WVA_BLOCK_EXACT]++;
                    }
                }
                out[n] = v;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        unsigned long long c = cnt[k];
        for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
        if ((threadIdx.x & 31) == 0 && c) atomicAdd(&bp.counts[k], c);
    }
}

// (sl, a, r, b) of a candidate id; the output slot is the id itself (plane) or the server (winners)
__device__ __forceinline__ void block_decode(const BlockParams& bp, int A, unsigned long long id, int& sl, int& a, int& r, int& b) {
    const int B = bp.b_max, R = bp.r_max;
    b = (int)(id % B) + 1;
    r = (int)((id / B) % R) + 1;
    const long long pair = (long long)(id / ((unsigned long long)B * R));
    sl = (int)(pair / A); a = (int)(pair % A);
}

// The reference's untruncated chain (mm1modelstatedependent.go:77-111) for one analysed candidate, streamed: p[n+1]
// = (p[n] * lambda) / sRate, sum = p[0] + ... + p[K] in index order, p[K] / sum.  No truncation rule: every one of the K
// steps runs.  A rescale predicate (:84, :95) sends the candidate to the literal list.
__global__ void __launch_bounds__(128)
k_block_exact(DevSystem sys, BlockParams bp, const unsigned long long* __restrict__ list, int n, float* __restrict__ out,
              int by_server) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const unsigned long long id = list[t];
    int sl, a, r, b;
    block_decode(bp, sys.A, id, sl, a, r, b);
    const size_t slot = by_server ? (size_t)sl : (size_t)id;
    GridServer gs;
    if (grid_pair_status(sys, bp.s0 + sl, a, gs) != WVA_CAND_OK) { out[slot] = __uint_as_float(WVA_BLOCK_NAN); return; }
    ServFormula sf; sf.init(gs.sp, gs.inTok, gs.outTok);
    const float lambda = (gs.totalRate / (float)r) / 1000.0f;
    const double lam = (double)lambda;
    const int N = b, K = 11 * b;
    const double sTail = (double)sf.rate(N);
    double p = 1.0, sum = 1.0;
    for (int k = 0; k < K; ++k) {
        const double sRate = k < N ? (double)sf.rate(k + 1) : sTail;
        const double q = p * lam;
        p = q / sRate;
        sum += p;
        if (!(p >= 0.0) || !(p < CUDART_INF) || !(sum < CUDART_INF)) {
            block_append(bp.lit_list, bp.lit_cap, bp.list_count + 1, id);
            return;
        }
    }
    out[slot] = (float)(p / sum);
}

// The materialised path: Analyze through analyze_candidate with a p[] scratch row (solve_literal, rescales included).
// p_block is its normalised p[K]; NaN when Analyze does not accept the candidate.
__global__ void __launch_bounds__(128)
k_block_literal(DevSystem sys, BlockParams bp, const unsigned long long* __restrict__ list, int n, double* scratch,
                long long stride, float* __restrict__ out, int by_server) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const unsigned long long id = list[t];
    int sl, a, r, b;
    block_decode(bp, sys.A, id, sl, a, r, b);
    double* row = scratch + (size_t)t * stride;
    GridServer gs; wva_metrics m; float rate, rateTPS; int fault = 0; unsigned long long steps = 0;
    const int st = analyze_candidate(sys, bp.s0 + sl, a, r, b, nullptr, row, gs, m, rate, rateTPS, fault, steps);
    out[by_server ? (size_t)sl : (size_t)id] = (st == WVA_CAND_OK) ? (float)row[11 * b] : __uint_as_float(WVA_BLOCK_NAN);
}

}  // namespace wva
