// wva_oracle.cpp — CPU restatement of the reference's Analyze -> Optimize path.
//
// THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load it.  The shipped library
// (libwva_b200.so) never links, loads or calls anything in oracle/.
//
// The reference is Go and no Go toolchain exists in this image, so the reference itself
// cannot be executed here.  Parity status: the restatement is pinned against every exact
// value the reference's own tests hold for this path (tests/test_oracle_golden.py lists them
// with file:line); all other values are defined by fidelity to the cited source lines
// ("parity unpinned" beyond those vectors, see DESIGN.md).
//
// Typing rule: every arithmetic operation below is performed in the type the Go source
// performs it in (float32 / float64 / int = int64), one rounding per operation.  Build with
//   g++ -O2 -ffp-contract=off -fno-fast-math -fexcess-precision=standard
// (x86-64 SSE2: no x87 excess precision, no FMA contraction; Go on amd64 does not fuse).
//
// Citations are file:line relative to the reference tree.

#include "../include/wva_b200.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <thread>
#include <vector>

namespace {

// ---------------------------------------------------------------------------------------
// Go semantics helpers
// ---------------------------------------------------------------------------------------

// Go builtin min/max on floats: NaN if any argument is NaN; -0 < +0 (Go spec, "Min and max").
inline float go_minf(float a, float b) {
    if (a != a || b != b) return std::numeric_limits<float>::quiet_NaN();
    if (a == 0.0f && b == 0.0f) return std::signbit(a) ? a : b;
    return a < b ? a : b;
}
inline float go_maxf(float a, float b) {
    if (a != a || b != b) return std::numeric_limits<float>::quiet_NaN();
    if (a == 0.0f && b == 0.0f) return std::signbit(a) ? b : a;
    return a > b ? a : b;
}
inline int64_t go_maxi(int64_t a, int64_t b) { return a > b ? a : b; }
inline int64_t go_mini(int64_t a, int64_t b) { return a < b ? a : b; }

// Go int(float64) on amd64 (CVTTSD2SQ): out-of-range, Inf and NaN give MinInt64.
inline int64_t go_f64_to_int(double x) {
    if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return INT64_MIN;
    return (int64_t)x;
}
// Go int multiplication wraps.
inline int64_t go_muli(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }
// Go int division truncates toward zero; MinInt64 / -1 wraps to MinInt64 (no panic for non-constants).
inline int64_t go_divi(int64_t a, int64_t b) {
    if (a == INT64_MIN && b == -1) return INT64_MIN;
    return a / b;
}
// cmp.Compare for floats: NaN is less than any non-NaN, NaN == NaN, -0 == +0.
inline int go_cmpf(float x, float y) {
    bool xn = x != x, yn = y != y;
    if (xn) return yn ? 0 : -1;
    if (yn) return +1;
    if (x < y) return -1;
    if (x > y) return +1;
    return 0;
}
inline int go_cmpi(int64_t x, int64_t y) { return x < y ? -1 : (x > y ? +1 : 0); }

// instrumentation: overflow-rescale branches taken, the chain's (mm1modelstatedependent.go:84-89) and the
// normalising sum's (:95-104) apart
std::atomic<uint64_t> g_rescale_chain{0};
std::atomic<uint64_t> g_rescale_sum{0};
const float kMaxFloat32 = std::numeric_limits<float>::max();
const double kMaxFloat64 = std::numeric_limits<double>::max();

// ---------------------------------------------------------------------------------------
// pkg/analyzer: MM1ModelStateDependent on top of MM1KModel / QueueModel
// ---------------------------------------------------------------------------------------

// State of one model instance.  p[] persists across Solve calls (the stale-p[0] validity
// quirk of pkg/analyzer/queuemodel.go:30 + mm1modelstatedependent.go:33-35 needs it).
struct StateDependentModel {
    int64_t K = 0;                 // MM1KModel.K                       mm1kmodel.go:12
    std::vector<double> p;         // MM1KModel.p, K+1 zeros at start   mm1kmodel.go:22
    std::vector<float> servRate;   // mm1modelstatedependent.go:10
    float lambda = 0, mu = 0, rho = 0;
    float avgRespTime = 0, avgWaitTime = 0, avgServTime = 0, avgNumInSystem = 0, avgQueueLength = 0;
    float avgNumInServers = 0, throughput = 0;
    bool isValid = false;
    uint64_t steps = 0;            // instrumentation only: chain steps executed

    // NewMM1ModelStateDependent, mm1modelstatedependent.go:15-26 (+ NewMM1KModel mm1kmodel.go:18-30)
    void init(int64_t K_, std::vector<float>&& serv) {
        K = K_;
        p.assign((size_t)K + 1, 0.0);
        servRate = std::move(serv);
    }

    // MM1ModelStateDependent.ComputeRho, mm1modelstatedependent.go:33-35
    float computeRho() const { return 1.0f - (float)p[0]; }
    // MM1KModel.GetRhoMax, mm1kmodel.go:47-49
    float rhoMax() const { return (float)K; }

    // QueueModel.Solve, queuemodel.go:27-37
    void solve(float lambda_, float mu_) {
        lambda = lambda_;
        mu = mu_;
        rho = computeRho();
        if ((rho < 0) || (rho >= rhoMax()) || (lambda_ < 0) || (mu_ <= 0)) {
            isValid = false;
        } else {
            isValid = true;
            computeStatistics();
        }
    }

    // computeProbabilities, mm1modelstatedependent.go:70-116
    void computeProbabilities() {
        p[0] = 1;
        const double scale = kMaxFloat64 / (double)K;                          // :74
        double sRate = 0;
        const int64_t num = (int64_t)servRate.size();
        for (int64_t n = 0; n < K; n++) {                                       // :77
            if (n < num) sRate = (double)servRate[(size_t)n];
            else         sRate = (double)servRate[(size_t)num - 1];
            double t = p[n] * (double)lambda;                                   // :83, (p*lambda)/s
            p[n + 1] = t / sRate;
            while (p[n + 1] < 0 || std::isinf(p[n + 1]) || std::isnan(p[n + 1])) {   // :84
                g_rescale_chain++;
                for (int64_t i = 0; i <= n; i++) p[i] /= scale;
                double t2 = p[n] * (double)lambda;
                p[n + 1] = t2 / sRate;
            }
        }
        double sum = 0;                                                         // :92
        for (int64_t n = 0; n <= K; n++) {
            sum += p[n];
            if (sum < 0 || std::isinf(sum)) {                                   // :95
                g_rescale_sum++;
                sum = 0;
                for (int64_t i = 0; i <= K; i++) {
                    p[i] /= scale;
                    if (i <= n) sum += p[i];
                }
            }
        }
        for (int64_t n = 0; n <= K; n++) p[n] /= sum;                           // :108-111 (sumP unused)
        rho = computeRho();                                                     // :114
        steps += 2 * (uint64_t)(K + 1);
    }

    // computeStatistics, mm1modelstatedependent.go:38-67
    void computeStatistics() {
        if (!isValid) return;
        computeProbabilities();
        const int64_t num = (int64_t)servRate.size();
        double inServ = 0, inSys = 0;
        double sumP = p[0];
        for (int64_t i = 1; i <= K; i++) {
            double term = (double)i * p[i];
            inSys += term;
            sumP += p[i];
            if (i == num) {
                double rest = (1 - sumP) * (double)num;
                inServ = inSys + rest;
            }
        }
        avgNumInServers = (float)inServ;
        avgNumInSystem = (float)inSys;
        throughput = lambda * (1 - (float)p[K]);                                // :59
        avgRespTime = avgNumInSystem / throughput;
        avgServTime = avgNumInServers / throughput;
        avgWaitTime = avgRespTime - avgServTime;
        if (avgWaitTime < 0) avgWaitTime = 0;
        avgQueueLength = throughput * avgWaitTime;
    }
};

// MM1KModel, mm1kmodel.go:10-93 (closed form; the one place math.Pow appears; not on the
// CreateAllocation path — kept for API completeness and as an independent check of the chain).
struct MM1KClosedForm {
    int64_t K = 0;
    std::vector<double> p;
    float lambda = 0, mu = 0, rho = 0, throughput = 0;
    float avgRespTime = 0, avgWaitTime = 0, avgServTime = 0, avgNumInSystem = 0, avgQueueLength = 0;
    bool isValid = false;
    explicit MM1KClosedForm(int64_t K_) : K(K_), p((size_t)K_ + 1, 0.0) {}
    float computeRho() const { return lambda == mu ? 1.0f : lambda / mu; }              // :38-44
    void solve(float l, float m) {                                                       // queuemodel.go:27-37
        lambda = l; mu = m; rho = computeRho();
        if ((rho < 0) || (rho >= (float)K) || (l < 0) || (m <= 0)) { isValid = false; return; }
        isValid = true;
        if (rho == 1) p[0] = 1 / (double)(K + 1);                                        // :60-64
        else p[0] = (1 - (double)rho) / (1 - std::pow((double)rho, (double)(K + 1)));
        for (int64_t i = 0; i <= K; i++) p[(size_t)i] = p[0] * std::pow((double)rho, (double)i);   // :67-70
        double temp = 0;
        for (int64_t i = 0; i <= K; i++) temp += (double)i * p[(size_t)i];               // :79-82
        avgNumInSystem = (float)temp;
        throughput = lambda * (1 - (float)p[(size_t)K]);
        avgRespTime = avgNumInSystem / throughput;
        avgServTime = 1 / mu;
        avgWaitTime = avgRespTime - avgServTime;
        if (avgWaitTime < 0) avgWaitTime = 0;
        avgQueueLength = throughput * avgWaitTime;
    }
};

struct ServiceParms { float alpha, beta, gamma, delta; };

// PrefillParms.PrefillTime, queueanalyzer.go:257-262
inline float prefillTime(const ServiceParms& sp, int64_t avgInputTokens, float batchSize) {
    if (avgInputTokens == 0) return 0;
    float t = sp.delta * (float)avgInputTokens;
    t = t * batchSize;
    return sp.gamma + t;
}
// DecodeParms.DecodeTime, queueanalyzer.go:264-266
inline float decodeTime(const ServiceParms& sp, float batchSize) {
    float t = sp.beta * batchSize;
    return sp.alpha + t;
}

// EffectiveConcurrency, queueanalyzer.go:296-302
inline float effectiveConcurrency(float avgServiceTime, const ServiceParms& sp, int64_t inTok, int64_t outTok,
                                  int64_t maxBatchSize) {
    float tokens = (float)(outTok - 1);
    float at = sp.alpha * tokens;
    float base = sp.gamma + at;
    float numerator = avgServiceTime - base;
    float d1 = sp.delta * (float)inTok;
    float d2 = sp.beta * tokens;
    float denominator = d1 + d2;
    float n = numerator / denominator;
    return go_minf(go_maxf(n, 0.0f), (float)maxBatchSize);
}

struct QueueAnalyzer {
    int64_t maxBatchSize = 0, maxQueueSize = 0;
    ServiceParms sp{};
    int64_t inTok = 0, outTok = 0;
    StateDependentModel model;
    float rateMin = 0, rateMax = 0;   // RateRange, req/sec
};

// Configuration.check + RequestSize.check, queueanalyzer.go:337-352
inline bool configOk(int64_t N, int64_t maxQueue, int64_t inTok, int64_t outTok) {
    if (N <= 0 || maxQueue < 0) return false;
    if (inTok < 0 || outTok < 1) return false;
    return true;
}

// BuildModel, queueanalyzer.go:99-131
void buildModel(QueueAnalyzer& qa, int64_t N, int64_t maxQueue, const ServiceParms& sp, int64_t inTok, int64_t outTok) {
    std::vector<float> servRate((size_t)N);
    for (int64_t n = 1; n <= N; n++) {
        float pre = prefillTime(sp, inTok, (float)n);
        int64_t numDecode = outTok - 1;
        if (inTok == 0 && outTok == 1) numDecode = 1;
        float dec = (float)numDecode * decodeTime(sp, (float)n);
        float tot = pre + dec;
        servRate[(size_t)n - 1] = (float)n / tot;
    }
    float lambdaMin = servRate[0] * WVA_EPSILON;
    float lambdaMax = servRate[(size_t)N - 1] * (1.0f - WVA_EPSILON);
    qa.rateMin = lambdaMin * 1000.0f;
    qa.rateMax = lambdaMax * 1000.0f;
    qa.maxBatchSize = N;
    qa.maxQueueSize = maxQueue;
    qa.sp = sp;
    qa.inTok = inTok;
    qa.outTok = outTok;
    qa.model.init(maxQueue + N, std::move(servRate));
}

// QueueAnalyzer.Analyze, queueanalyzer.go:134-174.  Returns WVA_CAND_OK or an error status.
int analyze(QueueAnalyzer& qa, float requestRate, wva_metrics* m) {
    if (requestRate <= 0) return WVA_CAND_ERR_RATE_LE0;
    if (requestRate > qa.rateMax) return WVA_CAND_ERR_RATE_MAX;
    qa.model.solve(requestRate / 1000.0f, 1.0f);
    if (!qa.model.isValid) return WVA_CAND_ERR_MODEL;
    float avgNumInServ = qa.model.avgNumInServers;
    float effConc = effectiveConcurrency(qa.model.avgServTime, qa.sp, qa.inTok, qa.outTok, qa.maxBatchSize);
    float pre = prefillTime(qa.sp, qa.inTok, effConc);
    float tok = decodeTime(qa.sp, effConc);
    float rho = avgNumInServ / (float)qa.maxBatchSize;
    rho = go_minf(go_maxf(rho, 0.0f), 1.0f);
    m->throughput = qa.model.throughput * 1000.0f;
    m->avg_resp_time = qa.model.avgRespTime;
    m->avg_wait_time = qa.model.avgWaitTime;
    m->avg_num_in_serv = avgNumInServ;
    m->avg_prefill_time = pre;
    m->avg_token_time = tok;
    m->max_rate = qa.rateMax;
    m->rho = rho;
    return WVA_CAND_OK;
}

// WithinTolerance, utils.go:12-20
inline bool withinTolerance(float x, float value, float tolerance) {
    if (x == value) return true;
    if (value == 0 || tolerance < 0) return false;
    float d = x - value;
    float q = d / value;
    return std::fabs((double)q) <= (double)tolerance;
}

// EvalTTFT / EvalITL, queueanalyzer.go:270-290.  Returns false on "invalid model".
enum EvalKind { EVAL_TTFT, EVAL_ITL };
inline bool evalTarget(QueueAnalyzer& qa, EvalKind kind, float x, float* y) {
    qa.model.solve(x, 1.0f);
    if (!qa.model.isValid) return false;
    float effConc = effectiveConcurrency(qa.model.avgServTime, qa.sp, qa.inTok, qa.outTok, qa.maxBatchSize);
    if (kind == EVAL_TTFT) *y = qa.model.avgWaitTime + prefillTime(qa.sp, qa.inTok, effConc);
    else                   *y = decodeTime(qa.sp, effConc);
    return true;
}

// BinarySearch, utils.go:26-70.  Returns false on error; ind in {-1,0,+1}.
// `eval(x, &y)` returns false for the reference's "invalid function evaluation" error.
template <class Eval>
bool binarySearchGeneric(Eval eval, float xMin, float xMax, float yTarget, float* xOut, int* ind) {
    *xOut = 0; *ind = 0;
    if (xMin > xMax) return false;
    float yBounds[2];
    const float xs[2] = {xMin, xMax};
    for (int i = 0; i < 2; i++) {
        if (!eval(xs[i], &yBounds[i])) return false;
        if (withinTolerance(yBounds[i], yTarget, WVA_BISECT_TOL)) { *xOut = xs[i]; *ind = 0; return true; }
    }
    bool increasing = yBounds[0] < yBounds[1];
    if ((increasing && yTarget < yBounds[0]) || (!increasing && yTarget > yBounds[0])) { *xOut = xMin; *ind = -1; return true; }
    if ((increasing && yTarget > yBounds[1]) || (!increasing && yTarget < yBounds[1])) { *xOut = xMax; *ind = +1; return true; }
    float xStar = 0, yStar = 0;
    for (int it = 0; it < WVA_BISECT_MAXIT; it++) {
        xStar = 0.5f * (xMin + xMax);
        if (!eval(xStar, &yStar)) return false;
        if (withinTolerance(yStar, yTarget, WVA_BISECT_TOL)) break;
        if ((increasing && yTarget < yStar) || (!increasing && yTarget > yStar)) xMax = xStar;
        else xMin = xStar;
    }
    *xOut = xStar; *ind = 0;
    return true;
}
bool binarySearch(QueueAnalyzer& qa, EvalKind kind, float xMin, float xMax, float yTarget, float* xOut, int* ind) {
    return binarySearchGeneric([&](float x, float* y) { return evalTarget(qa, kind, x, y); }, xMin, xMax, yTarget, xOut, ind);
}

// QueueAnalyzer.Size, queueanalyzer.go:185-255.  Returns false on any error.
bool sizeQueue(QueueAnalyzer& qa, float targetTTFT, float targetITL, float targetTPS,
               float rates[3], wva_metrics* metrics, float achieved[3]) {
    if (targetITL < 0 || targetTTFT < 0 || targetTPS < 0) return false;       // TargetPerf.check :355-362
    float lambdaMin = qa.rateMin / 1000.0f;
    float lambdaMax = qa.rateMax / 1000.0f;
    int ind = 0;
    float lambdaStarTTFT = lambdaMax;
    if (targetTTFT > 0) {
        bool ok = binarySearch(qa, EVAL_TTFT, lambdaMin, lambdaMax, targetTTFT, &lambdaStarTTFT, &ind);
        if (ind < 0) ok = false;
        if (!ok) return false;
    }
    float lambdaStarITL = lambdaMax;
    if (targetITL > 0) {
        bool ok = binarySearch(qa, EVAL_ITL, lambdaMin, lambdaMax, targetITL, &lambdaStarITL, &ind);
        if (ind < 0) ok = false;
        if (!ok) return false;
    }
    float lambdaStarTPS = lambdaMax;
    if (targetTPS > 0) lambdaStarTPS = lambdaMax * (1.0f - WVA_STABILITY_SAFETY);
    float lambda = go_minf(go_minf(lambdaStarTTFT, lambdaStarITL), lambdaStarTPS);
    float requestRate = lambda * 1000.0f;
    if (analyze(qa, requestRate, metrics) != WVA_CAND_OK) return false;
    rates[0] = lambdaStarTTFT * 1000.0f;
    rates[1] = lambdaStarITL * 1000.0f;
    rates[2] = lambdaStarTPS * 1000.0f;
    achieved[0] = metrics->avg_wait_time + metrics->avg_prefill_time;
    achieved[1] = metrics->avg_token_time;
    achieved[2] = metrics->throughput * (float)qa.outTok;
    return true;
}

// ---------------------------------------------------------------------------------------
// pkg/core
// ---------------------------------------------------------------------------------------

struct Alloc {                 // core.Allocation, allocation.go:13-24
    int32_t acc = WVA_ACC_NONE;
    int64_t numReplicas = 0, batchSize = 0;
    float cost = 0, value = 0, itl = 0, ttft = 0, rho = 0, maxArrv = 0;
};

// Allocation.TransitionPenalty, allocation.go:291-300 (a = current, b = candidate).
// Accelerator names compare as strings; index equality is the same thing once interned
// (WVA_ACC_NONE == "" on both sides; WVA_ACC_UNKNOWN never equals a candidate).
inline float transitionPenalty(int32_t aAcc, int64_t aRep, float aCost, const Alloc& b) {
    if (aAcc == b.acc && aAcc != WVA_ACC_UNKNOWN) {
        if (aRep == b.numReplicas) return 0;
        return b.cost - aCost;
    }
    float s = aCost + b.cost;
    float p = WVA_ACCEL_PENALTY_FACTOR * s;
    float d = b.cost - aCost;
    return p + d;
}

inline int64_t numInstances(const wva_system_soa* sys, int32_t m, int32_t a) {   // model.go:45-54
    int32_t c = sys->perf_acc_count[(size_t)m * sys->n_accels + a];
    return c <= 0 ? 1 : c;
}

// lookups of CreateAllocation, allocation.go:41-70 (everything that yields nil before any math)
inline bool pairLookupsOk(const wva_system_soa* sys, int32_t s, int32_t a) {
    if (sys->srv_arrival_rpm[s] < 0 || sys->srv_in_tokens[s] < 0 || sys->srv_out_tokens[s] < 0) return false;
    int32_t m = sys->srv_model[s];
    if (m < 0 || m >= sys->n_models) return false;
    if (!sys->perf_valid[(size_t)m * sys->n_accels + a]) return false;
    if (!sys->srv_target_valid[s]) return false;
    return true;
}

// Server.GetCandidateAccelerators, server.go:70-82
inline bool isCandidateAccel(const wva_system_soa* sys, int32_t s, int32_t a) {
    if (sys->srv_keep_acc[s]) {
        int32_t cur = sys->srv_cur_acc[s];
        if (cur != WVA_ACC_NONE) return cur == a;   // WVA_ACC_UNKNOWN: empty candidate map
    }
    return true;
}

// zeroLoadAllocation, allocation.go:259-288
Alloc zeroLoadAllocation(const wva_system_soa* sys, int32_t s, int32_t a) {
    Alloc out;
    int64_t numReplicas = sys->srv_min_replicas[s];
    if (numReplicas == 0) return out;     // accelerator "", everything zero
    int32_t m = sys->srv_model[s];
    size_t pi = (size_t)m * sys->n_accels + a;
    int64_t maxBatchSize = sys->perf_max_batch[pi];
    if (sys->srv_max_batch[s] > 0) maxBatchSize = sys->srv_max_batch[s];
    int64_t total = go_muli(numInstances(sys, m, a), numReplicas);
    float cost = sys->acc_cost[a] * (float)total;
    float alpha = sys->perf_alpha[pi], beta = sys->perf_beta[pi], gamma = sys->perf_gamma[pi], delta = sys->perf_delta[pi];
    float decode = alpha + beta;
    float bb = beta * (float)maxBatchSize;
    float maxDecode = alpha + bb;
    float prefill = gamma + delta;
    float maxServ = prefill + maxDecode;
    float maxArrv = (float)maxBatchSize / maxServ;
    out.acc = a; out.numReplicas = numReplicas; out.batchSize = maxBatchSize;
    out.cost = cost; out.itl = decode; out.ttft = prefill; out.rho = 0; out.maxArrv = maxArrv;
    out.value = cost;
    return out;
}

// CreateAllocation, allocation.go:27-163.  Returns false for nil.
bool createAllocation(const wva_system_soa* sys, int32_t s, int32_t a, Alloc* out, uint64_t* steps) {
    if (!pairLookupsOk(sys, s, a)) return false;
    const float arrival = sys->srv_arrival_rpm[s];
    const int64_t inTok = sys->srv_in_tokens[s], outTok = sys->srv_out_tokens[s];
    if (arrival == 0 || outTok == 0) { *out = zeroLoadAllocation(sys, s, a); return true; }   // :73
    int32_t m = sys->srv_model[s];
    size_t pi = (size_t)m * sys->n_accels + a;
    const int64_t K = outTok;
    int64_t N;
    if (sys->srv_max_batch[s] > 0) N = sys->srv_max_batch[s];
    else N = go_maxi(go_divi(go_muli(sys->perf_max_batch[pi], sys->perf_at_tokens[pi]), K), 1);   // :85
    int64_t maxQueue = go_muli(N, WVA_MAX_QUEUE_TO_BATCH_RATIO);
    ServiceParms sp{sys->perf_alpha[pi], sys->perf_beta[pi], sys->perf_gamma[pi], sys->perf_delta[pi]};
    if (!configOk(N, maxQueue, inTok, K)) return false;
    QueueAnalyzer qa;
    buildModel(qa, N, maxQueue, sp, inTok, K);
    float rates[3], achieved[3];
    wva_metrics metrics;
    bool ok = sizeQueue(qa, sys->srv_slo_ttft[s], sys->srv_slo_itl[s], sys->srv_slo_tps[s], rates, &metrics, achieved);
    if (steps) *steps += qa.model.steps;
    if (!ok) return false;
    float rateStar = metrics.throughput;
    float totalRate;
    if (sys->srv_slo_tps[s] == 0) totalRate = arrival / 60.0f;
    else totalRate = sys->srv_slo_tps[s] / (float)K;
    int64_t numReplicas = go_f64_to_int(std::ceil((double)totalRate / (double)rateStar));   // :140
    numReplicas = go_maxi(numReplicas, sys->srv_min_replicas[s]);
    int64_t totalNumInstances = go_muli(numInstances(sys, m, a), numReplicas);
    float cost = sys->acc_cost[a] * (float)totalNumInstances;
    float rate = totalRate / (float)numReplicas;
    uint64_t before = qa.model.steps;
    if (analyze(qa, rate, &metrics) != WVA_CAND_OK) return false;
    if (steps) *steps += qa.model.steps - before;
    out->acc = a; out->numReplicas = numReplicas; out->batchSize = N;
    out->cost = cost; out->itl = metrics.avg_token_time;
    out->ttft = metrics.avg_wait_time + metrics.avg_prefill_time;
    out->rho = metrics.rho; out->maxArrv = rateStar / 1000.0f;
    out->value = cost;
    return true;
}

// Server.Calculate for one (server, accelerator): CreateAllocation + penalty, server.go:55-67
bool calculatePair(const wva_system_soa* sys, int32_t s, int32_t a, Alloc* out, uint64_t* steps) {
    if (!isCandidateAccel(sys, s, a)) return false;
    if (!createAllocation(sys, s, a, out, steps)) return false;
    out->value = transitionPenalty(sys->srv_cur_acc[s], sys->srv_cur_replicas[s], sys->srv_cur_cost[s], *out);
    return true;
}

inline void storeAlloc(wva_alloc_soa* o, size_t i, const Alloc& a) {
    o->acc[i] = a.acc; o->num_replicas[i] = a.numReplicas; o->batch_size[i] = a.batchSize;
    o->cost[i] = a.cost; o->value[i] = a.value; o->itl[i] = a.itl; o->ttft[i] = a.ttft; o->rho[i] = a.rho;
    o->max_arrv_rate_per_replica[i] = a.maxArrv;
}
inline Alloc loadAlloc(const wva_alloc_soa* o, size_t i) {
    Alloc a;
    a.acc = o->acc[i]; a.numReplicas = o->num_replicas[i]; a.batchSize = o->batch_size[i];
    a.cost = o->cost[i]; a.value = o->value[i]; a.itl = o->itl[i]; a.ttft = o->ttft[i]; a.rho = o->rho[i];
    a.maxArrv = o->max_arrv_rate_per_replica[i];
    return a;
}

template <class F>
void parallelFor(int64_t n, int threads, F f) {
    if (threads <= 1 || n <= 1) { for (int64_t i = 0; i < n; i++) f(i); return; }
    std::atomic<int64_t> next{0};
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; t++)
        pool.emplace_back([&] { for (;;) { int64_t i = next.fetch_add(1); if (i >= n) break; f(i); } });
    for (auto& th : pool) th.join();
}

// ---------------------------------------------------------------------------------------
// pkg/solver
// ---------------------------------------------------------------------------------------

struct ServerEntry {           // greedy.go:15-21
    int32_t server;
    int64_t priority;
    int64_t curIndex;
    std::vector<int32_t> allocs;   // keys (accelerator index) ordered by value
    float delta;
};

struct GreedyState {
    const wva_system_soa* sys;
    std::vector<Alloc> cand;          // S*A working copies (best effort mutates them in place, greedy.go:208-212)
    const uint8_t* feasible;
    std::vector<int32_t> chosen;      // S, key of chosen candidate or -1
    std::vector<int64_t> available;   // T
    Alloc& alloc(int32_t s, int32_t key) { return cand[(size_t)s * sys->n_accels + key]; }
};

// orderFunc, greedy.go:76-85
int orderFunc(GreedyState& g, const ServerEntry* a, const ServerEntry* b) {
    if (a->priority == b->priority) {
        if (a->delta == b->delta) {
            return go_cmpf(g.alloc(b->server, b->allocs[(size_t)b->curIndex]).value,
                           g.alloc(a->server, a->allocs[(size_t)a->curIndex]).value);
        }
        return go_cmpf(b->delta, a->delta);
    }
    return go_cmpi(a->priority, b->priority);
}

// units needed by one replica: model.NumInstances(gName) * acc.Spec().Multiplicity, greedy.go:136
inline int64_t unitsPerReplica(const wva_system_soa* sys, int32_t s, int32_t accIdx) {
    return go_muli(numInstances(sys, sys->srv_model[s], accIdx), sys->acc_multiplicity[accIdx]);
}

// allocate, greedy.go:107-166
std::vector<ServerEntry*> allocate(GreedyState& g, std::vector<ServerEntry*> entries) {
    std::vector<ServerEntry*> unallocated;
    const wva_system_soa* sys = g.sys;
    while (!entries.empty()) {
        ServerEntry* top = entries.front();
        entries.erase(entries.begin());
        if (top->allocs.empty()) continue;
        int32_t s = top->server;
        int32_t m = sys->srv_model[s];
        if (m < 0) continue;                                     // GetModel == nil
        int32_t key = top->allocs[(size_t)top->curIndex];
        Alloc& al = g.alloc(s, key);
        int32_t gi = al.acc;                                     // alloc.Accelerator()
        if (gi < 0) continue;                                    // GetAccelerator("") == nil, :130-133
        int32_t t = sys->acc_type[gi];
        int64_t upr = unitsPerReplica(sys, s, gi);
        int64_t count = go_muli(al.numReplicas, upr);
        if (g.available[(size_t)t] >= count) {
            g.available[(size_t)t] -= count;
            g.chosen[(size_t)s] = key;
        } else {
            top->curIndex++;
            int64_t len = (int64_t)top->allocs.size();
            if (top->curIndex + 1 < len) {
                top->delta = g.alloc(s, top->allocs[(size_t)top->curIndex + 1]).value -
                             g.alloc(s, top->allocs[(size_t)top->curIndex]).value;
            } else if (top->curIndex == len) {
                unallocated.push_back(top);
                continue;
            } else {
                top->delta = kMaxFloat32;
            }
            // slices.BinarySearchFunc: leftmost i with orderFunc(entries[i], top) >= 0
            size_t lo = 0, hi = entries.size();
            while (lo < hi) {
                size_t mid = lo + (hi - lo) / 2;
                if (orderFunc(g, entries[mid], top) < 0) lo = mid + 1; else hi = mid;
            }
            entries.insert(entries.begin() + (ptrdiff_t)lo, top);
        }
    }
    return unallocated;
}

// allocateMaximally, greedy.go:194-223
void allocateMaximally(GreedyState& g, const std::vector<ServerEntry*>& entries) {
    const wva_system_soa* sys = g.sys;
    for (ServerEntry* e : entries) {
        int32_t s = e->server;
        for (int32_t key : e->allocs) {
            Alloc& al = g.alloc(s, key);
            int32_t gi = al.acc;
            if (gi < 0 || sys->srv_model[s] < 0) continue;
            int64_t upr = unitsPerReplica(sys, s, gi);
            if (upr > 0) {
                int32_t t = sys->acc_type[gi];
                int64_t maxReplicas = go_divi(g.available[(size_t)t], upr);
                maxReplicas = go_mini(maxReplicas, al.numReplicas);
                if (maxReplicas > 0) {
                    int64_t cur = al.numReplicas;
                    float factor = (float)maxReplicas / (float)cur;
                    al.cost = al.cost * factor;
                    al.value = al.value * factor;
                    al.numReplicas = maxReplicas;
                    g.chosen[(size_t)s] = key;
                    g.available[(size_t)t] -= go_muli(maxReplicas, upr);
                    break;
                }
            }
        }
    }
}

// allocateEqually, greedy.go:239-316
void allocateEqually(GreedyState& g, const std::vector<ServerEntry*>& entries) {
    const wva_system_soa* sys = g.sys;
    struct Ticket { bool present = false, active = false, allocated = false; int32_t type = 0; int64_t upr = 0, numReplicas = 0; int32_t key = -1; };
    std::vector<Ticket> tickets(entries.size());
    size_t live = 0;
    for (size_t i = 0; i < entries.size(); i++) {
        if (sys->srv_model[entries[i]->server] < 0) continue;
        tickets[i].present = true; live++;
    }
    while (live > 0) {
        for (size_t i = 0; i < entries.size(); i++) {
            Ticket& tk = tickets[i];
            if (!tk.present) continue;
            ServerEntry* e = entries[i];
            int32_t s = e->server;
            if (!tk.active) {
                for (int32_t key : e->allocs) {
                    Alloc& al = g.alloc(s, key);
                    int32_t gi = al.acc;
                    if (gi < 0) continue;
                    int64_t upr = unitsPerReplica(sys, s, gi);
                    int32_t t = sys->acc_type[gi];
                    if (upr > 0 && g.available[(size_t)t] >= upr) {
                        tk.active = true; tk.type = t; tk.upr = upr; tk.key = key;
                        break;
                    }
                }
                if (!tk.active) { tk.present = false; live--; continue; }
            }
            int64_t replicasAvailable = go_divi(g.available[(size_t)tk.type], tk.upr);
            int64_t allocatable = go_mini(replicasAvailable, g.alloc(s, tk.key).numReplicas);
            if (allocatable > 0) {
                tk.numReplicas++;
                g.available[(size_t)tk.type] -= tk.upr;
                tk.allocated = true;
            } else {
                tk.present = false; live--;
            }
        }
    }
    for (size_t i = 0; i < entries.size(); i++) {
        Ticket& tk = tickets[i];
        if (!tk.allocated) continue;
        int32_t s = entries[i]->server;
        Alloc& al = g.alloc(s, tk.key);
        int64_t cur = al.numReplicas;
        float factor = (float)tk.numReplicas / (float)cur;
        al.cost = al.cost * factor;
        al.value = al.value * factor;
        al.numReplicas = tk.numReplicas;
        g.chosen[(size_t)s] = tk.key;
    }
}

// makePriorityGroups, greedy.go:321-341
std::vector<std::vector<ServerEntry*>> makePriorityGroups(const std::vector<ServerEntry*>& entries) {
    std::vector<std::vector<ServerEntry*>> groups;
    size_t index = 0, n = entries.size();
    while (index < n) {
        std::vector<ServerEntry*> group;
        group.push_back(entries[index]);
        int64_t pr = entries[index]->priority;
        index++;
        while (index < n && entries[index]->priority == pr) { group.push_back(entries[index]); index++; }
        groups.push_back(std::move(group));
    }
    return groups;
}

// bestEffort, greedy.go:169-190
void bestEffort(GreedyState& g, const std::vector<ServerEntry*>& unallocated, int policy) {
    switch (policy) {
        case WVA_POLICY_PRIORITY_EXHAUSTIVE: allocateMaximally(g, unallocated); break;
        case WVA_POLICY_PRIORITY_ROUND_ROBIN:
            for (auto& grp : makePriorityGroups(unallocated)) allocateEqually(g, grp);
            break;
        case WVA_POLICY_ROUND_ROBIN: allocateEqually(g, unallocated); break;
        default: break;
    }
}

}  // namespace

// =======================================================================================
// exported test API (prefix wvao_: "wva oracle")
// =======================================================================================
extern "C" {

int wvao_queue_analyze_mt(int32_t n, const wva_queue_config* cfg, const float* rate, wva_metrics* metrics, uint8_t* status, int threads) {
    parallelFor(n, threads, [&](int64_t i) {
        std::memset(&metrics[i], 0, sizeof(wva_metrics));
        const wva_queue_config& c = cfg[i];
        if (!configOk(c.max_batch_size, c.max_queue_size, c.avg_input_tokens, c.avg_output_tokens)) {
            status[i] = WVA_CAND_ERR_CONFIG; return;
        }
        QueueAnalyzer qa;
        buildModel(qa, c.max_batch_size, c.max_queue_size, ServiceParms{c.alpha, c.beta, c.gamma, c.delta},
                   c.avg_input_tokens, c.avg_output_tokens);
        status[i] = (uint8_t)analyze(qa, rate[i], &metrics[i]);
    });
    return WVA_OK;
}
int wvao_queue_analyze(int32_t n, const wva_queue_config* cfg, const float* rate, wva_metrics* metrics, uint8_t* status) {
    return wvao_queue_analyze_mt(n, cfg, rate, metrics, status, 1);
}

int wvao_queue_size_mt(int32_t n, const wva_queue_config* cfg, const float* target, float* rates, wva_metrics* metrics,
                       float* achieved, uint8_t* status, int threads) {
    parallelFor(n, threads, [&](int64_t i) {
        std::memset(&metrics[i], 0, sizeof(wva_metrics));
        for (int k = 0; k < 3; k++) { rates[3 * i + k] = 0; achieved[3 * i + k] = 0; }
        const wva_queue_config& c = cfg[i];
        if (!configOk(c.max_batch_size, c.max_queue_size, c.avg_input_tokens, c.avg_output_tokens)) { status[i] = 1; return; }
        QueueAnalyzer qa;
        buildModel(qa, c.max_batch_size, c.max_queue_size, ServiceParms{c.alpha, c.beta, c.gamma, c.delta},
                   c.avg_input_tokens, c.avg_output_tokens);
        bool ok = sizeQueue(qa, target[3 * i], target[3 * i + 1], target[3 * i + 2], &rates[3 * i], &metrics[i], &achieved[3 * i]);
        if (!ok) { std::memset(&metrics[i], 0, sizeof(wva_metrics)); for (int k = 0; k < 3; k++) { rates[3 * i + k] = 0; achieved[3 * i + k] = 0; } }
        status[i] = ok ? 0 : 1;
    });
    return WVA_OK;
}
int wvao_queue_size(int32_t n, const wva_queue_config* cfg, const float* target, float* rates, wva_metrics* metrics,
                    float* achieved, uint8_t* status) {
    return wvao_queue_size_mt(n, cfg, target, rates, metrics, achieved, status, 1);
}

// A persistent analyzer handle so tests can exercise the stale-p[0] validity state
// (queuemodel.go:30) and the raw model outputs the reference's unit tests assert on.
struct wvao_analyzer { QueueAnalyzer qa; };
wvao_analyzer* wvao_analyzer_new(const wva_queue_config* c) {
    if (!configOk(c->max_batch_size, c->max_queue_size, c->avg_input_tokens, c->avg_output_tokens)) return nullptr;
    auto* h = new wvao_analyzer;
    buildModel(h->qa, c->max_batch_size, c->max_queue_size, ServiceParms{c->alpha, c->beta, c->gamma, c->delta},
               c->avg_input_tokens, c->avg_output_tokens);
    return h;
}
void wvao_analyzer_free(wvao_analyzer* h) { delete h; }
int wvao_analyzer_analyze(wvao_analyzer* h, float rate, wva_metrics* m) { std::memset(m, 0, sizeof(*m)); return analyze(h->qa, rate, m); }
void wvao_analyzer_rate_range(wvao_analyzer* h, float* lo, float* hi) { *lo = h->qa.rateMin; *hi = h->qa.rateMax; }
int wvao_analyzer_serv_rate(wvao_analyzer* h, float* out, int32_t n) {
    int32_t k = (int32_t)std::min<size_t>((size_t)n, h->qa.model.servRate.size());
    for (int32_t i = 0; i < k; i++) out[i] = h->qa.model.servRate[(size_t)i];
    return k;
}
// raw model Solve: out = {isValid, rho, avgRespTime, avgWaitTime, avgServTime, avgNumInSystem, avgQueueLength, avgNumInServers, throughput}
void wvao_analyzer_solve(wvao_analyzer* h, float lambda, float mu, float* out9) {
    StateDependentModel& m = h->qa.model;
    m.solve(lambda, mu);
    out9[0] = m.isValid ? 1.0f : 0.0f; out9[1] = m.rho; out9[2] = m.avgRespTime; out9[3] = m.avgWaitTime; out9[4] = m.avgServTime;
    out9[5] = m.avgNumInSystem; out9[6] = m.avgQueueLength; out9[7] = m.avgNumInServers; out9[8] = m.throughput;
}
int64_t wvao_analyzer_probabilities(wvao_analyzer* h, double* out, int64_t n) {
    int64_t k = std::min<int64_t>(n, (int64_t)h->qa.model.p.size());
    for (int64_t i = 0; i < k; i++) out[i] = h->qa.model.p[(size_t)i];
    return (int64_t)h->qa.model.p.size();
}

// Raw MM1ModelStateDependent handle: NewMM1ModelStateDependent(K, servRate), mm1modelstatedependent.go:15
struct wvao_model { StateDependentModel m; };
wvao_model* wvao_model_new(int64_t K, const float* servRate, int32_t n) {
    if (K < 0 || n <= 0) return nullptr;
    auto* h = new wvao_model;
    h->m.init(K, std::vector<float>(servRate, servRate + n));
    return h;
}
void wvao_model_free(wvao_model* h) { delete h; }
void wvao_model_solve(wvao_model* h, float lambda, float mu, float* out9) {
    StateDependentModel& m = h->m;
    m.solve(lambda, mu);
    out9[0] = m.isValid ? 1.0f : 0.0f; out9[1] = m.rho; out9[2] = m.avgRespTime; out9[3] = m.avgWaitTime; out9[4] = m.avgServTime;
    out9[5] = m.avgNumInSystem; out9[6] = m.avgQueueLength; out9[7] = m.avgNumInServers; out9[8] = m.throughput;
}
int64_t wvao_model_probabilities(wvao_model* h, double* out, int64_t n) {
    int64_t k = std::min<int64_t>(n, (int64_t)h->m.p.size());
    for (int64_t i = 0; i < k; i++) out[i] = h->m.p[(size_t)i];
    return (int64_t)h->m.p.size();
}
// MM1KModel(K).Solve(lambda, mu): out = {isValid, rho, resp, wait, serv, inSystem, queueLen, throughput}; p (may be NULL) gets K+1 doubles
void wvao_mm1k_solve(int64_t K, float lambda, float mu, float* out8, double* p) {
    MM1KClosedForm m(K);
    m.solve(lambda, mu);
    out8[0] = m.isValid ? 1.0f : 0.0f; out8[1] = m.rho; out8[2] = m.avgRespTime; out8[3] = m.avgWaitTime; out8[4] = m.avgServTime;
    out8[5] = m.avgNumInSystem; out8[6] = m.avgQueueLength; out8[7] = m.throughput;
    if (p) for (int64_t i = 0; i <= K; i++) p[i] = m.p[(size_t)i];
}
// analyzer.BinarySearch with the evaluation functions of the reference's own unit test
// (pkg/analyzer/utils_test.go:72-223): 0: x*x, 1: 2*x, 2: -x, 3: x (error when x > 5).
int wvao_binary_search_testfunc(int func, float xMin, float xMax, float yTarget, float* x, int* ind) {
    auto eval = [&](float v, float* y) {
        switch (func) {
            case 0: *y = v * v; return true;
            case 1: *y = 2 * v; return true;
            case 2: *y = -v; return true;
            default: if (v > 5.0f) return false; *y = v; return true;
        }
    };
    return binarySearchGeneric(eval, xMin, xMax, yTarget, x, ind) ? 0 : 1;
}
float wvao_prefill_time(float gamma, float delta, int32_t inTok, float batch) { return prefillTime(ServiceParms{0, 0, gamma, delta}, inTok, batch); }
float wvao_decode_time(float alpha, float beta, float batch) { return decodeTime(ServiceParms{alpha, beta, 0, 0}, batch); }
float wvao_effective_concurrency(float servTime, float alpha, float beta, float gamma, float delta, int32_t inTok, int32_t outTok, int32_t maxBatch) {
    return effectiveConcurrency(servTime, ServiceParms{alpha, beta, gamma, delta}, inTok, outTok, maxBatch);
}

// analyzer.BinarySearch on the model (utils.go:26-70) with EvalTTFT (kind 0) / EvalITL (kind 1)
int wvao_analyzer_binary_search(wvao_analyzer* h, int kind, float xMin, float xMax, float yTarget, float* x, int* ind) {
    return binarySearch(h->qa, kind == 0 ? EVAL_TTFT : EVAL_ITL, xMin, xMax, yTarget, x, ind) ? 0 : 1;
}
// EvalTTFT (kind 0) / EvalITL (kind 1) at x on the handle's model: 0 and *y, or 1 for "invalid model"
int wvao_analyzer_eval(wvao_analyzer* h, int kind, float x, float* y) {
    *y = 0;
    return evalTarget(h->qa, kind == 0 ? EVAL_TTFT : EVAL_ITL, x, y) ? 0 : 1;
}
int wvao_within_tolerance(float x, float v, float tol) { return withinTolerance(x, v, tol) ? 1 : 0; }
float wvao_transition_penalty(int32_t aAcc, int64_t aRep, float aCost, int32_t bAcc, int64_t bRep, float bCost) {
    Alloc b; b.acc = bAcc; b.numReplicas = bRep; b.cost = bCost;
    return transitionPenalty(aAcc, aRep, aCost, b);
}

// Server.Calculate for every server: S*A records + feasible flags.  threads>1 shards servers
// over host threads (the reference itself is single-goroutine).  steps (may be NULL) receives the
// number of chain-state updates executed, for throughput accounting.
int wvao_analyze_pairs(const wva_system_soa* sys, wva_alloc_soa* out, uint8_t* feasible, int threads, uint64_t* steps) {
    const int32_t S = sys->n_servers, A = sys->n_accels;
    std::atomic<uint64_t> total{0};
    parallelFor((int64_t)S * A, threads, [&](int64_t i) {      // one work item per (server, accelerator) pair
        uint64_t st = 0;
        const int32_t s = (int32_t)(i / A), a = (int32_t)(i % A);
        Alloc al;
        bool ok = calculatePair(sys, s, a, &al, &st);
        if (!ok) al = Alloc{};
        storeAlloc(out, (size_t)i, al);
        feasible[i] = ok ? 1 : 0;
        total += st;
    });
    if (steps) *steps = total.load();
    return WVA_OK;
}

// Candidate sweep oracle: the reference's own QueueAnalyzer API at (N=b, maxQueue=10b, rate=total/r).
// One candidate = one fresh NewQueueAnalyzer + Analyze (queueanalyzer.go:87-174); SLO tests as in
// allocation.go:134-139 / queueanalyzer.go:231-246; value = TransitionPenalty of the candidate's cost.
struct GridCand {
    wva_metrics m; int status; bool feas; float value, cost, ttft, itl; uint64_t steps;
};
static void gridCandidate(const wva_system_soa* sys, int32_t s, int32_t a, int32_t r, int32_t b, GridCand* o) {
    const int32_t A = sys->n_accels;
    std::memset(&o->m, 0, sizeof(o->m));
    o->feas = false; o->value = 0; o->cost = 0; o->ttft = 0; o->itl = 0; o->steps = 0;
    const bool pairOk = pairLookupsOk(sys, s, a) && isCandidateAccel(sys, s, a);
    const float arrival = sys->srv_arrival_rpm[s];
    const int64_t inTok = sys->srv_in_tokens[s], outTok = sys->srv_out_tokens[s];
    const float sloTTFT = sys->srv_slo_ttft[s], sloITL = sys->srv_slo_itl[s], sloTPS = sys->srv_slo_tps[s];
    float rate = 0, rateTPS = 0;
    if (!pairOk) { o->status = WVA_CAND_ERR_PAIR; return; }
    if (!configOk(b, (int64_t)b * WVA_MAX_QUEUE_TO_BATCH_RATIO, inTok, outTok) || sloTTFT < 0 || sloITL < 0 || sloTPS < 0) {
        o->status = WVA_CAND_ERR_CONFIG; return;
    }
    const size_t pi = (size_t)sys->srv_model[s] * A + a;
    const ServiceParms sp{sys->perf_alpha[pi], sys->perf_beta[pi], sys->perf_gamma[pi], sys->perf_delta[pi]};
    const int64_t ninst = numInstances(sys, sys->srv_model[s], a);
    QueueAnalyzer qa;
    buildModel(qa, b, (int64_t)b * WVA_MAX_QUEUE_TO_BATCH_RATIO, sp, inTok, outTok);
    float totalRate = (sloTPS == 0) ? arrival / 60.0f : sloTPS / (float)outTok;   // allocation.go:134-139
    rate = totalRate / (float)r;
    o->status = analyze(qa, rate, &o->m);
    o->steps = qa.model.steps;
    float lamMax = qa.rateMax / 1000.0f;
    rateTPS = (lamMax * (1.0f - WVA_STABILITY_SAFETY)) * 1000.0f;   // TargetRate.RateTargetTPS, :231-234,:246
    if (o->status != WVA_CAND_OK) { std::memset(&o->m, 0, sizeof(o->m)); return; }
    o->ttft = o->m.avg_wait_time + o->m.avg_prefill_time;
    o->itl = o->m.avg_token_time;
    o->feas = (!(sloTTFT > 0) || o->ttft <= sloTTFT) && (!(sloITL > 0) || o->itl <= sloITL) &&
              (!(sloTPS > 0) || rate <= rateTPS) && ((int64_t)r >= (int64_t)sys->srv_min_replicas[s]);
    if (o->feas) {
        Alloc cand; cand.acc = a; cand.numReplicas = r;
        cand.cost = sys->acc_cost[a] * (float)go_muli(ninst, r);
        o->cost = cand.cost;
        float value = transitionPenalty(sys->srv_cur_acc[s], sys->srv_cur_replicas[s], sys->srv_cur_cost[s], cand);
        o->value = value + 0.0f;   // canonical +0
    }
}

// server range [s0, s1) so callers can bound the work.  best/cube/status indexed as in wva_analyze_grid
// but relative to s0.  Host threads work on (server, accelerator, replicas) rows; the per-server winner is
// then reduced in the loop order of the sweep (a, r, b ascending, strict <), so the result does not depend
// on the thread count.
int wvao_analyze_grid(const wva_system_soa* sys, int32_t s0, int32_t s1, int32_t r_max, int32_t b_max,
                      wva_grid_best* best, wva_metrics* cube, uint8_t* status, int threads, uint64_t* steps) {
    const int32_t A = sys->n_accels;
    const int64_t ns = s1 - s0;
    const int64_t nRows = ns * A * r_max;
    std::atomic<uint64_t> total{0};
    struct RowBest { bool have; wva_grid_best bb; };
    std::vector<RowBest> rows(best ? (size_t)nRows : 0);
    parallelFor(nRows, threads, [&](int64_t row) {
        const int32_t r = (int32_t)(row % r_max) + 1;
        const int32_t a = (int32_t)((row / r_max) % A);
        const int64_t si = row / ((int64_t)r_max * A);
        const int32_t s = s0 + (int32_t)si;
        uint64_t st = 0;
        RowBest rb; rb.have = false; std::memset(&rb.bb, 0, sizeof(rb.bb)); rb.bb.acc = -1;
        for (int32_t b = 1; b <= b_max; b++) {
            const size_t ci = (size_t)row * b_max + (b - 1);
            GridCand gc;
            gridCandidate(sys, s, a, r, b, &gc);
            st += gc.steps;
            if (gc.feas && gc.value == gc.value) {          // NaN values are never selected
                if (!rb.have || gc.value < rb.bb.value) {
                    rb.have = true;
                    rb.bb.acc = a; rb.bb.replicas = r; rb.bb.batch = b; rb.bb.cost = gc.cost; rb.bb.value = gc.value;
                    rb.bb.itl = gc.itl; rb.bb.ttft = gc.ttft; rb.bb.rho = gc.m.rho;
                }
            }
            if (cube) cube[ci] = gc.m;
            if (status) status[ci] = (uint8_t)(gc.status | (gc.feas ? WVA_CAND_FEASIBLE : 0));
        }
        if (best) rows[(size_t)row] = rb;
        total += st;
    });
    if (best) {
        for (int64_t si = 0; si < ns; si++) {
            wva_grid_best bb; std::memset(&bb, 0, sizeof(bb)); bb.acc = -1;
            bool have = false;
            for (int64_t k = 0; k < (int64_t)A * r_max; k++) {     // (a, r) ascending
                const RowBest& rb = rows[(size_t)(si * A * r_max + k)];
                if (rb.have && (!have || rb.bb.value < bb.value)) { have = true; bb = rb.bb; }
            }
            best[si] = bb;
        }
    }
    if (steps) *steps = total.load();
    return WVA_OK;
}

// A list of sweep candidates (s, a, r, b), each evaluated exactly like the loop body above.
// out_value / out_feasible may be NULL.
int wvao_grid_candidates(const wva_system_soa* sys, int64_t n, const int32_t* s, const int32_t* a, const int32_t* r,
                         const int32_t* b, wva_metrics* metrics, uint8_t* status, int threads) {
    parallelFor(n, threads, [&](int64_t i) {
        GridCand gc;
        gridCandidate(sys, s[i], a[i], r[i], b[i], &gc);
        metrics[i] = gc.m;
        status[i] = (uint8_t)(gc.status | (gc.feas ? WVA_CAND_FEASIBLE : 0));
    });
    return WVA_OK;
}

// value (TransitionPenalty of cost = acc.Cost * float32(numInstances * r), canonical +0) of every sweep row
// (s, a, r), s in [s0, s1): what orders the candidates of a server.  NaN for rows whose pair lookups fail.
int wvao_grid_row_values(const wva_system_soa* sys, int32_t s0, int32_t s1, int32_t r_max, float* value) {
    const int32_t A = sys->n_accels;
    for (int32_t s = s0; s < s1; s++)
        for (int32_t a = 0; a < A; a++) {
            const bool pairOk = pairLookupsOk(sys, s, a) && isCandidateAccel(sys, s, a);
            const int64_t ninst = pairOk ? numInstances(sys, sys->srv_model[s], a) : 1;
            for (int32_t r = 1; r <= r_max; r++) {
                float v = std::numeric_limits<float>::quiet_NaN();
                if (pairOk) {
                    Alloc cand; cand.acc = a; cand.numReplicas = r;
                    cand.cost = sys->acc_cost[a] * (float)go_muli(ninst, r);
                    v = transitionPenalty(sys->srv_cur_acc[s], sys->srv_cur_replicas[s], sys->srv_cur_cost[s], cand) + 0.0f;
                }
                value[((size_t)(s - s0) * A + a) * r_max + (r - 1)] = v;
            }
        }
    return WVA_OK;
}

// For each listed row (s, a, r): how many of its candidates b in [b_lo, b_hi] the reference API finds feasible.
int wvao_grid_rows_feasible(const wva_system_soa* sys, int64_t n, const int32_t* s, const int32_t* a, const int32_t* r,
                            const int32_t* b_lo, const int32_t* b_hi, int32_t* n_feasible, int threads) {
    parallelFor(n, threads, [&](int64_t i) {
        int32_t cnt = 0;
        for (int32_t b = b_lo[i]; b <= b_hi[i]; b++) {
            GridCand gc;
            gridCandidate(sys, s[i], a[i], r[i], b, &gc);
            if (gc.feas && gc.value == gc.value) cnt++;
        }
        n_feasible[i] = cnt;
    });
    return WVA_OK;
}

// Solver.Solve over the candidates produced by wvao_analyze_pairs.
int wvao_solve(const wva_system_soa* sys, const wva_alloc_soa* pairs, const uint8_t* feasible,
               const wva_optimizer_spec* spec, int32_t* chosen_acc, wva_alloc_soa* chosen) {
    const int32_t S = sys->n_servers, A = sys->n_accels, T = sys->n_types;
    GreedyState g;
    g.sys = sys; g.feasible = feasible;
    g.cand.resize((size_t)S * A);
    for (size_t i = 0; i < (size_t)S * A; i++) g.cand[i] = loadAlloc(pairs, i);
    g.chosen.assign((size_t)S, -1);
    if (spec->unlimited) {
        // SolveUnlimited, solver.go:63-79; canonical iteration = ascending accelerator index
        for (int32_t s = 0; s < S; s++) {
            float minVal = kMaxFloat32;
            int32_t minKey = -1;
            for (int32_t a = 0; a < A; a++) {
                if (!feasible[(size_t)s * A + a]) continue;
                float v = g.alloc(s, a).value;
                if (v < minVal) { minVal = v; minKey = a; }
            }
            g.chosen[(size_t)s] = minKey;
        }
    } else {
        // SolveGreedy, greedy.go:35-104
        g.available.assign((size_t)T, 0);
        for (int32_t t = 0; t < T; t++) g.available[(size_t)t] = sys->type_capacity[t];
        std::vector<ServerEntry> store; store.reserve((size_t)S);
        for (int32_t s = 0; s < S; s++) {
            ServerEntry e; e.server = s; e.priority = sys->srv_priority[s]; e.curIndex = 0; e.delta = 0;
            for (int32_t a = 0; a < A; a++) if (feasible[(size_t)s * A + a]) e.allocs.push_back(a);
            if (e.allocs.empty()) continue;
            // slices.SortFunc by value (cmp.Compare); canonical = stable on accelerator index
            std::stable_sort(e.allocs.begin(), e.allocs.end(), [&](int32_t x, int32_t y) {
                return go_cmpf(g.alloc(s, x).value, g.alloc(s, y).value) < 0;
            });
            if (e.allocs.size() > 1) e.delta = g.alloc(s, e.allocs[1]).value - g.alloc(s, e.allocs[0]).value;
            else e.delta = kMaxFloat32;
            store.push_back(std::move(e));
        }
        std::vector<ServerEntry*> entries;
        for (auto& e : store) entries.push_back(&e);
        std::stable_sort(entries.begin(), entries.end(), [&](ServerEntry* x, ServerEntry* y) { return orderFunc(g, x, y) < 0; });
        if (spec->delayed_best_effort) {
            auto un = allocate(g, entries);
            bestEffort(g, un, spec->saturation_policy);
        } else {
            for (auto& grp : makePriorityGroups(entries)) {
                auto un = allocate(g, grp);
                bestEffort(g, un, spec->saturation_policy);
            }
        }
    }
    for (int32_t s = 0; s < S; s++) {
        int32_t key = g.chosen[(size_t)s];
        chosen_acc[s] = key;
        storeAlloc(chosen, (size_t)s, key >= 0 ? g.alloc(s, key) : Alloc{});
    }
    return WVA_OK;
}

// System.AllocateByType, system.go:271-300; canonical summation order = ascending server index.
int wvao_allocate_by_type(const wva_system_soa* sys, int32_t s0, int32_t s1, const int32_t* chosen_acc,
                          const wva_alloc_soa* chosen, int64_t* count, float* cost) {
    const int32_t T = sys->n_types;
    for (int32_t t = 0; t < T; t++) { count[t] = 0; cost[t] = 0; }
    for (int32_t s = s0; s < s1; s++) {
        if (chosen_acc[s] < 0) continue;                     // server.Allocation() == nil
        int32_t gi = chosen->acc[s];                         // serverAlloc.accelerator
        int32_t m = sys->srv_model[s];
        if (gi < 0 || m < 0) continue;                       // acc == nil || model == nil
        int32_t t = sys->acc_type[gi];
        int64_t units = go_muli(go_muli(chosen->num_replicas[s], numInstances(sys, m, gi)), sys->acc_multiplicity[gi]);
        count[t] += units;
        cost[t] = cost[t] + chosen->cost[s];
    }
    return WVA_OK;
}

// number of overflow-rescale branches (mm1modelstatedependent.go:84-89, :96-104) taken since load
uint64_t wvao_rescale_events(void) { return g_rescale_chain.load() + g_rescale_sum.load(); }
// the same, per branch: the chain's (:84-89) and the normalising sum's (:95-104)
void wvao_rescale_counts(uint64_t* chain, uint64_t* sum) { *chain = g_rescale_chain.load(); *sum = g_rescale_sum.load(); }

int wvao_hardware_threads(void) { unsigned n = std::thread::hardware_concurrency(); return n ? (int)n : 1; }

}  // extern "C"
