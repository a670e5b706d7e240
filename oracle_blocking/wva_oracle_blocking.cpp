// Blocking probability of sweep candidates from the CPU oracle (test infrastructure only).
//
// wvao_grid_candidates_blocking is the sibling of the oracle's wvao_grid_candidates: every candidate (s, a, r, b) goes
// through that very entry point (status and metrics), and an analysed one also through the oracle's QueueAnalyzer
// handle (NewQueueAnalyzer({b, 10 b}, {in, out}) + Analyze(totalRate / float32(r)), queueanalyzer.go:87-174), whose
// model state then holds the normalised p[] of computeProbabilities (mm1modelstatedependent.go:70-112).  p_block is
// float32 of its p[K], K = 11 b; the quiet NaN 0x7fc00000 where the status is not WVA_CAND_OK.  No arithmetic of the
// model is restated here: both numbers come from libwva_oracle.so.
#include <atomic>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../include/wva_b200.h"

extern "C" {
struct wvao_analyzer;
wvao_analyzer* wvao_analyzer_new(const wva_queue_config* c);
void wvao_analyzer_free(wvao_analyzer* h);
int wvao_analyzer_analyze(wvao_analyzer* h, float rate, wva_metrics* m);
int64_t wvao_analyzer_probabilities(wvao_analyzer* h, double* out, int64_t n);
int wvao_grid_candidates(const wva_system_soa* sys, int64_t n, const int32_t* s, const int32_t* a, const int32_t* r,
                         const int32_t* b, wva_metrics* metrics, uint8_t* status, int threads);
}

namespace {

float quiet_nan() {
    const uint32_t bits = 0x7fc00000u;
    float f;
    std::memcpy(&f, &bits, 4);
    return f;
}

// p_block of one candidate whose oracle status is WVA_CAND_OK; returns false if the analyzer disagrees
bool candidate_p_block(const wva_system_soa* sys, int32_t s, int32_t a, int32_t r, int32_t b, std::vector<double>& p, float* out) {
    const int32_t A = sys->n_accels;
    const size_t pi = (size_t)sys->srv_model[s] * A + a;
    wva_queue_config c;
    c.max_batch_size = b;
    c.max_queue_size = b * WVA_MAX_QUEUE_TO_BATCH_RATIO;
    c.alpha = sys->perf_alpha[pi]; c.beta = sys->perf_beta[pi]; c.gamma = sys->perf_gamma[pi]; c.delta = sys->perf_delta[pi];
    c.avg_input_tokens = sys->srv_in_tokens[s];
    c.avg_output_tokens = sys->srv_out_tokens[s];
    wvao_analyzer* h = wvao_analyzer_new(&c);
    if (!h) return false;
    const float sloTPS = sys->srv_slo_tps[s];
    const float totalRate = (sloTPS == 0) ? sys->srv_arrival_rpm[s] / 60.0f : sloTPS / (float)sys->srv_out_tokens[s];   // allocation.go:134-139
    wva_metrics m;
    const int st = wvao_analyzer_analyze(h, totalRate / (float)r, &m);
    const int64_t K = (int64_t)b * (WVA_MAX_QUEUE_TO_BATCH_RATIO + 1);
    p.assign((size_t)K + 1, 0.0);
    const int64_t n = wvao_analyzer_probabilities(h, p.data(), K + 1);
    wvao_analyzer_free(h);
    if (st != WVA_CAND_OK || n != K + 1) return false;
    *out = (float)p[(size_t)K];
    return true;
}

}  // namespace

extern "C" {

// Candidates (s[i], a[i], r[i], b[i]) -> metrics[i], status[i] (exactly wvao_grid_candidates) and p_block[i].
// Returns WVA_OK, or WVA_EINVAL if the analyzer handle rejects a candidate the oracle's sweep accepted.
int wvao_grid_candidates_blocking(const wva_system_soa* sys, int64_t n, const int32_t* s, const int32_t* a, const int32_t* r,
                                  const int32_t* b, wva_metrics* metrics, uint8_t* status, float* p_block, int threads) {
    std::atomic<int64_t> next{0};
    std::atomic<int> bad{0};
    auto work = [&] {
        std::vector<double> p;
        for (;;) {
            const int64_t i = next.fetch_add(1);
            if (i >= n) return;
            wvao_grid_candidates(sys, 1, s + i, a + i, r + i, b + i, metrics + i, status + i, 1);
            p_block[i] = quiet_nan();
            if ((status[i] & ~WVA_CAND_FEASIBLE) == WVA_CAND_OK && !candidate_p_block(sys, s[i], a[i], r[i], b[i], p, &p_block[i]))
                bad.store(1);
        }
    };
    if (threads <= 1 || n <= 1) {
        work();
    } else {
        std::vector<std::thread> pool;
        for (int t = 0; t < threads; ++t) pool.emplace_back(work);
        for (auto& t : pool) t.join();
    }
    return bad.load() ? WVA_EINVAL : WVA_OK;
}

}  // extern "C"
