/* cabi_test.c — the C-ABI seen from plain C99, the way a cgo preamble sees it.
 *
 * (1) include/wva_b200.h compiles as C (cgo compiles the preamble with the C compiler, not C++);
 * (2) struct layouts are the natural-alignment ones cgo mirrors into Go (every field at a multiple of
 *     its size, no packing pragmas): offsets are asserted so that a change of the header that would
 *     silently change the Go-side layout fails here;
 * (3) on a box with an H100: the *_arrays entry points (what go/internal/native calls -- no struct of
 *     pointers crosses the boundary) give the same bytes as the struct forms.
 * Exit code 0 = ok (prints "no device" and stops after (2) when CUDA is unavailable). */
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "wva_b200.h"

#define CHECK(c) do { if (!(c)) { fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

_Static_assert(sizeof(wva_metrics) == 32, "wva_metrics");
_Static_assert(sizeof(wva_grid_best) == 32, "wva_grid_best");
_Static_assert(sizeof(wva_queue_config) == 32, "wva_queue_config");
_Static_assert(sizeof(wva_optimizer_spec) == 12, "wva_optimizer_spec");
_Static_assert(offsetof(wva_system_soa, acc_cost) == 16, "4 x int32 header, then pointers");
_Static_assert(sizeof(wva_system_soa) == 16 + 27 * sizeof(void*), "27 array pointers");
_Static_assert(offsetof(wva_system_soa, srv_cur_cost) == 16 + 26 * sizeof(void*), "last pointer");
_Static_assert(sizeof(wva_alloc_soa) == 9 * sizeof(void*), "9 array pointers");
_Static_assert(offsetof(wva_alloc_soa, max_arrv_rate_per_replica) == 8 * sizeof(void*), "last pointer");
_Static_assert(WVA_COMM_ID_BYTES == 128, "ncclUniqueId");
_Static_assert(sizeof(wva_pair_rec) == 48, "wva_pair_rec");
_Static_assert(offsetof(wva_pair_rec, num_replicas) == 8 && offsetof(wva_pair_rec, max_arrv_rate_per_replica) == 44, "wva_pair_rec");

enum { S = 6, A = 3, M = 6, T = 2 };

int main(void) {
    CHECK(wva_abi_version() == WVA_ABI_VERSION);
    wva_ctx* ctx = NULL;
    int rc = wva_ctx_create(0, &ctx);
    if (rc != WVA_OK) {
        CHECK(rc == WVA_ECUDA && ctx == NULL && strlen(wva_last_error(NULL)) > 0);   /* fails loudly, no CPU fallback */
        printf("cabi_test: layout ok; no device (%s)\n", wva_last_error(NULL));
        return 0;
    }
    /* a tiny system, every array a separate allocation (as Go slices are) */
    float acc_cost[A] = {40.0f, 75.5f, 110.0f}; int32_t acc_mult[A] = {1, 2, 1}, acc_type[A] = {0, 1, 0};
    int64_t cap[T] = {0, 0};
    float al[M * A], be[M * A], ga[M * A], de[M * A]; int32_t mb[M * A], at[M * A], ac[M * A]; uint8_t pv[M * A];
    for (int i = 0; i < M * A; ++i) {
        al[i] = 6.0f + (float)(i % 7); be[i] = 0.05f + 0.03f * (float)(i % 5); ga[i] = 20.0f + 9.0f * (float)(i % 4);
        de[i] = 0.001f * (float)(1 + i % 3); mb[i] = 16 + 8 * (i % 5); at[i] = 256; ac[i] = 1 + (i % 2); pv[i] = 1;
    }
    int32_t sm[S], sin[S], sout[S], spr[S], smr[S], smb[S], sca[S], scr[S]; uint8_t stv[S], ska[S];
    float sar[S], stt[S], sit[S], stp[S], scc[S];
    for (int s = 0; s < S; ++s) {
        sm[s] = s; sar[s] = 30.0f * (float)(s + 1) * (float)(s + 1); sin[s] = 128 * (s + 1); sout[s] = 64 + 32 * s;
        stt[s] = 1000.0f; sit[s] = 80.0f; stp[s] = 0.0f; stv[s] = 1; spr[s] = 1 + s; smr[s] = s & 1; smb[s] = 0; ska[s] = 0;
        sca[s] = (s % 3 == 0) ? WVA_ACC_NONE : (s % A); scr[s] = (s % 3 == 0) ? 0 : 2; scc[s] = (s % 3 == 0) ? 0.0f : 150.0f;
    }
    sar[4] = 0.0f;   /* a zero-load server */
    CHECK(wva_system_upload_arrays(ctx, S, A, M, T, acc_cost, acc_mult, acc_type, cap, al, be, ga, de, mb, at, ac, pv, sm, sar, sin, sout,
                                   stt, sit, stp, stv, spr, smr, smb, ska, sca, scr, scc) == WVA_OK);
    int32_t acc1[S * A]; int64_t rep1[S * A], bat1[S * A]; float f1[6][S * A]; uint8_t fe1[S * A];
    CHECK(wva_analyze_pairs_arrays(ctx, acc1, rep1, bat1, f1[0], f1[1], f1[2], f1[3], f1[4], f1[5], fe1) == WVA_OK);
    int32_t key1[S], cacc1[S]; int64_t crep1[S], cbat1[S]; float cf1[6][S];
    CHECK(wva_solve_arrays(ctx, 1, 0, WVA_POLICY_NONE, key1, cacc1, crep1, cbat1, cf1[0], cf1[1], cf1[2], cf1[3], cf1[4], cf1[5]) == WVA_OK);

    /* the struct forms on the same inputs */
    wva_system_soa h;
    h.n_servers = S; h.n_accels = A; h.n_models = M; h.n_types = T;
    h.acc_cost = acc_cost; h.acc_multiplicity = acc_mult; h.acc_type = acc_type; h.type_capacity = cap;
    h.perf_alpha = al; h.perf_beta = be; h.perf_gamma = ga; h.perf_delta = de; h.perf_max_batch = mb; h.perf_at_tokens = at;
    h.perf_acc_count = ac; h.perf_valid = pv; h.srv_model = sm; h.srv_arrival_rpm = sar; h.srv_in_tokens = sin; h.srv_out_tokens = sout;
    h.srv_slo_ttft = stt; h.srv_slo_itl = sit; h.srv_slo_tps = stp; h.srv_target_valid = stv; h.srv_priority = spr;
    h.srv_min_replicas = smr; h.srv_max_batch = smb; h.srv_keep_acc = ska; h.srv_cur_acc = sca; h.srv_cur_replicas = scr; h.srv_cur_cost = scc;
    CHECK(wva_system_upload(ctx, &h) == WVA_OK);
    int32_t acc2[S * A]; int64_t rep2[S * A], bat2[S * A]; float f2[6][S * A]; uint8_t fe2[S * A];
    wva_alloc_soa o2 = {acc2, rep2, bat2, f2[0], f2[1], f2[2], f2[3], f2[4], f2[5]};
    CHECK(wva_analyze_pairs(ctx, &o2, fe2) == WVA_OK);
    int32_t key2[S], cacc2[S]; int64_t crep2[S], cbat2[S]; float cf2[6][S];
    wva_alloc_soa c2 = {cacc2, crep2, cbat2, cf2[0], cf2[1], cf2[2], cf2[3], cf2[4], cf2[5]};
    wva_optimizer_spec spec = {1, 0, WVA_POLICY_NONE};
    CHECK(wva_solve(ctx, &spec, key2, &c2) == WVA_OK);
    CHECK(!memcmp(acc1, acc2, sizeof acc1) && !memcmp(rep1, rep2, sizeof rep1) && !memcmp(bat1, bat2, sizeof bat1));
    CHECK(!memcmp(f1, f2, sizeof f1) && !memcmp(fe1, fe2, sizeof fe1));
    CHECK(!memcmp(key1, key2, sizeof key1) && !memcmp(cacc1, cacc2, sizeof cacc1) && !memcmp(crep1, crep2, sizeof crep1) && !memcmp(cf1, cf2, sizeof cf1));
    int nfe = 0; for (int i = 0; i < S * A; ++i) nfe += fe1[i];
    CHECK(nfe > 0);
    int64_t cnt[T]; float cst[T];
    CHECK(wva_allocate_by_type(ctx, cnt, cst) == WVA_OK);
    /* pair sizing over a batch-size list: column j equals wva_pairs_fetch after an upload with that override */
    const int32_t batch[3] = {8, 24, 40};
    wva_pair_rec plane[S * A * 3], best[S];
    CHECK(wva_analyze_pairs_batches(ctx, 3, batch, plane, best) == WVA_OK);
    for (int s = 0; s < S; ++s) smb[s] = batch[1];
    CHECK(wva_system_upload(ctx, &h) == WVA_OK);
    CHECK(wva_analyze_pairs(ctx, NULL, NULL) == WVA_OK);
    CHECK(wva_pairs_fetch(ctx, &o2, fe2) == WVA_OK);
    int nb = 0;
    for (int i = 0; i < S * A; ++i) {
        const wva_pair_rec* r = &plane[i * 3 + 1];
        CHECK(r->acc == acc2[i] && r->feasible == fe2[i] && r->num_replicas == rep2[i] && r->batch_size == bat2[i]);
        CHECK(!memcmp(&r->cost, &f2[0][i], 4) && !memcmp(&r->value, &f2[1][i], 4) && !memcmp(&r->itl, &f2[2][i], 4));
        CHECK(!memcmp(&r->ttft, &f2[3][i], 4) && !memcmp(&r->rho, &f2[4][i], 4) && !memcmp(&r->max_arrv_rate_per_replica, &f2[5][i], 4));
        nb += r->feasible;
    }
    CHECK(nb > 0);
    /* pair sizing over arrival-rate scenarios: column j equals wva_pairs_fetch after an upload with that rate, and best
     * equals wva_solve(unlimited)'s choice on that image */
    enum { L = 3 };
    const float fac[L] = {0.5f, 2.0f, 7.0f};
    float rpm[S * L];
    for (int s = 0; s < S; ++s)
        for (int j = 0; j < L; ++j) rpm[s * L + j] = sar[s] * fac[j];
    rpm[1 * L + 0] = -1.0f;      /* nil */
    wva_pair_rec lplane[S * L * A], lbest[S * L];
    CHECK(wva_analyze_pairs_loads(ctx, L, rpm, lplane, lbest) == WVA_OK);
    uint64_t lcnt[5];
    CHECK(wva_pairs_loads_counters(ctx, lcnt) == WVA_OK && lcnt[0] == 1 && lcnt[1] > 0 && lcnt[2] > 0);
    CHECK(wva_analyze_pairs_loads(ctx, 0, rpm, NULL, NULL) == WVA_EINVAL && wva_analyze_pairs_loads(ctx, L, NULL, NULL, NULL) == WVA_EINVAL);
    int nl = 0;
    for (int j = 0; j < L; ++j) {
        for (int s = 0; s < S; ++s) sar[s] = rpm[s * L + j];
        CHECK(wva_system_upload(ctx, &h) == WVA_OK);
        CHECK(wva_analyze_pairs(ctx, &o2, fe2) == WVA_OK);
        CHECK(wva_solve(ctx, &spec, key2, &c2) == WVA_OK);
        for (int s = 0; s < S; ++s) {
            for (int a = 0; a < A; ++a) {
                const int i = s * A + a;
                const wva_pair_rec* r = &lplane[(s * L + j) * A + a];
                CHECK(r->acc == acc2[i] && r->feasible == fe2[i] && r->num_replicas == rep2[i] && r->batch_size == bat2[i]);
                CHECK(!memcmp(&r->cost, &f2[0][i], 4) && !memcmp(&r->value, &f2[1][i], 4) && !memcmp(&r->itl, &f2[2][i], 4));
                CHECK(!memcmp(&r->ttft, &f2[3][i], 4) && !memcmp(&r->rho, &f2[4][i], 4) && !memcmp(&r->max_arrv_rate_per_replica, &f2[5][i], 4));
                nl += r->feasible;
            }
            const wva_pair_rec* b = &lbest[s * L + j];
            if (key2[s] < 0) { CHECK(b->acc == WVA_ACC_NONE && b->feasible == 0); continue; }
            CHECK(b->feasible == 1 && b->acc == cacc2[s] && b->num_replicas == crep2[s] && b->batch_size == cbat2[s]);
            CHECK(!memcmp(&b->cost, &cf2[0][s], 4) && !memcmp(&b->value, &cf2[1][s], 4) && !memcmp(&b->itl, &cf2[2][s], 4));
            CHECK(!memcmp(&b->ttft, &cf2[3][s], 4) && !memcmp(&b->rho, &cf2[4][s], 4) && !memcmp(&b->max_arrv_rate_per_replica, &cf2[5][s], 4));
        }
    }
    CHECK(nl > 0);
    printf("cabi_test: ok (%d feasible pairs, type counts %lld %lld, %d at batch size 24, %d over %d arrival-rate scenarios)\n",
           nfe, (long long)cnt[0], (long long)cnt[1], nb, nl, (int)L);
    wva_ctx_destroy(ctx);
    return 0;
}
