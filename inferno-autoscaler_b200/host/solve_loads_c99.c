/* The arrival-rate scenario solve through plain C99, the way a cgo preamble compiles the header: the declarations are
 * valid C, the symbols link, and every entry point rejects a missing context without touching a device. */
#include <stdint.h>
#include <stdio.h>

#include "wva_b200.h"

int main(void) {
    int (*solve)(wva_ctx*, const wva_optimizer_spec*, int32_t, const float*, int32_t*, wva_pair_rec*, int64_t*, float*) =
        wva_solve_loads;
    wva_optimizer_spec spec = {0, 0, WVA_POLICY_NONE};
    float rpm[2] = {60.0f, 120.0f};
    uint64_t counters[6];
    if (WVA_SOLVE_MAX_LOADS != 8192) { printf("bad limit\n"); return 1; }
    if (solve(NULL, &spec, 2, rpm, NULL, NULL, NULL, NULL) != WVA_EINVAL) { printf("solve(NULL)\n"); return 1; }
    if (wva_solve_loads_counters(NULL, counters) != WVA_EINVAL) { printf("counters(NULL)\n"); return 1; }
    if (wva_solve_loads_set_budget(NULL, 0) != WVA_EINVAL) { printf("set_budget(NULL)\n"); return 1; }
    printf("solve_loads c99: ok\n");
    return 0;
}
