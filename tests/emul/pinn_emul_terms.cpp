// TEST INFRASTRUCTURE ONLY — host emulation of the constraint-term points of the persistent multi-step kernels.
//
// Compiles pydens_b200/csrc/pinn_device.cuh and pinn_host_plan.h with g++ and runs point_step<..., TERMS = true> — the
// per-point code the multi-step kernel runs at a constraint point — for a term plan next to the equation's plan, built
// and checked by build_dev_term as pinn_multi_step_terms builds and checks it.  The storage is laid out as on the device
// (rows of 32 lanes, the point in one lane): every lane starts with finite stale rows, every other lane holds NaN.
// Never loaded by the product.
#include <vector>
#include <limits>
#include <string.h>
#include "../../pydens_b200/csrc/pinn_host_plan.h"

using namespace pinn;

static const int EMUL_RS = 32;
static const float EMUL_STALE = -7.25e3f;

template <int NF, int NS>
static void run_terms(const DevPlan& P, int rows, const DevTerm& T, const float* sw, const float* params,
                      const float* points, long long n, float* out, float* residual) {
    std::vector<float> st((size_t)rows * EMUL_RS, std::numeric_limits<float>::quiet_NaN());
    GradSink sink;
    sink.wacc = out;
    sink.atomic = false;
    sink.dump = P.n_params + 2;
    PointPartials<NF, NS> part;
    part.loss = 0.0f; part.sbar = 0.0f;
    for (int i = 0; i < PINN_MAX_VARS; ++i) part.vbar[i] = 0.0f;
    for (long long p = 0; p < n; ++p) {
        float* lane = st.data() + (p % EMUL_RS);
        for (int r = 0; r < rows; ++r) lane[(size_t)r * EMUL_RS] = EMUL_STALE;
        for (int k = 0; k < P.total; ++k) lane[(size_t)k * EMUL_RS] = points[p * P.total + k];
        // the batch's point weight is passed as NaN: a term point must take its own (T.weight)
        const float r = point_step<NF, NS, 16, true, false, true>(P, sw, params, lane, EMUL_RS, true,
                                                                 std::numeric_limits<float>::quiet_NaN(), sink, part, &T);
        for (int q = 0; q < rows; ++q) lane[(size_t)q * EMUL_RS] = std::numeric_limits<float>::quiet_NaN();
        if (residual) residual[p] = r;
    }
    out[P.n_params] += part.loss;
    out[P.log_scale_off] += part.sbar;
    for (int i = 0; i < P.n_vars; ++i) out[P.var_off[i]] += part.vbar[i];
}

// rc of build_dev_term for `term` next to `plan` (PINN_E_INVALID: pinn_multi_step_terms refuses the pair).
extern "C" int emul_term_check(const PinnSpec* plan, const PinnSpec* term, char* msg, int msg_len) {
    DevPlan h, g;
    int fr, fs;
    int rc = build_dev_plan(plan, h, fr, fs, msg, (size_t)msg_len);
    if (rc) return rc;
    rc = build_dev_plan(term, g, fr, fs, msg, (size_t)msg_len);
    if (rc) return rc;
    static DevTerm t;
    return build_dev_term(h, spec_order(plan), g, spec_order(term), t, msg, (size_t)msg_len);
}

// The term points `points` [n, total] of `term` under the equation's `plan`, point weight `weight`: out = [grads | loss].
extern "C" int emul_term_step(const PinnSpec* plan, const PinnSpec* term, const float* params, const float* points,
                              long long n, float weight, float* out, float* residual, char* msg, int msg_len) {
    DevPlan P, G;
    int fr, fs;
    int rc = build_dev_plan(plan, P, fr, fs, msg, (size_t)msg_len);
    if (rc) return rc;
    rc = build_dev_plan(term, G, fr, fs, msg, (size_t)msg_len);
    if (rc) return rc;
    static DevTerm T;
    rc = build_dev_term(P, spec_order(plan), G, spec_order(term), T, msg, (size_t)msg_len);
    if (rc) return rc;
    T.weight = weight;
    // the scratch rows cover the larger of the two programs, as multi_setup sizes them
    const int rows = P.row_scr + G.n_slots > P.rows_total ? P.row_scr + G.n_slots : P.rows_total;
    std::vector<float> sw(P.weights_floats + 16);
    host_stage_weights(P, params, sw.data());
    for (int i = 0; i < P.n_params + 4; ++i) out[i] = 0.0f;
#define CASE(NF_, NS_) if (P.nf == NF_ && P.ns == NS_) { run_terms<NF_, NS_>(P, rows, T, sw.data(), params, points, n, out, residual); return 0; }
    CASE(0, 0) CASE(1, 0) CASE(1, 1) CASE(2, 0) CASE(2, 1) CASE(2, 2)
    CASE(3, 0) CASE(3, 1) CASE(3, 2) CASE(3, 3)
    CASE(4, 0) CASE(4, 1) CASE(4, 2) CASE(4, 3) CASE(4, 4)
#undef CASE
    snprintf(msg, msg_len, "no persistent variant nf=%d ns=%d", P.nf, P.ns);
    return PINN_E_UNSUPPORTED;
}
