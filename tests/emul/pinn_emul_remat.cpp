// TEST INFRASTRUCTURE ONLY — host build of the twelve-warp step kernel's compact per-point layout (build_remat_plan,
// point_step<…, REMAT0 = true>), driven like pinn_emul.cpp: one point per lane of a 32-lane storage block, the other
// lanes NaN, the point's own lane stale at the start of every point.  tests/test_occupancy_layout.py compiles it into a
// temporary directory and compares the compact layout with the plan's own, bit for bit.
#include <vector>
#include <limits>
#include <string.h>
#include "../../pydens_b200/csrc/pinn_host_plan.h"

using namespace pinn;

static const int RS_ = 32;
static const float STALE = -7.25e3f;

template <int NF, int NS, bool REMAT0>
static void run(const DevPlan& P, const float* sw, const float* params, const float* points, long long n, float inv_n,
                float* out, float* residual) {
    std::vector<float> st((size_t)P.rows_total * RS_, std::numeric_limits<float>::quiet_NaN());
    GradSink sink;
    sink.wacc = out;
    sink.atomic = false;
    sink.dump = P.n_params + 2;
    PointPartials<NF, NS> part;
    part.loss = 0.0f; part.sbar = 0.0f;
    for (int i = 0; i < PINN_MAX_VARS; ++i) part.vbar[i] = 0.0f;
    for (long long p = 0; p < n; ++p) {
        float* lane = st.data() + (p % RS_);
        for (int r = 0; r < P.rows_total; ++r) lane[(size_t)r * RS_] = STALE;
        for (int k = 0; k < P.total; ++k) lane[(size_t)k * RS_] = points[p * P.total + k];
        const float r = point_step<NF, NS, 16, false, false, false, REMAT0>(P, sw, params, lane, RS_, true, inv_n, sink, part);
        for (int q = 0; q < P.rows_total; ++q) lane[(size_t)q * RS_] = std::numeric_limits<float>::quiet_NaN();
        residual[p] = r;
    }
    out[P.n_params] += part.loss;
    out[P.log_scale_off] += part.sbar;
    for (int i = 0; i < P.n_vars; ++i) out[P.var_off[i]] += part.vbar[i];
}

// rows[0]: rows per point of the plan's layout; rows[1]: of the compact layout, or -1 where it does not apply
extern "C" int remat_rows(const PinnSpec* spec, int* rows, char* msg, int msg_len) {
    DevPlan P, Pc;
    int fr, fs;
    const int rc = build_dev_plan(spec, P, fr, fs, msg, (size_t)msg_len);
    if (rc) return rc;
    rows[0] = P.rows_total;
    rows[1] = build_remat_plan(P, Pc) ? Pc.rows_total : -1;
    return 0;
}

// One step over `n` points on the plan's layout (compact = 0) or on the compact one (compact = 1, plain plans only).
extern "C" int remat_step(const PinnSpec* spec, int compact, const float* params, const float* points, long long n,
                          float* out, float* residual, char* msg, int msg_len) {
    DevPlan P, Pc;
    int fr, fs;
    const int rc = build_dev_plan(spec, P, fr, fs, msg, (size_t)msg_len);
    if (rc) return rc;
    if (P.general) { snprintf(msg, msg_len, "a general plan"); return PINN_E_UNSUPPORTED; }
    if (compact && !build_remat_plan(P, Pc)) { snprintf(msg, msg_len, "no compact layout"); return PINN_E_UNSUPPORTED; }
    std::vector<float> sw(P.weights_floats + 16);
    host_stage_weights(P, params, sw.data());
    for (int i = 0; i < P.n_params + 4; ++i) out[i] = 0.0f;
    const float inv_n = 1.0f / (float)n;
#define CASE(NF_, NS_)                                                                                         \
    if (P.nf == NF_ && P.ns == NS_) {                                                                          \
        if (compact) run<NF_, NS_, true>(Pc, sw.data(), params, points, n, inv_n, out, residual);             \
        else         run<NF_, NS_, false>(P, sw.data(), params, points, n, inv_n, out, residual);             \
        return 0;                                                                                              \
    }
    CASE(0, 0) CASE(1, 0) CASE(1, 1) CASE(2, 0) CASE(2, 1) CASE(2, 2)
    CASE(3, 0) CASE(3, 1) CASE(3, 2) CASE(3, 3)
    CASE(4, 0) CASE(4, 1) CASE(4, 2) CASE(4, 3) CASE(4, 4)
#undef CASE
    snprintf(msg, msg_len, "no variant nf=%d ns=%d", P.nf, P.ns);
    return PINN_E_UNSUPPORTED;
}
