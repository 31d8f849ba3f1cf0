// TEST INFRASTRUCTURE ONLY — host emulation of the per-point device code of networks with 2..4 outputs (coupled systems).
//
// The companion of pinn_emul.cpp for the k-output form of point_step / point_forward (what coupled_step_kernel and
// coupled_forward_kernel run per thread), driven the same way: one point at a time in lane p % 32 of device-shaped
// storage rows, every other lane poisoned with NaN, the warp reduction replaced by direct accumulation.
// Never loaded by the product (pydens_b200/_native.py loads only libpinn_b200.so).
#include <vector>
#include <limits>
#include <string.h>
#include "../../pydens_b200/csrc/pinn_host_plan.h"

using namespace pinn;

static const int EMUL_RS = 32;                       // the device's row stride (pinn_step_kernel.cuh: RS)
static const float EMUL_STALE = -7.25e3f;            // what a lane holds when a point starts (leftovers of the previous tile)

static std::vector<float> poisoned_rows(int rows) {
    return std::vector<float>((size_t)rows * EMUL_RS, std::numeric_limits<float>::quiet_NaN());
}

static int plan_k(const PinnSpec* spec, DevPlan& P, int& fwd_rows, int& fwd_row_scr, char* msg, int msg_len) {
    int rc = build_dev_plan(spec, P, fwd_rows, fwd_row_scr, msg, (size_t)msg_len, 4);
    if (rc) return rc;
    if (P.layer[P.n_layers - 1].n_out < 2) {
        snprintf(msg, msg_len, "a network of one output: emul_step of pinn_emul.cpp");
        return PINN_E_UNSUPPORTED;
    }
    return PINN_OK;
}

template <int NF, int NS>
static void run_step(const DevPlan& P, const float* sw, const float* params, const float* points, long long n,
                     float inv_n, float* out, float* residual) {
    std::vector<float> st = poisoned_rows(P.rows_total);
    GradSink sink;
    sink.wacc = out;
    sink.atomic = false;
    sink.dump = P.n_params + 2;
    PointPartials<NF, NS> part;
    part.loss = 0.0f; part.sbar = 0.0f;
    for (int i = 0; i < PINN_MAX_VARS; ++i) part.vbar[i] = 0.0f;
    for (long long p = 0; p < n; ++p) {
        float* lane = st.data() + (p % EMUL_RS);
        for (int r = 0; r < P.rows_total; ++r) lane[(size_t)r * EMUL_RS] = EMUL_STALE;
        for (int k = 0; k < P.total; ++k) lane[(size_t)k * EMUL_RS] = points[p * P.total + k];
        const float r = point_step<NF, NS, 16, true, true>(P, sw, params, lane, EMUL_RS, true, inv_n, sink, part);
        for (int q = 0; q < P.rows_total; ++q) lane[(size_t)q * EMUL_RS] = std::numeric_limits<float>::quiet_NaN();
        if (residual) residual[p] = r;
    }
    out[P.n_params] += part.loss;
    out[P.log_scale_off] += part.sbar;
    for (int i = 0; i < P.n_vars; ++i) out[P.var_off[i]] += part.vbar[i];
}

extern "C" int emul_coupled_step(const PinnSpec* spec, const float* params, const float* points, long long n, float inv_n,
                                 float* out, float* residual, char* msg, int msg_len) {
    DevPlan P;
    int fr, fs;
    int rc = plan_k(spec, P, fr, fs, msg, msg_len);
    if (rc) return rc;
    std::vector<float> sw(P.weights_floats + 16);
    host_stage_weights(P, params, sw.data());
    for (int i = 0; i < P.n_params + 4; ++i) out[i] = 0.0f;
#define CASE(NF_, NS_) if (P.nf == NF_ && P.ns == NS_) { run_step<NF_, NS_>(P, sw.data(), params, points, n, inv_n, out, residual); return 0; }
    CASE(0, 0) CASE(1, 0) CASE(1, 1) CASE(2, 0) CASE(2, 1) CASE(2, 2)
    CASE(3, 0) CASE(3, 1) CASE(3, 2) CASE(3, 3)
    CASE(4, 0) CASE(4, 1) CASE(4, 2) CASE(4, 3) CASE(4, 4)
#undef CASE
    snprintf(msg, msg_len, "no variant nf=%d ns=%d", P.nf, P.ns);
    return PINN_E_UNSUPPORTED;
}

// u_out [n, k]: what coupled_forward_kernel writes.
extern "C" int emul_coupled_forward(const PinnSpec* spec, const float* params, const float* points, long long n,
                                    float* u_out, char* msg, int msg_len) {
    DevPlan P;
    int fwd_rows, fwd_row_scr;
    int rc = plan_k(spec, P, fwd_rows, fwd_row_scr, msg, msg_len);
    if (rc) return rc;
    const int k = P.layer[P.n_layers - 1].n_out;
    std::vector<float> sw(P.weights_floats + 16);
    host_stage_weights(P, params, sw.data());
    std::vector<float> st = poisoned_rows(fwd_rows);
    for (long long p = 0; p < n; ++p) {
        float* lane = st.data() + (p % EMUL_RS);
        for (int r = 0; r < fwd_rows; ++r) lane[(size_t)r * EMUL_RS] = EMUL_STALE;
        for (int c = 0; c < P.total; ++c) lane[(size_t)c * EMUL_RS] = points[p * P.total + c];
        point_forward<16, true>(P, sw.data(), params, lane, EMUL_RS, fwd_row_scr);
        for (int j = 0; j < k; ++j) u_out[p * k + j] = lane[(size_t)(fwd_row_scr + j) * EMUL_RS];
        for (int r = 0; r < fwd_rows; ++r) lane[(size_t)r * EMUL_RS] = std::numeric_limits<float>::quiet_NaN();
    }
    return 0;
}
