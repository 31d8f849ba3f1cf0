// TEST INFRASTRUCTURE ONLY — host emulation of the per-point device code.
//
// Compiles pydens_b200/csrc/pinn_device.cuh (the very functions the CUDA kernel runs per thread)
// with g++ and drives them one point at a time, so the forward jets, ansatz, residual programs and
// the hand-derived reverse sweep can be checked against the oracle on a machine without a GPU.
// The warp-level gradient reduction is replaced by direct accumulation (emit_entries' host branch).
// The per-point storage is laid out as on the device: rows of 32 lanes (row stride RS = 32), the point in one lane,
// every other lane poisoned with NaN — an access that forgets the row stride or strays into a neighbour's lane shows
// up as NaN in the result instead of passing by accident.
// Never loaded by the product (pydens_b200/_native.py loads only libpinn_b200.so).
#include <vector>
#include <limits>
#include <string.h>
#include "../../pydens_b200/csrc/pinn_host_plan.h"
#include "../../pydens_b200/csrc/pinn_device_hi.cuh"

using namespace pinn;

static const int EMUL_RS = 32;                       // the device's row stride (pinn_step_kernel.cuh: RS)
// what a lane holds when a point starts: on the device the leftovers of the previous tile (finite, arbitrary) — results must
// not depend on them
static const float EMUL_STALE = -7.25e3f;

// storage of `rows` rows x 32 lanes, all NaN; the point of index p lives in lane p % 32
static std::vector<float> poisoned_rows(int rows) {
    return std::vector<float>((size_t)rows * EMUL_RS, std::numeric_limits<float>::quiet_NaN());
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
        // both instantiations the CUDA build uses: the plain one when the plan allows it, else the general one
        // (more than 4 directions: the CUDA build has the general instantiation only, also for plain plans)
        float r;
        if constexpr (NF > 4) r = point_step<NF, NS, 16, true>(P, sw, params, lane, EMUL_RS, true, inv_n, sink, part);
        else r = P.general ? point_step<NF, NS, 16, true>(P, sw, params, lane, EMUL_RS, true, inv_n, sink, part)
                           : point_step<NF, NS, 16, false>(P, sw, params, lane, EMUL_RS, true, inv_n, sink, part);
        for (int q = 0; q < P.rows_total; ++q) lane[(size_t)q * EMUL_RS] = std::numeric_limits<float>::quiet_NaN();
        if (residual) residual[p] = r;
    }
    out[P.n_params] += part.loss;
    out[P.log_scale_off] += part.sbar;
    for (int i = 0; i < P.n_vars; ++i) out[P.var_off[i]] += part.vbar[i];
}

// derivatives of order 3 / 4: the whole-jet code of pinn_device_hi.cuh, driven the same way
template <int NF, int K>
static void run_step_hi(const DevPlan& P, const float* sw, const float* params, const float* points, long long n,
                        float inv_n, float* out, float* residual) {
    std::vector<float> st = poisoned_rows(P.rows_total);
    GradSink sink;
    sink.wacc = out;
    sink.atomic = false;
    sink.dump = P.n_params + 2;
    hi::PartialsHi part;
    part.loss = 0.0f; part.sbar = 0.0f;
    for (int i = 0; i < PINN_MAX_VARS; ++i) part.vbar[i] = 0.0f;
    for (long long p = 0; p < n; ++p) {
        float* lane = st.data() + (p % EMUL_RS);
        for (int r = 0; r < P.rows_total; ++r) lane[(size_t)r * EMUL_RS] = EMUL_STALE;
        for (int k = 0; k < P.total; ++k) lane[(size_t)k * EMUL_RS] = points[p * P.total + k];
        float r = hi::point_step<NF, K>(P, sw, params, lane, EMUL_RS, true, inv_n, sink, part);
        for (int q = 0; q < P.rows_total; ++q) lane[(size_t)q * EMUL_RS] = std::numeric_limits<float>::quiet_NaN();
        if (residual) residual[p] = r;
    }
    out[P.n_params] += part.loss;
    out[P.log_scale_off] += part.sbar;
    for (int i = 0; i < P.n_vars; ++i) out[P.var_off[i]] += part.vbar[i];
}

extern "C" int emul_step(const PinnSpec* spec, const float* params, const float* points, long long n, float inv_n,
                         float* out, float* residual, char* msg, int msg_len) {
    DevPlan P;
    int fr, fs;
    int rc = build_dev_plan(spec, P, fr, fs, msg, (size_t)msg_len);
    if (rc) return rc;
    std::vector<float> sw(P.weights_floats + 16);
    host_stage_weights(P, params, sw.data());
    for (int i = 0; i < P.n_params + 4; ++i) out[i] = 0.0f;
#define CASE_HI(NF_, K_) if (spec_order(spec) == K_ && P.nf == NF_) { run_step_hi<NF_, K_>(P, sw.data(), params, points, n, inv_n, out, residual); return 0; }
    CASE_HI(1, 3) CASE_HI(2, 3) CASE_HI(3, 3) CASE_HI(4, 3) CASE_HI(1, 4) CASE_HI(2, 4) CASE_HI(3, 4) CASE_HI(4, 4)
#undef CASE_HI
    if (spec_order(spec) >= 3) { snprintf(msg, msg_len, "no hi variant nf=%d order=%d", P.nf, spec_order(spec)); return PINN_E_UNSUPPORTED; }
#define CASE(NF_, NS_) if (P.nf == NF_ && P.ns == NS_) { run_step<NF_, NS_>(P, sw.data(), params, points, n, inv_n, out, residual); return 0; }
    CASE(0, 0) CASE(1, 0) CASE(1, 1) CASE(2, 0) CASE(2, 1) CASE(2, 2)
    CASE(3, 0) CASE(3, 1) CASE(3, 2) CASE(3, 3)
    CASE(4, 0) CASE(4, 1) CASE(4, 2) CASE(4, 3) CASE(4, 4)
    CASE(5, 5) CASE(6, 6)
#undef CASE
    snprintf(msg, msg_len, "no variant nf=%d ns=%d", P.nf, P.ns);
    return PINN_E_UNSUPPORTED;
}

extern "C" int emul_forward(const PinnSpec* spec, const float* params, const float* points, long long n,
                            float* u_out, char* msg, int msg_len) {
    DevPlan P;
    int fwd_rows, fwd_row_scr;
    int rc = build_dev_plan(spec, P, fwd_rows, fwd_row_scr, msg, (size_t)msg_len);
    if (rc) return rc;
    std::vector<float> sw(P.weights_floats + 16);
    host_stage_weights(P, params, sw.data());
    std::vector<float> st = poisoned_rows(fwd_rows);
    for (long long p = 0; p < n; ++p) {
        float* lane = st.data() + (p % EMUL_RS);
        for (int r = 0; r < fwd_rows; ++r) lane[(size_t)r * EMUL_RS] = EMUL_STALE;
        for (int k = 0; k < P.total; ++k) lane[(size_t)k * EMUL_RS] = points[p * P.total + k];
        u_out[p] = point_forward<16>(P, sw.data(), params, lane, EMUL_RS, fwd_row_scr);
        for (int r = 0; r < fwd_rows; ++r) lane[(size_t)r * EMUL_RS] = std::numeric_limits<float>::quiet_NaN();
    }
    return 0;
}

// Philox / sampler restatement check: same code path as sample_kernel.
extern "C" void emul_sample(const PinnColumn* cols, int total, unsigned long long seed, unsigned long long step,
                            unsigned long long point_offset, long long n, float* out) {
    for (long long p = 0; p < n; ++p) {
        const uint64_t gidx = point_offset + (uint64_t)p;
        Philox4 b0 = philox_block(gidx, step, seed, 0u);
        Philox4 b1 = b0;
        if (total > 4) b1 = philox_block(gidx, step, seed, 1u);
        for (int k = 0; k < total; ++k) out[p * total + k] = sample_column(cols[k], k, gidx, step, seed, b0, b1);
    }
}
