// pinn_host_plan.h — host-side validation of a PinnSpec and construction of the device plan
// (layer table, shared-memory weight layout, per-point storage rows).  Plain C++: included by
// pinn_kernels.cu and by the test-only emulation harness (tests/emul/pinn_emul.cpp).
#pragma once

#include <stdio.h>
#include <string.h>
#include "pinn_device.cuh"

namespace pinn {

inline int round_up_i(int x, int m) { return (x + m - 1) / m * m; }

#define PINN_PLAN_FAIL(code, ...)                   \
    do {                                            \
        snprintf(msg, msg_len, __VA_ARGS__);        \
        return (code);                              \
    } while (0)

inline int validate_prog(const PinnInstr* prog, int n, int n_slots, int total, int n_vars, const char* name,
                         char* msg, size_t msg_len) {
    if (n < 0 || n > PINN_MAX_PROG) PINN_PLAN_FAIL(PINN_E_INVALID, "%s: %d instructions (max %d)", name, n, PINN_MAX_PROG);
    for (int i = 0; i < n; ++i) {
        const PinnInstr& in = prog[i];
        if (in.op >= PINN_OP_COUNT_) PINN_PLAN_FAIL(PINN_E_INVALID, "%s[%d]: bad opcode %d", name, i, in.op);
        if (in.dst >= n_slots) PINN_PLAN_FAIL(PINN_E_INVALID, "%s[%d]: dst slot %d >= n_slots %d", name, i, in.dst, n_slots);
        if (in.op == PINN_OP_COORD && in.a >= total) PINN_PLAN_FAIL(PINN_E_INVALID, "%s[%d]: coord %d", name, i, in.a);
        if (in.op == PINN_OP_VAR && in.a >= n_vars) PINN_PLAN_FAIL(PINN_E_INVALID, "%s[%d]: var %d", name, i, in.a);
        if (in.op >= PINN_OP_ADD) {
            if (in.a >= n_slots) PINN_PLAN_FAIL(PINN_E_INVALID, "%s[%d]: src slot", name, i);
            bool binary = in.op == PINN_OP_ADD || in.op == PINN_OP_SUB || in.op == PINN_OP_MUL ||
                          in.op == PINN_OP_DIV || in.op == PINN_OP_POW;
            if (binary && in.b >= n_slots) PINN_PLAN_FAIL(PINN_E_INVALID, "%s[%d]: src slot", name, i);
        }
    }
    return PINN_OK;
}

// Derivative order of a spec: 2 (value / first / second channels), or 3 / 4 (whole jets per direction, pinn_device_hi.cuh).
inline int spec_order(const PinnSpec* s) { return s->order >= 3 ? s->order : 2; }
inline int spec_channels(const PinnSpec* s) { return s->order >= 3 ? 1 + s->nf * s->order : 1 + s->nf + s->ns; }

// Fills `h` (device plan, minus anything that needs a device) and the forward-only row layout.  `max_out`: the most
// network outputs the caller's kernels take — 1 for the one-output code, 4 where the coupled form runs too.
inline int build_dev_plan(const PinnSpec* s, DevPlan& h, int& fwd_rows, int& fwd_row_scr, char* msg, size_t msg_len,
                          int max_out = 1) {
    if (s->abi_version != PINN_ABI_VERSION)
        PINN_PLAN_FAIL(PINN_E_INVALID, "spec abi_version %d != library %d", s->abi_version, PINN_ABI_VERSION);
    const int Ln = s->n_layers;
    if (Ln < 1 || Ln > PINN_MAX_LAYERS) PINN_PLAN_FAIL(PINN_E_INVALID, "n_layers %d", Ln);
    const int total = s->ndims + s->nparams;
    if (s->ndims < 1 || s->nparams < 0 || total > PINN_MAX_DIMS) PINN_PLAN_FAIL(PINN_E_INVALID, "ndims/nparams");
    if (s->widths[0] != total) PINN_PLAN_FAIL(PINN_E_INVALID, "widths[0]=%d != ndims+nparams=%d", s->widths[0], total);
    const int n_out = s->widths[Ln];
    if (n_out < 1 || n_out > max_out) PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "output width %d (1..%d)", n_out, max_out);
    if (s->act[Ln - 1] != PINN_ACT_NONE) PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "activation after the last layer");
    if (s->n_params <= 0 || (s->n_params & 3)) PINN_PLAN_FAIL(PINN_E_INVALID, "n_params must be a positive multiple of 4");
    if (s->nf < 0 || s->nf > PINN_MAX_DIRS || s->ns < 0 || s->ns > s->nf) PINN_PLAN_FAIL(PINN_E_INVALID, "jet set nf=%d ns=%d", s->nf, s->ns);
    if (s->n_vars < 0 || s->n_vars > PINN_MAX_VARS) PINN_PLAN_FAIL(PINN_E_INVALID, "n_vars");
    if (s->order != 0 && (s->order < 2 || s->order > 4)) PINN_PLAN_FAIL(PINN_E_INVALID, "derivative order %d (2..4)", s->order);
    const bool hi = s->order >= 3;
    if (hi) {
        // whole-jet plans (pinn_device_hi.cuh): what that code covers
        if (s->nf < 1 || s->nf > 4) PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "order %d with %d derivative directions (1..4)", s->order, s->nf);
        if (s->ns != 0) PINN_PLAN_FAIL(PINN_E_INVALID, "order %d: ns must be 0 (every direction carries its whole jet)", s->order);
        for (int d = 0; d < s->nf; ++d)
            for (int e = 0; e < d; ++e)
                if (s->dir_col[d] >= 0 && s->dir_col[e] == s->dir_col[d])
                    PINN_PLAN_FAIL(PINN_E_INVALID, "order %d: directions %d and %d coincide", s->order, e, d);
    }
    const int C = spec_channels(s);
    // networks of k > 1 outputs (coupled systems): the thread kernel's second-order form only
    if (n_out > 1 && (hi || s->nf > 4))
        PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "a network of %d outputs with %s: only derivatives up to order 2 along at most 4 directions",
                       n_out, hi ? "derivatives of order 3 / 4" : "more than 4 derivative directions");
    if (1 + C + s->n_vars > (int)(sizeof(s->eq_out) / sizeof(s->eq_out[0])))
        PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "%d jet channels + %d variables exceed the program's outputs", C, s->n_vars);
    if (s->has_ic && C * (1 + (s->ic_has_vars ? s->n_vars : 0)) > (int)(sizeof(s->ic_out) / sizeof(s->ic_out[0])))
        PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "%d jet channels x (1 + %d variables) exceed the initial condition's outputs", C, s->n_vars);
    for (int d = 0; d < s->nf; ++d) {
        if (s->dir_col[d] >= total) PINN_PLAN_FAIL(PINN_E_INVALID, "dir_col[%d]", d);
        bool any = false;
        for (int k = 0; k < total; ++k) {
            const float v = s->dir_vec[d][k];
            if (!(v == v) || v > 1e6f || v < -1e6f) PINN_PLAN_FAIL(PINN_E_INVALID, "dir_vec[%d][%d]", d, k);
            any = any || v != 0.0f;
            if (s->dir_col[d] >= 0 && v != (k == s->dir_col[d] ? 1.0f : 0.0f))
                PINN_PLAN_FAIL(PINN_E_INVALID, "dir_vec[%d] is not the unit vector of column %d", d, s->dir_col[d]);
        }
        if (!any) PINN_PLAN_FAIL(PINN_E_INVALID, "dir_vec[%d] is zero", d);
    }
    if (s->n_slots < C * n_out || s->n_slots > PINN_MAX_SLOTS) PINN_PLAN_FAIL(PINN_E_INVALID, "n_slots %d", s->n_slots);
    int rc;
    if ((rc = validate_prog(s->eq_prog, s->n_eq, s->n_slots, total, s->n_vars, "eq_prog", msg, msg_len))) return rc;
    if (s->has_ic && (rc = validate_prog(s->ic_prog, s->n_ic, s->n_slots, total, s->n_vars, "ic_prog", msg, msg_len))) return rc;
    for (int i = 0; i < 1 + C + s->n_vars; ++i)
        if (s->eq_out[i] < 0 || s->eq_out[i] >= s->n_slots) PINN_PLAN_FAIL(PINN_E_INVALID, "eq_out[%d]", i);
    if (n_out > 1) {                                   // the partials of the k components: one contiguous block of k*C slots
        if (s->eq_out[1] + C * n_out > s->n_slots) PINN_PLAN_FAIL(PINN_E_INVALID, "eq_out[1]: the partial block of %d slots ends past n_slots", C * n_out);
        for (int c = 0; c < C; ++c)
            if (s->eq_out[1 + c] != s->eq_out[1] + c) PINN_PLAN_FAIL(PINN_E_INVALID, "eq_out[%d] != eq_out[1] + %d", 1 + c, c);
    }
    if (s->has_ic)
        for (int c = 0; c < C * (1 + (s->ic_has_vars ? s->n_vars : 0)); ++c)
            if (s->ic_out[c] < 0 || s->ic_out[c] >= s->n_slots) PINN_PLAN_FAIL(PINN_E_INVALID, "ic_out[%d]", c);
    if (s->log_scale_off < 0 || s->log_scale_off >= s->n_params) PINN_PLAN_FAIL(PINN_E_INVALID, "log_scale_off");
    for (int i = 0; i < s->n_vars; ++i)
        if (s->var_off[i] < 0 || s->var_off[i] >= s->n_params) PINN_PLAN_FAIL(PINN_E_INVALID, "var_off[%d]", i);

    memset(&h, 0, sizeof(h));
    h.n_layers = Ln; h.total = total; h.ndims = s->ndims; h.nparams = s->nparams;
    h.has_bc = s->has_bc ? 1 : 0; h.has_ic = s->has_ic ? 1 : 0;
    h.nsp = s->has_ic ? s->ndims - 1 : s->ndims;
    h.nf = s->nf; h.ns = hi ? 0 : s->ns; h.n_params = s->n_params; h.log_scale_off = s->log_scale_off;
    h.n_vars = s->n_vars; h.n_eq = s->n_eq; h.n_ic = s->has_ic ? s->n_ic : 0; h.n_slots = s->n_slots;
    h.bc = s->bc_value;
    h.ic_has_vars = (s->has_ic && s->ic_has_vars) ? 1 : 0;
    h.t0 = s->dom_lo[s->ndims - 1];
    for (int d = 0; d < PINN_MAX_DIRS; ++d) {
        h.dir_col[d] = d < s->nf ? s->dir_col[d] : 0;
        for (int k = 0; k < PINN_MAX_DIMS; ++k) h.dir_vec[d][k] = (d < s->nf && k < total) ? s->dir_vec[d][k] : 0.0f;
    }
    for (int i = 0; i < PINN_MAX_VARS; ++i) h.var_off[i] = i < s->n_vars ? s->var_off[i] : 0;
    for (int i = 0; i < PINN_MAX_DIMS; ++i) {
        h.lo[i] = s->dom_lo[i]; h.hi[i] = s->dom_hi[i];
        float w = s->dom_hi[i] - s->dom_lo[i];
        h.inv_w2[i] = (i < s->ndims && w != 0.0f) ? 1.0f / (w * w) : 0.0f;
        memset(&h.cols[i], 0, sizeof(PinnColumn));
        h.cols[i].kind = PINN_COL_UNIFORM; h.cols[i].a = 0.0f; h.cols[i].b = 1.0f;
    }
    memcpy(h.eq_out, s->eq_out, sizeof(h.eq_out));
    memcpy(h.ic_out, s->ic_out, sizeof(h.ic_out));
    memcpy(h.eq, s->eq_prog, sizeof(h.eq));
    memcpy(h.ic, s->ic_prog, sizeof(h.ic));

    int sw = 0, units = 0;
    for (int l = 0; l < Ln; ++l) {
        DevLayer& L = h.layer[l];
        L.n_in = s->widths[l]; L.n_out = s->widths[l + 1]; L.act = s->act[l];
        if (L.n_in < 1 || L.n_out < 1) PINN_PLAN_FAIL(PINN_E_INVALID, "layer %d width", l);
        if (L.act < 0 || L.act > PINN_ACT_GELU) PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "layer %d: activation %d is not covered by the fused kernel", l, L.act);
        L.w_off = s->w_off[l]; L.b_off = s->b_off[l];
        if (L.w_off < 0 || L.w_off + L.n_in * L.n_out > s->n_params || L.b_off < 0 || L.b_off + L.n_out > s->n_params)
            PINN_PLAN_FAIL(PINN_E_INVALID, "layer %d offsets out of range", l);
        L.n_out_p4 = round_up_i(L.n_out, 4);
        L.n_in_p8 = round_up_i(L.n_in + 1, 8);          // + the (zero) bias column of the reverse sweep
        L.wt_s = sw; sw += L.n_in * L.n_out_p4;
        L.w_s = sw;  sw += L.n_out_p4 * L.n_in_p8;
        L.b_s = sw;  sw += L.n_out_p4;
        L.unit_base = units; units += L.n_out;
        L.post_base = -1; L.skip_src = -1; L.adj_from = -1;
    }
    for (int l = 0; l < Ln; ++l) {
        const int src = s->skip_src[l];
        if (src < 0) continue;
        DevLayer& L = h.layer[l];
        if (l == Ln - 1) PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "skip connection into the output layer");
        if (src >= l) PINN_PLAN_FAIL(PINN_E_INVALID, "skip_src[%d] = %d must be an earlier layer", l, src);
        if (h.layer[src].n_out != L.n_out) PINN_PLAN_FAIL(PINN_E_INVALID, "skip %d -> %d: widths %d and %d differ", src, l, h.layer[src].n_out, L.n_out);
        if (h.layer[src].adj_from >= 0) PINN_PLAN_FAIL(PINN_E_UNSUPPORTED, "layer %d is the source of two skip connections", src);
        L.skip_src = src; L.post_base = units; units += L.n_out;
        h.layer[src].adj_from = l;
    }
    h.general = h.ic_has_vars;
    for (int l = 0; l < Ln; ++l) if (h.layer[l].skip_src >= 0) h.general = 1;
    for (int l = 0; l < Ln; ++l) if (h.layer[l].act >= PINN_ACT_SIN) h.general = 1;     // z-stored activations
    for (int d = 0; d < s->nf; ++d) if (s->dir_col[d] < 0) h.general = 1;
    h.weights_floats = round_up_i(sw, 4);
    h.n_units = units;
    h.row_units = total;
    h.row_scr = total + units * C;
    h.rows_total = h.row_scr + s->n_slots;
    fwd_row_scr = total + units;
    fwd_rows = fwd_row_scr + s->n_slots;
    return PINN_OK;
}

// The step kernel's compact per-point layout (point_step<…, REMAT0 = true>), for plain one-output networks of two hidden
// layers or more.  The first layer's jet is never kept: its first-order channels are the same for every point and its
// second-order ones vanish, and its values cost one tiny layer over the coordinates, so the forward pass builds it in rows
// that the second hidden layer takes over later, and the reverse pass rebuilds it, bit for bit, in the same rows once
// that layer's adjoint is spent.  The output layer's adjoint and the rows that swallow masked-off stores share the
// program's scratch rows, which are dead by then.  Per point: the coordinates, hidden layers 1 .. n-2 (at least as many
// rows as layers 0 and 1 take together), and max(n_slots, 2 C) scratch rows — cfg2 ([2, 10, 12, 15, 1], C = 5): 147 rows
// instead of 200.
// Fills `c` from the plan `h` and returns true, or returns false where the compact layout does not apply.
inline bool build_remat_plan(const DevPlan& h, DevPlan& c) {
    const int Ln = h.n_layers;
    if (h.general || Ln < 3 || h.layer[Ln - 1].n_out != 1) return false;
    const int C = 1 + h.nf + h.ns;
    c = h;
    int units = 0;
    for (int l = 1; l < Ln - 1; ++l) { c.layer[l].unit_base = units; units += h.layer[l].n_out; }
    c.layer[0].unit_base = h.layer[1].n_out;                  // behind layer 1 (over layer 2's rows, if that is hidden)
    c.layer[Ln - 1].unit_base = 0;                            // unused: the output layer's adjoint lives in the scratch rows
    const int first_end = h.layer[1].n_out + h.layer[0].n_out;
    c.row_scr = h.total + C * (units > first_end ? units : first_end);
    c.rows_total = c.row_scr + (h.n_slots > 2 * C ? h.n_slots : 2 * C);
    return true;
}

// Re-layout of the flat parameters into the weight area (what stage_plan_and_weights does on the GPU).
inline void host_stage_weights(const DevPlan& P, const float* params, float* sw) {
    for (int i = 0; i < P.weights_floats; ++i) sw[i] = 0.0f;
    for (int l = 0; l < P.n_layers; ++l) {
        const DevLayer& L = P.layer[l];
        for (int j = 0; j < L.n_out; ++j) {
            for (int k = 0; k < L.n_in; ++k) {
                float w = params[L.w_off + j * L.n_in + k];
                sw[L.wt_s + k * L.n_out_p4 + j] = w;
                sw[L.w_s + j * L.n_in_p8 + k] = w;
            }
            sw[L.b_s + j] = params[L.b_off + j];
        }
    }
}

// A constraint term's plan `g` (spec order `g_order`) next to the plan `h` it trains with: the same network, parameter
// layout and ansatz, variables among h's, and a jet set the kernels run its program on — no derivative directions
// (C = 1), or exactly h's (nf, ns, directions, order 2).  Fills `t` (var_map: h's variable of every term variable).
inline int build_dev_term(const DevPlan& h, int h_order, const DevPlan& g, int g_order, DevTerm& t, char* msg,
                          size_t msg_len) {
    if (g.n_layers != h.n_layers || memcmp(g.layer, h.layer, sizeof(DevLayer) * h.n_layers) != 0)
        PINN_PLAN_FAIL(PINN_E_INVALID, "constraint term: its layer table differs from the plan's");
    if (g.n_params != h.n_params || g.log_scale_off != h.log_scale_off)
        PINN_PLAN_FAIL(PINN_E_INVALID, "constraint term: n_params / log_scale_off differ from the plan's");
    const bool value_only = g.nf == 0 && g.ns == 0 && g_order == 2;
    const bool same_jets = g.nf == h.nf && g.ns == h.ns && g_order == 2 && h_order == 2 &&
                           memcmp(g.dir_vec, h.dir_vec, sizeof(h.dir_vec[0]) * h.nf) == 0;
    if (!value_only && !same_jets)
        PINN_PLAN_FAIL(PINN_E_INVALID, "constraint term: its plan carries derivative directions other than the plan's");
    if (g.total != h.total || g.nsp != h.nsp || g.has_bc != h.has_bc || g.has_ic != h.has_ic || g.bc != h.bc ||
        g.t0 != h.t0 || memcmp(g.lo, h.lo, sizeof(h.lo)) != 0 || memcmp(g.hi, h.hi, sizeof(h.hi)) != 0)
        PINN_PLAN_FAIL(PINN_E_INVALID, "constraint term: its ansatz differs from the plan's");
    memset(&t, 0, sizeof(t));
    t.n_eq = g.n_eq; t.n_vars = g.n_vars;
    t.C = 1 + g.nf + g.ns;
    for (int i = 0; i < g.n_vars; ++i) {
        t.var_off[i] = g.var_off[i];
        t.var_map[i] = -1;
        for (int j = 0; j < h.n_vars; ++j) if (h.var_off[j] == g.var_off[i]) t.var_map[i] = j;
        if (t.var_map[i] < 0) PINN_PLAN_FAIL(PINN_E_INVALID, "constraint term: variable %d is not one of the plan's", i);
    }
    for (int i = 0; i < 1 + t.C + g.n_vars; ++i) t.eq_out[i] = g.eq_out[i];     // r, dr/dchannel_c, dr/dV_i
    memcpy(t.eq, g.eq, sizeof(t.eq));
    return PINN_OK;
}

}  // namespace pinn
