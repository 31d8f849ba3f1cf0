// L-BFGS state machine: torch.optim.LBFGS.step(closure) (torch 2.11, torch/optim/lbfgs.py) restated so that its state
// lives in one buffer and every evaluation of the objective is an exit point (include/pinn_b200.h: pinn_lbfgs_advance).
//
// Two halves, both templated on the vector type T (float on the device, double in the host build the tests run):
//   lbfgs_control  the scalar logic of torch's step, line search and exit tests, one branch for each of torch's; it
//                  runs on one thread and asks for one vector pass (or an evaluation) at a time;
//   lbfgs_pass     the vector passes over the n_params entries, written once for a CTA and for one host thread (Exec).
// The two-loop recursion runs without vectors (Chen, Wang, Zhou, NeurIPS 2014): the state keeps the Gram entries
// s_p . y_q and y_p . y_q of the ring, a new pair adds one row and column, and one pass over the history gives every
// dot product the recursion needs; the recursion itself is scalar (one warp), and one more pass forms
// d = hg g + sum_i cs_i s_i + cy_i y_i.
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/pinn_b200.h"

#if defined(__CUDACC__)
#define LB_HD __host__ __device__ __forceinline__
#else
#define LB_HD inline
#endif

namespace pinn {
namespace lbfgs {

// gradient references: the evaluation just made ([grads | loss]), prev_flat_grad, three line-search copies
enum { REF_OUT = 0, REF_PG = 1, REF_POOL = 2, N_REF = 5 };
// vector slots of the state buffer (pinn_b200.h)
enum { V_D = 0, V_PG = 1, V_X = 2, V_POOL = 3, V_RING = 6 };
// control phases; PH_START, PH_FIX_EVAL and PH_LS_EVAL wait for an evaluation
enum { PH_START = 0, PH_E0_STAT, PH_ITER, PH_HIST_DONE, PH_DIR_DONE, PH_FIX_EVAL, PH_FIX_STAT, PH_CHECKS, PH_LS_EVAL,
       PH_LS_STAT, PH_ZOOM_TOP, PH_FINISH };
// what the control asks for next
enum { ACT_DONE = 0, ACT_GSTAT, ACT_HIST, ACT_DIR, ACT_MOVE, ACT_LSEVAL };

static const double C1 = 1e-4, C2 = 0.9;             // _strong_wolfe defaults

LB_HD int64_t padded(int64_t n) { return (n + 3) / 4 * 4; }
LB_HD size_t fp64_count(int m) { size_t S = (size_t)m + 1; return 2 * S * S + 5 * S; }
LB_HD size_t vector_offset(int m) { return (PINN_LBFGS_HEADER_BYTES + 8 * fp64_count(m) + 255) / 256 * 256; }
template <class T>
LB_HD size_t state_bytes(int64_t n, int m) {
    return vector_offset(m) + sizeof(T) * (size_t)padded(n) * (size_t)(V_RING + 2 * (m + 1));
}

// max as torch's .max() reduces: a NaN wins
LB_HD double nan_max(double a, double b) { return (b > a || b != b) ? b : a; }

// Python's max(a, b) / min(a, b): the first argument unless the second compares greater / smaller (NaN stays put)
LB_HD double py_max(double a, double b) { return b > a ? b : a; }
LB_HD double py_min(double a, double b) { return b < a ? b : a; }

// torch.optim.lbfgs._cubic_interpolate; bounded: (lo, hi) as given, else the sorted pair (x1, x2)
LB_HD double cubic_interpolate(double x1, double f1, double g1, double x2, double f2, double g2, bool bounded,
                               double lo, double hi) {
    double xmin = bounded ? lo : (x1 <= x2 ? x1 : x2);
    double xmax = bounded ? hi : (x1 <= x2 ? x2 : x1);
    double d1 = g1 + g2 - 3 * (f1 - f2) / (x1 - x2);
    double d2_square = d1 * d1 - g1 * g2;
    if (d2_square >= 0) {
        double d2 = sqrt(d2_square), min_pos;
        if (x1 <= x2) min_pos = x2 - (x2 - x1) * ((g2 + d2 - d1) / (g2 - g1 + 2 * d2));
        else min_pos = x1 - (x1 - x2) * ((g1 + d2 - d1) / (g1 - g2 + 2 * d2));
        return py_min(py_max(min_pos, xmin), xmax);
    }
    return (xmin + xmax) / 2.0;
}

// The parts of one state buffer.
template <class T>
struct View {
    double *sy, *yy, *sg, *yg, *al, *cs, *cy;
    T* vec;
    int64_t nv;
    int S;
    LB_HD View(void* state, int64_t n, int m) {
        S = m + 1;
        double* f = (double*)((char*)state + PINN_LBFGS_HEADER_BYTES);
        sy = f; yy = sy + S * S; sg = yy + S * S; yg = sg + S; al = yg + S; cs = al + S; cy = cs + S;
        vec = (T*)((char*)state + vector_offset(m));
        nv = padded(n);
    }
    LB_HD T* v(int k) const { return vec + (int64_t)k * nv; }
    LB_HD T* s(int p) const { return v(V_RING + p); }
    LB_HD T* y(int p) const { return v(V_RING + S + p); }
    LB_HD int phys(const PinnLbfgsState* h, int i) const { return (h->ring_head + i) % S; }
    LB_HD int spare(const PinnLbfgsState* h) const { return (h->ring_head + h->ring_count) % S; }
};

LB_HD int ask(PinnLbfgsState* h, int phase, int action, int arg = 0, int eval = 0) {
    h->phase = phase; h->action = action; h->act_arg = arg; h->act_eval = eval;
    return action;
}

// The first line-search copy no bracket entry (or g_prev) refers to.
LB_HD int free_copy(const PinnLbfgsState* h) {
    for (int r = REF_POOL; r < N_REF; ++r) {
        bool live = h->ls_zoom ? (h->br_g[0] == r || h->br_g[1] == r) : h->gp_ref == r;
        if (!live) return r;
    }
    return REF_POOL;                                   // unreachable: at most two references are live
}

LB_HD void set_bracket(PinnLbfgsState* h, int k, double t, double f, double gtd, int g) {
    h->br_t[k] = t; h->br_f[k] = f; h->br_gtd[k] = gtd; h->br_g[k] = g;
}

LB_HD void zoom_start(PinnLbfgsState* h) {
    h->ls_zoom = 1;
    h->low = h->br_f[0] <= h->br_f[1] ? 0 : 1;
    h->high = 1 - h->low;
    h->phase = PH_ZOOM_TOP;
}

// Runs torch's step from h->phase until it needs a vector pass or the step is over (ACT_DONE).  An ACT_MOVE with
// act_eval set ends the advance: the caller evaluates at the new params.  `loss` is that evaluation's loss (read where a
// phase consumes it).
LB_HD int lbfgs_control(const PinnLbfgs& c, PinnLbfgsState* h, const double* sy, const double* yy, double loss, int S) {
    for (;;) {
        switch (h->phase) {
        case PH_START:                                 // orig_loss = closure(); flat_grad
            return ask(h, PH_E0_STAT, ACT_GSTAT, REF_OUT);
        case PH_E0_STAT:
            h->loss = h->first_loss = loss;
            h->current_evals = 1;
            h->func_evals += 1;
            h->g_src = REF_OUT;
            h->ref_gmax[REF_OUT] = h->r_max;
            h->gsum_g = h->r_l1;
            h->opt_cond = 0;
            h->cur_iter = 0;
            h->phase = h->r_max <= c.tolerance_grad ? PH_FINISH : PH_ITER;
            break;
        case PH_ITER:
            h->cur_iter += 1;
            h->n_iter += 1;
            if (h->n_iter == 1) {                      // d = -g: the two-loop over an empty history with H_diag = 1
                h->ring_count = 0; h->ring_head = 0; h->H_diag = 1;
                return ask(h, PH_DIR_DONE, ACT_DIR, h->g_src);
            }
            return ask(h, PH_HIST_DONE, ACT_HIST, h->g_src);
        case PH_HIST_DONE: {                           // the new pair sits in the spare slot; keep it if ys > 1e-10
            int sp = (h->ring_head + h->ring_count) % S;
            double ys = sy[sp * S + sp];
            if (ys > 1e-10) {
                if (h->ring_count == S - 1) h->ring_head = (h->ring_head + 1) % S;
                else h->ring_count += 1;
                h->H_diag = ys / yy[sp * S + sp];
            }
            return ask(h, PH_DIR_DONE, ACT_DIR, h->g_src);
        }
        case PH_DIR_DONE:                              // d formed, prev_flat_grad = g, x = params (line search)
            h->gtd = h->r_dot;
            h->d_norm = h->r_max;
            h->ref_gmax[REF_PG] = h->ref_gmax[h->g_src];
            h->prev_loss = h->loss;
            h->t = h->n_iter == 1 ? py_min(1.0, 1.0 / h->gsum_g) * c.lr : c.lr;
            if (h->gtd > -c.tolerance_change) { h->phase = PH_FINISH; break; }
            if (c.line_search) {                       // _strong_wolfe(obj, x, t, d, loss, g, gtd, max_ls)
                h->max_ls = c.max_eval - h->current_evals;
                h->ls_iter = 0; h->ls_evals = 0; h->ls_done = 0; h->ls_zoom = 0; h->insuf = 0;
                h->t_prev = 0; h->f_prev = h->loss; h->gtd_prev = h->gtd; h->gp_ref = REF_PG;
                return ask(h, PH_LS_EVAL, ACT_MOVE, 1, 1);
            }
            if (h->cur_iter != c.max_iter) return ask(h, PH_FIX_EVAL, ACT_MOVE, 0, 1);
            h->ls_evals = 0;                           // last inner iteration: no re-evaluation
            return ask(h, PH_CHECKS, ACT_MOVE, 0, 0);
        case PH_FIX_EVAL:
            return ask(h, PH_FIX_STAT, ACT_GSTAT, REF_OUT);
        case PH_FIX_STAT:
            h->loss = loss;
            h->g_src = REF_OUT;
            h->ref_gmax[REF_OUT] = h->r_max;
            h->opt_cond = h->r_max <= c.tolerance_grad;
            h->ls_evals = 1;
            h->phase = PH_CHECKS;
            break;
        case PH_CHECKS:
            h->current_evals += h->ls_evals;
            h->func_evals += h->ls_evals;
            if (h->cur_iter == c.max_iter || h->current_evals >= c.max_eval || h->opt_cond
                    || h->d_norm * fabs(h->t) <= c.tolerance_change || fabs(h->loss - h->prev_loss) < c.tolerance_change)
                h->phase = PH_FINISH;
            else
                h->phase = PH_ITER;
            break;
        case PH_LS_EVAL:                               // an evaluation at x + t d: keep a copy of its gradient
            h->new_ref = free_copy(h);
            return ask(h, PH_LS_STAT, ACT_LSEVAL, h->new_ref);
        case PH_LS_STAT: {
            h->f_new = loss;
            h->gtd_new = h->r_dot;
            h->ref_gmax[h->new_ref] = h->r_max;
            if (h->ls_evals == 0) h->ls_evals = 1;
            else { h->ls_evals += 1; h->ls_iter += 1; }
            double armijo = h->loss + C1 * h->t * h->gtd;
            if (h->ls_zoom) {
                if (h->f_new > armijo || h->f_new >= h->br_f[h->low]) {
                    set_bracket(h, h->high, h->t, h->f_new, h->gtd_new, h->new_ref);
                    h->low = h->br_f[0] <= h->br_f[1] ? 0 : 1;
                    h->high = 1 - h->low;
                } else {
                    if (fabs(h->gtd_new) <= -C2 * h->gtd) h->ls_done = 1;
                    else if (h->gtd_new * (h->br_t[h->high] - h->br_t[h->low]) >= 0)
                        set_bracket(h, h->high, h->br_t[h->low], h->br_f[h->low], h->br_gtd[h->low], h->br_g[h->low]);
                    set_bracket(h, h->low, h->t, h->f_new, h->gtd_new, h->new_ref);
                }
                h->phase = PH_ZOOM_TOP;
                break;
            }
            if (h->ls_iter < h->max_ls) {              // the bracket phase
                bool wolfe = fabs(h->gtd_new) <= -C2 * h->gtd;
                if (h->f_new > armijo || (h->ls_iter > 1 && h->f_new >= h->f_prev) || (!wolfe && h->gtd_new >= 0)) {
                    set_bracket(h, 0, h->t_prev, h->f_prev, h->gtd_prev, h->gp_ref);
                    set_bracket(h, 1, h->t, h->f_new, h->gtd_new, h->new_ref);
                    zoom_start(h);
                    break;
                }
                if (wolfe) {
                    set_bracket(h, 0, h->t, h->f_new, h->gtd_new, h->new_ref);
                    set_bracket(h, 1, h->t, h->f_new, h->gtd_new, h->new_ref);
                    h->ls_done = 1;
                    zoom_start(h);
                    break;
                }
                double min_step = h->t + 0.01 * (h->t - h->t_prev), max_step = h->t * 10, tmp = h->t;
                h->t = cubic_interpolate(h->t_prev, h->f_prev, h->gtd_prev, h->t, h->f_new, h->gtd_new, true,
                                         min_step, max_step);
                h->t_prev = tmp; h->f_prev = h->f_new; h->gp_ref = h->new_ref; h->gtd_prev = h->gtd_new;
                return ask(h, PH_LS_EVAL, ACT_MOVE, 1, 1);
            }
            // ls_iter == max_ls: bracket [0, t] (its gtd is never read: the zoom loop does not run)
            set_bracket(h, 0, 0.0, h->loss, 0.0, REF_PG);
            set_bracket(h, 1, h->t, h->f_new, h->gtd_new, h->new_ref);
            zoom_start(h);
            break;
        }
        case PH_ZOOM_TOP: {
            if (!h->ls_done && h->ls_iter < h->max_ls
                    && !(fabs(h->br_t[1] - h->br_t[0]) * h->d_norm < c.tolerance_change)) {
                double t = cubic_interpolate(h->br_t[0], h->br_f[0], h->br_gtd[0], h->br_t[1], h->br_f[1],
                                             h->br_gtd[1], false, 0.0, 0.0);
                double bmax = py_max(h->br_t[0], h->br_t[1]), bmin = py_min(h->br_t[0], h->br_t[1]);
                double eps = 0.1 * (bmax - bmin);
                if (py_min(bmax - t, t - bmin) < eps) {
                    if (h->insuf || t >= bmax || t <= bmin) {
                        t = fabs(t - bmax) < fabs(t - bmin) ? bmax - eps : bmin + eps;
                        h->insuf = 0;
                    } else {
                        h->insuf = 1;
                    }
                } else {
                    h->insuf = 0;
                }
                h->t = t;
                return ask(h, PH_LS_EVAL, ACT_MOVE, 1, 1);
            }
            // the line search returns the low bracket point; params = x + t d
            h->t = h->br_t[h->low];
            h->loss = h->br_f[h->low];
            h->g_src = h->br_g[h->low];
            h->opt_cond = h->ref_gmax[h->g_src] <= c.tolerance_grad;
            return ask(h, PH_CHECKS, ACT_MOVE, 1, 0);
        }
        default:                                       // PH_FINISH
            if (c.losses_ring) {
                uint64_t k = *c.step_counter;
                c.losses_ring[k % (uint64_t)c.ring_len] = (float)h->first_loss;
            }
            *c.step_counter += 1;
            return ask(h, PH_START, ACT_DONE);
        }
    }
}

// Where the vector passes run: a CTA (CtaExec below) or one host thread (HostExec below).  Exec provides tid /
// nt (thread and thread count), lane / nl / warp / nw, wsum (warp sum, the same value in every lane), bsum / bmax
// (block reductions, the same value in every thread), bsync, wsync.

// The two-loop recursion on the Gram entries (warp 0 of the CTA, or the host thread): al (torch's `al`), and the
// coefficients of d = hg g + sum_i cs[i] s_i + cy[i] y_i.
//   q = -g - sum_{j>i} al_j y_j:             al_i = ro_i s_i . q = ro_i (-s_i . g - sum_{j>i} al_j s_i . y_j)
//   r = H q + sum_{j<i} c_j s_j:             be_i = ro_i y_i . r,  c_i = al_i - be_i
template <class T, class E>
LB_HD void two_loop(E& ex, PinnLbfgsState* h, const View<T>& v) {
    const int S = v.S, k = h->ring_count;
    const double H = h->H_diag;
    for (int i = k - 1; i >= 0; --i) {
        int pi = v.phys(h, i);
        double acc = 0;
        for (int j = i + 1 + ex.lane; j < k; j += ex.nl) acc += v.al[j] * v.sy[pi * S + v.phys(h, j)];
        acc = ex.wsum(acc);
        double ro = 1.0 / v.sy[pi * S + pi];
        if (ex.lane == 0) v.al[i] = (-v.sg[pi] - acc) * ro;
        ex.wsync();
    }
    for (int i = 0; i < k; ++i) {
        int pi = v.phys(h, i);
        double a1 = 0, a2 = 0;
        for (int j = ex.lane; j < k; j += ex.nl) {
            int pj = v.phys(h, j);
            a1 += v.al[j] * v.yy[pi * S + pj];
            if (j < i) a2 += v.cs[j] * v.sy[pj * S + pi];
        }
        a1 = ex.wsum(a1);
        a2 = ex.wsum(a2);
        double be = (H * (-v.yg[pi] - a1) + a2) * (1.0 / v.sy[pi * S + pi]);
        if (ex.lane == 0) { v.cs[i] = v.al[i] - be; v.cy[i] = -H * v.al[i]; }
        ex.wsync();
    }
    if (ex.lane == 0) h->hg = -H;
    ex.wsync();
}

// The gradient an action reads: the evaluation's (masked as it is read), prev_flat_grad or a line-search copy.
template <class T>
LB_HD const T* grad_of(const View<T>& v, int ref, const T* out) {
    return ref == REF_OUT ? out : v.v(ref == REF_PG ? V_PG : V_POOL + ref - REF_POOL);
}

// One vector pass (h->action) over the n entries.  `stage`: 3 nv values of shared memory for g, y, s, or null.
template <class T, class E>
LB_HD void lbfgs_pass(E& ex, const PinnLbfgs& c, PinnLbfgsState* h, const View<T>& v, int64_t n, T* params,
                      const T* out, const T* mask, T* stage) {
    const int S = v.S;
    const int64_t nv = v.nv;
    switch (h->action) {
    case ACT_GSTAT: {                                  // max|g|, |g|_1
        double mx = 0, l1 = 0;
        for (int64_t e = ex.tid; e < n; e += ex.nt) {
            if (mask[e] == T(0)) continue;
            double a = fabs((double)out[e]);
            mx = nan_max(mx, a);
            l1 += a;
        }
        mx = ex.bmax(mx);
        l1 = ex.bsum(l1);
        if (ex.tid == 0) { h->r_max = mx; h->r_l1 = l1; }
        break;
    }
    case ACT_HIST: {                                   // y = g - prev_flat_grad, s = t d into the spare slot; dots
        const T* g = grad_of(v, h->act_arg, out);
        const int sp = v.spare(h);
        T *ys = v.y(sp), *ss = v.s(sp), *pg = v.v(V_PG), *d = v.v(V_D);
        const T tt = (T)h->t;
        T *gq = stage ? stage : nullptr, *yq = stage ? stage + nv : ys, *sq = stage ? stage + 2 * nv : ss;
        for (int64_t e = ex.tid; e < nv; e += ex.nt) {
            T ge = (e < n && mask[e] != T(0)) ? g[e] : T(0);
            T ye = ge - pg[e], se = d[e] * tt;
            ys[e] = ye; ss[e] = se;
            if (stage) { gq[e] = ge; yq[e] = ye; sq[e] = se; }
        }
        ex.bsync();
        const int k = h->ring_count;
        for (int task = ex.warp; task <= k; task += ex.nw) {
            double a0 = 0, a1 = 0, a2 = 0, a3 = 0, a4 = 0;
            if (task < k) {                            // s_p . g, y_p . g, s_p . y, y_p . y, y_p . s
                int p = v.phys(h, task);
                const T *sp_ = v.s(p), *yp_ = v.y(p);
                for (int64_t e = ex.lane; e < n; e += ex.nl) {
                    double ge = stage ? (double)gq[e] : (mask[e] != T(0) ? (double)g[e] : 0.0);
                    double se = sp_[e], ye = yp_[e], yn = yq[e], sn = sq[e];
                    a0 += se * ge; a1 += ye * ge; a2 += se * yn; a3 += ye * yn; a4 += ye * sn;
                }
                a0 = ex.wsum(a0); a1 = ex.wsum(a1); a2 = ex.wsum(a2); a3 = ex.wsum(a3); a4 = ex.wsum(a4);
                if (ex.lane == 0) {
                    v.sg[p] = a0; v.yg[p] = a1;
                    v.sy[p * S + sp] = a2; v.yy[p * S + sp] = a3; v.yy[sp * S + p] = a3; v.sy[sp * S + p] = a4;
                }
            } else {                                   // s . g, y . g, s . y, y . y of the new pair
                for (int64_t e = ex.lane; e < n; e += ex.nl) {
                    double ge = stage ? (double)gq[e] : (mask[e] != T(0) ? (double)g[e] : 0.0);
                    double sn = sq[e], yn = yq[e];
                    a0 += sn * ge; a1 += yn * ge; a2 += sn * yn; a3 += yn * yn;
                }
                a0 = ex.wsum(a0); a1 = ex.wsum(a1); a2 = ex.wsum(a2); a3 = ex.wsum(a3);
                if (ex.lane == 0) { v.sg[sp] = a0; v.yg[sp] = a1; v.sy[sp * S + sp] = a2; v.yy[sp * S + sp] = a3; }
            }
        }
        break;
    }
    case ACT_DIR: {                                    // two-loop on the Gram entries, then d; prev_flat_grad = g
        if (ex.warp == 0) two_loop(ex, h, v);
        ex.bsync();
        const T* g = grad_of(v, h->act_arg, out);
        T *d = v.v(V_D), *pg = v.v(V_PG), *x = v.v(V_X);
        const int k = h->ring_count;
        const double hg = h->hg;
        double gtd = 0, mx = 0;
        for (int64_t e = ex.tid; e < nv; e += ex.nt) {
            bool in = e < n && mask[e] != T(0);
            T ge = in ? g[e] : T(0), de = T(0);
            if (in) {
                double acc = hg * (double)ge;
                for (int i = 0; i < k; ++i) {
                    int p = v.phys(h, i);
                    acc += v.cs[i] * (double)v.s(p)[e] + v.cy[i] * (double)v.y(p)[e];
                }
                de = (T)acc;
            }
            d[e] = de;
            pg[e] = ge;                                // a self-copy when g is prev_flat_grad
            if (c.line_search && e < n) x[e] = params[e];
            gtd += (double)ge * (double)de;
            double a = fabs((double)de);
            mx = nan_max(mx, a);
        }
        gtd = ex.bsum(gtd);
        mx = ex.bmax(mx);
        if (ex.tid == 0) { h->r_dot = gtd; h->r_max = mx; }
        break;
    }
    case ACT_MOVE: {                                   // params = base + t d (base: x, or params in place)
        const T* d = v.v(V_D);
        const T* base = h->act_arg ? v.v(V_X) : params;
        const T tt = (T)h->t;
        for (int64_t e = ex.tid; e < n; e += ex.nt)
            if (mask[e] != T(0)) params[e] = base[e] + tt * d[e];
        break;
    }
    case ACT_LSEVAL: {                                 // copy of the new gradient; g_new . d, max|g_new|
        T* dst = v.v(V_POOL + h->act_arg - REF_POOL);
        const T* d = v.v(V_D);
        double gtd = 0, mx = 0;
        for (int64_t e = ex.tid; e < nv; e += ex.nt) {
            T ge = (e < n && mask[e] != T(0)) ? out[e] : T(0);
            dst[e] = ge;
            gtd += (double)ge * (double)d[e];
            double a = fabs((double)ge);
            mx = nan_max(mx, a);
        }
        gtd = ex.bsum(gtd);
        mx = ex.bmax(mx);
        if (ex.tid == 0) { h->r_dot = gtd; h->r_max = mx; }
        break;
    }
    default:
        break;
    }
}

#if defined(__CUDACC__)
// Reductions of the CTA in a fixed order: lanes by a shuffle tree into lane 0, warps by thread 0 in warp order.
struct CtaExec {
    int tid, nt, lane, nl, warp, nw;
    double* red;                                      // shared [2 * nw]
    __device__ CtaExec(double* red_) : red(red_) {
        tid = threadIdx.x; nt = blockDim.x; lane = tid & 31; nl = 32; warp = tid >> 5; nw = nt >> 5;
    }
    __device__ double wsum(double v) {
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        return __shfl_sync(0xffffffffu, v, 0);
    }
    __device__ double wmax(double v) {
        for (int o = 16; o > 0; o >>= 1) v = nan_max(v, __shfl_down_sync(0xffffffffu, v, o));
        return __shfl_sync(0xffffffffu, v, 0);
    }
    __device__ double block(double v, bool is_max) {
        v = is_max ? wmax(v) : wsum(v);
        __syncthreads();
        if (lane == 0) red[warp] = v;
        __syncthreads();
        if (tid == 0) {
            double a = red[0];
            for (int w = 1; w < nw; ++w) a = is_max ? nan_max(a, red[w]) : a + red[w];
            red[nw] = a;
        }
        __syncthreads();
        return red[nw];
    }
    __device__ double bsum(double v) { return block(v, false); }
    __device__ double bmax(double v) { return block(v, true); }
    __device__ void bsync() { __syncthreads(); }
    __device__ void wsync() { __syncwarp(); }
};
#endif

#if !defined(__CUDACC__)
struct HostExec {
    int tid = 0, nt = 1, lane = 0, nl = 1, warp = 0, nw = 1;
    double wsum(double v) { return v; }
    double bsum(double v) { return v; }
    double bmax(double v) { return v; }
    void bsync() {}
    void wsync() {}
};

// One pinn_lbfgs_advance on one host thread (the host build of the tests): fp64 vectors, the same control and passes.
inline int advance_host(const PinnLbfgs& c, int64_t n, double* params, const double* grads_and_loss, void* state,
                        const double* mask) {
    PinnLbfgsState* h = (PinnLbfgsState*)state;
    View<double> v(state, n, c.history_size);
    HostExec ex;
    for (;;) {
        int a = lbfgs_control(c, h, v.sy, v.yy, grads_and_loss[n], v.S);
        if (a == ACT_DONE) return PINN_LBFGS_DONE;
        lbfgs_pass(ex, c, h, v, n, params, grads_and_loss, mask, (double*)nullptr);
        if (a == ACT_MOVE && h->act_eval) return PINN_LBFGS_EVALUATE;
    }
}
#endif

}  // namespace lbfgs
}  // namespace pinn
