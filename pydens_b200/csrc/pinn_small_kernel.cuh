// pinn_small_kernel.cuh — the fit loop for TINY batches (README example: batch_size = 100, niters = 1500;
// reference pydens/model_torch.py:426-464 including optimizer.step() :461).
//
// At batch 100 the thread-per-point kernel is pure latency: one 32-point tile per warp is one warp walking ~14 000
// dependent instructions (~36 us), whoever launches it — measured: 1500 steps in ONE launch of multi_step_kernel take
// as long as 1500 graph-replayed launches.  Here the work of a step is decomposed the other way round: ONE CTA of 512
// threads, every linear layer is split over (point, output unit) pairs, every weight gradient over (output unit, input
// unit) entries, with __syncthreads between the layers — ~15 short phases per step instead of one long chain.
// Parameters, Adam moments, the stored jets of every level and the gradient live in shared memory for all `k_steps`
// steps of a launch.  Same math as pinn_device.cuh (the jet / activation / ansatz helpers are shared), same Adam as
// multi_step_kernel.
//
// One SM still has to do all of a step's arithmetic, so the batch is further spread over a THREAD-BLOCK CLUSTER of up
// to 8 CTAs (8 SMs): each CTA keeps a full replica of the parameters and Adam state and takes a contiguous slice of the
// points; once per step the CTAs exchange their gradient partials through DISTRIBUTED SHARED MEMORY (every CTA sums
// the 8 partials in rank order, so all replicas apply bit-identical updates) — one cluster barrier per step (the partial
// buffers alternate), nothing leaves the SMs.
//
// Covered: batches of at most 128 points per CTA (1024 per launch), dense chains without residual wiring whose state
// fits shared memory (everything the README / tutorial problems need).  Selected by pinn_multi_step for such batches.
//
// Constraint terms (pinn_multi_step_terms, a.terms): their fixed points are columns n_points .. n_points + a.terms.n_points - 1
// behind the batch, split over the CTAs with it.  Such a column runs the same forward jets; in the residual phase it
// evaluates its term's program on the value channel, with the term's weight and zero seeds on the derivative channels.
//
// The body is three pieces: small_batch (a step's columns), small_gradient (one evaluation, ending in the all-reduce)
// and the optimizer.  The Adam forms below run all three once per step; the L-BFGS form (pinn_small_lbfgs.cuh) runs
// small_gradient once per evaluation of a step.
#pragma once

#include <cooperative_groups.h>
#include "pinn_step_kernel.cuh"

namespace pinn {
namespace small {
namespace cg = cooperative_groups;

constexpr int BP = 128;                 // points (padded)
constexpr int SR = BP + 4;              // row stride of every [row][point] array: rows land 4 banks apart
constexpr int NT = 512;

struct Layout {
    int flat, m1, m2, g, gsum, x, scr, red, lev[PINN_MAX_LAYERS + 2], post[PINN_MAX_LAYERS + 2], total;   // float offsets
};
__host__ __device__ inline Layout make_layout(const DevPlan& P) {
    const int C = 1 + P.nf + P.ns;
    Layout L;
    int o = 0;
    const int np4 = (P.n_params + 3) & ~3;
    L.flat = o; o += np4;
    L.m1 = o; o += np4;
    L.m2 = o; o += np4;
    L.g = o; o += 2 * (np4 + 4);                        // two partial-gradient buffers, alternating by step parity
    L.gsum = o; o += np4 + 4;
    L.x = o; o += PINN_MAX_DIMS * SR;
    L.scr = o; o += P.n_slots * SR;
    L.red = o; o += (2 + PINN_MAX_VARS) * SR;           // per point: loss, d/dlog_scale, d/dV_i
    L.lev[0] = 0; L.post[0] = 0;
    for (int l = 0; l < P.n_layers; ++l) {              // level l+1 = output of layer l, rows (unit, channel)
        L.lev[l + 1] = o; o += P.layer[l].n_out * C * SR;
        // post-activation jets of every hidden level stay too: the forward feeds the next layer from them, the
        // reverse sweep its weight gradients — no recomputation phase, one barrier less per layer
        L.post[l + 1] = o; if (l + 1 < P.n_layers) o += P.layer[l].n_out * C * SR;
    }
    L.total = o;
    return L;
}

// Which columns a CTA of the cluster takes: the batch, then the constraint terms' points, split in contiguous slices
struct Slice {
    int crank, csize;               // rank of this CTA in its cluster, CTAs in the cluster
    int B, base, Bp;                // points of this CTA (may be 0), index of its first column, B rounded up to 4
    int ps_log, PS;                 // item decomposition: point stride PS = 2^ps_log >= Bp
};
__device__ __forceinline__ Slice make_slice(const MultiArgs& a) {
    cg::cluster_group cluster = cg::this_cluster();
    Slice S;
    S.crank = (int)cluster.block_rank(); S.csize = (int)cluster.num_blocks();
    const int n_cols = (int)a.n_points + a.terms.n_points;
    const int q_pts = n_cols / S.csize, r_pts = n_cols % S.csize;
    S.B = q_pts + (S.crank < r_pts ? 1 : 0);
    S.base = S.crank * q_pts + (S.crank < r_pts ? S.crank : r_pts);
    S.Bp = (S.B + 3) & ~3;
    S.ps_log = 2;
    while ((1 << S.ps_log) < S.Bp) ++S.ps_log;
    S.PS = 1 << S.ps_log;
    return S;
}

// The batch of step `step` (the s-th of the launch) into X: coordinates of point p in X[k][p]; padded points replay the
// last one (their adjoint seed is 0).  `mb` holds the fit's explicit batches (or null) and its seed.
template <class MB>
__device__ __forceinline__ void small_batch(const DevPlan& P, const MultiArgs& a, const MB& mb, const Slice& S, float* X,
                                            int s, uint64_t step) {
    if (threadIdx.x < BP && S.B > 0) {
        const int p = threadIdx.x, pe = S.base + (p < S.B ? p : S.B - 1);
        if (pe >= a.n_points) {                                      // a constraint point: fixed, no sampler draw
            for (int k = 0; k < P.total; ++k) X[k * SR + p] = a.terms.x[pe - a.n_points][k];
        } else if (mb.points) {
            const float* src = mb.points + ((size_t)s * a.n_points + (size_t)pe) * P.total;
            for (int k = 0; k < P.total; ++k) X[k * SR + p] = __ldg(src + k);
        } else {
            const uint64_t gidx = (uint64_t)pe;
            const uint32_t c3 = (uint32_t)(((step >> 32) & 0xffffu) << 16);
            Philox4 b0 = philox4x32_10((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)step, c3, (uint32_t)mb.seed, (uint32_t)(mb.seed >> 32));
            Philox4 b1 = b0;
            if (P.total > 4)
                b1 = philox4x32_10((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)step, c3 | 1u, (uint32_t)mb.seed, (uint32_t)(mb.seed >> 32));
            for (int k = 0; k < P.total; ++k) X[k * SR + p] = sample_column(P.cols[k], k, gidx, step, mb.seed, b0, b1);
        }
    }
}

// One evaluation of the objective at the parameters `flat`, on the batch in X and the constraint terms' points:
// [grads | loss] of the whole cluster, summed over its CTAs in rank order, into gsum (the same bits in every CTA).  g is
// this CTA's partial buffer (a peer may still read the other one), zeroed by the caller before a barrier of the CTA.
// Ends with a barrier of the CTA.
template <int NF, int NS>
__device__ __forceinline__ void small_gradient(const DevPlan& P, const MultiArgs& a, const Layout& Y, const Slice& S,
                                               const float* flat, float* g, float* gsum) {
    constexpr int C = 1 + NF + NS;
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x;
    const float* X = smem + Y.x;
    float* scr = smem + Y.scr;
    float* red = smem + Y.red;
    const int Ln = P.n_layers;
    const int n_out_floats = P.n_params + 4;
    cg::cluster_group cluster = cg::this_cluster();
    const int csize = S.csize, B = S.B, base = S.base, Bp = S.Bp, ps_log = S.ps_log, PS = S.PS;
    // ---- forward: layer l over (output unit j, point p) pairs ------------------------------------------------
    for (int l = 0; l < Ln; ++l) {
        const DevLayer& L = P.layer[l];
        float* out = smem + Y.lev[l + 1];
        const float* in_post = smem + Y.post[l];            // post-activation jets of level l (written in the previous pass)
        float* out_post = smem + Y.post[l + 1];
        const ActC kc = make_actc(L.act);
        const float* W = flat + L.w_off;
        for (int i = tid; i < L.n_out * PS; i += NT) {
            const int j = i >> ps_log, p = i & (PS - 1);
            if (p >= Bp) continue;
            float acc[C];
            acc[0] = flat[L.b_off + j];
#pragma unroll
            for (int c = 1; c < C; ++c) acc[c] = 0.0f;
            if (l == 0) {
                for (int k = 0; k < L.n_in; ++k) {
                    const float w = W[j * L.n_in + k];
                    acc[0] = fmaf(w, X[k * SR + p], acc[0]);
#pragma unroll
                    for (int d = 0; d < NF; ++d) acc[1 + d] = fmaf(w, P.dir_vec[d][k], acc[1 + d]);
                }
            } else {
#pragma unroll 4
                for (int m = 0; m < L.n_in; ++m) {
                    const float w = W[j * L.n_in + m];
                    const float* r = in_post + (size_t)m * C * SR + p;
#pragma unroll
                    for (int c = 0; c < C; ++c) acc[c] = fmaf(w, r[c * SR], acc[c]);
                }
            }
            float* row = out + (size_t)j * C * SR + p;
            if (l + 1 < Ln) {
                row[0] = act_store<true>(kc, acc[0]);
#pragma unroll
                for (int c = 1; c < C; ++c) row[c * SR] = acc[c];
                float pj[C];
                load_post_jet<NF, NS, true>(row, SR, kc, pj);
                float* pr = out_post + (size_t)j * C * SR + p;
#pragma unroll
                for (int c = 0; c < C; ++c) pr[c * SR] = pj[c];
            } else {
#pragma unroll
                for (int c = 0; c < C; ++c) row[c * SR] = acc[c];      // the network jet N
            }
        }
        __syncthreads();
    }

    // ---- ansatz, residual, adjoint seed: one thread per point ----------------------------------------------------
    if (tid < Bp) {
        const int p = tid;
        const bool valid = p < B;
        const int q = base + (valid ? p : B - 1);            // its column (a padded one replays the last)
        const DevTerm* term = q >= a.n_points ? &a.terms.t[term_of(a.terms, q - (int)a.n_points)] : nullptr;
        float* nrow = smem + Y.lev[Ln] + p;                  // level Ln: one unit, C channels
        float N[C];
#pragma unroll
        for (int c = 0; c < C; ++c) N[c] = nrow[c * SR];
        const float* coords = X + p;
        float* sc = scr + p;
        float icj[C];
#pragma unroll
        for (int c = 0; c < C; ++c) icj[c] = 0.0f;
        if (P.has_ic) {
            eval_prog(P.ic, P.n_ic, sc, SR, coords, flat, P.var_off);
#pragma unroll
            for (int c = 0; c < C; ++c) icj[c] = sc[(size_t)P.ic_out[c] * SR];
        }
        AnsatzState<NF, NS> as;
        float u[C];
        ansatz_forward<NF, NS, true>(P, coords, SR, flat[P.log_scale_off], N, icj, as, u);
        float ub[C];
        if (term) {
#pragma unroll
            for (int c = 0; c < C; ++c)
                if (c < term->C) sc[(size_t)c * SR] = u[c];         // the channels its program reads
            eval_prog(term->eq, term->n_eq, sc, SR, coords, flat, term->var_off);
            const float r = sc[(size_t)term->eq_out[0] * SR];
            const float rb = valid ? 2.0f * r * term->weight : 0.0f;
            red[0 * SR + p] = valid ? r * term->weight * r : 0.0f;
            PointPartials<NF, NS> part;
#pragma unroll
            for (int i = 0; i < PINN_MAX_VARS; ++i) part.vbar[i] = 0.0f;
            term_seeds<NF, NS>(P, *term, sc, SR, rb, ub, part);
            if (P.ic_has_vars) {
                eval_prog(P.ic, P.n_ic, sc, SR, coords, flat, P.var_off);
                term_ic_partials<NF, NS>(P, *term, sc, SR, ub, part);
            }
#pragma unroll
            for (int i = 0; i < PINN_MAX_VARS; ++i) red[(2 + i) * SR + p] = part.vbar[i];
        } else {
#pragma unroll
            for (int c = 0; c < C; ++c) sc[(size_t)c * SR] = u[c];
            eval_prog(P.eq, P.n_eq, sc, SR, coords, flat, P.var_off);
            const float r = sc[(size_t)P.eq_out[0] * SR];
            const float rb = valid ? 2.0f * r * a.inv_n : 0.0f;
            red[0 * SR + p] = valid ? r * a.inv_n * r : 0.0f;
#pragma unroll
            for (int c = 0; c < C; ++c) ub[c] = rb * sc[(size_t)P.eq_out[1 + c] * SR];
#pragma unroll
            for (int i = 0; i < PINN_MAX_VARS; ++i) {
                float v = 0.0f;
                if (i < P.n_vars) {
                    v = rb * sc[(size_t)P.eq_out[1 + C + i] * SR];
                    if (P.ic_has_vars) {
#pragma unroll
                        for (int c = 0; c < C; ++c) v = fmaf(ub[c], sc[(size_t)P.ic_out[C * (1 + i) + c] * SR], v);
                    }
                }
                red[(2 + i) * SR + p] = v;
            }
        }
        float Nb[C];
        red[1 * SR + p] = ansatz_adjoint<NF, NS>(P, as, ub, Nb);
#pragma unroll
        for (int c = 0; c < C; ++c) nrow[c * SR] = Nb[c];    // in place: the adjoint of the network jet
    }
    __syncthreads();
    if (tid < 2 + PINN_MAX_VARS) {                           // scalars: fixed summation order
        float t = 0.0f;
        for (int p = 0; p < B; ++p) t += red[tid * SR + p];
        if (tid == 0) g[P.n_params] = t;
        else if (tid == 1) g[P.log_scale_off] += t;
        else if (tid - 2 < P.n_vars) g[P.var_off[tid - 2]] += t;
    }

    // ---- reverse: layer l; its output adjoints sit in level l+1 ---------------------------------------------------
    for (int l = Ln - 1; l >= 0; --l) {
        const DevLayer& L = P.layer[l];
        float* dl = smem + Y.lev[l + 1];
        float* cur = smem + Y.lev[l];                        // level l (l >= 1): stored jets, turned into adjoints in place
        const float* W = flat + L.w_off;
        const float* pa = smem + Y.post[l];                  // (a) post-activation jets of level l: kept by the forward sweep
        // (b) weight and bias gradients: entry (j, m), four lanes share the points of an entry
        const int n_e = L.n_out * (L.n_in + 1);
        for (int it = tid; it < ((n_e * 4 + 31) & ~31); it += NT) {
            const int e = it >> 2, sub = it & 3;
            float sum = 0.0f;
            int j = 0, m = 0;
            if (e < n_e) {
                j = e / (L.n_in + 1); m = e - j * (L.n_in + 1);
                const float* dr = dl + (size_t)j * C * SR;
                if (m == L.n_in) {
                    for (int p = sub; p < Bp; p += 4) sum += dr[p];
                } else if (l == 0) {
                    for (int p = sub; p < Bp; p += 4) {
                        float t = dr[p] * X[m * SR + p];
#pragma unroll
                        for (int d = 0; d < NF; ++d) t = fmaf(dr[(1 + d) * SR + p], P.dir_vec[d][m], t);
                        sum += t;
                    }
                } else {
                    const float* ar = pa + (size_t)m * C * SR;
#pragma unroll 4
                    for (int p = sub; p < Bp; p += 4) {
                        float t = 0.0f;
#pragma unroll
                        for (int c = 0; c < C; ++c) t = fmaf(dr[c * SR + p], ar[c * SR + p], t);
                        sum += t;
                    }
                }
            }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            if (e < n_e && sub == 0) g[(m == L.n_in) ? L.b_off + j : L.w_off + j * L.n_in + m] = sum;
        }
        // (c) data gradient through the layer, then through the activation of level l (in place)
        if (l >= 1) {
            const ActC kin = make_actc(P.layer[l - 1].act);
            for (int i = tid; i < L.n_in * PS; i += NT) {
                const int m = i >> ps_log, p = i & (PS - 1);
                if (p >= Bp) continue;
                float ab[C];
#pragma unroll
                for (int c = 0; c < C; ++c) ab[c] = 0.0f;
#pragma unroll 4
                for (int j = 0; j < L.n_out; ++j) {
                    const float w = W[j * L.n_in + m];
                    const float* dr = dl + (size_t)j * C * SR + p;
#pragma unroll
                    for (int c = 0; c < C; ++c) ab[c] = fmaf(w, dr[c * SR], ab[c]);
                }
                float* row = cur + (size_t)m * C * SR + p;
                float pre[C], zb[C];
#pragma unroll
                for (int c = 0; c < C; ++c) pre[c] = row[c * SR];
                const ActD f = act_from_stored(kin, pre[0]);
                act_adjoint<NF, NS>(f, pre, ab, zb);
#pragma unroll
                for (int c = 0; c < C; ++c) row[c * SR] = zb[c];
            }
        }
        __syncthreads();
    }

    // ---- gradient all-reduce over the cluster through distributed shared memory, in rank order ------------------------
    if (csize > 1) {
        cluster.sync();                                      // every CTA's partial [grads | loss] is complete
        for (int i = tid; i < n_out_floats; i += NT) {
            float v[8];                                      // the remote loads go out together, the sum stays in rank order
#pragma unroll
            for (int r = 0; r < 8; ++r) v[r] = (r < csize) ? cluster.map_shared_rank(g, r)[i] : 0.0f;
            float t = 0.0f;
#pragma unroll
            for (int r = 0; r < 8; ++r) t += v[r];
            gsum[i] = t;
        }
    } else {
        for (int i = tid; i < n_out_floats; i += NT) gsum[i] = g[i];
    }
    __syncthreads();
}

// The body of both Adam forms: the fields of `mb` (MultiArgs itself, or one row of the member table) are the fit's own
// state, and those of `hy` (MultiArgs itself, or the member's row of hyper-parameters) its Adam hyper-parameters.
template <int NF, int NS, class MB, class HY>
__device__ __forceinline__ void small_step_body(const DevPlan& P, const MultiArgs& a, const MB& mb, const HY& hy) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x;
    const Layout Y = make_layout(P);
    float* flat = smem + Y.flat;
    float* mom1 = smem + Y.m1;
    float* mom2 = smem + Y.m2;
    const int g_stride = ((P.n_params + 3) & ~3) + 4;
    float* gsum = smem + Y.gsum;
    const Slice S = make_slice(a);
    cg::cluster_group cluster = cg::this_cluster();
    const int crank = S.crank, csize = S.csize;

    for (int i = tid; i < P.n_params; i += NT) { flat[i] = mb.params[i]; mom1[i] = mb.exp_avg[i]; mom2[i] = mb.exp_avg_sq[i]; }
    const unsigned long long step0 = *mb.step_counter;
    __syncthreads();

    for (int s = 0; s < a.k_steps; ++s) {
        small_batch(P, a, mb, S, smem + Y.x, s, step0 + (unsigned long long)s);
        // the partial gradient alternates between two buffers: a CTA that runs ahead into step s+1 never touches the
        // buffer its peers may still be reading for step s, so ONE cluster barrier per step is enough
        float* g = smem + Y.g + (s & 1) * g_stride;
        for (int i = tid; i < P.n_params + 4; i += NT) g[i] = 0.0f;
        // Adam's bias corrections do not depend on the gradient: computed here, off the critical path
        const float t_opt = mb.opt_step0 + (float)(s + 1);
        const float bc1 = 1.0f - powf(hy.beta1, t_opt);
        const float bc2_sqrt = sqrtf(1.0f - powf(hy.beta2, t_opt));
        const float step_size = hy.lr / bc1;
        __syncthreads();
        small_gradient<NF, NS>(P, a, Y, S, flat, g, gsum);
        // ---- Adam (torch.optim.Adam, fused form) on the flat copy ------------------------------------------------------
        {
            for (int i = tid; i < P.n_params; i += NT) {
                if (mb.mask[i] != 0.0f) {
                    float gi = gsum[i];
                    const float pv = flat[i];
                    if (hy.weight_decay != 0.0f) gi = fmaf(hy.weight_decay, pv, gi);
                    const float m1 = fmaf(1.0f - hy.beta1, gi - mom1[i], mom1[i]);
                    const float m2 = fmaf(hy.beta2, mom2[i], (1.0f - hy.beta2) * gi * gi);
                    flat[i] = pv - step_size * m1 / (sqrtf(m2) / bc2_sqrt + hy.eps);
                    mom1[i] = m1; mom2[i] = m2;
                }
            }
            if (tid == 0 && crank == 0) mb.losses_ring[(step0 + (unsigned long long)s) % (unsigned long long)a.ring_len] = gsum[P.n_params];
        }
        __syncthreads();
    }
    if (csize > 1) cluster.sync();                               // every CTA has read the step counter before rank 0 advances it
    if (crank == 0) {                                            // the replicas are bit-identical: rank 0 writes them back
        for (int i = tid; i < P.n_params; i += NT) { mb.params[i] = flat[i]; mb.exp_avg[i] = mom1[i]; mb.exp_avg_sq[i] = mom2[i]; }
        for (int i = tid; i < mb.n_step_tensors; i += NT) mb.step_tensors[i] += (float)a.k_steps;
        if (tid == 0) *mb.step_counter = step0 + (unsigned long long)a.k_steps;
    }
}

template <int NF, int NS>
__global__ void __launch_bounds__(NT, 1) small_step_kernel(const __grid_constant__ DevPlan P, const __grid_constant__ MultiArgs a) {
    small_step_body<NF, NS>(P, a, a, a);
}

// The ensemble form (pinn_multi_step_ensemble_adam): cluster c trains member c of the table with its Adam
// hyper-parameters m.h[c].  Its CTAs exchange their partials with each other only, in rank order, so each member's
// steps are those of its solo launch at the same cluster size.
template <int NF, int NS>
__global__ void __launch_bounds__(NT, 1) small_step_ensemble_kernel(const __grid_constant__ DevPlan P, const __grid_constant__ MultiArgs a,
                                                                    const __grid_constant__ DevMembers m) {
    const unsigned c = blockIdx.x / cg::this_cluster().num_blocks();
    const PinnAdamHyper h = m.h[c];               // once, at entry: not an indexed parameter load per Adam element
    small_step_body<NF, NS>(P, a, m.m[c], h);
}

}  // namespace small
}  // namespace pinn
