// pinn_small_lbfgs.cuh — L-BFGS in the tiny-batch cluster kernel (pinn_lbfgs_multi, pinn_lbfgs_multi_ensemble).
//
// pinn_lbfgs_advance runs the L-BFGS state machine (pinn_lbfgs.cuh) one launch per evaluation of the objective, and the
// host reads a status word after each one to know whether the step goes on.  At batch 100 an evaluation is a few tens of
// microseconds of latency-bound work, so the launches and that read dominate.  Here the whole loop stays in the
// cluster kernel of pinn_small_kernel.cuh: every CTA evaluates its slice of the columns (small_gradient: the same code
// as the Adam form, ending in the rank-ordered DSMEM all-reduce into gsum), then cluster rank 0 runs lbfgs_control and
// lbfgs_pass, unchanged, on 512 threads with its shared-memory parameters as `params` and gsum as `grads_and_loss`.
// When the control asks for an evaluation (an ACT_MOVE with act_eval) or ends the step (ACT_DONE, which logs the loss
// and advances the step counter), the other ranks copy the parameters from rank 0 through DSMEM behind a cluster
// barrier.  The history, the Gram entries and the vectors stay in the state buffer in global memory, in the layout of
// pinn_lbfgs_advance; the header lives in rank 0's shared memory for the launch.
//
// Barriers: the all-reduce's cluster barrier orders every CTA's partial before the sums; the barrier after the control
// orders rank 0's new parameters before the copies.  A CTA reads rank 0's parameters only between that barrier and the
// next all-reduce barrier, and rank 0 changes them only after it: one buffer is enough.
#pragma once

#include "pinn_small_kernel.cuh"
#include "pinn_lbfgs.cuh"

namespace pinn {
namespace small {

template <int NF, int NS>
__device__ __forceinline__ void small_lbfgs_body(const DevPlan& P, const MultiArgs& a, const PinnLbfgs& shared_cfg,
                                                 const PinnLbfgsMember& mb) {
    using namespace lbfgs;
    extern __shared__ __align__(16) float smem[];
    __shared__ PinnLbfgsState h;                    // rank 0: the state header, for the launch
    __shared__ PinnLbfgs c;                         // the fit's settings: shared ones with the member's own
    __shared__ double red[NT / 32 + 1];
    __shared__ int more;                            // rank 0's verdict: 1 = evaluate again, 0 = the step is done
    const int tid = threadIdx.x;
    const Layout Y = make_layout(P);
    float* flat = smem + Y.flat;
    float* gsum = smem + Y.gsum;
    const int g_stride = ((P.n_params + 3) & ~3) + 4;
    const Slice S = make_slice(a);
    cg::cluster_group cluster = cg::this_cluster();
    const View<float> v(mb.state, P.n_params, shared_cfg.history_size);
    CtaExec ex(red);

    for (int i = tid; i < P.n_params; i += NT) flat[i] = mb.params[i];
    if (tid == 0) {
        c = shared_cfg;
        c.lr = mb.lr; c.mask = mb.mask; c.losses_ring = mb.losses_ring; c.step_counter = mb.step_counter;
        if (S.crank == 0) h = *(const PinnLbfgsState*)mb.state;
    }
    // every CTA reads the counter before its first all-reduce barrier; rank 0 advances it only after that barrier
    const unsigned long long step0 = *mb.step_counter;
    __syncthreads();

    int ev = 0;
    for (int s = 0; s < a.k_steps; ++s) {
        small_batch(P, a, mb, S, smem + Y.x, s, step0 + (unsigned long long)s);
        for (;;) {
            float* g = smem + Y.g + (ev++ & 1) * g_stride;
            for (int i = tid; i < P.n_params + 4; i += NT) g[i] = 0.0f;
            __syncthreads();
            small_gradient<NF, NS>(P, a, Y, S, flat, g, gsum);
            if (S.crank == 0) {                     // pinn_lbfgs_advance on this evaluation
                const double loss = (double)gsum[P.n_params];
                for (;;) {
                    if (tid == 0) lbfgs_control(c, &h, v.sy, v.yy, loss, v.S);
                    __syncthreads();
                    const int act = h.action, eval = h.act_eval;
                    if (act == ACT_DONE) break;
                    lbfgs_pass(ex, c, &h, v, (int64_t)P.n_params, flat, gsum, c.mask, (float*)nullptr);
                    __syncthreads();
                    if (act == ACT_MOVE && eval) break;
                }
                if (tid == 0) more = h.action != ACT_DONE;
            }
            if (S.csize > 1) {
                cluster.sync();                     // rank 0's parameters and verdict are final
                if (S.crank != 0) {
                    const float* src = cluster.map_shared_rank(flat, 0);
                    for (int i = tid; i < P.n_params; i += NT) flat[i] = src[i];
                    if (tid == 0) more = *cluster.map_shared_rank(&more, 0);
                }
            }
            __syncthreads();
            if (!more) break;
        }
    }
    if (S.csize > 1) cluster.sync();                // no CTA leaves while a peer may still read its shared memory
    if (S.crank == 0) {
        for (int i = tid; i < P.n_params; i += NT) mb.params[i] = flat[i];
        if (tid == 0) *(PinnLbfgsState*)mb.state = h;
    }
}

// Cluster c trains member c of the table (a solo fit: a table of one).  Its CTAs exchange partials and parameters with
// each other only, so each member's steps are those of its solo launch at the same cluster size.
template <int NF, int NS>
__global__ void __launch_bounds__(NT, 1) small_lbfgs_kernel(const __grid_constant__ DevPlan P, const __grid_constant__ MultiArgs a,
                                                            const __grid_constant__ DevLbfgsMembers m) {
    const unsigned c = blockIdx.x / cg::this_cluster().num_blocks();
    small_lbfgs_body<NF, NS>(P, a, m.cfg, m.m[c]);
}

}  // namespace small
}  // namespace pinn
