// pinn_hi_kernel.cuh — the fit-step kernel for derivatives of order 3 / 4 (per-point math: pinn_device_hi.cuh).
//
// Same skeleton as step_kernel (pinn_step_kernel.cuh), of which it reuses every shared piece — the TMA staging of the
// parameters, the in-kernel Philox sampler, the per-warp gradient accumulators, the deterministic grid fold with the
// NVLink all-reduce, Adam and the loss log in its tail: one thread per point, persistent grid of one CTA per SM,
// per-point state (1 + NF*K jet channels per unit) in the per-warp global area.
#pragma once

#include "pinn_step_kernel.cuh"
#include "pinn_device_hi.cuh"

namespace pinn {
namespace hi {

template <int NF, int K>
__global__ void __launch_bounds__(256, 1) hi_step_kernel(const __grid_constant__ DevPlan P, const StepArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int n_out_floats = P.n_params + 4;
    const SmemLayout SL = smem_layout(P.weights_floats, n_out_floats, a.wacc ? 0 : nwarps, P.n_params);
    stage_weights(smem, SL, P, a.params);
    const float* sw = smem + SL.weights_f;
    float* wacc_all = warp_accumulators(a, smem, SL, n_out_floats, nwarps);

    GradSink sink;
    sink.wacc = wacc_all + warp * n_out_floats;
    sink.dump = P.n_params + 2;

    const long long gw = (long long)blockIdx.x * nwarps + warp;
    const long long total_warps = (long long)gridDim.x * nwarps;
    float* st = a.spill + (size_t)gw * a.rows_total * RS + lane;

    const uint64_t step = a.step_ptr ? *a.step_ptr : a.step_val;
    const long long n_tiles = (a.n_points + 31) / 32;
    PartialsHi part;
    part.loss = 0.0f; part.sbar = 0.0f;
#pragma unroll
    for (int i = 0; i < PINN_MAX_VARS; ++i) part.vbar[i] = 0.0f;

    for (long long tile = (long long)warp * gridDim.x + blockIdx.x; tile < n_tiles; tile += total_warps) {
        const long long pl = tile * 32 + lane;
        const bool valid = pl < a.n_points;
        const long long pe = valid ? pl : a.n_points - 1;     // masked lanes replay the last point
        if (a.points) {
            const float* src = a.points + (size_t)pe * P.total;
            for (int k = 0; k < P.total; ++k) st[k * RS] = __ldg(src + k);
        } else {
            const uint64_t gidx = a.point_offset + (uint64_t)pe;
            Philox4 b0 = philox_block(gidx, step, a.seed, 0u);
            Philox4 b1 = b0;
            if (P.total > 4) b1 = philox_block(gidx, step, a.seed, 1u);
            for (int k = 0; k < P.total; ++k) st[k * RS] = sample_column(P.cols[k], k, gidx, step, a.seed, b0, b1);
        }
        float r = point_step<NF, K>(P, sw, a.params, st, RS, valid, a.inv_n, sink, part);
        if (a.residual && valid) a.residual[pl] = r;
    }

    {
        float v = warp_sum(part.loss);
        if (lane == 0) sink.add(P.n_params, v);
        v = warp_sum(part.sbar);
        if (lane == 0) sink.add(P.log_scale_off, v);
#pragma unroll
        for (int i = 0; i < PINN_MAX_VARS; ++i) {
            if (i < P.n_vars) {
                float t = warp_sum(part.vbar[i]);
                if (lane == 0) sink.add(P.var_off[i], t);
            }
        }
    }
    __syncthreads();

    cta_partial(a, wacc_all, n_out_floats, nwarps);
    finish_grid(a, n_out_floats);
}

}  // namespace hi
}  // namespace pinn
