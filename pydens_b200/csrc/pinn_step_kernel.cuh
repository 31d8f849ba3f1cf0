// pinn_step_kernel.cuh — the fused fit-step kernel template and its shared-memory staging helpers.
// Included by pinn_kernels.cu (host API, forward/sampling kernels) and by the build units of
// pinn_instances.cu, which instantiate the kernels so the build can run in parallel.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include "pinn_device.cuh"

#ifndef PINN_COMM_MAX_RANKS
#define PINN_COMM_MAX_RANKS 8
#endif

namespace pinn {

constexpr int RS = 32;                    // row stride of per-point storage: one warp tile

struct StepArgs {
    const float* params;
    const float* points;
    uint64_t seed;
    const uint64_t* step_ptr;
    uint64_t step_val;
    uint64_t point_offset;
    long long n_points;
    float inv_n;
    float* out;
    float* residual;
    float* partials;
    unsigned int* ticket;
    float* spill;
    float* wacc;                           // per-warp gradient accumulators in the workspace [grid][warps][n_out_floats],
                                           // or nullptr: in shared memory
    int rows_total;
    // in-kernel all-reduce over NVLink peer memory (comm_world == 0: off)
    char* comm_peers[PINN_COMM_MAX_RANKS]; // exchange buffer of every rank, mapped through CUDA IPC
    int comm_rank, comm_world;
    long long comm_timeout;                // clock64 ticks a rank waits for its peers before poisoning the step
    // optimizer.step() fused into the tail of the step (pinn_step_adam; adam_m == nullptr: off): torch.optim.Adam on
    // the flat parameter vector, state shared with the torch optimizer object (its state tensors are views of these)
    float* adam_m;                         // exp_avg [n_params]
    float* adam_v;                         // exp_avg_sq [n_params]
    const float* adam_mask;                // 1 = trainable
    float* adam_steps;                     // the optimizer's per-parameter step counters (float, device), each += 1
    int adam_n_steps;
    float adam_lr, adam_beta1, adam_beta2, adam_eps, adam_wd;
    float* ring;                           // loss log: ring[step % ring_len] = loss, then the step counter += 1
    long long ring_len;
};

// Layout of one rank's exchange buffer (pinn_comm_create): epoch counter, arrival flags, slots.
constexpr int PINN_COMM_FLAGS_OFF = 256;
constexpr int PINN_COMM_SLOTS_OFF = 1024;
__host__ __device__ inline size_t comm_slot_floats(int n_out_floats) { return (size_t)((n_out_floats + 31) & ~31); }
// Small vectors travel in the "LL" form: every float rides in an 8-byte word next to the epoch it belongs to, so a
// word validates itself — no fence, no separate flag, ONE NVLink traversal between the last fold and the sum.
constexpr int PINN_COMM_LL_MAX_FLOATS = 4096;
__host__ __device__ inline bool comm_uses_ll(int n_out_floats) { return n_out_floats <= PINN_COMM_LL_MAX_FLOATS; }
__host__ __device__ inline size_t comm_bytes(int n_out_floats, int world) {
    const size_t per_float = comm_uses_ll(n_out_floats) ? 2 * sizeof(float) : sizeof(float);
    return PINN_COMM_SLOTS_OFF + 2 * (size_t)world * comm_slot_floats(n_out_floats) * per_float;
}
// one 8-byte SCALAR access each way: value in the low word, epoch in the high word (single-copy atomic)
__device__ __forceinline__ void st_relaxed_sys_v2(unsigned long long* p, unsigned int lo, unsigned int hi) {
    const unsigned long long w = (unsigned long long)lo | ((unsigned long long)hi << 32);
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ void ld_relaxed_sys_v2(const unsigned long long* p, unsigned int& lo, unsigned int& hi) {
    unsigned long long w;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
    lo = (unsigned int)w; hi = (unsigned int)(w >> 32);
}

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}


struct FwdArgs {
    const float* params;
    const float* points;
    long long n_points;
    float* u_out;
    float* spill;
    int rows_total;
    int row_scr;
};

// ---- PTX helpers: mbarrier + 1-D TMA bulk copy (global -> shared) ---------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// Shared-memory carve-up (in floats) common to both kernels.
struct SmemLayout {
    int weights_f, wacc_f, bar_f, storage_f, total_f;
};
__host__ __device__ inline int align4(int x) { return (x + 3) & ~3; }
__host__ __device__ inline SmemLayout smem_layout(int weights_floats, int n_out_floats, int n_wacc,
                                                  int storage_floats) {
    SmemLayout L;
    L.weights_f = 0;
    L.wacc_f = L.weights_f + align4(weights_floats);
    L.bar_f = L.wacc_f + align4(n_out_floats * n_wacc);
    L.storage_f = L.bar_f + 4;
    L.total_f = L.storage_f + align4(storage_floats);
    return L;
}

// Stage the parameters into shared memory: one TMA bulk copy of the flat buffer, then a re-layout
// into the padded forward / reverse weight matrices.  Returns with __syncthreads() done.
// The plan itself is a __grid_constant__ kernel parameter: every loop bound and program word is read
// through the constant bank, i.e. provably warp-uniform.
__device__ __forceinline__ void stage_weights(float* smem, const SmemLayout& SL, const DevPlan& P,
                                              const float* params) {
    const int tid = threadIdx.x, nt = blockDim.x;
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + SL.bar_f);
    if (tid == 0) mbar_init(bar, 1);
    __syncthreads();
    float* stage = smem + SL.storage_f;           // parameters land here first
    if (tid == 0) {
        uint32_t bytes = (uint32_t)P.n_params * 4u;
        mbar_expect_tx(bar, bytes);
        tma_bulk_g2s(stage, params, bytes, bar);
    }
    float* sw = smem + SL.weights_f;
    for (int i = tid; i < P.weights_floats; i += nt) sw[i] = 0.0f;
    mbar_wait(bar, 0);
    __syncthreads();
    for (int l = 0; l < P.n_layers; ++l) {
        const DevLayer& L = P.layer[l];
        const int n = L.n_in * L.n_out;
        for (int i = tid; i < n; i += nt) {
            int j = i / L.n_in, k = i - j * L.n_in;
            float w = stage[L.w_off + i];
            sw[L.wt_s + k * L.n_out_p4 + j] = w;
            sw[L.w_s + j * L.n_in_p8 + k] = w;
        }
        for (int j = tid; j < L.n_out; j += nt) sw[L.b_s + j] = stage[L.b_off + j];
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// Grid tail shared by every step kernel: the CTA has written its partial [n_out_floats] to
// a.partials[blockIdx.x]; the last CTA to arrive (ticket) folds all partials in block order and — in
// data-parallel runs — exchanges the folded vector with the peers over NVLink.
// ---------------------------------------------------------------------------------------------------
constexpr int FOLD_GROUP = 12;           // CTAs per first-level fold group (148 CTAs -> 13 groups)

// sum of `n` partial vectors (stride n_out_floats) at element i, fixed order, four loads in flight
__device__ __forceinline__ float fold_column(const float* __restrict__ src, int n, int n_out_floats) {
    float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
    int b = 0;
    for (; b + 3 < n; b += 4) {
        s0 += __ldcg(src + (size_t)(b + 0) * n_out_floats);
        s1 += __ldcg(src + (size_t)(b + 1) * n_out_floats);
        s2 += __ldcg(src + (size_t)(b + 2) * n_out_floats);
        s3 += __ldcg(src + (size_t)(b + 3) * n_out_floats);
    }
    for (; b < n; ++b) s0 += __ldcg(src + (size_t)b * n_out_floats);
    return (s0 + s1) + (s2 + s3);
}

// Programmatic dependent launch: consecutive steps are launched with programmatic stream serialization, so the CTAs of
// step s+1 are placed on the SMs as the CTAs of step s drain (fold, all-reduce and Adam run in ONE last CTA) instead
// of after the whole grid has retired.  pdl_wait() blocks until the previous grid has completed and its writes
// (parameters, step counter, ticket words) are visible; without the launch attribute both are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// optimizer.step() (reference model_torch.py:461) inside the step kernel: torch.optim.Adam's update, element by element,
// applied by the thread that has just produced the reduced gradient element.
struct AdamHyper { float step_size, bc2_sqrt; };
struct AdamPre { float mk, m0, v0, pv; };
__device__ __forceinline__ AdamHyper adam_hyper(const StepArgs& a) {
    AdamHyper h;
    h.step_size = 0.0f; h.bc2_sqrt = 1.0f;
    if (a.adam_m) {
        float t = 0.0f;
        for (int i = 0; i < a.adam_n_steps; ++i) t = fmaxf(t, a.adam_steps[i]);
        t += 1.0f;
        h.step_size = a.adam_lr / (1.0f - powf(a.adam_beta1, t));
        h.bc2_sqrt = sqrtf(1.0f - powf(a.adam_beta2, t));
    }
    return h;
}
// the state of element i: loaded BEFORE the gradient element is folded / waited for, so that the latencies overlap
__device__ __forceinline__ AdamPre adam_load(const StepArgs& a, int i, int n_params) {
    AdamPre q;
    q.mk = 0.0f; q.m0 = 0.0f; q.v0 = 0.0f; q.pv = 0.0f;
    if (a.adam_m && i < n_params) { q.mk = a.adam_mask[i]; q.m0 = a.adam_m[i]; q.v0 = a.adam_v[i]; q.pv = a.params[i]; }
    return q;
}
__device__ __forceinline__ void adam_apply(const StepArgs& a, int i, float g, const AdamPre& q, const AdamHyper& h,
                                           int n_params) {
    if (a.adam_m && i == n_params && a.step_ptr) {
        // element n_params is the loss: `losses.append` (:464) and the step counter, by the thread that produced it
        // (every CTA read the counter when it started; the next launch is stream-ordered)
        const unsigned long long s = *a.step_ptr;
        if (a.ring) a.ring[s % (unsigned long long)a.ring_len] = g;
        *const_cast<unsigned long long*>(reinterpret_cast<const unsigned long long*>(a.step_ptr)) = s + 1ull;
    }
    if (q.mk != 0.0f) {
        if (a.adam_wd != 0.0f) g = fmaf(a.adam_wd, q.pv, g);
        const float m1 = fmaf(1.0f - a.adam_beta1, g - q.m0, q.m0);
        const float m2 = fmaf(a.adam_beta2, q.v0, (1.0f - a.adam_beta2) * g * g);
        const_cast<float*>(a.params)[i] = q.pv - h.step_size * m1 / (sqrtf(m2) / h.bc2_sqrt + a.adam_eps);
        a.adam_m[i] = m1; a.adam_v[i] = m2;
    }
}

__device__ __forceinline__ void finish_grid(const StepArgs& a, const int n_out_floats) {
    const int tid = threadIdx.x;
    // Two-level fold, fixed order: the last CTA of every group of FOLD_GROUP consecutive CTAs sums its group into
    // the group's first slot; the last GROUP to finish sums the group results.  (One CTA folding all 148 partials
    // was a 7 us serial tail at cfg2 and > 100 us for a 51 KB gradient vector.)
    const int n_groups = ((int)gridDim.x + FOLD_GROUP - 1) / FOLD_GROUP;
    const int group = (int)blockIdx.x / FOLD_GROUP;
    const int n_params = n_out_floats - 4;
    const AdamHyper hy = adam_hyper(a);          // bias corrections: every CTA, before it knows whether it is the last
    const int g_first = group * FOLD_GROUP;
    const int g_size = min(FOLD_GROUP, (int)gridDim.x - g_first);
    __threadfence();
    __syncthreads();
    __shared__ unsigned int s_last;
    if (tid == 0) {
        unsigned int t = atomicAdd(a.ticket + 1 + group, 1u);
        s_last = (t == (unsigned int)g_size - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (n_groups > 1) {
        float* gdst = a.partials + (size_t)g_first * n_out_floats;
        for (int i = tid; i < n_out_floats; i += blockDim.x) {
            const float t = fold_column(a.partials + (size_t)g_first * n_out_floats + i, g_size, n_out_floats);
            gdst[i] = t;                                 // this thread read every partial's element i before writing it
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            a.ticket[1 + group] = 0u;
            unsigned int t = atomicAdd(a.ticket, 1u);
            s_last = (t == (unsigned int)n_groups - 1) ? 1u : 0u;
        }
        __syncthreads();
        if (!s_last) return;
        __threadfence();
    } else if (tid == 0) {
        a.ticket[1] = 0u;
    }
    const int n_fold = (n_groups > 1) ? n_groups : g_size;
    const size_t fold_stride = (n_groups > 1) ? (size_t)FOLD_GROUP * n_out_floats : (size_t)n_out_floats;
    {
        // --- data-parallel runs: the all-reduce of [grads | loss] happens right here, over NVLink peer
        // memory.  This rank's folded vector is stored into its slot in EVERY rank's exchange buffer, an
        // arrival flag follows (release, system scope), and once all flags of this epoch are in, every
        // rank sums the slots in rank order — identical bits everywhere, no second kernel, no NCCL call.
        // Slots and flags are double-buffered by epoch parity: a rank can be at most one step ahead.
        __shared__ unsigned int s_epoch;
        __shared__ int s_timeout;
        if (tid == 0) s_timeout = 0;
        float* slot_base = nullptr;
        unsigned int epoch = 0;
        int par = 0;
        const size_t slot_f = comm_slot_floats(n_out_floats);
        if (a.comm_world > 1) {
            if (tid == 0) {
                unsigned int* ep = reinterpret_cast<unsigned int*>(a.comm_peers[a.comm_rank]);
                s_epoch = *ep + 1u;
                *ep = s_epoch;
            }
            __syncthreads();
            epoch = s_epoch;
            par = (int)(epoch & 1u);
            slot_base = reinterpret_cast<float*>(a.comm_peers[a.comm_rank] + PINN_COMM_SLOTS_OFF);
        }
        const bool ll = a.comm_world > 1 && comm_uses_ll(n_out_floats);
        for (int i = tid; i < n_out_floats; i += blockDim.x) {
            const AdamPre pre = (a.comm_world > 1) ? AdamPre{0.0f, 0.0f, 0.0f, 0.0f} : adam_load(a, i, n_params);
            // partial vectors to fold: the group results (stride FOLD_GROUP slots), or the CTAs of the only group
            float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
            int b = 0;
            const float* src = a.partials + i;
            for (; b + 3 < n_fold; b += 4) {
                s0 += __ldcg(src + (size_t)(b + 0) * fold_stride);
                s1 += __ldcg(src + (size_t)(b + 1) * fold_stride);
                s2 += __ldcg(src + (size_t)(b + 2) * fold_stride);
                s3 += __ldcg(src + (size_t)(b + 3) * fold_stride);
            }
            for (; b < n_fold; ++b) s0 += __ldcg(src + (size_t)b * fold_stride);
            const float total = (s0 + s1) + (s2 + s3);
            if (ll) {
                for (int r = 0; r < a.comm_world; ++r) {       // peer stores over NVLink: (value, epoch) in one 8-byte word
                    unsigned long long* dst = reinterpret_cast<unsigned long long*>(a.comm_peers[r] + PINN_COMM_SLOTS_OFF) +
                                              ((size_t)par * a.comm_world + a.comm_rank) * slot_f;
                    st_relaxed_sys_v2(dst + i, __float_as_uint(total), epoch);
                }
            } else if (a.comm_world > 1) {
                for (int r = 0; r < a.comm_world; ++r) {       // peer stores over NVLink
                    float* dst = reinterpret_cast<float*>(a.comm_peers[r] + PINN_COMM_SLOTS_OFF) +
                                 ((size_t)par * a.comm_world + a.comm_rank) * slot_f;
                    dst[i] = total;
                }
            } else {
                a.out[i] = total;
                adam_apply(a, i, total, pre, hy, n_params);
            }
        }
        if (ll) {
            // every word carries its epoch: spin on the data itself, sum in rank order (bit-identical on every rank)
            const unsigned long long* slots = reinterpret_cast<const unsigned long long*>(a.comm_peers[a.comm_rank] + PINN_COMM_SLOTS_OFF) +
                                              (size_t)par * a.comm_world * slot_f;
            volatile unsigned int* aborted = reinterpret_cast<volatile unsigned int*>(a.comm_peers[a.comm_rank]) + 1;
            for (int i = tid; i < n_out_floats; i += blockDim.x) {
                const AdamPre pre = adam_load(a, i, n_params);
                float sum = 0.0f;
                bool dead = false;
                for (int r = 0; r < a.comm_world; ++r) {
                    unsigned int lo, hi;
                    ld_relaxed_sys_v2(slots + (size_t)r * slot_f + i, lo, hi);
                    if (hi != epoch) {
                        const long long t0 = clock64();
                        do {
                            if (*aborted || clock64() - t0 > a.comm_timeout) { *aborted = 1u; dead = true; break; }
                            ld_relaxed_sys_v2(slots + (size_t)r * slot_f + i, lo, hi);
                        } while (hi != epoch);
                    }
                    sum += __uint_as_float(lo);
                }
                const float val = dead ? __int_as_float(0x7fc00000) : sum;
                a.out[i] = val;
                adam_apply(a, i, val, pre, hy, n_params);
            }
        } else if (a.comm_world > 1) {
            __threadfence_system();
            __syncthreads();
            if (tid < a.comm_world) {
                unsigned int* flag = reinterpret_cast<unsigned int*>(a.comm_peers[tid] + PINN_COMM_FLAGS_OFF) +
                                     par * PINN_COMM_MAX_RANKS + a.comm_rank;
                st_release_sys(flag, epoch);
                const unsigned int* mine_f = reinterpret_cast<const unsigned int*>(a.comm_peers[a.comm_rank] + PINN_COMM_FLAGS_OFF) +
                                             par * PINN_COMM_MAX_RANKS + tid;
                // a peer that never arrives (crashed rank) must not hang the GPU: give up after the time limit, and make
                // that sticky (word 1 of the local buffer) so that the remaining steps fail fast
                volatile unsigned int* aborted = reinterpret_cast<volatile unsigned int*>(a.comm_peers[a.comm_rank]) + 1;
                const long long t0 = clock64();
                while (ld_acquire_sys(mine_f) != epoch) {
                    if (*aborted || clock64() - t0 > a.comm_timeout) { *aborted = 1u; s_timeout = 1; break; }
                }
            }
            __syncthreads();
            const float* slots = slot_base + (size_t)par * a.comm_world * slot_f;
            for (int i = tid; i < n_out_floats; i += blockDim.x) {
                const AdamPre pre = adam_load(a, i, n_params);
                float s = 0.0f;
                for (int r = 0; r < a.comm_world; ++r) s += __ldcv(slots + (size_t)r * slot_f + i);
                const float val = s_timeout ? __int_as_float(0x7fc00000) : s;   // poison instead of hanging
                a.out[i] = val;
                adam_apply(a, i, val, pre, hy, n_params);
            }
        }
        if (tid == 0) *a.ticket = 0u;
        // optimizer.step() (:461) happened element by element above (adam_apply), by the CTA that holds the reduced
        // gradient: every other CTA of this launch has finished (it took its ticket after its last read of the
        // parameters), the next launch is stream-ordered.  Left: the optimizer's step counters (every thread of this
        // CTA read them in adam_hyper, before the barriers above).
        if (a.adam_m && tid < a.adam_n_steps) a.adam_steps[tid] += 1.0f;
    }
}

// The gradient accumulators of a step: one per warp, [warps][n_out_floats], zeroed.  In shared memory behind the
// weights, or, when the placement left no room there (a.wacc set), in this CTA's slice of the workspace.  Every warp
// adds into its own accumulator only, and cta_partial sums them in warp order: the result does not depend on timing.
__device__ __forceinline__ float* warp_accumulators(const StepArgs& a, float* smem, const SmemLayout& SL,
                                                    int n_out_floats, int nwarps) {
    float* w = a.wacc ? a.wacc + (size_t)blockIdx.x * nwarps * n_out_floats : smem + SL.wacc_f;
    for (int i = threadIdx.x; i < n_out_floats * nwarps; i += blockDim.x) w[i] = 0.0f;
    __syncthreads();
    return w;
}
// The CTA's partial [n_out_floats] -> a.partials[blockIdx.x]: the warps' accumulators summed in warp order.
__device__ __forceinline__ void cta_partial(const StepArgs& a, const float* wacc_all, int n_out_floats, int nwarps) {
    float* mine = a.partials + (size_t)blockIdx.x * n_out_floats;
    for (int i = threadIdx.x; i < n_out_floats; i += blockDim.x) {
        float s = 0.0f;
        for (int w = 0; w < nwarps; ++w) s += wacc_all[w * n_out_floats + i];
        mine[i] = s;
    }
}

// ---------------------------------------------------------------------------------------------------
// The fit-step kernel.
// ---------------------------------------------------------------------------------------------------
template <int NF, int NS, bool GMEM, int MAXT, int JF, bool GEN>
__global__ void __launch_bounds__(MAXT, 1) step_kernel(const __grid_constant__ DevPlan P, const StepArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;

    const int n_out_floats = P.n_params + 4;
    const SmemLayout SL = smem_layout(P.weights_floats, n_out_floats, a.wacc ? 0 : nwarps,
                                      GMEM ? P.n_params : max(P.n_params, a.rows_total * RS * nwarps));
    pdl_wait();                                    // the previous step (its parameter update) is complete and visible
    pdl_launch_dependents();                       // the next step's CTAs may take the SMs as ours leave them
    stage_weights(smem, SL, P, a.params);
    const float* sw = smem + SL.weights_f;
    float* wacc_all = warp_accumulators(a, smem, SL, n_out_floats, nwarps);

    GradSink sink;
    sink.wacc = wacc_all + warp * n_out_floats;
    sink.dump = P.n_params + 2;                    // spare float behind the loss slot

    const long long gw = (long long)blockIdx.x * nwarps + warp;         // global warp id
    const long long total_warps = (long long)gridDim.x * nwarps;
    float* st = (GMEM ? a.spill + (size_t)gw * a.rows_total * RS : smem + SL.storage_f + (size_t)warp * a.rows_total * RS) + lane;

    const uint64_t step = a.step_ptr ? *a.step_ptr : a.step_val;
    const long long n_tiles = (a.n_points + 31) / 32;
    PointPartials<NF, NS> part;
    part.loss = 0.0f; part.sbar = 0.0f;
#pragma unroll
    for (int i = 0; i < PINN_MAX_VARS; ++i) part.vbar[i] = 0.0f;

    // tiles are dealt warp-slot-major (slot w of every CTA before slot w+1 of any): the last, partial round of tiles
    // spreads over all SMs instead of filling the first CTAs and leaving the others idle
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
        float r = point_step<NF, NS, JF, GEN>(P, sw, a.params, st, RS, valid, a.inv_n, sink, part);
        if (a.residual && valid) a.residual[pl] = r;
    }

    // per-thread scalars -> accumulator
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

    // CTA partial -> global, then the last CTA folds all partials in block order
    cta_partial(a, wacc_all, n_out_floats, nwarps);
    finish_grid(a, n_out_floats);
}


// ---------------------------------------------------------------------------------------------------
// Persistent multi-step kernel for the small-batch regime (README example: batch 100 x 1500 iterations,
// reference loop pydens/model_torch.py:426-464 INCLUDING optimizer.step() :461): ONE CTA runs `k_steps`
// whole optimizer steps per launch.  Parameters, Adam moments and the gradient live in shared memory
// between the steps; every step is  sample / read points -> forward jets -> residual -> reverse ->
// CTA-wide fixed-order reduction -> Adam (torch.optim.Adam semantics, fused/capturable form) -> re-layout
// of the weights, with no launch and no trip to global memory in between.  Opt-in:
// Solver.fit(..., steps_per_launch=k).
// ---------------------------------------------------------------------------------------------------
struct MultiArgs {
    float* params;                 // [n_params] in/out
    float* exp_avg;                // [n_params] in/out (Adam first moment)
    float* exp_avg_sq;             // [n_params] in/out (Adam second moment)
    const float* mask;             // [n_params] 1 = trainable (requires_grad), 0 = frozen
    float* step_tensors;           // [n_step_tensors] the optimizer's per-parameter step counters (float), += k_steps
    int n_step_tensors;
    const float* points;           // [k_steps][n_points][total] explicit batches, or nullptr: sample in-kernel
    uint64_t seed;
    unsigned long long* step_counter;   // device step number (Philox counter word, ring index); += k_steps
    long long n_points;
    float inv_n;
    int k_steps;
    float lr, beta1, beta2, eps, weight_decay;
    float opt_step0;               // optimizer steps taken before this launch
    float* losses_ring;
    long long ring_len;
    int rows_total;
};

template <int NF, int NS, int MAXT, int JF>
__global__ void __launch_bounds__(MAXT, 1) multi_step_kernel(const __grid_constant__ DevPlan P, const MultiArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int n_out_floats = P.n_params + 4;
    const int storage_f = max(P.n_params, a.rows_total * RS * nwarps);
    const SmemLayout SL = smem_layout(P.weights_floats, n_out_floats, nwarps, storage_f);
    // behind the single-step layout: flat parameters, both Adam moments, the folded gradient
    float* flat = smem + SL.total_f;
    float* mom1 = flat + align4(P.n_params);
    float* mom2 = mom1 + align4(P.n_params);
    float* gsum = mom2 + align4(P.n_params);
    stage_weights(smem, SL, P, a.params);
    float* sw = smem + SL.weights_f;
    float* wacc_all = smem + SL.wacc_f;
    for (int i = tid; i < P.n_params; i += blockDim.x) {
        flat[i] = a.params[i]; mom1[i] = a.exp_avg[i]; mom2[i] = a.exp_avg_sq[i];
    }
    __syncthreads();

    GradSink sink;
    sink.wacc = wacc_all + warp * n_out_floats;
    sink.dump = P.n_params + 2;
    float* st = smem + SL.storage_f + (size_t)warp * a.rows_total * RS + lane;
    const unsigned long long step0 = *a.step_counter;
    const long long n_tiles = (a.n_points + 31) / 32;

    for (int s = 0; s < a.k_steps; ++s) {
        for (int i = tid; i < n_out_floats * nwarps; i += blockDim.x) wacc_all[i] = 0.0f;
        __syncthreads();
        const uint64_t step = step0 + (unsigned long long)s;
        PointPartials<NF, NS> part;
        part.loss = 0.0f; part.sbar = 0.0f;
#pragma unroll
        for (int i = 0; i < PINN_MAX_VARS; ++i) part.vbar[i] = 0.0f;
        for (long long tile = warp; tile < n_tiles; tile += nwarps) {
            const long long pl = tile * 32 + lane;
            const bool valid = pl < a.n_points;
            const long long pe = valid ? pl : a.n_points - 1;
            if (a.points) {
                const float* src = a.points + ((size_t)s * a.n_points + (size_t)pe) * P.total;
                for (int k = 0; k < P.total; ++k) st[k * RS] = __ldg(src + k);
            } else {
                const uint64_t gidx = (uint64_t)pe;
                Philox4 b0 = philox_block(gidx, step, a.seed, 0u);
                Philox4 b1 = b0;
                if (P.total > 4) b1 = philox_block(gidx, step, a.seed, 1u);
                for (int k = 0; k < P.total; ++k) st[k * RS] = sample_column(P.cols[k], k, gidx, step, a.seed, b0, b1);
            }
            point_step<NF, NS, JF, true>(P, sw, flat, st, RS, valid, a.inv_n, sink, part);
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
        // fold the warps in warp order, then Adam on the flat copy
        const float t_opt = a.opt_step0 + (float)(s + 1);
        const float bc1 = 1.0f - powf(a.beta1, t_opt);
        const float bc2_sqrt = sqrtf(1.0f - powf(a.beta2, t_opt));
        const float step_size = a.lr / bc1;
        for (int i = tid; i < n_out_floats; i += blockDim.x) {
            float g = 0.0f;
            for (int w = 0; w < nwarps; ++w) g += wacc_all[w * n_out_floats + i];
            gsum[i] = g;
            if (i < P.n_params && a.mask[i] != 0.0f) {
                float pv = flat[i];
                if (a.weight_decay != 0.0f) g = fmaf(a.weight_decay, pv, g);
                const float m1 = fmaf(1.0f - a.beta1, g - mom1[i], mom1[i]);
                const float m2 = fmaf(a.beta2, mom2[i], (1.0f - a.beta2) * g * g);
                const float denom = sqrtf(m2) / bc2_sqrt + a.eps;
                flat[i] = pv - step_size * m1 / denom;
                mom1[i] = m1; mom2[i] = m2;
            }
        }
        __syncthreads();
        if (tid == 0) a.losses_ring[(step0 + (unsigned long long)s) % (unsigned long long)a.ring_len] = gsum[P.n_params];
        // the new parameters in both weight layouts (what stage_weights does after its TMA copy)
        for (int l = 0; l < P.n_layers; ++l) {
            const DevLayer& L = P.layer[l];
            const int n = L.n_in * L.n_out;
            for (int i = tid; i < n; i += blockDim.x) {
                const int j = i / L.n_in, k = i - j * L.n_in;
                const float w = flat[L.w_off + i];
                sw[L.wt_s + k * L.n_out_p4 + j] = w;
                sw[L.w_s + j * L.n_in_p8 + k] = w;
            }
            for (int j = tid; j < L.n_out; j += blockDim.x) sw[L.b_s + j] = flat[L.b_off + j];
        }
        __syncthreads();
    }
    for (int i = tid; i < P.n_params; i += blockDim.x) {
        a.params[i] = flat[i]; a.exp_avg[i] = mom1[i]; a.exp_avg_sq[i] = mom2[i];
    }
    for (int i = tid; i < a.n_step_tensors; i += blockDim.x) a.step_tensors[i] += (float)a.k_steps;
    if (tid == 0) *a.step_counter = step0 + (unsigned long long)a.k_steps;
}

typedef void (*MultiKernelFn)(const DevPlan, const MultiArgs);

typedef void (*StepKernelFn)(const DevPlan, const StepArgs);

// Every kernel instantiation of one jet set: (nf, ns) for second-order problems, (nf, order) for orders 3 / 4.
// The build units of pinn_instances.cu fill the sets during static initialisation; a null entry has no instantiation.
struct KernelSet {
    StepKernelFn step[2][2];                 // step_kernel [GEN][GMEM]; GEN = 0: plain problems (no residual wiring /
                                             // oblique directions / IC variables / z-stored activations), 1: everything.
                                             // Five / six directions and orders 3 / 4 have step[1][1] only (orders 3 / 4:
                                             // hi_step_kernel), which serves plain plans too.
    MultiKernelFn multi;                     // persistent multi-step kernel (general form, smem-resident)
    MultiKernelFn small;                     // tiny-batch cluster kernel (pinn_small_kernel.cuh)
    StepKernelFn wide[2];                    // tensor-core tile kernel (pinn_wide_kernel.cuh), [0]: 512, [1]: 256 threads
    int maxt;                                // threads per CTA the step kernels are compiled for
    StepKernelFn wide128;                    // the tile kernel's class for hidden widths up to 128, 512 threads
};

// The set of a jet set, or nullptr when none was built: 0 <= ns <= nf <= PINN_MAX_DIRS for order 2; 1 <= nf <= 4 and
// ns = 0 for orders 3 / 4 (their plans carry no second-order channels).  Defined in pinn_kernels.cu.
const KernelSet* kernels(int nf, int ns, int order);
// The writable entry of a jet set, for the build units' static initialisers (same key, not range-checked).
KernelSet& kernel_slot(int nf, int ns, int order);

template <int NF, int NS>
struct VariantCfg {
    static constexpr int C = 1 + NF + NS;
    static constexpr int MAXT = (C <= 3) ? 512 : 256;
    static constexpr int JF = 16;
};

}  // namespace pinn
