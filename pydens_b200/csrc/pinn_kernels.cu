// pinn_kernels.cu — sm_90a kernels and the C ABI (include/pinn_b200.h) of the fused PINN fit step.
//
// One launch of step_kernel does, for every collocation point of the batch, everything the
// reference does between sampling and loss.backward() (pydens/model_torch.py:430-460):
//   * coordinates are sampled in-kernel (Philox4x32-10) or read coalesced from HBM;
//   * the flat parameter buffer is staged into shared memory with one TMA bulk copy
//     (cp.async.bulk + mbarrier) and re-laid out for broadcast 128-bit reads;
//   * one thread per point: forward jets -> ansatz -> residual program -> reverse sweep
//     (pinn_device.cuh), all per-point state resident in shared memory (or, for networks too wide
//     for that, in a global spill area);
//   * weight gradients are reduced warp -> CTA -> grid (last-arriving CTA folds the per-CTA
//     partials in a fixed order, so results are run-to-run deterministic).
// Persistent grid: one CTA per SM, every warp strides over 32-point tiles.

#include <cuda_runtime.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>
#include <stdlib.h>
#include <memory>
#include <new>

#include "pinn_step_kernel.cuh"
#include "pinn_wide_kernel.cuh"
#include "pinn_small_kernel.cuh"
#include "pinn_lbfgs.cuh"
#include "pinn_host_plan.h"

namespace pinn {

// The kernel table, filled by the build units of pinn_instances.cu during static initialisation.  A function-local
// static is initialised on first use, so the order in which the units initialise does not matter.
KernelSet& kernel_slot(int nf, int ns, int order) {
    static KernelSet table[3][PINN_MAX_DIRS + 1][PINN_MAX_DIRS + 1];      // [order - 2][nf][ns]
    return table[order - 2][nf][ns];
}

const KernelSet* kernels(int nf, int ns, int order) {
    if (order < 2 || order > 4 || nf < 0 || nf > PINN_MAX_DIRS || ns < 0 || ns > nf) return nullptr;
    const KernelSet& k = kernel_slot(nf, ns, order);
    return k.step[1][1] ? &k : nullptr;
}

// ---------------------------------------------------------------------------------------------------
// Forward-only kernel (predict): u for explicit points; MULTI: the k components of every point, u_out [n_points, k].
// ---------------------------------------------------------------------------------------------------
template <bool GMEM, bool MULTI>
__device__ __forceinline__ void forward_body(const DevPlan& P, const FwdArgs& a) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const SmemLayout SL = smem_layout(P.weights_floats, 0, 0,
                                      GMEM ? P.n_params : max(P.n_params, a.rows_total * RS * nwarps));
    stage_weights(smem, SL, P, a.params);
    const float* sw = smem + SL.weights_f;
    const long long gw = (long long)blockIdx.x * nwarps + warp;
    const long long total_warps = (long long)gridDim.x * nwarps;
    float* st = (GMEM ? a.spill + (size_t)gw * a.rows_total * RS : smem + SL.storage_f + (size_t)warp * a.rows_total * RS) + lane;
    const long long n_tiles = (a.n_points + 31) / 32;
    for (long long tile = gw; tile < n_tiles; tile += total_warps) {
        const long long pl = tile * 32 + lane;
        const bool valid = pl < a.n_points;
        const long long pe = valid ? pl : a.n_points - 1;
        const float* src = a.points + (size_t)pe * P.total;
        for (int k = 0; k < P.total; ++k) st[k * RS] = __ldg(src + k);
        float u = point_forward<16, MULTI>(P, sw, a.params, st, RS, a.row_scr);
        if constexpr (MULTI) {
            const int k = P.layer[P.n_layers - 1].n_out;
            for (int j = 0; j < k; ++j)
                if (valid) a.u_out[(size_t)pl * k + j] = st[(size_t)(a.row_scr + j) * RS];
        } else {
            if (valid) a.u_out[pl] = u;
        }
    }
}

template <bool GMEM>
__global__ void __launch_bounds__(256, 1) forward_kernel(const __grid_constant__ DevPlan P, const FwdArgs a) {
    forward_body<GMEM, false>(P, a);
}

template <bool GMEM>
__global__ void __launch_bounds__(256, 1) coupled_forward_kernel(const __grid_constant__ DevPlan P, const FwdArgs a) {
    forward_body<GMEM, true>(P, a);
}

// The forward-only form of the 128-wide tile kernel (declared in pinn_wide_kernel.cuh).
__global__ void __launch_bounds__(512, 1) wide::wide128_forward_kernel(const __grid_constant__ DevPlan P, const StepArgs a) {
    wide::wide_step<0, 0, 128, true>(P, a);
}
// ... and of its coupled form: u_out [n, k]
__global__ void __launch_bounds__(512, 1) wide::wide128_coupled_forward_kernel(const __grid_constant__ DevPlan P, const StepArgs a) {
    wide::wide_step<0, 0, 128, true, true>(P, a);
}

// Points the in-kernel sampler produces (for tests / replay).
struct SampleCols { PinnColumn c[PINN_MAX_DIMS]; int total; };

__global__ void sample_kernel(const __grid_constant__ SampleCols cols, uint64_t seed, const uint64_t* step_ptr,
                              uint64_t step_val, uint64_t point_offset, long long n_points, float* out) {
    const uint64_t step = step_ptr ? *step_ptr : step_val;
    const int total = cols.total;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n_points;
         p += (long long)gridDim.x * blockDim.x) {
        const uint64_t gidx = point_offset + (uint64_t)p;
        const uint32_t c3 = (uint32_t)(((step >> 32) & 0xffffu) << 16);
        Philox4 b0 = philox4x32_10((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)step, c3, (uint32_t)seed,
                                   (uint32_t)(seed >> 32));
        Philox4 b1 = b0;
        if (total > 4)
            b1 = philox4x32_10((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)step, c3 | 1u, (uint32_t)seed,
                               (uint32_t)(seed >> 32));
        for (int k = 0; k < total; ++k)
            out[(size_t)p * total + k] = sample_column(cols.c[k], k, gidx, step, seed, b0, b1);
    }
}

__global__ void record_loss_kernel(const float* out, int loss_idx, float* ring, long long ring_len,
                                   unsigned long long* step) {
    unsigned long long s = *step;
    ring[s % (unsigned long long)ring_len] = out[loss_idx];
    *step = s + 1ull;
}

}  // namespace pinn

// ===================================================================================================
// Host side: plan construction, kernel selection, C ABI.
// ===================================================================================================
using namespace pinn;

static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CUDA_TRY(expr)                                                                   \
    do {                                                                                 \
        cudaError_t e_ = (expr);                                                         \
        if (e_ != cudaSuccess) return fail(PINN_E_CUDA, "%s: %s", #expr, cudaGetErrorString(e_)); \
    } while (0)

// The tensor-core tile kernel (pinn_wide_kernel.cuh) covers plain dense chains with polynomial-family activations
// and hidden widths <= 128, in two width classes (<= 64 and 65..128); it pays off once the layers are wide enough to
// be real GEMMs.  Networks of 2..4 outputs pass the same rules; only the 128-wide class has their (coupled) form.
// *max_width: the widest hidden layer.
static bool wide_eligible(const pinn::DevPlan& h, int* max_width) {
    if (h.n_layers < 2 || h.n_layers > pinn::wide::MAX_LAYERS) return false;
    if (h.layer[h.n_layers - 1].n_out > 4) return false;
    int mw = 0;
    for (int l = 0; l < h.n_layers; ++l) {
        const pinn::DevLayer& L = h.layer[l];
        if (L.skip_src >= 0 || L.post_base >= 0) return false;
        if (L.act != PINN_ACT_NONE && L.act != PINN_ACT_TANH && L.act != PINN_ACT_SIGMOID) return false;
        if (l + 1 < h.n_layers) { if (L.n_out > pinn::wide::Tile<128>::KW) return false; if (L.n_out > mw) mw = L.n_out; }
    }
    *max_width = mw;
    return true;
}

// The launch of pinn_step / pinn_step_allreduce / pinn_step_adam.
struct StepLaunch {
    StepKernelFn fn;
    DevPlan plan;                            // the plan fn runs on: h, or its compact layout (build_remat_plan) under
                                             // step_kernel_w12
    int threads, smem, regs;
    int points_per_cta;                      // per round: threads (thread kernels), Tile<KW>::T (tile kernels)
    int tensor_core;                         // 0: a thread kernel; 1 / 2: the 64- / 128-wide tile kernel, whose grid
                                             // PINN_WIDE_CTAS caps
    bool state_in_smem;                      // the per-point state lives in shared memory, not in the spill area
    size_t wacc_floats, spill_floats;        // workspace per CTA: gradient accumulators, spill area
};

// The launch of pinn_forward: a thread-forward kernel (FwdArgs) or the 128-wide tile kernel's forward-only form (StepArgs).
struct ForwardLaunch {
    void (*fn)(const DevPlan, const FwdArgs);
    StepKernelFn tile_fn;
    int threads, smem, points_per_cta, rows, row_scr;
    size_t spill_floats;                     // workspace per CTA
};

// A persistent kernel (multi_step_kernel, or the tiny-batch cluster kernel) and its ensemble form; null where they do
// not fit.  budget: the dynamic shared memory they can take (constraint programs with more slots).
struct PersistentLaunch {
    MultiKernelFn solo;
    EnsembleKernelFn ensemble;
    int threads, smem, budget;
};

// The L-BFGS form of the cluster kernel (pinn_lbfgs_multi): null where the cluster kernel is, or where its static shared
// memory leaves no room for the cluster kernel's layout.
struct LbfgsLaunch {
    LbfgsKernelFn fn;
    int threads, smem, budget;
};

struct PinnPlan {
    PinnSpec spec;
    DevPlan h;
    int device;
    const KernelSet* ks;                     // the kernels of this plan's jet set
    bool coupled;                            // a network of 2..4 outputs: coupled_step_kernel / coupled_forward_kernel,
                                             // or the coupled form of the 128-wide tile kernel
    int sm_count;
    int smem_optin;
    StepLaunch step;
    ForwardLaunch fwd;
    PersistentLaunch multi, small;
    LbfgsLaunch small_lbfgs;
};

extern "C" const char* pinn_last_error(void) { return g_err; }
// the error message of the other build units (pinn_lbfgs.cu)
int pinn_fail_message(int code, const char* msg) { return fail(code, "%s", msg); }
extern "C" int pinn_abi_version(void) { return PINN_ABI_VERSION; }

// The dynamic shared-memory limit is an attribute of the KERNEL, shared by every plan that uses the same
// instantiation: raise it to the device maximum once instead of to this plan's size, so that creating a second
// plan (another Solver, a constraint plan) can never lower it under a plan that is still in use.
static cudaError_t allow_max_smem(const void* fn, int smem_optin) {
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, fn);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin - (int)fa.sharedSizeBytes);
}

// Warps per CTA a kernel compiled for `maxt` threads can run at its register count (one CTA per SM).
static int max_warps(const cudaFuncAttributes& fa, int maxt) {
    const int by_regs = 65536 / (fa.numRegs * 32);
    return by_regs < maxt / 32 ? by_regs : maxt / 32;
}

// Floats of the per-point storage area for `nw` warps of `rows` rows; the area holds at least the flat parameters.
static int storage_floats(const DevPlan& h, int rows, int nw) {
    return rows * RS * nw > h.n_params ? rows * RS * nw : h.n_params;
}

// A kernel's attributes, and the dynamic shared memory it can take beside its static shared memory (64 B spare).
static cudaError_t kernel_budget(const void* fn, int smem_optin, cudaFuncAttributes& fa, int& budget) {
    const cudaError_t e = cudaFuncGetAttributes(&fa, fn);
    if (e == cudaSuccess) budget = smem_optin - (int)fa.sharedSizeBytes - 64;
    return e;
}

// Dynamic shared memory of a thread step kernel on `plan` at `nw` warps with `nwacc` gradient accumulators there (the
// others live in the workspace); gmem: the per-point state lives in the spill area.
static int step_smem_bytes(const DevPlan& plan, int nw, int nwacc, bool gmem) {
    return smem_layout(plan.weights_floats, plan.n_params + 4, nwacc,
                       gmem ? plan.n_params : storage_floats(plan, plan.rows_total, nw)).total_f * 4;
}

static StepLaunch thread_step(StepKernelFn fn, const DevPlan& plan, int regs, int nw, int nwacc, bool gmem) {
    StepLaunch s = {};
    s.fn = fn; s.plan = plan; s.regs = regs;
    s.threads = s.points_per_cta = nw * 32;
    s.smem = step_smem_bytes(plan, nw, nwacc, gmem);
    s.state_in_smem = !gmem;
    s.wacc_floats = nwacc ? 0 : (size_t)nw * (plan.n_params + 4);
    s.spill_floats = gmem ? (size_t)nw * plan.rows_total * RS : 0;
    return s;
}

// Thread kernel: per-point state in shared memory at the largest warp count that fits, or in the global spill area.
// Every warp has a gradient accumulator of its own: in shared memory when it fits there too, else in the workspace.
// fn_smem / fn_gmem: the pair matching this plan (plain or general, or coupled_step_kernel); fn_smem may be null.
static int place_thread_step(const PinnPlan* p, StepKernelFn fn_smem, StepKernelFn fn_gmem, StepLaunch& s) {
    const DevPlan& h = p->h;
    cudaFuncAttributes fa;
    int budget;
    cudaError_t e = kernel_budget((const void*)(fn_smem ? fn_smem : fn_gmem), p->smem_optin, fa, budget);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncGetAttributes: %s", cudaGetErrorString(e));
    const int max_nw = max_warps(fa, p->ks->maxt);
    int best_nw = 0, best_nwacc = 0;                 // best_nwacc: accumulators in smem (best_nw), or 0 (workspace)
    for (int nw = max_nw; nw >= 1 && !best_nw; --nw)
        for (int nwacc : {nw, 0})
            if (!best_nw && step_smem_bytes(h, nw, nwacc, false) <= budget) { best_nw = nw; best_nwacc = nwacc; }
    // PINN_FORCE_MODE=smem|gmem overrides the placement heuristic (experiments only)
    const char* force = getenv("PINN_FORCE_MODE");
    const bool force_gmem = force && !strcmp(force, "gmem");
    bool use_smem = best_nw >= 4 || (best_nw >= 2 && max_nw <= 4);
    if (force && !strcmp(force, "smem") && best_nw >= 1) use_smem = true;
    if (force_gmem || !fn_smem) use_smem = false;
    // three warps per scheduler: the twelve-warp form on the compact per-point layout, where its 384 threads fit (register
    // count, and the storage of twelve warps with their accumulators in shared memory or else in the workspace) and
    // outnumber the warps placed above (cfg2: 12 instead of 8)
    DevPlan hc;
    const StepKernelFn f12 = p->coupled ? nullptr : p->ks->step_w12;
    bool w12 = false;
    if (f12 && !force_gmem && build_remat_plan(h, hc) && (!use_smem || best_nw < 12)) {
        cudaFuncAttributes f12a;
        int budget12;
        e = kernel_budget((const void*)f12, p->smem_optin, f12a, budget12);
        if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncGetAttributes: %s", cudaGetErrorString(e));
        for (int nwacc : {12, 0})
            if (!w12 && max_warps(f12a, 384) == 12 && step_smem_bytes(hc, 12, nwacc, false) <= budget12) {
                s = thread_step(f12, hc, f12a.numRegs, 12, nwacc, false);
                w12 = true;
            }
    }
    if (!w12 && use_smem) {
        s = thread_step(fn_smem, h, fa.numRegs, best_nw, best_nwacc, false);
    } else if (!w12) {
        // activations spill to a global workspace; accumulators: in smem if they fit, else in the workspace too
        e = cudaFuncGetAttributes(&fa, (const void*)fn_gmem);
        if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncGetAttributes: %s", cudaGetErrorString(e));
        int nw = max_warps(fa, p->ks->maxt);
        { const char* e2 = getenv("PINN_GMEM_WARPS"); if (e2 && atoi(e2) >= 1 && atoi(e2) <= nw) nw = atoi(e2); }   // experiments
        const int nwacc = step_smem_bytes(h, nw, nw, true) <= budget ? nw : 0;
        if (step_smem_bytes(h, nw, nwacc, true) > budget)
            return fail(PINN_E_UNSUPPORTED, "network too large: %d B of weights do not fit shared memory", step_smem_bytes(h, nw, 0, true));
        s = thread_step(fn_gmem, h, fa.numRegs, nw, nwacc, true);
    }
    e = allow_max_smem((const void*)s.fn, p->smem_optin);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncSetAttribute(smem=%d): %s", s.smem, cudaGetErrorString(e));
    return PINN_OK;
}

// Forward kernel: eight warps, per-point state (`rows` rows) in shared memory when it fits, else in the global spill area.
static int place_forward_kernel(const PinnPlan* p, int rows, int row_scr, ForwardLaunch& f) {
    const DevPlan& h = p->h;
    const int nw = 8;
    int smem = smem_layout(h.weights_floats, 0, 0, storage_floats(h, rows, nw)).total_f * 4;
    const bool gmem = smem > p->smem_optin - 64;
    if (gmem) smem = smem_layout(h.weights_floats, 0, 0, h.n_params).total_f * 4;
    if (smem > p->smem_optin - 64) return fail(PINN_E_UNSUPPORTED, "network too large for shared memory");
    f = {};
    f.fn = p->coupled ? (gmem ? coupled_forward_kernel<true> : coupled_forward_kernel<false>)
                      : (gmem ? forward_kernel<true> : forward_kernel<false>);
    f.threads = f.points_per_cta = nw * 32; f.smem = smem; f.rows = rows; f.row_scr = row_scr;
    f.spill_floats = gmem ? (size_t)nw * rows * RS : 0;
    const cudaError_t e = allow_max_smem((const void*)f.fn, p->smem_optin);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncSetAttribute(fwd): %s", cudaGetErrorString(e));
    return PINN_OK;
}

// Dynamic shared memory of multi_step_kernel at `nw` warps and `rows` per-point rows.
static int multi_smem_bytes(const DevPlan& h, int nw, int rows) {
    const int n_out_floats = h.n_params + 4;
    const int extra = 3 * align4(h.n_params) + align4(n_out_floats);
    return (smem_layout(h.weights_floats, n_out_floats, nw, storage_floats(h, rows, nw)).total_f + extra) * 4;
}

// A persistent kernel `f` (compiled for maxt threads) at the most warps whose dynamic shared memory, bytes(nw), fits, and
// its ensemble form `fe` where that runs as many threads in at least as much shared memory.  Null where the jet set has
// none or they do not fit.
template <class Bytes>
static PersistentLaunch place_persistent(const PinnPlan* p, MultiKernelFn f, EnsembleKernelFn fe, int maxt, Bytes bytes) {
    PersistentLaunch k = {};
    cudaFuncAttributes fa;
    int budget;
    if (f && kernel_budget((const void*)f, p->smem_optin, fa, budget) == cudaSuccess)
        for (int nw = max_warps(fa, maxt); nw >= 1; --nw) {
            if (bytes(nw) > budget) continue;
            if (allow_max_smem((const void*)f, p->smem_optin) == cudaSuccess) k = {f, nullptr, nw * 32, bytes(nw), budget};
            break;
        }
    if (k.solo && fe && kernel_budget((const void*)fe, p->smem_optin, fa, budget) == cudaSuccess &&
        max_warps(fa, k.threads) * 32 >= k.threads && budget >= k.budget && allow_max_smem((const void*)fe, p->smem_optin) == cudaSuccess)
        k.ensemble = fe;
    (void)cudaGetLastError();
    return k;
}

// The L-BFGS form of the cluster kernel, where it runs NT threads in the `smem` bytes of the cluster kernel's layout.
static LbfgsLaunch place_lbfgs(const PinnPlan* p, LbfgsKernelFn f, int smem) {
    LbfgsLaunch k = {};
    cudaFuncAttributes fa;
    int budget;
    if (kernel_budget((const void*)f, p->smem_optin, fa, budget) == cudaSuccess && max_warps(fa, small::NT) * 32 >= small::NT &&
        smem <= budget && allow_max_smem((const void*)f, p->smem_optin) == cudaSuccess)
        k = {f, small::NT, smem, budget};
    (void)cudaGetLastError();
    return k;
}

// Wide networks: the tensor-core tile kernel takes the step (PINN_FORCE_KERNEL=thread|wide|wide128 overrides).
// thread_rc is how the thread kernel's placement (step and forward) went: a network whose weights do not fit its
// shared memory goes to the 128-wide class when that class covers it; otherwise that failure is the plan's.
// Fills `s` where the tile kernel takes the step; returns thread_rc where it does not.
static int place_tile_step(const PinnPlan* p, int order, int thread_rc, StepLaunch& s) {
    int mw = 0;
    const char* fk = getenv("PINN_FORCE_KERNEL");
    const bool eligible = order < 3 && wide_eligible(p->h, &mw);
    // networks of 2..4 outputs: the coupled form of the 128-wide class only
    const StepKernelFn f128 = p->coupled ? p->ks->coupled_wide128 : p->ks->wide128;
    const bool eligible64 = eligible && !p->coupled;
    const bool eligible128 = eligible && mw > 64 && f128;
    // the tile kernel wins from 64-wide layers with many jet channels on (H100 80GB HBM3 at 700 W, cfg5: 21.1 ms
    // vs 32.3 ms per step); for narrower networks the per (unit, channel) operand handling costs as much as the
    // FMA row it replaces, and the CUDA-core kernel keeps them.  Networks of 65-128 units the thread kernel holds
    // stay there: the 128-wide class takes only what the thread kernel refuses.
    bool want = eligible64 && mw <= 64 && mw >= 48 && (1 + p->spec.nf + p->spec.ns) >= 5;
    int kw = 64;
    if (thread_rc != PINN_OK) { want = eligible128; kw = 128; }
    if (fk && !strcmp(fk, "thread")) want = false;
    if (fk && !strcmp(fk, "wide")) {
        if (!eligible64 || mw > 64) return fail(PINN_E_UNSUPPORTED, "PINN_FORCE_KERNEL=wide: this network is outside what the tile kernel covers");
        want = true; kw = 64;
    }
    if (fk && !strcmp(fk, "wide128")) {
        if (!eligible128) return fail(PINN_E_UNSUPPORTED, "PINN_FORCE_KERNEL=wide128: this network is outside what the 128-wide tile kernel covers");
        want = true; kw = 128;
    }
    const StepKernelFn f = kw == 128 ? f128 : p->ks->wide;
    if (!want || !f || (thread_rc != PINN_OK && kw != 128)) return thread_rc;
    const int smem = kw == 128 ? (p->coupled ? wide::Tile<128, true>::SMEM_BYTES : wide::Tile<128>::SMEM_BYTES)
                               : wide::Tile<64>::SMEM_BYTES;
    cudaError_t e = cudaFuncSetAttribute((const void*)f, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncSetAttribute(wide, smem=%d): %s", smem, cudaGetErrorString(e));
    cudaFuncAttributes fa;
    e = cudaFuncGetAttributes(&fa, (const void*)f);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncGetAttributes(wide): %s", cudaGetErrorString(e));
    s = {};
    s.fn = f; s.plan = p->h; s.threads = wide::NT; s.smem = smem; s.regs = fa.numRegs;
    s.points_per_cta = kw == 128 ? wide::Tile<128>::T : wide::Tile<64>::T;
    s.tensor_core = kw == 128 ? 2 : 1;
    s.wacc_floats = kw == 128 ? wide::Tile<128>::WACC_FLOATS : 0;
    s.spill_floats = wide::spill_floats_per_cta(p->h.n_layers, 1 + p->h.nf + p->h.ns);
    return PINN_OK;
}

// The 128-wide tile kernel's forward-only form, for the networks the thread-forward kernel does not hold.
static int place_tile_forward(const PinnPlan* p, ForwardLaunch& f) {
    const StepKernelFn ff = p->coupled ? wide::wide128_coupled_forward_kernel : wide::wide128_forward_kernel;
    const int smem = p->coupled ? wide::Tile<128, true>::SMEM_BYTES : wide::Tile<128>::SMEM_BYTES;
    const cudaError_t e = cudaFuncSetAttribute((const void*)ff, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncSetAttribute(wide forward, smem=%d): %s", smem, cudaGetErrorString(e));
    f = {};
    f.tile_fn = ff; f.threads = wide::NT; f.smem = smem; f.points_per_cta = wide::Tile<128>::T;
    return PINN_OK;
}

extern "C" int pinn_plan_create(const PinnSpec* s, int device, PinnPlan** out) {
    if (!s || !out) return fail(PINN_E_INVALID, "null argument");
    std::unique_ptr<PinnPlan> p(new (std::nothrow) PinnPlan());
    if (!p) return fail(PINN_E_INVALID, "out of memory");
    int fwd_rows, fwd_row_scr;
    {
        char msg[256];
        const int rc = build_dev_plan(s, p->h, fwd_rows, fwd_row_scr, msg, sizeof(msg), 4);
        if (rc) return fail(rc, "%s", msg);
    }
    // orders 3 / 4 take whole jets per direction (pinn_hi_kernel.cuh), one kernel per (nf, order); their plans have ns = 0
    const int order = spec_order(s);
    p->ks = kernels(p->h.nf, p->h.ns, order);
    if (!p->ks && order >= 3)
        return fail(PINN_E_UNSUPPORTED, "no kernel for derivative order %d with %d directions", order, s->nf);
    if (!p->ks)
        return fail(PINN_E_UNSUPPORTED, "no kernel variant for nf=%d ns=%d%s", s->nf, s->ns,
                    s->nf > 4 ? " (more than 4 derivative directions: every direction must carry its second derivative, ns = nf)" : "");
    // a set with the general global-memory form only serves plain plans with it
    const int gen = p->h.general ? 1 : 0;
    StepKernelFn fn_smem = p->ks->step[gen][0];
    StepKernelFn fn_gmem = p->ks->step[gen][1] ? p->ks->step[gen][1] : p->ks->step[1][1];
    // networks of 2..4 outputs: their own step kernels (build_dev_plan has refused what those do not cover)
    p->coupled = p->h.layer[p->h.n_layers - 1].n_out > 1;
    if (p->coupled) {
        if (!p->ks->coupled[1]) return fail(PINN_E_UNSUPPORTED, "no kernel for a network of several outputs with nf=%d ns=%d", p->h.nf, p->h.ns);
        fn_smem = p->ks->coupled[0];
        fn_gmem = p->ks->coupled[1];
    }
    p->spec = *s;
    p->device = device;

    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0) return fail(PINN_E_UNSUPPORTED, "device sm_%d%d: this library is built for sm_90a only", prop.major, prop.minor);
    p->sm_count = prop.multiProcessorCount;
    p->smem_optin = (int)prop.sharedMemPerBlockOptin;

    // the thread kernels (step and forward); a network whose weights do not fit their shared memory can still go to
    // the 128-wide tile kernel, which stages one layer at a time (place_tile_step)
    StepLaunch thread = {}, tile = {};
    int thread_rc = place_thread_step(p.get(), fn_smem, fn_gmem, thread);
    if (thread_rc == PINN_OK) thread_rc = place_forward_kernel(p.get(), fwd_rows, fwd_row_scr, p->fwd);
    if (thread_rc != PINN_OK && thread_rc != PINN_E_UNSUPPORTED) return thread_rc;
    if (!p->coupled) {                           // the persistent multi-step kernels take networks of one output only
        // multi_step_kernel (small batches): per-point state + parameters + Adam moments in shared memory
        const DevPlan& h = p->h;
        p->multi = place_persistent(p.get(), p->ks->multi, p->ks->multi_ensemble, p->ks->maxt,
                                    [&](int nw) { return multi_smem_bytes(h, nw, h.rows_total); });
        // tiny batches: the (point, unit)-parallel cluster kernel, for plain dense chains whose jets fit shared memory
        bool chain = true;
        for (int l = 0; l < h.n_layers; ++l) chain = chain && h.layer[l].skip_src < 0 && h.layer[l].post_base < 0;
        if (chain)
            p->small = place_persistent(p.get(), p->ks->small, p->ks->small_ensemble, small::NT,
                                        [&](int) { return small::make_layout(h).total * 4; });
        if (p->small.solo && p->ks->small_lbfgs) p->small_lbfgs = place_lbfgs(p.get(), p->ks->small_lbfgs, p->small.smem);
    }
    if (int rc = place_tile_step(p.get(), order, thread_rc, tile)) return rc;
    p->step = tile.fn ? tile : thread;
    if (tile.fn && thread_rc != PINN_OK)          // the forward kernel does not hold this network either
        if (int rc = place_tile_forward(p.get(), p->fwd)) return rc;
    *out = p.release();
    return PINN_OK;
}

extern "C" int pinn_plan_destroy(PinnPlan* p) {
    if (!p) return PINN_OK;
    delete p;
    return PINN_OK;
}

// CTAs of a launch over n points at `per_cta` points per CTA and round, at most `cap`.
static int ctas(long long n_points, int per_cta, int cap) {
    const long long c = (n_points + per_cta - 1) / per_cta;
    return (int)(c < cap ? c : cap);
}

// workspace layout: [ticket: 256 B][partials: sm_count x n_out_floats][accumulators][spill]; the accumulators are the
// thread kernel's per-warp gradient accumulators (sm_count x warps x n_out_floats) when they do not fit shared memory,
// or the 128-wide tile kernel's hidden->hidden weight gradients (sm_count x 4 x 128 x 128, 256 KB per CTA); the spill
// area is shared by the step and forward launches.
static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
static size_t ws_wacc_off(const PinnPlan* p) { return align256(256 + (size_t)p->sm_count * (p->h.n_params + 4) * sizeof(float)); }
static size_t ws_spill_off(const PinnPlan* p) {
    return align256(ws_wacc_off(p) + (size_t)p->sm_count * p->step.wacc_floats * sizeof(float));
}

extern "C" size_t pinn_workspace_bytes(const PinnPlan* p, int64_t n_points) {
    if (!p) return 0;
    (void)n_points;
    const size_t spill = p->step.spill_floats > p->fwd.spill_floats ? p->step.spill_floats : p->fwd.spill_floats;
    return ws_spill_off(p) + (size_t)p->sm_count * spill * sizeof(float);
}

extern "C" int pinn_out_floats(const PinnPlan* p) { return p ? p->h.n_params + 4 : 0; }

// The sampler columns of a call are written into a by-value copy of the plan (kernel parameter).
static int resolve_cols(const PinnPlan* p, const PinnColumn* cols, PinnColumn* out) {
    for (int i = 0; i < PINN_MAX_DIMS; ++i) {
        memset(&out[i], 0, sizeof(PinnColumn));
        if (cols && i < p->h.total) out[i] = cols[i];
        else { out[i].kind = PINN_COL_UNIFORM; out[i].a = 0.0f; out[i].b = 1.0f; }
        const PinnColumn& c = out[i];
        if (c.kind < 0 || c.kind > PINN_COL_TNORMAL) return fail(PINN_E_INVALID, "column %d kind %d", i, c.kind);
        if (c.kind == PINN_COL_TNORMAL && !(c.comp_a[0] <= c.comp_b[0]))
            return fail(PINN_E_INVALID, "column %d: truncated normal with low %g > high %g", i, c.comp_a[0], c.comp_b[0]);
        if (c.kind == PINN_COL_MIXTURE) {
            if (c.n_comp < 2 || c.n_comp > PINN_MAX_MIX || c.group < 0 || c.group >= PINN_MAX_DIMS)
                return fail(PINN_E_INVALID, "column %d: mixture of %d components in group %d", i, c.n_comp, c.group);
            float prev = 0.0f;
            for (int j = 0; j < c.n_comp; ++j) {
                if (c.comp_kind[j] < 0 || c.comp_kind[j] > PINN_COL_CONST || !(c.cum_w[j] >= prev) || c.cum_w[j] > 1.0f + 1e-6f)
                    return fail(PINN_E_INVALID, "column %d: mixture component %d", i, j);
                prev = c.cum_w[j];
            }
        }
    }
    return PINN_OK;
}

static bool aligned16(const void* p) { return (((uintptr_t)p) & 15u) == 0; }

struct PinnComm {
    int rank, world, device;
    char* local;                              // this rank's exchange buffer (cudaMalloc)
    char* peers[PINN_COMM_MAX_RANKS];         // every rank's buffer as mapped here (peers[rank] == local)
    bool connected;
    size_t bytes;
};

extern "C" int pinn_comm_create(const PinnPlan* p, int rank, int world, PinnComm** out,
                                unsigned char handle_out[PINN_COMM_HANDLE_BYTES]) {
    if (!p || !out || !handle_out) return fail(PINN_E_INVALID, "null argument");
    if (world < 2 || world > PINN_COMM_MAX_RANKS || rank < 0 || rank >= world)
        return fail(PINN_E_INVALID, "rank %d / world %d (2..%d ranks of one node)", rank, world, PINN_COMM_MAX_RANKS);
    static_assert(sizeof(cudaIpcMemHandle_t) == PINN_COMM_HANDLE_BYTES, "IPC handle size");
    PinnComm* c = new (std::nothrow) PinnComm();
    if (!c) return fail(PINN_E_INVALID, "out of memory");
    c->rank = rank; c->world = world; c->device = p->device; c->connected = false; c->local = nullptr;
    for (int r = 0; r < PINN_COMM_MAX_RANKS; ++r) c->peers[r] = nullptr;
    c->bytes = comm_bytes(p->h.n_params + 4, world);
    cudaError_t e = cudaSetDevice(p->device);
    if (e == cudaSuccess) e = cudaMalloc(&c->local, c->bytes);
    if (e == cudaSuccess) e = cudaMemset(c->local, 0, c->bytes);
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, c->local);
    if (e != cudaSuccess) {
        if (c->local) cudaFree(c->local);
        delete c;
        return fail(PINN_E_CUDA, "pinn_comm_create: %s", cudaGetErrorString(e));
    }
    memcpy(handle_out, &h, PINN_COMM_HANDLE_BYTES);
    c->peers[rank] = c->local;
    *out = c;
    return PINN_OK;
}

extern "C" int pinn_comm_connect(PinnComm* c, const unsigned char* handles) {
    if (!c || !handles) return fail(PINN_E_INVALID, "null argument");
    if (c->connected) return PINN_OK;
    CUDA_TRY(cudaSetDevice(c->device));
    for (int r = 0; r < c->world; ++r) {
        if (r == c->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, handles + (size_t)r * PINN_COMM_HANDLE_BYTES, PINN_COMM_HANDLE_BYTES);
        void* ptr = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e));
        c->peers[r] = static_cast<char*>(ptr);
    }
    c->connected = true;
    return PINN_OK;
}

extern "C" int pinn_comm_destroy(PinnComm* c) {
    if (!c) return PINN_OK;
    cudaSetDevice(c->device);
    for (int r = 0; r < c->world; ++r)
        if (r != c->rank && c->peers[r]) cudaIpcCloseMemHandle(c->peers[r]);
    if (c->local) cudaFree(c->local);
    delete c;
    return PINN_OK;
}

extern "C" int pinn_comm_status(PinnComm* c, int* aborted, int reset) {
    if (!c || !aborted) return fail(PINN_E_INVALID, "null argument");
    CUDA_TRY(cudaSetDevice(c->device));
    unsigned int word = 0;
    CUDA_TRY(cudaMemcpy(&word, c->local + 4, 4, cudaMemcpyDeviceToHost));
    *aborted = (int)word;
    if (reset && word) { word = 0; CUDA_TRY(cudaMemcpy(c->local + 4, &word, 4, cudaMemcpyHostToDevice)); }
    return PINN_OK;
}

// ---------------------------------------------------------------------------------------------------
// Host-batch pipeline (see the header): staging buffers, copy / read-back streams, events.
// ---------------------------------------------------------------------------------------------------
#define PINN_PIPE_MAX_STAGE 8
struct PinnPipe {
    int device, n_stage;
    size_t bytes;                                  // one staging buffer
    float* buf[PINN_PIPE_MAX_STAGE];
    cudaEvent_t copied[PINN_PIPE_MAX_STAGE];       // H2D into buf[k] has completed
    cudaEvent_t freed[PINN_PIPE_MAX_STAGE];        // the compute stream no longer reads buf[k]
    cudaStream_t copy_stream, d2h_stream;
};

extern "C" int pinn_pipe_destroy(PinnPipe* q) {
    if (!q) return PINN_OK;
    cudaSetDevice(q->device);
    if (q->copy_stream) cudaStreamSynchronize(q->copy_stream);
    if (q->d2h_stream) cudaStreamSynchronize(q->d2h_stream);
    for (int k = 0; k < q->n_stage; ++k) {
        if (q->buf[k]) cudaFree(q->buf[k]);
        if (q->copied[k]) cudaEventDestroy(q->copied[k]);
        if (q->freed[k]) cudaEventDestroy(q->freed[k]);
    }
    if (q->copy_stream) cudaStreamDestroy(q->copy_stream);
    if (q->d2h_stream) cudaStreamDestroy(q->d2h_stream);
    delete q;
    return PINN_OK;
}

extern "C" int pinn_pipe_create(const PinnPlan* p, int n_stage, int64_t local_n, PinnPipe** out) {
    if (!p || !out) return fail(PINN_E_INVALID, "null argument");
    if (n_stage < 1 || n_stage > PINN_PIPE_MAX_STAGE || local_n <= 0)
        return fail(PINN_E_INVALID, "pinn_pipe_create: n_stage %d (1..%d), local_n %lld", n_stage, PINN_PIPE_MAX_STAGE, (long long)local_n);
    PinnPipe* q = new (std::nothrow) PinnPipe();
    if (!q) return fail(PINN_E_INVALID, "out of memory");
    memset(q, 0, sizeof(*q));
    q->device = p->device; q->n_stage = n_stage;
    q->bytes = (size_t)local_n * p->h.total * sizeof(float);
    cudaError_t e = cudaSetDevice(p->device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&q->copy_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&q->d2h_stream, cudaStreamNonBlocking);
    for (int k = 0; k < n_stage && e == cudaSuccess; ++k) {
        e = cudaMalloc(&q->buf[k], q->bytes);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&q->copied[k], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&q->freed[k], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { pinn_pipe_destroy(q); return fail(PINN_E_CUDA, "pinn_pipe_create: %s", cudaGetErrorString(e)); }
    *out = q;
    return PINN_OK;
}

extern "C" float* pinn_pipe_buffer(PinnPipe* q, int slot) {
    return (q && slot >= 0 && slot < q->n_stage) ? q->buf[slot] : nullptr;
}

extern "C" int pinn_pipe_finish(PinnPipe* q, int slot, const float* ring_src, float* loss_dst, void* stream) {
    if (!q || slot < 0 || slot >= q->n_stage) return fail(PINN_E_INVALID, "pinn_pipe_finish: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(cudaEventRecord(q->freed[slot], st));
    if (ring_src && loss_dst) {
        // the step's loss travels on its own stream so that the read-back never sits between two steps
        CUDA_TRY(cudaStreamWaitEvent(q->d2h_stream, q->freed[slot], 0));
        CUDA_TRY(cudaMemcpyAsync(loss_dst, ring_src, sizeof(float), cudaMemcpyDeviceToHost, q->d2h_stream));
    }
    return PINN_OK;
}

extern "C" int pinn_pipe_step(PinnPipe* q, int slot, const float* host_points, void* graph_exec,
                              const float* ring_src, float* loss_dst, void* stream) {
    if (!q || slot < 0 || slot >= q->n_stage || !host_points) return fail(PINN_E_INVALID, "pinn_pipe_step: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(cudaStreamWaitEvent(q->copy_stream, q->freed[slot], 0));
    CUDA_TRY(cudaMemcpyAsync(q->buf[slot], host_points, q->bytes, cudaMemcpyHostToDevice, q->copy_stream));
    CUDA_TRY(cudaEventRecord(q->copied[slot], q->copy_stream));
    CUDA_TRY(cudaStreamWaitEvent(st, q->copied[slot], 0));
    if (!graph_exec) return PINN_OK;
    CUDA_TRY(cudaGraphLaunch((cudaGraphExec_t)graph_exec, st));
    return pinn_pipe_finish(q, slot, ring_src, loss_dst, stream);
}

extern "C" int pinn_pipe_wait(PinnPipe* q, int slot) {
    if (!q || slot < 0 || slot >= q->n_stage) return fail(PINN_E_INVALID, "pinn_pipe_wait: bad argument");
    CUDA_TRY(cudaEventSynchronize(q->copied[slot]));
    return PINN_OK;
}

extern "C" int pinn_pipe_sync(PinnPipe* q) {
    if (!q) return fail(PINN_E_INVALID, "null argument");
    CUDA_TRY(cudaStreamSynchronize(q->copy_stream));
    CUDA_TRY(cudaStreamSynchronize(q->d2h_stream));
    return PINN_OK;
}

static int launch_step(StepKernelFn fn, int grid, int threads, int smem_bytes, cudaStream_t st, const DevPlan& plan,
                       const StepArgs& a) {
    fn<<<grid, threads, smem_bytes, st>>>(plan, a);
    CUDA_TRY(cudaGetLastError());
    return PINN_OK;
}

static int step_impl(const PinnPlan* cp, const PinnComm* comm, const float* params, const float* points,
                     const PinnColumn* cols, uint64_t seed, const uint64_t* step_counter, uint64_t step_value,
                     uint64_t point_offset, int64_t n_points, float inv_global_n, float* grads_and_loss,
                     float* residual_out, void* workspace, size_t workspace_bytes, void* stream,
                     const PinnAdam* adam = nullptr) {
    PinnPlan* p = const_cast<PinnPlan*>(cp);
    if (!p || !params || !grads_and_loss || !workspace) return fail(PINN_E_INVALID, "null argument");
    if (n_points <= 0) return fail(PINN_E_INVALID, "n_points must be positive");
    if (!aligned16(params) || !aligned16(grads_and_loss) || !aligned16(workspace))
        return fail(PINN_E_ALIGN, "params / grads_and_loss / workspace must be 16-byte aligned");
    if (points && (((uintptr_t)points) & 3u)) return fail(PINN_E_ALIGN, "points must be 4-byte aligned");
    if (workspace_bytes < pinn_workspace_bytes(p, n_points))
        return fail(PINN_E_WORKSPACE, "workspace %zu B < required %zu B", workspace_bytes, pinn_workspace_bytes(p, n_points));
    if (comm && (!comm->connected || comm->bytes != comm_bytes(p->h.n_params + 4, comm->world)))
        return fail(PINN_E_INVALID, "communicator is not connected or belongs to another plan");
    cudaStream_t st = (cudaStream_t)stream;
    const StepLaunch& s = p->step;
    DevPlan plan = s.plan;
    if (!points) { int rc = resolve_cols(p, cols, plan.cols); if (rc) return rc; }
    StepArgs a;
    a.params = params; a.points = points; a.seed = seed;
    a.step_ptr = step_counter; a.step_val = step_value; a.point_offset = point_offset;
    a.n_points = n_points; a.inv_n = inv_global_n; a.out = grads_and_loss; a.residual = residual_out;
    a.ticket = reinterpret_cast<unsigned int*>(workspace);
    a.partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
    a.spill = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws_spill_off(p));
    a.wacc = s.wacc_floats ? reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws_wacc_off(p)) : nullptr;
    a.rows_total = s.plan.rows_total;
    a.adam_m = nullptr; a.adam_v = nullptr; a.adam_mask = nullptr; a.adam_steps = nullptr; a.adam_n_steps = 0;
    a.adam_lr = a.adam_beta1 = a.adam_beta2 = a.adam_eps = a.adam_wd = 0.0f;
    a.ring = nullptr; a.ring_len = 1;
    if (adam) {
        if (!adam->exp_avg || !adam->exp_avg_sq || !adam->mask || !adam->step_tensors || adam->n_step_tensors < 1)
            return fail(PINN_E_INVALID, "PinnAdam: null state pointer");
        if (!step_counter) return fail(PINN_E_INVALID, "pinn_step_adam needs the device step counter");
        if (adam->losses_ring && adam->ring_len <= 0) return fail(PINN_E_INVALID, "PinnAdam: ring_len must be positive");
        a.adam_m = adam->exp_avg; a.adam_v = adam->exp_avg_sq; a.adam_mask = adam->mask;
        a.adam_steps = adam->step_tensors; a.adam_n_steps = adam->n_step_tensors;
        a.adam_lr = adam->lr; a.adam_beta1 = adam->beta1; a.adam_beta2 = adam->beta2; a.adam_eps = adam->eps;
        a.adam_wd = adam->weight_decay;
        a.ring = adam->losses_ring; a.ring_len = adam->losses_ring ? adam->ring_len : 1;
    }
    static long long comm_timeout = 0;
    if (!comm_timeout) {
        const char* e = getenv("PINN_COMM_TIMEOUT_S");
        double sec = e ? atof(e) : 60.0;
        if (!(sec > 0.0)) sec = 60.0;
        comm_timeout = (long long)(sec * 1.9e9);          // SM clock ticks (clock64), ~1.9 GHz
    }
    a.comm_timeout = comm_timeout;
    a.comm_rank = comm ? comm->rank : 0;
    a.comm_world = comm ? comm->world : 0;
    for (int r = 0; r < PINN_COMM_MAX_RANKS; ++r) a.comm_peers[r] = comm ? comm->peers[r] : nullptr;
    int cap = p->sm_count;
    if (s.tensor_core) { const char* e = getenv("PINN_WIDE_CTAS"); if (e && atoi(e) >= 1 && atoi(e) <= p->sm_count) cap = atoi(e); }   // experiments
    return launch_step(s.fn, ctas(n_points, s.points_per_cta, cap), s.threads, s.smem, st, plan, a);
}

extern "C" int pinn_step(const PinnPlan* plan, const float* params, const float* points, const PinnColumn* cols,
                         uint64_t seed, const uint64_t* step_counter, uint64_t step_value, uint64_t point_offset,
                         int64_t n_points, float inv_global_n, float* grads_and_loss, float* residual_out,
                         void* workspace, size_t workspace_bytes, void* stream) {
    return step_impl(plan, nullptr, params, points, cols, seed, step_counter, step_value, point_offset, n_points,
                     inv_global_n, grads_and_loss, residual_out, workspace, workspace_bytes, stream);
}

extern "C" int pinn_step_allreduce(const PinnPlan* plan, const PinnComm* comm, const float* params,
                                   const float* points, const PinnColumn* cols, uint64_t seed,
                                   const uint64_t* step_counter, uint64_t step_value, uint64_t point_offset,
                                   int64_t n_points, float inv_global_n, float* grads_and_loss, float* residual_out,
                                   void* workspace, size_t workspace_bytes, void* stream) {
    if (!comm) return fail(PINN_E_INVALID, "null communicator");
    return step_impl(plan, comm, params, points, cols, seed, step_counter, step_value, point_offset, n_points,
                     inv_global_n, grads_and_loss, residual_out, workspace, workspace_bytes, stream);
}

extern "C" int pinn_step_adam(const PinnPlan* plan, const PinnComm* comm, float* params, const float* points,
                              const PinnColumn* cols, uint64_t seed, uint64_t* step_counter, uint64_t point_offset,
                              int64_t n_points, float inv_global_n, float* grads_and_loss, float* residual_out,
                              void* workspace, size_t workspace_bytes, const PinnAdam* adam, void* stream) {
    if (!adam) return fail(PINN_E_INVALID, "null PinnAdam");
    return step_impl(plan, comm, params, points, cols, seed, step_counter, 0, point_offset, n_points, inv_global_n,
                     grads_and_loss, residual_out, workspace, workspace_bytes, stream, adam);
}

extern "C" int pinn_multi_step_max_points(const PinnPlan* p) {
    // one CTA walks the batch tile by tile: any batch works, but the kernel is meant for the launch-bound regime
    return (p && p->multi.solo) ? 4096 : ((p && p->small.solo) ? 8 * pinn::small::BP : 0);
}

// A constraint term's plan next to the plan it trains with (build_dev_term).
static int term_matches(const PinnPlan* p, const PinnPlan* q, DevTerm& t) {
    char msg[256];
    const int rc = build_dev_term(p->h, spec_order(&p->spec), q->h, spec_order(&q->spec), t, msg, sizeof(msg));
    return rc ? fail(rc, "%s", msg) : PINN_OK;
}

// What pinn_multi_step_terms and pinn_multi_step_ensemble share: the checks of the shared arguments and the terms, the
// by-value plan and arguments, and the kernel the columns go to — the cluster kernel at nc CTAs per member, or the
// multi-step kernel at one CTA per member (nc = 0).
struct MultiLaunch {
    DevPlan plan;
    MultiArgs a;
    const PersistentLaunch* k;
    int nc, smem;
};

// cluster_only: the cluster kernel whatever the batch (pinn_lbfgs_multi), for at most 8 x small::BP columns.
static int multi_setup(PinnPlan* p, int64_t n_points, int k_steps, int64_t ring_len, float point_weight, int n_terms,
                       const PinnTerm* terms, MultiLaunch& L, bool cluster_only = false) {
    if (!p->multi.solo && !p->small.solo) return fail(PINN_E_UNSUPPORTED, "the persistent multi-step kernels do not fit this network in shared memory");
    if (n_terms < 0 || n_terms > PINN_MAX_TERMS || (n_terms > 0 && !terms))
        return fail(PINN_E_INVALID, "pinn_multi_step_terms: %d terms (0..%d)", n_terms, PINN_MAX_TERMS);
    if (!(point_weight >= 0.0f) || point_weight > 3.0e38f) return fail(PINN_E_INVALID, "point_weight must be finite and >= 0");
    MultiArgs& a = L.a;
    memset(&a, 0, sizeof(a));
    a.terms.n_terms = n_terms;
    int rows = p->h.rows_total, n_slots = p->h.n_slots;             // scratch rows: the most any program needs
    for (int t = 0; t < n_terms; ++t) {
        const PinnTerm& T = terms[t];
        if (!T.plan || !T.points || T.n_points < 1 || a.terms.n_points + T.n_points > PINN_MAX_TERM_POINTS)
            return fail(PINN_E_INVALID, "constraint term %d: null plan / points, or more than %d points in all", t, PINN_MAX_TERM_POINTS);
        if (!(T.point_weight >= 0.0f) || T.point_weight > 3.0e38f) return fail(PINN_E_INVALID, "constraint term %d: point_weight", t);
        DevTerm& d = a.terms.t[t];
        const int rc = term_matches(p, T.plan, d);
        if (rc) return rc;
        d.weight = T.point_weight;
        a.terms.first[t] = a.terms.n_points;
        for (int i = 0; i < T.n_points; ++i)
            for (int k = 0; k < p->h.total; ++k) a.terms.x[a.terms.n_points + i][k] = T.points[(size_t)i * p->h.total + k];
        a.terms.n_points += T.n_points;
        if (T.plan->h.n_slots > n_slots) n_slots = T.plan->h.n_slots;
        if (p->h.row_scr + T.plan->h.n_slots > rows) rows = p->h.row_scr + T.plan->h.n_slots;
    }
    a.terms.first[n_terms] = a.terms.n_points;
    const long long n_cols = n_points + a.terms.n_points;
    const int max_cols = cluster_only ? 8 * pinn::small::BP : pinn_multi_step_max_points(p);
    if (n_points <= 0 || n_cols > max_cols || k_steps <= 0 || ring_len <= 0)
        return fail(PINN_E_INVALID, "pinn_multi_step: n_points %lld + %d constraint points (1..%d), k_steps %d", (long long)n_points,
                    a.terms.n_points, max_cols, k_steps);
    L.plan = p->h;
    L.plan.n_slots = n_slots;                                       // the small kernel's scratch rows
    a.n_points = n_points; a.inv_n = point_weight; a.k_steps = k_steps;
    a.ring_len = ring_len;
    a.rows_total = rows;
    // batches of at most 128 points: the (point, unit)-parallel kernel (PINN_MULTI_KERNEL=tile forces the other one)
    const char* mk = getenv("PINN_MULTI_KERNEL");
    const bool small = cluster_only || (p->small.solo && n_cols <= 8 * pinn::small::BP && (n_cols <= 256 || !p->multi.solo) &&
                                        !(mk && !strcmp(mk, "tile") && p->multi.solo));
    L.k = small ? &p->small : &p->multi;
    if (small) L.smem = n_slots == p->h.n_slots ? L.k->smem : small::make_layout(L.plan).total * 4;
    else       L.smem = rows == p->h.rows_total ? L.k->smem : multi_smem_bytes(p->h, L.k->threads / 32, rows);
    if (L.smem > L.k->budget) return fail(PINN_E_UNSUPPORTED, "the constraint programs' scratch slots do not fit shared memory");
    L.nc = 0;
    if (small) {
        // a cluster of up to 8 CTAs (8 SMs) shares the columns, ~16 per CTA at least; PINN_SMALL_CLUSTER overrides
        int nc = (int)((n_cols + 15) / 16);
        if (nc > 8) nc = 8;
        { const char* e = getenv("PINN_SMALL_CLUSTER"); if (e && atoi(e) >= 1 && atoi(e) <= 8) nc = atoi(e); }
        while ((n_cols + nc - 1) / nc > pinn::small::BP) ++nc;
        if (nc == 3) nc = 4; else if (nc > 4 && nc < 8) nc = 8;         // cluster sizes 1, 2, 4, 8
        L.nc = nc;
    }
    return PINN_OK;
}

// The persistent kernel of L for n_members members: the multi-step kernel on one CTA each, or the cluster kernel on
// n_members clusters of L.nc CTAs (member c: CTAs c * nc .. c * nc + nc - 1).
template <class... Args>
static int launch_persistent(void (*fn)(const DevPlan, const MultiArgs, Args...), const MultiLaunch& L, int n_members,
                             void* stream, const Args&... extra) {
    if (!L.nc) {
        fn<<<n_members, L.k->threads, L.smem, (cudaStream_t)stream>>>(L.plan, L.a, extra...);
        CUDA_TRY(cudaGetLastError());
        return PINN_OK;
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(L.nc * n_members); cfg.blockDim = dim3(L.k->threads); cfg.dynamicSmemBytes = L.smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = L.nc; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, fn, L.plan, L.a, extra...));
    CUDA_TRY(cudaGetLastError());
    return PINN_OK;
}

extern "C" int pinn_multi_step_terms(const PinnPlan* cp, float* params, float* exp_avg, float* exp_avg_sq, const float* mask,
                                     float* step_tensors, int n_step_tensors, const float* points, const PinnColumn* cols,
                                     uint64_t seed, uint64_t* step_counter, int64_t n_points, int k_steps,
                                     float lr, float beta1, float beta2, float eps, float weight_decay, float opt_step0,
                                     float* losses_ring, int64_t ring_len, float point_weight, int n_terms,
                                     const PinnTerm* terms, void* stream) {
    PinnPlan* p = const_cast<PinnPlan*>(cp);
    if (!p || !params || !exp_avg || !exp_avg_sq || !mask || !step_counter || !losses_ring)
        return fail(PINN_E_INVALID, "null argument");
    MultiLaunch L;
    if (int rc = multi_setup(p, n_points, k_steps, ring_len, point_weight, n_terms, terms, L))
        return rc;
    if (n_step_tensors < 0) return fail(PINN_E_INVALID, "pinn_multi_step: n_step_tensors %d", n_step_tensors);
    if (!aligned16(params)) return fail(PINN_E_ALIGN, "params must be 16-byte aligned");
    if (!points) { int rc = resolve_cols(p, cols, L.plan.cols); if (rc) return rc; }
    MultiArgs& a = L.a;
    a.params = params; a.exp_avg = exp_avg; a.exp_avg_sq = exp_avg_sq; a.mask = mask;
    a.step_tensors = step_tensors; a.n_step_tensors = n_step_tensors; a.points = points; a.seed = seed;
    a.step_counter = reinterpret_cast<unsigned long long*>(step_counter);
    a.opt_step0 = opt_step0;
    a.losses_ring = losses_ring;
    a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay;
    return launch_persistent(L.k->solo, L, 1, stream);
}

// The launch of both ensemble entry points: `hyper` holds n_members rows, already checked.
static int multi_step_ensemble(const PinnPlan* cp, int n_members, const PinnMember* members, const PinnAdamHyper* hyper,
                               int64_t n_points, int k_steps, int64_t ring_len, float point_weight, int n_terms,
                               const PinnTerm* terms, const PinnColumn* cols, void* stream) {
    PinnPlan* p = const_cast<PinnPlan*>(cp);
    if (!p || !members) return fail(PINN_E_INVALID, "null argument");
    if (n_members < 1 || n_members > PINN_MAX_MEMBERS)
        return fail(PINN_E_INVALID, "pinn_multi_step_ensemble: %d members (1..%d)", n_members, PINN_MAX_MEMBERS);
    bool sample = false;
    for (int j = 0; j < n_members; ++j) {
        const PinnMember& m = members[j];
        if (!m.params || !m.exp_avg || !m.exp_avg_sq || !m.mask || !m.step_counter || !m.losses_ring || m.n_step_tensors < 0 ||
            (m.n_step_tensors > 0 && !m.step_tensors))
            return fail(PINN_E_INVALID, "member %d: null pointer or n_step_tensors %d", j, m.n_step_tensors);
        if (!aligned16(m.params)) return fail(PINN_E_INVALID, "member %d: params must be 16-byte aligned", j);
        if (!m.points) sample = true;
    }
    static thread_local MultiLaunch L;                               // 13 KB: off the stack
    static thread_local DevMembers table;                            // 12.5 KB
    if (int rc = multi_setup(p, n_points, k_steps, ring_len, point_weight, n_terms, terms, L))
        return rc;
    if (!L.k->ensemble)
        return fail(PINN_E_UNSUPPORTED, "the ensemble form of the persistent kernel does not fit this network");
    if (sample) { int rc = resolve_cols(p, cols, L.plan.cols); if (rc) return rc; }
    memset(&table, 0, sizeof(table));
    memcpy(table.m, members, sizeof(PinnMember) * (size_t)n_members);
    memcpy(table.h, hyper, sizeof(PinnAdamHyper) * (size_t)n_members);
    return launch_persistent(L.k->ensemble, L, n_members, stream, table);
}

static bool finite_nonneg(float x) { return x >= 0.0f && x <= 3.4028235e38f; }   // false for NaN and inf

extern "C" int pinn_multi_step_ensemble_adam(const PinnPlan* plan, int n_members, const PinnMember* members,
                                             const PinnAdamHyper* hyper, int64_t n_points, int k_steps, int64_t ring_len,
                                             float point_weight, int n_terms, const PinnTerm* terms,
                                             const PinnColumn* cols, void* stream) {
    if (!hyper) return fail(PINN_E_INVALID, "pinn_multi_step_ensemble_adam: null hyper");
    for (int j = 0; j < n_members && j < PINN_MAX_MEMBERS; ++j) {   // torch.optim.Adam's checks, finite values only
        const PinnAdamHyper& h = hyper[j];
        if (!finite_nonneg(h.lr) || !(h.beta1 >= 0.0f && h.beta1 < 1.0f) || !(h.beta2 >= 0.0f && h.beta2 < 1.0f) ||
            !finite_nonneg(h.eps) || !finite_nonneg(h.weight_decay))
            return fail(PINN_E_INVALID, "member %d: lr %g, betas (%g, %g), eps %g, weight_decay %g (lr, eps, weight_decay "
                        "finite and >= 0, betas in [0, 1))", j, h.lr, h.beta1, h.beta2, h.eps, h.weight_decay);
    }
    return multi_step_ensemble(plan, n_members, members, hyper, n_points, k_steps, ring_len, point_weight, n_terms, terms,
                               cols, stream);
}

extern "C" int pinn_multi_step_ensemble(const PinnPlan* plan, int n_members, const PinnMember* members, int64_t n_points,
                                        int k_steps, float lr, float beta1, float beta2, float eps, float weight_decay,
                                        int64_t ring_len, float point_weight, int n_terms, const PinnTerm* terms,
                                        const PinnColumn* cols, void* stream) {
    static thread_local PinnAdamHyper rows[PINN_MAX_MEMBERS];
    for (int j = 0; j < PINN_MAX_MEMBERS; ++j) rows[j] = PinnAdamHyper{lr, beta1, beta2, eps, weight_decay};
    return multi_step_ensemble(plan, n_members, members, rows, n_points, k_steps, ring_len, point_weight, n_terms, terms,
                               cols, stream);
}

extern "C" int pinn_multi_step(const PinnPlan* p, float* params, float* exp_avg, float* exp_avg_sq, const float* mask,
                               float* step_tensors, int n_step_tensors, const float* points, const PinnColumn* cols,
                               uint64_t seed, uint64_t* step_counter, int64_t n_points, int k_steps,
                               float lr, float beta1, float beta2, float eps, float weight_decay, float opt_step0,
                               float* losses_ring, int64_t ring_len, void* stream) {
    return pinn_multi_step_terms(p, params, exp_avg, exp_avg_sq, mask, step_tensors, n_step_tensors, points, cols, seed,
                                 step_counter, n_points, k_steps, lr, beta1, beta2, eps, weight_decay, opt_step0,
                                 losses_ring, ring_len, n_points > 0 ? 1.0f / (float)n_points : 0.0f, 0, nullptr, stream);
}

// The launch of both L-BFGS entry points: cfg's shared settings as pinn_lbfgs_advance checks them, each member's own
// pointers and lr, then the columns as pinn_multi_step_terms checks them, on the cluster kernel only.
static int lbfgs_multi(const PinnPlan* cp, const PinnLbfgs* cfg, int n_members, const PinnLbfgsMember* members,
                       const PinnColumn* cols, int64_t n_points, int n_steps, float point_weight, int n_terms,
                       const PinnTerm* terms, void* stream) {
    PinnPlan* p = const_cast<PinnPlan*>(cp);
    if (!p || !cfg || !members) return fail(PINN_E_INVALID, "pinn_lbfgs_multi: null argument");
    if (!p->small_lbfgs.fn)
        return fail(PINN_E_UNSUPPORTED, "pinn_lbfgs_multi: the cluster kernel does not fit this network (small_batch_points = 0)");
    if (cfg->max_iter < 1 || cfg->max_eval < 1 || cfg->history_size < 1 || (cfg->line_search != 0 && cfg->line_search != 1) ||
        cfg->ring_len < 1)
        return fail(PINN_E_INVALID, "pinn_lbfgs_multi: invalid settings (max_iter %d, max_eval %d, history_size %d, line_search %d, "
                    "ring_len %lld)", cfg->max_iter, cfg->max_eval, cfg->history_size, cfg->line_search, (long long)cfg->ring_len);
    if (n_members < 1 || n_members > PINN_MAX_MEMBERS)
        return fail(PINN_E_INVALID, "pinn_lbfgs_multi_ensemble: %d members (1..%d)", n_members, PINN_MAX_MEMBERS);
    bool sample = false;
    for (int j = 0; j < n_members; ++j) {
        const PinnLbfgsMember& m = members[j];
        if (!m.params || !m.state || !m.mask || !m.step_counter || !m.losses_ring)
            return fail(PINN_E_INVALID, "pinn_lbfgs_multi: member %d: null pointer", j);
        if (!aligned16(m.params) || !aligned16(m.state))
            return fail(PINN_E_INVALID, "pinn_lbfgs_multi: member %d: params and state must be 16-byte aligned", j);
        if (!(m.lr >= 0.0)) return fail(PINN_E_INVALID, "pinn_lbfgs_multi: member %d: lr %g", j, m.lr);
        if (!m.points) sample = true;
    }
    if (n_steps < 1) return fail(PINN_E_INVALID, "pinn_lbfgs_multi: n_steps %d", n_steps);
    static thread_local MultiLaunch L;                               // 13 KB: off the stack
    static thread_local DevLbfgsMembers table;                       // 8 KB
    if (int rc = multi_setup(p, n_points, n_steps, cfg->ring_len, point_weight, n_terms, terms, L, true))
        return rc;
    if (L.smem > p->small_lbfgs.budget)
        return fail(PINN_E_UNSUPPORTED, "pinn_lbfgs_multi: the constraint programs' scratch slots do not fit shared memory");
    if (sample) { int rc = resolve_cols(p, cols, L.plan.cols); if (rc) return rc; }
    memset(&table, 0, sizeof(table));
    table.cfg = *cfg;
    memcpy(table.m, members, sizeof(PinnLbfgsMember) * (size_t)n_members);
    return launch_persistent(p->small_lbfgs.fn, L, n_members, stream, table);
}

extern "C" int pinn_lbfgs_multi(const PinnPlan* plan, const PinnLbfgs* cfg, float* params, void* state, const float* points,
                                const PinnColumn* cols, uint64_t seed, int64_t n_points, int n_steps, float point_weight,
                                int n_terms, const PinnTerm* terms, void* stream) {
    if (!cfg) return fail(PINN_E_INVALID, "pinn_lbfgs_multi: null argument");
    PinnLbfgsMember m;
    m.params = params; m.state = state; m.mask = cfg->mask; m.points = points; m.seed = seed;
    m.step_counter = cfg->step_counter; m.losses_ring = cfg->losses_ring; m.lr = cfg->lr;
    return lbfgs_multi(plan, cfg, 1, &m, cols, n_points, n_steps, point_weight, n_terms, terms, stream);
}

extern "C" int pinn_lbfgs_multi_ensemble(const PinnPlan* plan, const PinnLbfgs* cfg, int n_members,
                                         const PinnLbfgsMember* members, const PinnColumn* cols, int64_t n_points,
                                         int n_steps, float point_weight, int n_terms, const PinnTerm* terms, void* stream) {
    return lbfgs_multi(plan, cfg, n_members, members, cols, n_points, n_steps, point_weight, n_terms, terms, stream);
}

extern "C" int pinn_forward(const PinnPlan* p, const float* params, const float* points, int64_t n_points,
                            float* u_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!p || !params || !points || !u_out || !workspace) return fail(PINN_E_INVALID, "null argument");
    if (n_points <= 0) return fail(PINN_E_INVALID, "n_points must be positive");
    if (!aligned16(params) || !aligned16(workspace)) return fail(PINN_E_ALIGN, "params / workspace must be 16-byte aligned");
    if (((uintptr_t)points) & 3u) return fail(PINN_E_ALIGN, "points must be 4-byte aligned");
    if (workspace_bytes < pinn_workspace_bytes(p, n_points)) return fail(PINN_E_WORKSPACE, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const ForwardLaunch& f = p->fwd;
    const int grid = ctas(n_points, f.points_per_cta, p->sm_count);
    if (f.tile_fn) {                           // u of every point (coupled: u_out [n, k]) goes to `out` of the step arguments
        StepArgs w;
        memset(&w, 0, sizeof(w));
        w.params = params; w.points = points; w.n_points = n_points; w.out = u_out; w.ring_len = 1;
        return launch_step(f.tile_fn, grid, f.threads, f.smem, st, p->h, w);
    }
    FwdArgs a;
    a.params = params; a.points = points; a.n_points = n_points; a.u_out = u_out;
    a.spill = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws_spill_off(p));
    a.rows_total = f.rows; a.row_scr = f.row_scr;
    f.fn<<<grid, f.threads, f.smem, st>>>(p->h, a);
    CUDA_TRY(cudaGetLastError());
    return PINN_OK;
}

extern "C" int pinn_sample(const PinnPlan* cp, const PinnColumn* cols, uint64_t seed, const uint64_t* step_counter,
                           uint64_t step_value, uint64_t point_offset, int64_t n_points, float* points_out,
                           void* stream) {
    PinnPlan* p = const_cast<PinnPlan*>(cp);
    if (!p || !points_out) return fail(PINN_E_INVALID, "null argument");
    if (n_points <= 0) return fail(PINN_E_INVALID, "n_points must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    SampleCols sc;
    sc.total = p->h.total;
    int rc = resolve_cols(p, cols, sc.c);
    if (rc) return rc;
    long long blocks = (n_points + 255) / 256;
    if (blocks > 4 * p->sm_count) blocks = 4 * p->sm_count;
    sample_kernel<<<(int)blocks, 256, 0, st>>>(sc, seed, step_counter, step_value, point_offset, n_points, points_out);
    CUDA_TRY(cudaGetLastError());
    return PINN_OK;
}

extern "C" int pinn_record_loss(const PinnPlan* p, const float* grads_and_loss, float* losses_ring, int64_t ring_len,
                                uint64_t* step_counter, void* stream) {
    if (!p || !grads_and_loss || !losses_ring || !step_counter || ring_len <= 0) return fail(PINN_E_INVALID, "bad argument");
    record_loss_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(grads_and_loss, p->h.n_params, losses_ring, ring_len,
                                                         reinterpret_cast<unsigned long long*>(step_counter));
    CUDA_TRY(cudaGetLastError());
    return PINN_OK;
}

extern "C" int pinn_plan_info(const PinnPlan* p, PinnPlanInfo* info) {
    if (!p || !info) return fail(PINN_E_INVALID, "null argument");
    const int C = spec_channels(&p->spec);
    long long macs = 0;
    for (int l = 0; l < p->h.n_layers; ++l) macs += (long long)p->h.layer[l].n_in * p->h.layer[l].n_out;
    info->nf = p->h.nf; info->ns = p->h.ns; info->channels = C;
    info->threads_per_cta = p->step.threads; info->ctas_per_sm = 1;
    info->activations_in_smem = p->step.state_in_smem ? 1 : 0;
    info->tensor_core = p->step.tensor_core;
    info->small_batch_points = p->small.solo ? 8 * pinn::small::BP : 0;
    info->smem_bytes = p->step.smem; info->regs_per_thread = p->step.regs; info->sm_count = p->sm_count;
    info->rows_per_point = p->step.plan.rows_total;
    info->flops_per_point = 6ll * C * macs;
    info->bytes_per_point = 4 * p->h.total;
    return PINN_OK;
}
