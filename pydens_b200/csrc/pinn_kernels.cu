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
// Forward-only kernel (predict): u for explicit points.
// ---------------------------------------------------------------------------------------------------
template <bool GMEM>
__global__ void __launch_bounds__(256, 1) forward_kernel(const __grid_constant__ DevPlan P, const FwdArgs a) {
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
        float u = point_forward<16>(P, sw, a.params, st, RS, a.row_scr);
        if (valid) a.u_out[pl] = u;
    }
}

// The forward-only form of the 128-wide tile kernel (declared in pinn_wide_kernel.cuh).
__global__ void __launch_bounds__(512, 1) wide::wide128_forward_kernel(const __grid_constant__ DevPlan P, const StepArgs a) {
    wide::wide_step<0, 0, 512, 128, true>(P, a);
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
// be real GEMMs.  *max_width: the widest hidden layer.
static bool wide_eligible(const pinn::DevPlan& h, int* max_width) {
    if (h.n_layers < 2 || h.n_layers > pinn::wide::MAX_LAYERS) return false;
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

struct PinnPlan {
    PinnSpec spec;
    DevPlan h;
    int device;
    bool wide;                               // the tensor-core tile kernel runs the step
    int wide_kw;                             // its width class: 64 or 128
    StepKernelFn fn_wide;
    MultiKernelFn fn_multi;                  // persistent multi-step kernel, or nullptr when it does not fit
    int multi_threads, multi_smem;
    MultiKernelFn fn_small;                  // tiny-batch (<= 128 points) variant, or nullptr
    int small_smem;
    int wide_ctas;                           // CTAs the tile kernel runs on (<= sm_count)
    const KernelSet* ks;                     // the kernels of this plan's jet set
    StepKernelFn fn_smem, fn_gmem;           // the pair matching this plan (plain or general)
    int sm_count;
    int smem_optin;
    // step kernel launch config
    bool gmem;
    bool wacc_gmem;                          // the per-warp gradient accumulators live in the workspace, not in smem
    int threads, smem_bytes, regs;
    // forward kernel launch config
    bool fwd_gmem;
    bool fwd_wide;                           // pinn_forward runs the 128-wide tile kernel's forward-only form
    int fwd_threads, fwd_smem_bytes, fwd_rows, fwd_row_scr;
};


extern "C" const char* pinn_last_error(void) { return g_err; }
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

// Thread kernel: per-point state in shared memory at the largest warp count that fits, or in the global spill area.
// Every warp has a gradient accumulator of its own: in shared memory when it fits there too, else in the workspace.
static int place_step_kernel(PinnPlan* p) {
    const DevPlan& h = p->h;
    const int n_out_floats = h.n_params + 4;
    const bool has_smem_form = p->fn_smem != nullptr;
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, (const void*)(has_smem_form ? p->fn_smem : p->fn_gmem));
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncGetAttributes: %s", cudaGetErrorString(e));
    p->regs = fa.numRegs;
    const int max_nw = max_warps(fa, p->ks->maxt);
    const int budget = p->smem_optin - (int)fa.sharedSizeBytes - 64;
    int best_nw = 0, best_nwacc = 0;                 // best_nwacc: accumulators in smem (best_nw), or 0 (workspace)
    for (int nw = max_nw; nw >= 1 && !best_nw; --nw) {
        for (int pass = 0; pass < 2 && !best_nw; ++pass) {
            int nwacc = pass == 0 ? nw : 0;
            SmemLayout SL = smem_layout(h.weights_floats, n_out_floats, nwacc, storage_floats(h, h.rows_total, nw));
            if (SL.total_f * 4 <= budget) { best_nw = nw; best_nwacc = nwacc; }
        }
    }
    // PINN_FORCE_MODE=smem|gmem overrides the placement heuristic (experiments only)
    const char* force = getenv("PINN_FORCE_MODE");
    bool use_smem = best_nw >= 4 || (best_nw >= 2 && max_nw <= 4);
    if (force && !strcmp(force, "smem") && best_nw >= 1) use_smem = true;
    if (force && !strcmp(force, "gmem")) use_smem = false;
    if (!has_smem_form) use_smem = false;
    if (use_smem) {
        p->gmem = false; p->threads = best_nw * 32; p->wacc_gmem = best_nwacc == 0;
        SmemLayout SL = smem_layout(h.weights_floats, n_out_floats, best_nwacc, storage_floats(h, h.rows_total, best_nw));
        p->smem_bytes = SL.total_f * 4;
    } else {
        // activations spill to a global workspace; accumulators: in smem if they fit, else in the workspace too
        e = cudaFuncGetAttributes(&fa, (const void*)p->fn_gmem);
        if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncGetAttributes: %s", cudaGetErrorString(e));
        p->regs = fa.numRegs;
        int nw = max_warps(fa, p->ks->maxt);
        { const char* e2 = getenv("PINN_GMEM_WARPS"); if (e2 && atoi(e2) >= 1 && atoi(e2) <= nw) nw = atoi(e2); }   // experiments
        int nwacc = nw;
        SmemLayout SL = smem_layout(h.weights_floats, n_out_floats, nwacc, h.n_params);
        if (SL.total_f * 4 > budget) { nwacc = 0; SL = smem_layout(h.weights_floats, n_out_floats, 0, h.n_params); }
        if (SL.total_f * 4 > budget) return fail(PINN_E_UNSUPPORTED, "network too large: %d B of weights do not fit shared memory", SL.total_f * 4);
        p->gmem = true; p->threads = nw * 32; p->wacc_gmem = nwacc == 0; p->smem_bytes = SL.total_f * 4;
    }
    e = allow_max_smem((const void*)(p->gmem ? p->fn_gmem : p->fn_smem), p->smem_optin);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncSetAttribute(smem=%d): %s", p->smem_bytes, cudaGetErrorString(e));
    return PINN_OK;
}

// Forward kernel: eight warps, per-point state in shared memory when it fits, else in the global spill area.
static int place_forward_kernel(PinnPlan* p) {
    const DevPlan& h = p->h;
    const int nw = 8;
    SmemLayout SL = smem_layout(h.weights_floats, 0, 0, storage_floats(h, p->fwd_rows, nw));
    if (SL.total_f * 4 <= p->smem_optin - 64) { p->fwd_gmem = false; }
    else { p->fwd_gmem = true; SL = smem_layout(h.weights_floats, 0, 0, h.n_params); }
    p->fwd_threads = nw * 32; p->fwd_smem_bytes = SL.total_f * 4;
    if (p->fwd_smem_bytes > p->smem_optin - 64) return fail(PINN_E_UNSUPPORTED, "network too large for shared memory");
    const cudaError_t e = allow_max_smem((const void*)(p->fwd_gmem ? forward_kernel<true> : forward_kernel<false>), p->smem_optin);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncSetAttribute(fwd): %s", cudaGetErrorString(e));
    return PINN_OK;
}

// Persistent multi-step kernel (small batches): per-point state + parameters + Adam moments in shared memory.  Left
// out when the jet set has none or the network does not fit.
static void place_multi_kernel(PinnPlan* p) {
    p->fn_multi = nullptr; p->multi_threads = 0; p->multi_smem = 0;
    const MultiKernelFn f = p->ks->multi;
    if (!f) return;
    cudaFuncAttributes fm;
    if (cudaFuncGetAttributes(&fm, (const void*)f) == cudaSuccess) {
        const DevPlan& h = p->h;
        const int n_out_floats = h.n_params + 4;
        const int extra = 3 * align4(h.n_params) + align4(n_out_floats);
        const int mbudget = p->smem_optin - (int)fm.sharedSizeBytes - 64;
        for (int nw = max_warps(fm, p->ks->maxt); nw >= 1 && !p->fn_multi; --nw) {
            SmemLayout SL = smem_layout(h.weights_floats, n_out_floats, nw, storage_floats(h, h.rows_total, nw));
            if ((SL.total_f + extra) * 4 <= mbudget) {
                p->fn_multi = f; p->multi_threads = nw * 32;
                p->multi_smem = (SL.total_f + extra) * 4;
            }
        }
        if (p->fn_multi && allow_max_smem((const void*)f, p->smem_optin) != cudaSuccess) p->fn_multi = nullptr;
    }
    (void)cudaGetLastError();
}

// Tiny batches: the (point, unit)-parallel loop kernel, for plain dense chains whose jets fit shared memory.  Left out
// when the jet set has none (more than four directions, orders 3 / 4).
static void place_small_kernel(PinnPlan* p) {
    p->fn_small = nullptr; p->small_smem = 0;
    const MultiKernelFn f = p->ks->small;
    if (!f) return;
    const DevPlan& h = p->h;
    for (int l = 0; l < h.n_layers; ++l) if (h.layer[l].skip_src >= 0 || h.layer[l].post_base >= 0) return;
    const int bytes = small::make_layout(h).total * 4;
    cudaFuncAttributes fs;
    if (cudaFuncGetAttributes(&fs, (const void*)f) == cudaSuccess && bytes <= p->smem_optin - (int)fs.sharedSizeBytes - 64 &&
        allow_max_smem((const void*)f, p->smem_optin) == cudaSuccess) {
        p->fn_small = f; p->small_smem = bytes;
    }
    (void)cudaGetLastError();
}

// Wide networks: the tensor-core tile kernel takes the step (PINN_FORCE_KERNEL=thread|wide|wide128 overrides).
// thread_rc is how the thread kernel's placement (step and forward) went: a network whose weights do not fit its
// shared memory goes to the 128-wide class when that class covers it; otherwise that failure is the plan's.
static int place_wide_kernel(PinnPlan* p, int order, int thread_rc) {
    p->wide = false; p->fn_wide = nullptr; p->wide_ctas = p->sm_count; p->wide_kw = 64; p->fwd_wide = false;
    int mw = 0;
    const char* fk = getenv("PINN_FORCE_KERNEL");
    const bool eligible = order < 3 && wide_eligible(p->h, &mw);
    const bool eligible128 = eligible && mw > 64 && p->ks->wide128;
    // the tile kernel wins from 64-wide layers with many jet channels on (H100 80GB HBM3 at 700 W, cfg5: 21.1 ms
    // vs 32.3 ms per step); for narrower networks the per (unit, channel) operand handling costs as much as the
    // FMA row it replaces, and the CUDA-core kernel keeps them.  Networks of 65-128 units the thread kernel holds
    // stay there: the 128-wide class takes only what the thread kernel refuses.
    bool want = eligible && mw <= 64 && mw >= 48 && (1 + p->spec.nf + p->spec.ns) >= 5;
    int kw = 64;
    if (thread_rc != PINN_OK) { want = eligible128; kw = 128; }
    if (fk && !strcmp(fk, "thread")) want = false;
    if (fk && !strcmp(fk, "wide")) {
        if (!eligible || mw > 64) return fail(PINN_E_UNSUPPORTED, "PINN_FORCE_KERNEL=wide: this network is outside what the tile kernel covers");
        want = true; kw = 64;
    }
    if (fk && !strcmp(fk, "wide128")) {
        if (!eligible128) return fail(PINN_E_UNSUPPORTED, "PINN_FORCE_KERNEL=wide128: this network is outside what the 128-wide tile kernel covers");
        want = true; kw = 128;
    }
    int wide_threads = 512;                     // four threads per point; PINN_WIDE_THREADS=256: two (experiments, 64-wide class)
    { const char* wt = getenv("PINN_WIDE_THREADS"); if (wt && atoi(wt) == 256 && kw == 64) wide_threads = 256; }
    const StepKernelFn f = kw == 128 ? p->ks->wide128 : p->ks->wide[wide_threads == 256 ? 1 : 0];
    if (!want || !f || (thread_rc != PINN_OK && kw != 128)) return thread_rc;
    const int smem = kw == 128 ? wide::Tile<128>::SMEM_BYTES : wide::Tile<64>::SMEM_BYTES;
    cudaError_t e = cudaFuncSetAttribute((const void*)f, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncSetAttribute(wide, smem=%d): %s", smem, cudaGetErrorString(e));
    cudaFuncAttributes fa;
    e = cudaFuncGetAttributes(&fa, (const void*)f);
    if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncGetAttributes(wide): %s", cudaGetErrorString(e));
    p->fn_wide = f;
    p->wide = true; p->wide_kw = kw; p->gmem = true; p->threads = wide_threads; p->wacc_gmem = false;
    p->smem_bytes = smem; p->regs = fa.numRegs;
    if (thread_rc != PINN_OK) {                 // the forward kernel does not hold this network either
        e = cudaFuncSetAttribute((const void*)wide::wide128_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return fail(PINN_E_CUDA, "cudaFuncSetAttribute(wide forward, smem=%d): %s", smem, cudaGetErrorString(e));
        p->fwd_wide = true; p->fwd_gmem = false;
    }
    return PINN_OK;
}

extern "C" int pinn_plan_create(const PinnSpec* s, int device, PinnPlan** out) {
    if (!s || !out) return fail(PINN_E_INVALID, "null argument");
    std::unique_ptr<PinnPlan> p(new (std::nothrow) PinnPlan());
    if (!p) return fail(PINN_E_INVALID, "out of memory");
    {
        char msg[256];
        const int rc = build_dev_plan(s, p->h, p->fwd_rows, p->fwd_row_scr, msg, sizeof(msg));
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
    p->fn_smem = p->ks->step[gen][0];
    p->fn_gmem = p->ks->step[gen][1] ? p->ks->step[gen][1] : p->ks->step[1][1];
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
    // the 128-wide tile kernel, which stages one layer at a time (place_wide_kernel)
    int thread_rc = place_step_kernel(p.get());
    if (thread_rc == PINN_OK) thread_rc = place_forward_kernel(p.get());
    if (thread_rc != PINN_OK && thread_rc != PINN_E_UNSUPPORTED) return thread_rc;
    place_multi_kernel(p.get());
    place_small_kernel(p.get());
    if (int rc = place_wide_kernel(p.get(), order, thread_rc)) return rc;
    *out = p.release();
    return PINN_OK;
}

extern "C" int pinn_plan_destroy(PinnPlan* p) {
    if (!p) return PINN_OK;
    delete p;
    return PINN_OK;
}

static int grid_for(const PinnPlan* p, long long n_points, int threads) {
    long long tiles = (n_points + 31) / 32;
    long long ctas = (tiles + threads / 32 - 1) / (threads / 32);
    if (ctas > p->sm_count) ctas = p->sm_count;
    if (ctas < 1) ctas = 1;
    return (int)ctas;
}

// workspace layout: [ticket: 256 B][partials: sm_count x n_out_floats][accumulators][spill]; the accumulators are the
// thread kernel's per-warp gradient accumulators (sm_count x warps x n_out_floats) when they do not fit shared memory,
// or the 128-wide tile kernel's hidden->hidden weight gradients (sm_count x 4 x 128 x 128, 256 KB per CTA)
static size_t ws_partials_off() { return 256; }
static size_t ws_wacc_off(const PinnPlan* p) {
    size_t b = ws_partials_off() + (size_t)p->sm_count * (p->h.n_params + 4) * sizeof(float);
    return (b + 255) & ~(size_t)255;
}
static size_t ws_wacc_bytes(const PinnPlan* p) {
    if (p->wide) return p->wide_kw == 128 ? (size_t)p->sm_count * wide::Tile<128>::WACC_FLOATS * sizeof(float) : 0;
    return p->wacc_gmem ? (size_t)p->sm_count * (p->threads / 32) * (p->h.n_params + 4) * sizeof(float) : 0;
}
static size_t ws_spill_off(const PinnPlan* p) {
    size_t b = ws_wacc_off(p) + ws_wacc_bytes(p);
    return (b + 255) & ~(size_t)255;
}

extern "C" size_t pinn_workspace_bytes(const PinnPlan* p, int64_t n_points) {
    if (!p) return 0;
    size_t b = ws_spill_off(p);
    size_t spill = 0;
    if (p->wide) spill = (size_t)p->sm_count * pinn::wide::spill_floats_per_cta(p->h.n_layers, 1 + p->h.nf + p->h.ns) * sizeof(float);
    else if (p->gmem) spill = (size_t)p->sm_count * (p->threads / 32) * p->h.rows_total * RS * sizeof(float);
    if (p->fwd_gmem) {
        size_t f = (size_t)p->sm_count * (p->fwd_threads / 32) * p->fwd_rows * RS * sizeof(float);
        if (f > spill) spill = f;
    }
    (void)n_points;
    return b + spill;
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

// PINN_PDL=1 launches the step kernels with programmatic stream serialization (the kernel itself waits for its
// predecessor, griddepcontrol.wait, before it reads anything the predecessor wrote).  Graph-replayed steps (what
// `fit` runs) have no launch gap for it to hide, so it stays opt-in.
static int launch_step(StepKernelFn fn, int grid, int threads, int smem_bytes, cudaStream_t st, const DevPlan& plan,
                       const StepArgs& a) {
    static int pdl = -1;
    if (pdl < 0) { const char* e = getenv("PINN_PDL"); pdl = (e && !strcmp(e, "1")) ? 1 : 0; }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = (size_t)smem_bytes; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, fn, plan, a));
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
    DevPlan plan = p->h;
    if (!points) { int rc = resolve_cols(p, cols, plan.cols); if (rc) return rc; }
    StepArgs a;
    a.params = params; a.points = points; a.seed = seed;
    a.step_ptr = step_counter; a.step_val = step_value; a.point_offset = point_offset;
    a.n_points = n_points; a.inv_n = inv_global_n; a.out = grads_and_loss; a.residual = residual_out;
    a.ticket = reinterpret_cast<unsigned int*>(workspace);
    a.partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws_partials_off());
    a.spill = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws_spill_off(p));
    a.wacc = ws_wacc_bytes(p) ? reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws_wacc_off(p)) : nullptr;
    a.rows_total = p->h.rows_total;
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
    if (p->wide) {
        const int T = p->wide_kw == 128 ? wide::Tile<128>::T : wide::Tile<64>::T;
        long long tiles = (n_points + T - 1) / T;
        int max_ctas = p->wide_ctas;
        { const char* e = getenv("PINN_WIDE_CTAS"); if (e && atoi(e) >= 1 && atoi(e) <= p->sm_count) max_ctas = atoi(e); }   // experiments
        const int grid = (int)(tiles < max_ctas ? tiles : max_ctas);
        return launch_step(p->fn_wide, grid, p->threads, p->smem_bytes, st, plan, a);
    }
    const int grid = grid_for(p, n_points, p->threads);
    StepKernelFn fn = p->gmem ? p->fn_gmem : p->fn_smem;
    return launch_step(fn, grid, p->threads, p->smem_bytes, st, plan, a);
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
    return (p && p->fn_multi) ? 4096 : ((p && p->fn_small) ? 8 * pinn::small::BP : 0);
}

extern "C" int pinn_multi_step(const PinnPlan* cp, float* params, float* exp_avg, float* exp_avg_sq, const float* mask,
                               float* step_tensors, int n_step_tensors, const float* points, const PinnColumn* cols,
                               uint64_t seed, uint64_t* step_counter, int64_t n_points, int k_steps,
                               float lr, float beta1, float beta2, float eps, float weight_decay, float opt_step0,
                               float* losses_ring, int64_t ring_len, void* stream) {
    PinnPlan* p = const_cast<PinnPlan*>(cp);
    if (!p || !params || !exp_avg || !exp_avg_sq || !mask || !step_counter || !losses_ring)
        return fail(PINN_E_INVALID, "null argument");
    if (!p->fn_multi && !p->fn_small) return fail(PINN_E_UNSUPPORTED, "the persistent multi-step kernels do not fit this network in shared memory");
    if (n_points <= 0 || n_points > pinn_multi_step_max_points(p) || k_steps <= 0 || ring_len <= 0 || n_step_tensors < 0)
        return fail(PINN_E_INVALID, "pinn_multi_step: n_points %lld (1..%d), k_steps %d", (long long)n_points, pinn_multi_step_max_points(p), k_steps);
    if (!aligned16(params)) return fail(PINN_E_ALIGN, "params must be 16-byte aligned");
    DevPlan plan = p->h;
    if (!points) { int rc = resolve_cols(p, cols, plan.cols); if (rc) return rc; }
    MultiArgs a;
    a.params = params; a.exp_avg = exp_avg; a.exp_avg_sq = exp_avg_sq; a.mask = mask;
    a.step_tensors = step_tensors; a.n_step_tensors = n_step_tensors; a.points = points; a.seed = seed;
    a.step_counter = reinterpret_cast<unsigned long long*>(step_counter);
    a.n_points = n_points; a.inv_n = 1.0f / (float)n_points; a.k_steps = k_steps;
    a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay; a.opt_step0 = opt_step0;
    a.losses_ring = losses_ring; a.ring_len = ring_len;
    a.rows_total = p->h.rows_total;
    // batches of at most 128 points: the (point, unit)-parallel kernel (PINN_MULTI_KERNEL=tile forces the other one)
    const char* mk = getenv("PINN_MULTI_KERNEL");
    const bool small_ok = p->fn_small && n_points <= 8 * pinn::small::BP && (n_points <= 256 || !p->fn_multi) &&
                          !(mk && !strcmp(mk, "tile") && p->fn_multi);
    if (small_ok) {
        // a cluster of up to 8 CTAs (8 SMs) shares the batch, ~16 points per CTA at least; PINN_SMALL_CLUSTER overrides
        int nc = (int)((n_points + 15) / 16);
        if (nc > 8) nc = 8;
        { const char* e = getenv("PINN_SMALL_CLUSTER"); if (e && atoi(e) >= 1 && atoi(e) <= 8) nc = atoi(e); }
        while ((n_points + nc - 1) / nc > pinn::small::BP) ++nc;
        if (nc == 3) nc = 4; else if (nc > 4 && nc < 8) nc = 8;         // cluster sizes 1, 2, 4, 8
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3(nc); cfg.blockDim = dim3(pinn::small::NT); cfg.dynamicSmemBytes = p->small_smem;
        cfg.stream = (cudaStream_t)stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = nc; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        CUDA_TRY(cudaLaunchKernelEx(&cfg, p->fn_small, plan, a));
    } else {
        p->fn_multi<<<1, p->multi_threads, p->multi_smem, (cudaStream_t)stream>>>(plan, a);
    }
    CUDA_TRY(cudaGetLastError());
    return PINN_OK;
}

extern "C" int pinn_forward(const PinnPlan* p, const float* params, const float* points, int64_t n_points,
                            float* u_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!p || !params || !points || !u_out || !workspace) return fail(PINN_E_INVALID, "null argument");
    if (n_points <= 0) return fail(PINN_E_INVALID, "n_points must be positive");
    if (!aligned16(params) || !aligned16(workspace)) return fail(PINN_E_ALIGN, "params / workspace must be 16-byte aligned");
    if (((uintptr_t)points) & 3u) return fail(PINN_E_ALIGN, "points must be 4-byte aligned");
    if (workspace_bytes < pinn_workspace_bytes(p, n_points)) return fail(PINN_E_WORKSPACE, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    if (p->fwd_wide) {                         // u of every point goes to `out` of the step arguments
        StepArgs w;
        memset(&w, 0, sizeof(w));
        w.params = params; w.points = points; w.n_points = n_points; w.out = u_out; w.ring_len = 1;
        const long long tiles = (n_points + wide::Tile<128>::T - 1) / wide::Tile<128>::T;
        const int grid = (int)(tiles < p->sm_count ? tiles : p->sm_count);
        return launch_step(wide::wide128_forward_kernel, grid, 512, wide::Tile<128>::SMEM_BYTES, st, p->h, w);
    }
    FwdArgs a;
    a.params = params; a.points = points; a.n_points = n_points; a.u_out = u_out;
    a.spill = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ws_spill_off(p));
    a.rows_total = p->fwd_rows; a.row_scr = p->fwd_row_scr;
    const int grid = grid_for(p, n_points, p->fwd_threads);
    if (p->fwd_gmem) forward_kernel<true><<<grid, p->fwd_threads, p->fwd_smem_bytes, st>>>(p->h, a);
    else             forward_kernel<false><<<grid, p->fwd_threads, p->fwd_smem_bytes, st>>>(p->h, a);
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
    info->threads_per_cta = p->threads; info->ctas_per_sm = 1;
    info->activations_in_smem = p->gmem ? 0 : 1;
    info->tensor_core = p->wide ? (p->wide_kw == 128 ? 2 : 1) : 0;
    info->small_batch_points = p->fn_small ? 8 * pinn::small::BP : 0;
    info->smem_bytes = p->smem_bytes; info->regs_per_thread = p->regs; info->sm_count = p->sm_count;
    info->rows_per_point = p->h.rows_total;
    info->flops_per_point = 6ll * C * macs;
    info->bytes_per_point = 4 * p->h.total;
    return PINN_OK;
}
