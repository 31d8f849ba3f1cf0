// pinn_wide_kernel.cuh — the fit step for WIDE networks (hidden widths up to 128) on Hopper tensor cores.
//
// The thread-per-point kernel (pinn_step_kernel.cuh) runs every matrix product of the step on CUDA cores and has
// to keep `units x channels` floats of state per point; for a 64-wide network carrying 9 jet channels that is
// 2 300 floats per point and it does not fit on the SM.  Here the same step (reference pydens/model_torch.py:430-460:
// forward of ConvBlockModel :170-172 with the nested D() derivatives :174-178 carried as jet channels, ansatz
// :107-128, MSE :448, loss.backward() :460) is organised around warp-level tensor-core MMAs (mma.sync m16n8k8 tf32).
// Two width classes share one body (wide_step): KW = 64 (wide_step_kernel) and KW = 128 (wide128_step_kernel, for
// networks whose weights the thread kernel cannot hold in shared memory); the tile is T = 8192 / KW points.
//
//   * CTA tile = T collocation points (128 or 64); 512 threads: thread (p, part) owns point p and 16 of the KW hidden
//     units, so every per-(point, unit) quantity is thread-private (KW = 64 at 256 threads: 32 units each).
//   * Every hidden->hidden product, for every jet channel c, is one GEMM  Z_c[T x KW] = A_c[T x KW] . W^T
//     with A_c written row-per-thread into shared memory, W staged [n][k] in shared memory (one layer at a time), and
//     Z_c written back to shared memory, where the thread of each point reads its row.  The 16 x 32 blocks (16 of them
//     in both classes) are dealt to the warps.  Operands are split hi/lo as they are loaded and multiplied as 3xTF32
//     (lo.hi + hi.lo + hi.hi): fp32 grade — single-pass TF32 (7e-4 relative) cannot hold the 1e-4 bar.
//   * The reverse sweep is the same machinery: the data gradient  abar_{h-1} = delta_h . W  is again such a GEMM,
//     and EVERY reduction over points — weight gradients  Wbar = sum_p delta^T a  (M = KW output units, N = KW input
//     units, K = the T points of the tile, both operands read transposed from the same row-per-point buffers),
//     bias gradients, the first layer's and the output layer's weight gradients (small-N GEMMs against a
//     [16 x T] right-hand side) — runs on the tensor cores.  Each accumulator block belongs to one warp, which adds a
//     tile's product into an accumulator that lives for the whole kernel: no shuffles, no atomics, a fixed summation
//     order.  The accumulators are in shared memory, except the hidden->hidden weight gradients of the 128-wide class
//     (4 x 64 KB), which are in this CTA's area of the workspace.  They are read out once at the end of the kernel.
//   * Between the GEMMs the per-point state (a, z_d, z_dd per unit and channel) lives in a per-CTA slab of global
//     memory that is written and re-read by the same thread (L2-resident working set), T x KW floats per (channel,
//     level); the adjoint of a level overwrites the dead slot of the level above.
//   * wide128_forward_kernel is the forward-only form of the 128-wide class (pinn_forward): the value channel's
//     forward sweep and the ansatz, no slab.
//
// Covered: dense chains 'fa…f' with tanh / sigmoid / identity hidden activations, 2 to 6 linear layers (MAX_LAYERS),
// the jet sets NS <= NF <= 4, every ansatz / residual program / sampler the thread kernel covers; hidden widths <= 64
// (tests/test_gpu_tile.py) or <= 128 with at least one above 64 (tests/test_gpu_tile128.py).  Everything else
// (residual layouts, sin/softplus/SiLU/GELU, wider layers, more layers, orders 3 / 4) stays on the thread kernels.
#pragma once

#include "pinn_step_kernel.cuh"

namespace pinn {
namespace wide {

constexpr int NT_MAX = 512;            // threads per CTA (template NT = 256 or 512): thread = (point, 1/NH of the hidden units)
constexpr int MAX_LAYERS = 6;          // linear layers (hidden levels H <= 5, hidden->hidden layers <= 4)
constexpr int TILE_FLOATS = 8192;      // points per tile x padded width: the same for both width classes

__host__ __device__ constexpr int ilog2(int x) { return x <= 1 ? 0 : 1 + ilog2(x >> 1); }

// The geometry of one width class KW (padded hidden width, 64 or 128).  The tile shrinks as the width grows,
// T = 8192 / KW points, so that every [T][KW] operand, the slab block of a (level, channel) and the work-item count
// of the data-gradient GEMM stay the same size; a thread still owns 16 hidden units at 512 threads.
template <int KW_>
struct Tile {
    static constexpr int KW = KW_;
    static constexpr int T = TILE_FLOATS / KW;             // points per tile: 128 (KW = 64) or 64 (KW = 128)
    static constexpr int KSH = ilog2(KW), TSH = ilog2(T);
    static constexpr int LDS = KW + 4;                     // row stride (floats) of the [row][KW] operands: conflict-free fragment loads
    static constexpr int LXB = T + 4;                      // row stride of the small right-hand sides [16][T p]
    // the weight gradients of the hidden->hidden layers [4][KW j][KW m]: in shared memory at KW = 64; at KW = 128
    // (256 KB) in this CTA's area of the workspace
    static constexpr int WACC_FLOATS = (MAX_LAYERS - 2) * KW * KW;
    static constexpr bool WACC_SMEM = KW == 64;

    // ---- shared memory map (bytes) -----------------------------------------------------------------------------
    static constexpr int S_W = 0;                          // layer weights as B operand [KW n][LDS]
    static constexpr int S_A = S_W + KW * LDS * 4;         // A operand [T p][LDS]: jets (forward), delta (reverse)
    static constexpr int S_GB = S_A + T * LDS * 4;         // weight-gradient B operand: post-activation a_{h-1} [T p][LDS]
    static constexpr int S_D = S_GB + T * LDS * 4;         // GEMM result [T p][LDS]
    static constexpr int S_X = S_D + T * LDS * 4;          // exchange area between the threads of a point [24][T]
    static constexpr int S_XB = S_X + 24 * T * 4;          // small right-hand sides [16 rows][LXB]
    static constexpr int S_WACC = S_XB + 16 * LXB * 4;     // hidden->hidden weight gradients (KW = 64 only)
    static constexpr int S_SMALL1 = S_WACC + (WACC_SMEM ? WACC_FLOATS * 4 : 0);  // level 1: first-layer W / b gradients [KW k][16]
    static constexpr int S_OUT = S_SMALL1 + KW * 16 * 4;   // output-layer weight gradient [KW k][8]
    static constexpr int S_SMALLH = S_OUT + KW * 8 * 4;    // level h >= 2: bias gradient of layer h-1 [4][KW j][8]
    static constexpr int S_MISC = S_SMALLH + (MAX_LAYERS - 2) * KW * 8 * 4;   // biases, first-layer weights, scalars
    static constexpr int MISC_FLOATS = 24 * KW;
    static constexpr int SMEM_BYTES = S_MISC + MISC_FLOATS * 4;
    static constexpr int ACC_FLOATS = (S_MISC - S_WACC) / 4;   // every shared-memory accumulator, zeroed once per launch

    // misc area (float offsets)
    static constexpr int M_BIAS = 0;                           // [MAX_LAYERS][KW]
    static constexpr int M_W0 = M_BIAS + MAX_LAYERS * KW;      // first layer [KW][8]
    static constexpr int M_WD = M_W0 + KW * 8;                 // first layer applied to the direction vectors [6][KW]
    static constexpr int M_WOUT = M_WD + PINN_MAX_DIRS * KW;   // output layer weights [KW]
    static constexpr int M_SCAL = M_WOUT + KW;                 // per warp: loss, sbar, bout, vbar[4]  (8 floats each)
    static constexpr int M_END = M_SCAL + 8 * (NT_MAX / 32);

    static_assert(KW == 64 || KW == 128, "width classes");
    static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one CTA");
    static_assert(M_END <= MISC_FLOATS, "misc area");
};

// Split x into a TF32 high part and a TF32 remainder (3xTF32 products).
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(x - __uint_as_float(hi)));
}
__device__ __forceinline__ float tf32_rn(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// d += a . b as 3xTF32, small terms first
__device__ __forceinline__ void mma3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                     uint32_t bh0, uint32_t bh1, uint32_t bl0, uint32_t bl1) {
    mma_tf32(d, al, bh0, bh1);
    mma_tf32(d, ah, bl0, bl1);
    mma_tf32(d, ah, bh0, bh1);
}

// The slab block of one (level, channel) is laid out [k / 4][point][k % 4]: the 16-byte loads of a warp's 32
// points are contiguous (4 cache lines per request instead of 32 with one 256-byte row per point).
// `blk` points at this thread's first float4 of the block; units k0 .. k0+7 are two float4, T*4 floats apart.
template <int T>
__device__ __forceinline__ void ld8(const float* __restrict__ blk, int k0, float (&v)[8]) {
    const float* q = blk + (size_t)(k0 >> 2) * (T * 4);
    const float4 a = *reinterpret_cast<const float4*>(q), b = *reinterpret_cast<const float4*>(q + T * 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <int T>
__device__ __forceinline__ void st8(float* __restrict__ blk, int k0, const float (&v)[8]) {
    float* q = blk + (size_t)(k0 >> 2) * (T * 4);
    *reinterpret_cast<float4*>(q) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(q + T * 4) = make_float4(v[4], v[5], v[6], v[7]);
}
// units k0..k0+7 of row p of a [T][LDS] shared-memory operand
template <int LDS>
__device__ __forceinline__ void st_row8(uint8_t* base, int p, int k0, const float (&v)[8]) {
    float* q = reinterpret_cast<float*>(base) + p * LDS + k0;
    *reinterpret_cast<float4*>(q) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(q + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
template <int LDS>
__device__ __forceinline__ void ld_row8(const uint8_t* base, int p, int k0, float (&v)[8]) {
    const float* q = reinterpret_cast<const float*>(base) + p * LDS + k0;
    const float4 a = *reinterpret_cast<const float4*>(q), b = *reinterpret_cast<const float4*>(q + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__host__ __device__ inline int rup(int x, int m) { return (x + m - 1) / m * m; }
// Slab blocks per CTA: level 1 keeps only its activations (its first-order jets do not depend on the point, its
// second-order jets vanish), levels 2..H keep all C channels; the adjoint of level h-1 overwrites the dead slot (h, c).
// A block is T x KW floats, the same in both width classes.
__host__ __device__ inline size_t spill_floats_per_cta(int n_layers, int C) {
    const int upper = n_layers - 2 > 0 ? n_layers - 2 : 0;
    return (size_t)(1 + upper * C) * TILE_FLOATS;
}

// Stage one layer's weights as the B operand of a GEMM ([n][k], zero padded to KW x KW).
//   forward  (transpose = false): B[n = out unit j][k = in unit m] = W[j][m]
//   backward (transpose = true) : B[n = in unit m][k = out unit j] = W[j][m]
template <int KW>
__device__ __forceinline__ void stage_layer(uint8_t* smem, const float* __restrict__ params, const DevLayer& L, bool transpose) {
    using G = Tile<KW>;
    float* w_s = reinterpret_cast<float*>(smem + G::S_W);
    for (int i = threadIdx.x; i < KW * KW; i += blockDim.x) {
        const int n = i >> G::KSH, k = i & (KW - 1);
        const int j = transpose ? k : n, m = transpose ? n : k;
        w_s[n * G::LDS + k] = (j < L.n_out && m < L.n_in) ? __ldg(params + L.w_off + j * L.n_in + m) : 0.0f;
    }
}

// Fragment coordinates of mma.m16n8k8: g = row group, t = thread in group.
// Columns [0, np) of  D[T x np] = A[T x kp] . B[np x kp]^T  (A, D: [T][LDS], B: [KW][LDS]).
// Work items (16-row block, 32-column block: T/16 x KW/32 = 16 of them) are dealt to the warps.
template <int KW>
__device__ __forceinline__ void gemm_rows(const uint8_t* smem, int kp, int np, int warp, int n_warps) {
    using G = Tile<KW>;
    constexpr int LDS = G::LDS, CB = KW / 32;
    const float* A = reinterpret_cast<const float*>(smem + G::S_A);
    const float* B = reinterpret_cast<const float*>(smem + G::S_W);
    float* D = reinterpret_cast<float*>(const_cast<uint8_t*>(smem) + G::S_D);
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    for (int item = warp; item < (G::T / 16) * CB; item += n_warps) {
        const int r0 = (item >> ilog2(CB)) * 16, c0 = (item & (CB - 1)) * 32;
        if (c0 >= np) continue;
        float acc[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[nt][i] = 0.0f;
        for (int k0 = 0; k0 < kp; k0 += 8) {
            const float* pa = A + (r0 + g) * LDS + k0 + t;
            uint32_t ah[4], al[4];
            split_tf32(pa[0], ah[0], al[0]);
            split_tf32(pa[8 * LDS], ah[1], al[1]);
            split_tf32(pa[4], ah[2], al[2]);
            split_tf32(pa[8 * LDS + 4], ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                if (c0 + nt * 8 < np) {
                    const float* pb = B + (c0 + nt * 8 + g) * LDS + k0 + t;
                    uint32_t bh0, bl0, bh1, bl1;
                    split_tf32(pb[0], bh0, bl0);
                    split_tf32(pb[4], bh1, bl1);
                    mma3(acc[nt], ah, al, bh0, bh1, bl0, bl1);
                }
            }
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            if (c0 + nt * 8 < np) {
                float* pd = D + (r0 + g) * LDS + c0 + nt * 8 + 2 * t;
                *reinterpret_cast<float2*>(pd) = make_float2(acc[nt][0], acc[nt][1]);
                *reinterpret_cast<float2*>(pd + 8 * LDS) = make_float2(acc[nt][2], acc[nt][3]);
            }
        }
    }
}
// ACC[KW j x KW m] (row stride KW) += GA^T . GB over the T points of the tile (GA = S_A, GB = S_GB, both
// [T p][LDS]); rows j < mrows and columns m < ncols.  Work items: 16 x 16 blocks.  ACC is in shared memory
// (KW = 64) or in the workspace (KW = 128); either way each block has one owning warp, which adds the tiles in order.
template <int KW>
__device__ __forceinline__ void gemm_wgrad(uint8_t* smem, float* acc_s, int mrows, int ncols, int warp, int n_warps) {
    using G = Tile<KW>;
    constexpr int LDS = G::LDS, MB = KW / 16;
    const float* GA = reinterpret_cast<const float*>(smem + G::S_A);
    const float* GB = reinterpret_cast<const float*>(smem + G::S_GB);
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    for (int item = warp; item < MB * MB; item += n_warps) {
        const int j0 = (item >> ilog2(MB)) * 16, m0 = (item & (MB - 1)) * 16;
        if (j0 >= mrows || m0 >= ncols) continue;
        float acc[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[nt][i] = 0.0f;
#pragma unroll 2
        for (int p0 = 0; p0 < G::T; p0 += 8) {
            const float* pa = GA + (p0 + t) * LDS + j0 + g;
            uint32_t ah[4], al[4];
            split_tf32(pa[0], ah[0], al[0]);
            split_tf32(pa[8], ah[1], al[1]);
            split_tf32(pa[4 * LDS], ah[2], al[2]);
            split_tf32(pa[4 * LDS + 8], ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                const float* pb = GB + (p0 + t) * LDS + m0 + nt * 8 + g;
                uint32_t bh0, bl0, bh1, bl1;
                split_tf32(pb[0], bh0, bl0);
                split_tf32(pb[4 * LDS], bh1, bl1);
                mma3(acc[nt], ah, al, bh0, bh1, bl0, bl1);
            }
        }
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            float* q = acc_s + (j0 + g) * KW + m0 + nt * 8 + 2 * t;
            q[0] += acc[nt][0]; q[1] += acc[nt][1];
            q[8 * KW] += acc[nt][2]; q[8 * KW + 1] += acc[nt][3];
        }
    }
}
// ACC[KW j x n] (row stride n) += GA^T . XB^T over the tile (XB: [16 rows][LXB]), n = 8 or 16.  The work items
// (16 x 8 blocks) are dealt from the last warp down, so that they land beside the items of gemm_wgrad.
template <int KW>
__device__ __forceinline__ void gemm_small(uint8_t* smem, float* acc_s, int n, int warp, int n_warps) {
    using G = Tile<KW>;
    constexpr int LDS = G::LDS, MB = KW / 16;
    const float* GA = reinterpret_cast<const float*>(smem + G::S_A);
    const float* XB = reinterpret_cast<const float*>(smem + G::S_XB);
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int n_items = MB * (n >> 3);
    for (int item = n_warps - 1 - warp; item < n_items; item += n_warps) {
        const int j0 = (item & (MB - 1)) * 16, r0 = (item >> ilog2(MB)) * 8;
        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 2
        for (int p0 = 0; p0 < G::T; p0 += 8) {
            const float* pa = GA + (p0 + t) * LDS + j0 + g;
            uint32_t ah[4], al[4];
            split_tf32(pa[0], ah[0], al[0]);
            split_tf32(pa[8], ah[1], al[1]);
            split_tf32(pa[4 * LDS], ah[2], al[2]);
            split_tf32(pa[4 * LDS + 8], ah[3], al[3]);
            const float* pb = XB + (r0 + g) * G::LXB + p0 + t;
            uint32_t bh0, bl0, bh1, bl1;
            split_tf32(pb[0], bh0, bl0);
            split_tf32(pb[4], bh1, bl1);
            mma3(acc, ah, al, bh0, bh1, bl0, bl1);
        }
        float* q = acc_s + (j0 + g) * n + r0 + 2 * t;
        q[0] += acc[0]; q[1] += acc[1];
        q[8 * n] += acc[2]; q[8 * n + 1] += acc[3];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// The body of the kernels below.  KW: the width class (hidden widths <= 64 or <= 128).  FWD: the forward-only form
// (pinn_forward), with NF = NS = 0: forward sweep of the value channel, ansatz, u of every point to a.out; no slab, no
// reverse sweep.
template <int NF, int NS, int NT, int KW, bool FWD>
__device__ __forceinline__ void wide_step(const DevPlan& P, const StepArgs a) {
    using G = Tile<KW>;
    constexpr int T = G::T, LDS = G::LDS, LXB = G::LXB;
    constexpr int C = 1 + NF + NS;
    constexpr int NH = NT / T;               // threads per point: each owns KW / NH hidden units
    constexpr int QN = KW / NH / 8;          // 8-unit chunks per thread
    static_assert(NH * T == NT && QN * 8 * NH == KW, "threads per point");
    static_assert(!FWD || (NF == 0 && NS == 0), "the forward-only form carries the value channel only");
    extern __shared__ __align__(16) uint8_t smem[];
    float* misc = reinterpret_cast<float*>(smem + G::S_MISC);

    const int tid = threadIdx.x, p = tid & (T - 1), kh = tid >> G::TSH, warp = tid >> 5, lane = tid & 31;
    const int warp_u = __shfl_sync(0xffffffffu, tid >> 5, 0);        // the same number, provably warp-uniform
    const int Ln = P.n_layers, H = Ln - 1;
    const int n_out_floats = P.n_params + 4;
    // hidden->hidden weight-gradient accumulators [4][KW][KW]: shared memory, or this CTA's area of the workspace
    float* const wacc_base = G::WACC_SMEM ? reinterpret_cast<float*>(smem + G::S_WACC)
                                          : a.wacc + (size_t)blockIdx.x * G::WACC_FLOATS;

    pdl_wait();                                    // the previous step (its parameter update) is complete and visible
    pdl_launch_dependents();
    // ---- one-time setup: constants, zeroed accumulators -----------------------------------------------------------
    for (int i = tid; i < G::MISC_FLOATS; i += NT) misc[i] = 0.0f;
    for (int i = tid; i < 16 * LXB; i += NT) reinterpret_cast<float*>(smem + G::S_XB)[i] = 0.0f;
    for (int i = tid; i < G::ACC_FLOATS; i += NT) reinterpret_cast<float*>(smem + G::S_WACC)[i] = 0.0f;
    if constexpr (!G::WACC_SMEM && !FWD) {
        const int n4 = (Ln > 2 ? Ln - 2 : 0) * KW * KW / 4;          // the layers in use
        for (int i = tid; i < n4; i += NT) reinterpret_cast<float4*>(wacc_base)[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    __syncthreads();
    {
        // biases of every layer, first-layer weights and their products with the direction vectors, output weights
        for (int l = 0; l < Ln; ++l)
            for (int j = tid; j < P.layer[l].n_out; j += NT) misc[G::M_BIAS + l * KW + j] = __ldg(a.params + P.layer[l].b_off + j);
        const DevLayer& L0 = P.layer[0];
        for (int i = tid; i < L0.n_out * L0.n_in; i += NT) misc[G::M_W0 + (i / L0.n_in) * 8 + (i % L0.n_in)] = __ldg(a.params + L0.w_off + i);
        for (int i = tid; i < NF * KW; i += NT) {
            const int d = i >> G::KSH, k = i & (KW - 1);
            float sum = 0.0f;
            if (k < L0.n_out) for (int q = 0; q < L0.n_in; ++q) sum = fmaf(__ldg(a.params + L0.w_off + k * L0.n_in + q), P.dir_vec[d][q], sum);
            misc[G::M_WD + d * KW + k] = sum;
        }
        for (int k = tid; k < P.layer[H].n_in; k += NT) misc[G::M_WOUT + k] = __ldg(a.params + P.layer[H].w_off + k);
    }
    __syncthreads();

    // ---- per-thread views ----------------------------------------------------------------------------------------
    float* slab = a.spill + (size_t)blockIdx.x * spill_floats_per_cta(Ln, C);
    auto row = [&](int h, int c) -> float* {                 // block of (level h, channel c), at this thread's point
        const int b = (h == 1) ? 0 : 1 + (h - 2) * C + c;    // level 1 keeps channel 0 only
        return slab + (size_t)b * (T * KW) + p * 4;
    };
    float* Xbuf = reinterpret_cast<float*>(smem + G::S_X);      // exchange area between the threads of a point
    float* xb = reinterpret_cast<float*>(smem + G::S_XB);       // small right-hand sides [16][LXB]
    float* st = reinterpret_cast<float*>(smem + G::S_A) + p;    // ansatz / program scratch rows (stride T), A/GB area
    constexpr int RS = T;
    const int kbeg = kh * (KW / NH);

    const uint64_t step = a.step_ptr ? *a.step_ptr : a.step_val;
    const long long n_tiles = (a.n_points + T - 1) / T;
    float acc_loss = 0.0f, acc_sbar = 0.0f, acc_bout = 0.0f, acc_vbar[PINN_MAX_VARS];
#pragma unroll
    for (int i = 0; i < PINN_MAX_VARS; ++i) acc_vbar[i] = 0.0f;

    // One MMA phase: everybody's operand writes are complete -> every warp computes its share of the GEMMs (each
    // accumulator block belongs to exactly one warp, so the summation order is fixed) -> the results are visible.
    auto sync_issue = [&](auto&& issue) {
        __syncthreads();
        issue(warp_u);
        __syncthreads();
    };
    // stored jet channel c (>= 1) of level h, units k0..k0+7: level 1 is not stored — its first-order jets are the
    // first layer applied to the direction vectors (the same for every point), its second-order jets vanish
    auto ldz = [&](int h, int c, int k0, float (&v)[8]) {
        if (h == 1) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = (c <= NF) ? misc[G::M_WD + (c - 1) * KW + k0 + i] : 0.0f;
        } else {
            ld8<T>(row(h, c), k0, v);
        }
    };
    // A jet set is walked in GROUPS: group 0 = the value channel; group 1+d = direction d, i.e. its first-order
    // channel x = 1+d and (d < NS) its second-order partner y = 1+NF+d.  A pair shares its loads: both channels are
    // computed in one sweep, one goes to the tensor cores at once, the partner waits in registers (`stash`).
    auto group_x = [&](int g) { return g == 0 ? 0 : g; };
    auto group_y = [&](int g) { return (g >= 1 && g - 1 < NS) ? NF + g : -1; };
    // post-activation jets of group g at level h, units k0..k0+7 (a0 = the level's activations, kept in registers):
    // ax (channel x) and ay (partner, if any)
    auto post_group = [&](int h, int g, int k0, const ActC& kc, const float (&a0)[8], float (&ax)[8], float (&ay)[8]) {
        if (g == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) ax[i] = a0[i];
            return;
        }
        float zd[8];
        ldz(h, g, k0, zd);
        const bool pair = g - 1 < NS;
        float zdd[8];
        if (pair) ldz(h, NF + g, k0, zdd);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float s1 = fmaf(fmaf(kc.c2, a0[i], kc.c1), a0[i], kc.c0);
            ax[i] = s1 * zd[i];
            if (pair) {
                const float s2 = s1 * fmaf(kc.d1, a0[i], kc.d0);
                ay[i] = fmaf(s2 * zd[i], zd[i], s1 * zdd[i]);
            }
        }
    };
    auto put_A = [&](int k0, const float (&v)[8]) { st_row8<LDS>(smem + G::S_A, p, k0, v); };   // A operand of the next GEMM

    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long pl = tile * T + p;
        const bool valid = pl < a.n_points;
        const long long pe = valid ? pl : a.n_points - 1;         // masked lanes replay the last point
        float x[PINN_MAX_DIMS];
#pragma unroll
        for (int k = 0; k < PINN_MAX_DIMS; ++k) x[k] = 0.0f;
        if (a.points) {
            const float* src = a.points + (size_t)pe * P.total;
#pragma unroll
            for (int k = 0; k < PINN_MAX_DIMS; ++k) if (k < P.total) x[k] = __ldg(src + k);
        } else {
            const uint64_t gidx = a.point_offset + (uint64_t)pe;
            Philox4 b0 = philox_block(gidx, step, a.seed, 0u);
            Philox4 b1 = b0;
            if (P.total > 4) b1 = philox_block(gidx, step, a.seed, 1u);
#pragma unroll
            for (int k = 0; k < PINN_MAX_DIMS; ++k) if (k < P.total) x[k] = sample_column(P.cols[k], k, gidx, step, a.seed, b0, b1);
        }

        // =========================== forward ===========================
        // level 1: the first linear layer acts on (x, direction vectors, 0) — per thread, no GEMM; only the
        // activations are stored
        float a0h[QN][8];                                    // activations of the current level, this thread's units
        if (kh == 0) {                                       // the coordinates wait in the exchange area (rows 16..23)
#pragma unroll
            for (int k = 0; k < PINN_MAX_DIMS; ++k) Xbuf[(16 + k) * T + p] = x[k];
        }
        {
            const ActC kc = make_actc(P.layer[0].act);
#pragma unroll
            for (int q = 0; q < QN; ++q) {
                const int k0 = kbeg + q * 8;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float z = misc[G::M_BIAS + k0 + i];
#pragma unroll
                    for (int j = 0; j < PINN_MAX_DIMS; ++j) z = fmaf(misc[G::M_W0 + (k0 + i) * 8 + j], x[j], z);
                    a0h[q][i] = act_store<false>(kc, z);
                }
                if constexpr (!FWD) st8<T>(row(1, 0), k0, a0h[q]);
            }
        }
        // levels 2..H and the output: one GEMM per channel
        float N[C];
        for (int h = 1; h <= H; ++h) {
            const DevLayer& L = P.layer[h];                  // maps level h to level h+1 (h == H: the output)
            const int kp = rup(L.n_in, 8), np = rup(L.n_out, 16);
            const ActC kc = make_actc(P.layer[h - 1].act);
            const ActC kn = make_actc(L.act);
            __syncthreads();                                 // nobody reads the previous W any more
            stage_layer<KW>(smem, a.params, L, false);
            float a0n[QN][8];                                // activations of level h+1 as they come out of channel 0
            auto finish = [&](int c) {                       // accumulator -> level h+1 (or the network output)
                if (h < H) {
#pragma unroll
                    for (int q = 0; q < QN; ++q) {
                        const int n0 = kbeg + q * 8;
                        float z[8];
                        if (n0 < np) ld_row8<LDS>(smem + G::S_D, p, n0, z);
                        else {
#pragma unroll
                            for (int i = 0; i < 8; ++i) z[i] = 0.0f;
                        }
                        if (c == 0) {
#pragma unroll
                            for (int i = 0; i < 8; ++i) { z[i] = act_store<false>(kn, z[i] + misc[G::M_BIAS + h * KW + n0 + i]); a0n[q][i] = z[i]; }
                        }
                        if constexpr (!FWD) st8<T>(row(h + 1, c), n0, z);
                    }
                } else {
                    N[c] = reinterpret_cast<const float*>(smem + G::S_D)[p * LDS] + (c == 0 ? misc[G::M_BIAS + H * KW] : 0.0f);
                }
            };
            auto gemm = [&](int w) { gemm_rows<KW>(smem, kp, np, w, NT / 32); };
            for (int g = 0; g <= NF; ++g) {
                const int cy = group_y(g);
                float stash[QN][8];
#pragma unroll
                for (int q = 0; q < QN; ++q) {
                    const int k0 = kbeg + q * 8;
                    float ax[8];
                    post_group(h, g, k0, kc, a0h[q], ax, stash[q]);
                    put_A(k0, ax);
                }
                sync_issue(gemm);
                finish(group_x(g));
                if (cy >= 0) {
#pragma unroll
                    for (int q = 0; q < QN; ++q) put_A(kbeg + q * 8, stash[q]);
                    sync_issue(gemm);
                    finish(cy);
                }
            }
            if (h < H) {
#pragma unroll
                for (int q = 0; q < QN; ++q)
#pragma unroll
                    for (int i = 0; i < 8; ++i) a0h[q][i] = a0n[q][i];
            }
        }
        // a0h now holds the activations of the top level H

        // =========================== ansatz, residual, adjoint seed (one thread per point) ===========================
        __syncthreads();                                     // the A/GB area becomes program scratch
        if (kh == 0) {
            float Nb[C];
            float* coords = st;
            float* scr = st + (size_t)PINN_MAX_DIMS * RS;
#pragma unroll
            for (int k = 0; k < PINN_MAX_DIMS; ++k) coords[(size_t)k * RS] = Xbuf[(16 + k) * T + p];
            float icj[C];
#pragma unroll
            for (int c = 0; c < C; ++c) icj[c] = 0.0f;
            if (P.has_ic) {
                eval_prog(P.ic, P.n_ic, scr, RS, coords, a.params, P.var_off);
#pragma unroll
                for (int c = 0; c < C; ++c) icj[c] = scr[(size_t)P.ic_out[c] * RS];
            }
            const float log_scale = __ldg(a.params + P.log_scale_off);
            AnsatzState<NF, NS> as;
            float u[C];
            ansatz_forward<NF, NS, true>(P, coords, RS, log_scale, N, icj, as, u);
            if constexpr (FWD) {
                if (valid) a.out[pl] = u[0];
            } else {
#pragma unroll
                for (int c = 0; c < C; ++c) scr[(size_t)c * RS] = u[c];
                eval_prog(P.eq, P.n_eq, scr, RS, coords, a.params, P.var_off);
                const float r = scr[(size_t)P.eq_out[0] * RS];
                const float rb = valid ? 2.0f * r * a.inv_n : 0.0f;
                if (valid) acc_loss = fmaf(r * a.inv_n, r, acc_loss);
                if (a.residual && valid) a.residual[pl] = r;
                float ub[C];
#pragma unroll
                for (int c = 0; c < C; ++c) ub[c] = rb * scr[(size_t)P.eq_out[1 + c] * RS];
#pragma unroll
                for (int i = 0; i < PINN_MAX_VARS; ++i)
                    if (i < P.n_vars) acc_vbar[i] = fmaf(rb, scr[(size_t)P.eq_out[1 + C + i] * RS], acc_vbar[i]);
                if (P.ic_has_vars) {
#pragma unroll
                    for (int i = 0; i < PINN_MAX_VARS; ++i) {
                        if (i < P.n_vars) {
#pragma unroll
                            for (int c = 0; c < C; ++c)
                                acc_vbar[i] = fmaf(ub[c], scr[(size_t)P.ic_out[C * (1 + i) + c] * RS], acc_vbar[i]);
                        }
                    }
                }
                acc_sbar += ansatz_adjoint<NF, NS>(P, as, ub, Nb);
                acc_bout += Nb[0];
                // the adjoint seed of the point goes to the exchange area (rows 0..C-1): every thread of the point reads
                // it from there when it needs it, instead of carrying C registers through the reverse sweep
#pragma unroll
                for (int c = 0; c < C; ++c) Xbuf[c * T + p] = Nb[c];
            }
        }
        if constexpr (FWD) continue;                         // the forward-only form ends its tile here
        auto nb_of = [&](int c) { return Xbuf[c * T + p]; };
        __syncthreads();

        // =========================== reverse ===========================
        // the output layer (one unit): its weight gradient  Wbar_out[k] = sum_p sum_c Nb[c] a_{H,c}[k]  is ONE small
        // GEMM of the per-point sums against a column of ones; abar_{H,c}[k] = w_out[k] Nb[c] needs no GEMM at all
        {
            const ActC kc = make_actc(P.layer[H - 1].act);
#pragma unroll
            for (int q = 0; q < QN; ++q) {
                const int k0 = kbeg + q * 8;
                float t[8];
#pragma unroll
                const float nb0 = nb_of(0);
#pragma unroll
                for (int i = 0; i < 8; ++i) t[i] = nb0 * a0h[q][i];
                for (int g = 1; g <= NF; ++g) {
                    float ax[8], ay[8];
                    post_group(H, g, k0, kc, a0h[q], ax, ay);
                    const int cy = group_y(g);
#pragma unroll
                    const float nbx = nb_of(g), nby = cy >= 0 ? nb_of(cy) : 0.0f;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        t[i] = fmaf(nbx, ax[i], t[i]);
                        if (cy >= 0) t[i] = fmaf(nby, ay[i], t[i]);
                    }
                }
                put_A(k0, t);
            }
            if (kh == 0) xb[p] = 1.0f;
            sync_issue([&](int w) { gemm_small<KW>(smem, reinterpret_cast<float*>(smem + G::S_OUT), 8, w, NT / 32); });
        }
        // rounds H..1: adjoint through the activation of level h, then (h >= 2) through the linear layer below it
        for (int h = H; h >= 1; --h) {
            const ActC kc = make_actc(P.layer[h - 1].act);                   // activation of level h
            const ActC kb = make_actc(h >= 2 ? P.layer[h - 2].act : 0);      // activation of level h-1
            const DevLayer& L = P.layer[h - 1];                              // maps level h-1 to level h
            const int kp = rup(L.n_out, 8), np = rup(L.n_in, 16);
            if (h >= 2) {
                __syncthreads();
                stage_layer<KW>(smem, a.params, L, true);
            }
            if (h < H) {                                     // (at the top level the forward sweep left them in registers)
#pragma unroll
                for (int q = 0; q < QN; ++q) ld8<T>(row(h, 0), kbeg + q * 8, a0h[q]);
            }
            float R[QN][8];                                  // running sum of the value-channel adjoint
#pragma unroll
            for (int q = 0; q < QN; ++q)
#pragma unroll
                for (int i = 0; i < 8; ++i) R[q][i] = 0.0f;
            // adjoint of the post-activation jet channel c of level h, units k0..k0+7
            auto ld_ab = [&](int c, int k0, float (&v)[8]) {
                if (h == H) {
                    const float nb = nb_of(c);
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = misc[G::M_WOUT + k0 + i] * nb;
                } else {
                    ld8<T>(row(h + 1, c), k0, v);
                }
            };
            // operands of channel c are in place (A = GA = delta, and for h >= 2 GB = a_{h-1,c})
            auto run = [&](int c) {
                const int d = (c == 0) ? -1 : ((c <= NF) ? c - 1 : c - 1 - NF);
                if (kh == 0) {       // small right-hand side: row 0 = 1 for the value channel (bias gradient); level 1: the inputs
                    xb[p] = (c == 0) ? 1.0f : 0.0f;
                    if (h == 1) {
#pragma unroll
                        for (int i = 0; i < PINN_MAX_DIMS; ++i)
                            if (i < P.total) xb[(1 + i) * LXB + p] = (c == 0) ? Xbuf[(16 + i) * T + p] : ((c <= NF) ? P.dir_vec[d][i] : 0.0f);
                    }
                }
                if (h >= 2) {
                    // every warp takes its share of each GEMM's items: the data gradient (16 x 32 blocks), the
                    // weight gradient (16 x 16 blocks) and, on the value channel, the bias gradient (dealt from the
                    // last warp down)
                    sync_issue([&](int w) {
                        gemm_rows<KW>(smem, kp, np, w, NT / 32);
                        gemm_wgrad<KW>(smem, wacc_base + (h - 2) * KW * KW, L.n_out, L.n_in, w, NT / 32);
                        if (c == 0) gemm_small<KW>(smem, reinterpret_cast<float*>(smem + G::S_SMALLH) + (h - 2) * KW * 8, 8, w, NT / 32);
                    });
                    float* dst = row(h, c);                  // abar_{h-1,c} takes the dead slot of (h, c)
#pragma unroll
                    for (int q = 0; q < QN; ++q) {
                        const int n0 = kbeg + q * 8;
                        float z[8];
                        if (n0 < np) ld_row8<LDS>(smem + G::S_D, p, n0, z);
                        else {
#pragma unroll
                            for (int i = 0; i < 8; ++i) z[i] = 0.0f;
                        }
                        st8<T>(dst, n0, z);
                    }
                } else {                                     // level 1: only the first layer's own gradients
                    sync_issue([&](int w) { gemm_small<KW>(smem, reinterpret_cast<float*>(smem + G::S_SMALL1), 16, w, NT / 32); });
                }
            };
            auto put_ops = [&](int k0, const float (&delta)[8], const float (&below)[8]) {
                put_A(k0, delta);                            // A of the data gradient and GA of the reductions
                if (h >= 2) st_row8<LDS>(smem + G::S_GB, p, k0, below);
            };
            // directions first (pairs: second-order channel, then its first-order partner), the value channel last
            for (int gg = 1; gg <= NF + 1; ++gg) {
                const int g = (gg <= NF) ? gg : 0;
                const int cy = group_y(g);
                float sd[QN][8], sb[QN][8];                  // stash: delta and a_{h-1} of the first-order channel of a pair
#pragma unroll
                for (int q = 0; q < QN; ++q) {
                    const int k0 = kbeg + q * 8;
                    float dx[8], bx[8], by[8];
                    const float (&a0)[8] = a0h[q];
                    if (h >= 2) {
                        float a0l[8];
                        ld8<T>(row(h - 1, 0), k0, a0l);
                        post_group(h - 1, g, k0, kb, a0l, bx, by);
                    }
                    if (g == 0) {
                        float ab[8];
                        ld_ab(0, k0, ab);
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            const float s1 = fmaf(fmaf(kc.c2, a0[i], kc.c1), a0[i], kc.c0);
                            dx[i] = fmaf(s1, ab[i], R[q][i]);
                        }
                        put_ops(k0, dx, bx);
                    } else {
                        float zd[8], abx[8];
                        ldz(h, g, k0, zd);
                        ld_ab(g, k0, abx);
                        if (cy >= 0) {
                            float zdd[8], aby[8], dy[8];
                            ldz(h, cy, k0, zdd);
                            ld_ab(cy, k0, aby);
#pragma unroll
                            for (int i = 0; i < 8; ++i) {
                                const float s1 = fmaf(fmaf(kc.c2, a0[i], kc.c1), a0[i], kc.c0);
                                const float s2 = s1 * fmaf(kc.d1, a0[i], kc.d0);
                                const float s3 = s1 * fmaf(fmaf(kc.e2, a0[i], kc.e1), a0[i], kc.e0);
                                const float t = s2 * zd[i];
                                dy[i] = s1 * aby[i];
                                dx[i] = fmaf(2.0f * t, aby[i], s1 * abx[i]);
                                R[q][i] = fmaf(fmaf(s3 * zd[i], zd[i], s2 * zdd[i]), aby[i], fmaf(t, abx[i], R[q][i]));
                            }
                            put_ops(k0, dy, by);             // the second-order channel goes first
#pragma unroll
                            for (int i = 0; i < 8; ++i) { sd[q][i] = dx[i]; sb[q][i] = bx[i]; }
                        } else {
#pragma unroll
                            for (int i = 0; i < 8; ++i) {
                                const float s1 = fmaf(fmaf(kc.c2, a0[i], kc.c1), a0[i], kc.c0);
                                const float s2 = s1 * fmaf(kc.d1, a0[i], kc.d0);
                                dx[i] = s1 * abx[i];
                                R[q][i] = fmaf(s2 * zd[i], abx[i], R[q][i]);
                            }
                            put_ops(k0, dx, bx);
                        }
                    }
                }
                if (cy >= 0) {
                    if (h >= 2) run(cy);                     // level 1: a second-order channel feeds nothing below
#pragma unroll
                    for (int q = 0; q < QN; ++q) put_ops(kbeg + q * 8, sd[q], sb[q]);
                }
                run(group_x(g));
            }
        }
    }

    if constexpr (FWD) return;

    // ---- read the accumulators out: this CTA's partial [grads | loss] ------------------------------------------------
    float* mine = a.partials + (size_t)blockIdx.x * n_out_floats;
    for (int i = tid; i < n_out_floats; i += NT) mine[i] = 0.0f;
    {
        // per-warp slots, summed in warp order below: no float atomics, bit-reproducible run to run
        float* slot = misc + G::M_SCAL + 8 * warp;
        float v = warp_sum(acc_loss);
        if (lane == 0) slot[0] = v;
        v = warp_sum(acc_sbar);
        if (lane == 0) slot[1] = v;
        v = warp_sum(acc_bout);
        if (lane == 0) slot[2] = v;
#pragma unroll
        for (int i = 0; i < PINN_MAX_VARS; ++i) {
            v = warp_sum(acc_vbar[i]);
            if (lane == 0) slot[3 + i] = v;
        }
    }
    __syncthreads();
    {
        const float* wacc = wacc_base;
        const float* smallh = reinterpret_cast<const float*>(smem + G::S_SMALLH);
        for (int li = 0; li + 2 < Ln; ++li) {               // hidden->hidden layer li+1
            const DevLayer& L = P.layer[li + 1];
            for (int i = tid; i < L.n_out * L.n_in; i += NT)
                mine[L.w_off + i] = wacc[li * KW * KW + (i / L.n_in) * KW + i % L.n_in];
            for (int j = tid; j < L.n_out; j += NT) mine[L.b_off + j] = smallh[li * KW * 8 + j * 8];   // bias gradient
        }
        const float* small1 = reinterpret_cast<const float*>(smem + G::S_SMALL1);   // [j][0] bias, [j][1 + i] weights
        const DevLayer& L0 = P.layer[0];
        for (int j = tid; j < L0.n_out; j += NT) {
            mine[L0.b_off + j] = small1[j * 16];
            for (int i = 0; i < L0.n_in; ++i) mine[L0.w_off + j * L0.n_in + i] = small1[j * 16 + 1 + i];
        }
        const float* outw = reinterpret_cast<const float*>(smem + G::S_OUT);
        const DevLayer& LO = P.layer[H];
        for (int j = tid; j < LO.n_in; j += NT) mine[LO.w_off + j] = outw[j * 8];
    }
    if (tid == 0) {
        float sc[3 + PINN_MAX_VARS];
#pragma unroll
        for (int i = 0; i < 3 + PINN_MAX_VARS; ++i) {
            float t = 0.0f;
            for (int w = 0; w < NT / 32; ++w) t += misc[G::M_SCAL + 8 * w + i];
            sc[i] = t;
        }
        mine[P.n_params] = sc[0];
        mine[P.log_scale_off] = sc[1];
        mine[P.layer[H].b_off] = sc[2];
        for (int i = 0; i < P.n_vars; ++i) mine[P.var_off[i]] = sc[3 + i];
    }
    __syncthreads();
    finish_grid(a, n_out_floats);
}

// hidden widths <= 64: 128-point tiles, NT = 512 (four threads per point) or 256 (two)
template <int NF, int NS, int NT>
__global__ void __launch_bounds__(NT, 1) wide_step_kernel(const __grid_constant__ DevPlan P, const StepArgs a) {
    wide_step<NF, NS, NT, 64, false>(P, a);
}
// hidden widths <= 128: 64-point tiles, eight threads per point
template <int NF, int NS>
__global__ void __launch_bounds__(512, 1) wide128_step_kernel(const __grid_constant__ DevPlan P, const StepArgs a) {
    wide_step<NF, NS, 512, 128, false>(P, a);
}
// pinn_forward of the networks only the 128-wide class holds: u of every point to a.out
__global__ void __launch_bounds__(512, 1) wide128_forward_kernel(const __grid_constant__ DevPlan P, const StepArgs a);

}  // namespace wide
}  // namespace pinn
