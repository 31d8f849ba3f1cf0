// pinn_device.cuh — per-point math of the fused PINN fit step (sm_90a).
//
// Everything in this header is written per THREAD: one thread owns one collocation point and
// walks the whole step for it (MLP forward carrying a Taylor jet, ansatz, residual program,
// hand-derived reverse sweep).  The functions are `__host__ __device__` so the very same code
// can be compiled by g++ into the test-only emulation harness (tests/emul/) and checked against
// the fp64 oracle on a machine without a GPU.  Cross-lane work (the weight-gradient reduction)
// is isolated in emit_entries().
//
// Reference semantics being reproduced (analysiscenter/pydens, pydens/model_torch.py):
//   forward  :170-172 (MLP via batchflow Block) + anzatc :107-128
//   D()      :174-178 — nested autograd.grad == the jet channels carried here
//   loss     :448     — MSE of the residual
//   backward :460     — the reverse sweep below (SURVEY.md §3.3 has the derivation)
#pragma once

#include <stdint.h>
#include <math.h>
#include "../../include/pinn_b200.h"

#if defined(__CUDACC__)
#define PINN_HD __host__ __device__ __forceinline__
#define PINN_D  __device__ __forceinline__
#else
#define PINN_HD inline
#define PINN_D  inline
struct float4 { float x, y, z, w; };      // host emulation build only
struct float2 { float x, y; };
inline float2 make_float2(float x, float y) { float2 r; r.x = x; r.y = y; return r; }
#endif

// Unroll factors of the inner loops for many-channel (C >= 8) problems, whose per-point state lives in global memory.
#ifndef PINN_UNR_WIDE
#define PINN_UNR_WIDE 4
#endif
#ifndef PINN_BWD_UNR_WIDE
#define PINN_BWD_UNR_WIDE 1
#endif

// Pairwise FP32 arithmetic: the inner loops keep their accumulators as pairs of neighbouring output units.
// Hopper has no packed FP32x2 instruction, so each pair is two round-to-nearest scalar operations (the same
// results a packed instruction would give).
#define PINN_FFMA2(a2, s, c2) make_float2(fmaf((a2).x, (s), (c2).x), fmaf((a2).y, (s), (c2).y))
#define PINN_FMUL2(a2, s)     make_float2((a2).x * (s), (a2).y * (s))
#define PINN_FFMA2V(a2, b2, c2) make_float2(fmaf((a2).x, (b2).x, (c2).x), fmaf((a2).y, (b2).y, (c2).y))
#define PINN_FMUL2V(a2, b2)     make_float2((a2).x * (b2).x, (a2).y * (b2).y)

namespace pinn {

// ----------------------------------------------------------------------------------------------
// Device-side plan (lives in global memory, copied to shared memory by every CTA).
// ----------------------------------------------------------------------------------------------
struct DevLayer {
    int n_in, n_out, act;       // act = activation applied to this layer's output
    int w_off, b_off;           // offsets in the flat parameter buffer
    int wt_s;                   // smem float offset of Wt [n_in][n_out_p4]   (forward layout)
    int w_s;                    // smem float offset of W  [n_out_p4][n_in_p8] (reverse layout)
    int b_s;                    // smem float offset of bias [n_out_p4]
    int n_out_p4, n_in_p8;
    int unit_base;              // first unit index of this layer's output buffer (stored jet, later its adjoint)
    int post_base;              // residual layers: unit index of the buffer holding the activated output + skip, else -1
    int skip_src;               // layer whose output is added to this layer's activated output, or -1
    int adj_from;               // this layer feeds the skip of layer `adj_from` (whose post buffer carries the adjoint), or -1
    int pad_[2];
};

struct alignas(16) DevPlan {
    int n_layers;
    int total, ndims, nparams, nsp;     // nsp = number of spatial dims (ndims or ndims-1)
    int has_bc, has_ic;
    int nf, ns;
    int n_params;                       // floats in the flat buffer (multiple of 4)
    int log_scale_off;
    int n_vars;
    int n_eq, n_ic, n_slots;
    int row_units, row_scr, rows_total; // per-point storage rows
    int weights_floats;                 // floats of the smem weight area
    int n_units;
    float bc;
    float t0;
    int dir_col[PINN_MAX_DIRS];                       // unit-vector directions: their column; else -1
    float dir_vec[PINN_MAX_DIRS][PINN_MAX_DIMS];      // direction vectors in point-column space
    int var_off[PINN_MAX_VARS];
    float lo[PINN_MAX_DIMS], hi[PINN_MAX_DIMS], inv_w2[PINN_MAX_DIMS];
    int eq_out[1 + 1 + 2 * PINN_MAX_DIRS + PINN_MAX_VARS];
    int ic_out[(1 + 2 * PINN_MAX_DIRS) * (1 + PINN_MAX_VARS)];
    int ic_has_vars;
    int general;                // 1: residual layouts / non-axis directions / variables in the initial condition present
    PinnColumn cols[PINN_MAX_DIMS];     // sampler columns of the current call
    DevLayer layer[PINN_MAX_LAYERS];
    PinnInstr eq[PINN_MAX_PROG];
    PinnInstr ic[PINN_MAX_PROG];
};

// ----------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11) — counter-based RNG for in-kernel collocation sampling.
// Restated bit-exactly in oracle/philox.py.
// ----------------------------------------------------------------------------------------------
struct Philox4 { uint32_t x, y, z, w; };

PINN_HD uint32_t mulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

PINN_HD Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                              uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = mulhi32(M0, c0), lo0 = M0 * c0;
        uint32_t hi1 = mulhi32(M1, c2), lo1 = M1 * c2;
        uint32_t n0 = hi1 ^ c1 ^ k0;
        uint32_t n1 = lo1;
        uint32_t n2 = hi0 ^ c3 ^ k1;
        uint32_t n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    Philox4 o; o.x = c0; o.y = c1; o.z = c2; o.w = c3;
    return o;
}

PINN_HD float u01_from_bits(uint32_t w) { return (float)(w >> 8) * 5.9604644775390625e-08f; }  // [0,1)

PINN_HD uint32_t philox_word(const Philox4& p, int i) {
    return i == 0 ? p.x : (i == 1 ? p.y : (i == 2 ? p.z : p.w));
}

// Block `block` of the point with global index `gidx` at step `step`.
// Counter = (gidx lo, gidx hi, step lo, (step hi & 0xffff) << 16 | block); key = seed.
// block 0/1 serve uniform columns 0-3 / 4-7 (one word each); block 2+k serves normal column k (attempt t of a
// truncated normal: block 2+k | t << 8); block 10+g, word 0 picks the component of mixture group g.
PINN_HD Philox4 philox_block(uint64_t gidx, uint64_t step, uint64_t seed, uint32_t block) {
    return philox4x32_10((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)step,
                         (uint32_t)(((step >> 32) & 0xffffu) << 16) | block, (uint32_t)seed, (uint32_t)(seed >> 32));
}

// Coordinate k of the point with global index `gidx` at step `step` (blk0 / blk1: its blocks 0 and 1).
PINN_HD float sample_simple(int kind, float a, float b, int k, uint64_t gidx, uint64_t step, uint64_t seed,
                            const Philox4& blk0, const Philox4& blk1) {
    if (kind == PINN_COL_CONST) return a;
    if (kind == PINN_COL_UNIFORM) {
        uint32_t w = (k < 4) ? philox_word(blk0, k) : philox_word(blk1, k - 4);
        float u = u01_from_bits(w);
        return fmaf(b - a, u, a);
    }
    // normal: Box-Muller on a dedicated Philox block
    uint32_t c3 = (uint32_t)(((step >> 32) & 0xffffu) << 16) | (uint32_t)(2 + k);
    Philox4 p = philox4x32_10((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)step, c3,
                              (uint32_t)seed, (uint32_t)(seed >> 32));
    float u1 = ((float)(p.x >> 8) + 1.0f) * 5.9604644775390625e-08f;   // (0,1]
    float u2 = u01_from_bits(p.y);
    float rad = sqrtf(-2.0f * logf(u1));
    float z = rad * cosf(6.283185307179586f * u2);
    return fmaf(b, z, a);
}

// Truncated normal by rejection (batchflow `.truncate(high, low)` on a normal column): candidate t comes from words
// (0,1) / (2,3) of Philox block 2+k with the attempt number t/2 in bits 8..15 of the block word; the first candidate
// inside [lo, hi] wins; after 16 misses the mean is clamped into the interval (mass outside 16 sigma-ish only).
PINN_HD float sample_tnormal(float a, float b, float lo, float hi, int k, uint64_t gidx, uint64_t step, uint64_t seed) {
    for (int att = 0; att < 8; ++att) {
        const uint32_t c3 = (uint32_t)(((step >> 32) & 0xffffu) << 16) | (uint32_t)(att << 8) | (uint32_t)(2 + k);
        const Philox4 p = philox4x32_10((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)step, c3,
                                        (uint32_t)seed, (uint32_t)(seed >> 32));
        for (int half = 0; half < 2; ++half) {
            const uint32_t w1 = half ? p.z : p.x, w2 = half ? p.w : p.y;
            const float u1 = ((float)(w1 >> 8) + 1.0f) * 5.9604644775390625e-08f;   // (0,1]
            const float u2 = u01_from_bits(w2);
            const float z = sqrtf(-2.0f * logf(u1)) * cosf(6.283185307179586f * u2);
            const float v = fmaf(b, z, a);
            if (v >= lo && v <= hi) return v;
        }
    }
    return fminf(fmaxf(a, lo), hi);
}

PINN_HD float sample_column(const PinnColumn& col, int k, uint64_t gidx, uint64_t step, uint64_t seed,
                            const Philox4& blk0, const Philox4& blk1) {
    if (col.kind == PINN_COL_TNORMAL) return sample_tnormal(col.a, col.b, col.comp_a[0], col.comp_b[0], k, gidx, step, seed);
    if (col.kind != PINN_COL_MIXTURE) return sample_simple(col.kind, col.a, col.b, k, gidx, step, seed, blk0, blk1);
    uint32_t c3 = (uint32_t)(((step >> 32) & 0xffffu) << 16) | (uint32_t)(10 + col.group);
    Philox4 p = philox4x32_10((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)step, c3,
                              (uint32_t)seed, (uint32_t)(seed >> 32));
    const float u = u01_from_bits(p.x);
    int i = 0;
#pragma unroll
    for (int c = 0; c < PINN_MAX_MIX - 1; ++c) i += (c < col.n_comp - 1 && u >= col.cum_w[c]) ? 1 : 0;
    return sample_simple(col.comp_kind[i], col.comp_a[i], col.comp_b[i], k, gidx, step, seed, blk0, blk1);
}

// ----------------------------------------------------------------------------------------------
// Activations, branch-free.  A hidden unit stores its activation VALUE a; the derivatives of the
// activation are polynomials of a for tanh / sigmoid (constants for the identity), so ONE coefficient
// set per layer replaces every switch in the inner loops:
//     a   = ident ? z : p * tanh(q z) + r          (sigmoid(z) = 1/2 tanh(z/2) + 1/2)
//     s1  = c0 + c1 a + c2 a^2 ;  s2 = s1 (d0 + d1 a) ;  s3 = s1 (e0 + e1 a + e2 a^2)
// tanh   : s1 = 1 - a^2,  s2 = -2 a s1,         s3 = s1 (-2 + 6 a^2)
// sigmoid: s1 = a - a^2,  s2 = s1 (1 - 2 a),    s3 = s1 (1 - 6 a + 6 a^2)
// (s1, s2, s3 = first, second, third derivative of the activation w.r.t. its argument.)
//
// Activations outside that family (sin, softplus, SiLU, GELU) keep the pre-activation z itself in channel 0
// and rebuild (a, s1, s2, s3) from it wherever they are needed (act_terms_z): `zs` holds their id, 0 for the
// polynomial family.  Only the general kernel variants (template flag GEN) compile that path.
// ----------------------------------------------------------------------------------------------
struct ActD { float a, s1, s2, s3; };
struct ActC { float p, q, r, c0, c1, c2, d0, d1, e0, e1, e2; bool ident; int zs; };

PINN_HD ActC make_actc(int act) {
    const bool th = act == PINN_ACT_TANH, sg = act == PINN_ACT_SIGMOID;
    ActC k;
    k.zs = (act >= PINN_ACT_SIN && act <= PINN_ACT_GELU) ? act : 0;
    k.ident = !(th || sg);
    k.p = sg ? 0.5f : 1.0f; k.q = sg ? 0.5f : 1.0f; k.r = sg ? 0.5f : 0.0f;
    k.c0 = sg ? 0.0f : 1.0f; k.c1 = sg ? 1.0f : 0.0f; k.c2 = (th || sg) ? -1.0f : 0.0f;
    k.d0 = sg ? 1.0f : 0.0f; k.d1 = (th || sg) ? -2.0f : 0.0f;
    k.e0 = th ? -2.0f : (sg ? 1.0f : 0.0f); k.e1 = sg ? -6.0f : 0.0f; k.e2 = (th || sg) ? 6.0f : 0.0f;
    return k;
}

// tanh without branches: below 0.55 the odd polynomial x + x^3 q(x^2), q fitted (minimax over [0, 0.55]) so that the
// fp32 evaluation stays within 4.4e-8 absolute / 1.2e-7 relative of tanh; above, 1 - 2/(e^{2|x|}+1).
#define PINN_TANH_C0 (-3.3332759141921997e-1f)
#define PINN_TANH_C1 (1.3317519426345825e-1f)
#define PINN_TANH_C2 (-5.2506424486637115e-2f)
#define PINN_TANH_C3 (1.6171904280781746e-2f)
PINN_HD float tanh_acc(float x) {
    const float ax = fabsf(x);
    const float x2 = ax * ax;
    float p = fmaf(x2, PINN_TANH_C3, PINN_TANH_C2);
    p = fmaf(p, x2, PINN_TANH_C1);
    p = fmaf(p, x2, PINN_TANH_C0);
    const float small = fmaf(p * x2, ax, ax);
#if defined(__CUDA_ARCH__)
    float e;
    // volatile: without it the compiler turns the select below into a branch around the MUFU ops
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(ax * 2.8853900817779268f));
    const float big = fmaf(-2.0f, __frcp_rn(e + 1.0f), 1.0f);
#else
    const float e = exp2f(ax * 2.8853900817779268f);
    const float big = fmaf(-2.0f, 1.0f / (e + 1.0f), 1.0f);
#endif
    return copysignf(ax < 0.55f ? small : big, x);
}

// Value and first three derivatives of a z-stored activation at z.
//   sin      : a = sin z,            s1 = cos z,  s2 = -a,  s3 = -s1
//   softplus : a = log(1 + e^z),     s1 = sg(z),  s2 = s1 (1 - s1),  s3 = s2 (1 - 2 s1)         (sg = logistic)
//   SiLU     : a = z sg,  with g1 = sg (1 - sg), g2 = g1 (1 - 2 sg), g3 = g2 (1 - 2 sg) - 2 g1^2:
//              s1 = sg + z g1,  s2 = 2 g1 + z g2,  s3 = 3 g2 + z g3
//   GELU     : a = z Phi(z) (erf form),  s1 = Phi + z phi,  s2 = phi (2 - z^2),  s3 = phi z (z^2 - 4)
PINN_HD void act_terms_z(int kind, float z, float& a, float& s1, float& s2, float& s3) {
    if (kind == PINN_ACT_SIN) {
        float sn, cs;
#if defined(__CUDA_ARCH__)
        sincosf(z, &sn, &cs);
#else
        sn = sinf(z); cs = cosf(z);
#endif
        a = sn; s1 = cs; s2 = -sn; s3 = -cs;
    } else if (kind == PINN_ACT_GELU) {
        const float phi = 0.3989422804014327f * expf(-0.5f * z * z);
        const float Phi = 0.5f * erfcf(-0.7071067811865476f * z);
        const float z2 = z * z;
        a = z * Phi;
        s1 = fmaf(z, phi, Phi);
        s2 = phi * (2.0f - z2);
        s3 = phi * z * (z2 - 4.0f);
    } else {
        const float sg = fmaf(0.5f, tanh_acc(0.5f * z), 0.5f);
        const float g1 = sg * (1.0f - sg);
        const float om = fmaf(-2.0f, sg, 1.0f);
        const float g2 = g1 * om;
        if (kind == PINN_ACT_SOFTPLUS) {
            a = fmaxf(z, 0.0f) + log1pf(expf(-fabsf(z)));
            s1 = sg; s2 = g1; s3 = g2;
        } else {                                          // SiLU
            const float g3 = fmaf(g2, om, -2.0f * g1 * g1);
            a = z * sg;
            s1 = fmaf(z, g1, sg);
            s2 = fmaf(z, g2, 2.0f * g1);
            s3 = fmaf(z, g3, 3.0f * g2);
        }
    }
}

template <bool GEN = true>
PINN_HD float act_store(const ActC& k, float z) {
    const float t = fmaf(k.p, tanh_acc(k.q * z), k.r);
    return (k.ident || (GEN && k.zs)) ? z : t;
}

// act_store for two neighbouring units: the polynomial branch and the final blend run packed.
template <bool GEN = true>
PINN_HD float2 act_store2(const ActC& k, float2 z) {
    if (GEN && k.zs) return z;                            // z-stored family: channel 0 keeps z
    const float2 x = PINN_FMUL2(z, k.q);
    const float2 ax = make_float2(fabsf(x.x), fabsf(x.y));
    const float2 x2 = PINN_FMUL2V(ax, ax);
    float2 p = PINN_FFMA2(x2, PINN_TANH_C3, make_float2(PINN_TANH_C2, PINN_TANH_C2));
    p = PINN_FFMA2V(p, x2, make_float2(PINN_TANH_C1, PINN_TANH_C1));
    p = PINN_FFMA2V(p, x2, make_float2(PINN_TANH_C0, PINN_TANH_C0));
    const float2 small = PINN_FFMA2V(PINN_FMUL2V(p, x2), ax, ax);
#if defined(__CUDA_ARCH__)
    float e0, e1;
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(ax.x * 2.8853900817779268f));
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(ax.y * 2.8853900817779268f));
    const float2 r = make_float2(__frcp_rn(e0 + 1.0f), __frcp_rn(e1 + 1.0f));
#else
    const float2 r = make_float2(1.0f / (exp2f(ax.x * 2.8853900817779268f) + 1.0f),
                                 1.0f / (exp2f(ax.y * 2.8853900817779268f) + 1.0f));
#endif
    const float2 big = PINN_FFMA2(r, -2.0f, make_float2(1.0f, 1.0f));
    const float2 t = make_float2(copysignf(ax.x < 0.55f ? small.x : big.x, x.x),
                                 copysignf(ax.y < 0.55f ? small.y : big.y, x.y));
    const float2 out = PINN_FFMA2(t, k.p, make_float2(k.r, k.r));
    return k.ident ? z : out;
}

PINN_HD ActD act_from_stored(const ActC& k, float a) {
    ActD r;
    if (k.zs) { act_terms_z(k.zs, a, r.a, r.s1, r.s2, r.s3); return r; }
    r.a = a;
    r.s1 = fmaf(fmaf(k.c2, a, k.c1), a, k.c0);
    r.s2 = r.s1 * fmaf(k.d1, a, k.d0);
    r.s3 = r.s1 * fmaf(fmaf(k.e2, a, k.e1), a, k.e0);
    return r;
}

// Load the stored (pre-activation) jet of one hidden unit and turn it into the post-activation
// jet that feeds the next linear layer:  a, a_d = s1*z_d, a_dd = s2*z_d^2 + s1*z_dd.
template <int NF, int NS, bool GEN = true>
PINN_HD void load_post_jet(const float* __restrict__ row, int RS, const ActC& k, float (&a)[1 + NF + NS]) {
    float av = row[0];
    float s1 = fmaf(fmaf(k.c2, av, k.c1), av, k.c0);
    float s2 = s1 * fmaf(k.d1, av, k.d0);
    if (GEN && k.zs) { float s3; act_terms_z(k.zs, row[0], av, s1, s2, s3); }
    a[0] = av;
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        float zd = row[(1 + d) * RS];
        a[1 + d] = s1 * zd;
        if (d < NS) {
            float zdd = row[(1 + NF + d) * RS];
            a[1 + NF + d] = fmaf(s2 * zd, zd, s1 * zdd);
        }
    }
}

// The same for TWO units at once (rows of units A and B), on packed FP32x2 operations.
template <int NF, int NS, bool GEN = true>
PINN_HD void load_post_jet2(const float* __restrict__ rowa, const float* __restrict__ rowb, int RS, const ActC& k,
                            float2 (&a)[1 + NF + NS]) {
    float2 av = make_float2(rowa[0], rowb[0]);
    float2 s1 = PINN_FFMA2V(PINN_FFMA2(av, k.c2, make_float2(k.c1, k.c1)), av, make_float2(k.c0, k.c0));
    float2 s2 = PINN_FMUL2V(s1, PINN_FFMA2(av, k.d1, make_float2(k.d0, k.d0)));
    if (GEN && k.zs) {
        float s3;
        const float za = av.x, zb = av.y;
        act_terms_z(k.zs, za, av.x, s1.x, s2.x, s3);
        act_terms_z(k.zs, zb, av.y, s1.y, s2.y, s3);
    }
    a[0] = av;
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        const float2 zd = make_float2(rowa[(1 + d) * RS], rowb[(1 + d) * RS]);
        a[1 + d] = PINN_FMUL2V(s1, zd);
        if (d < NS) {
            const float2 zdd = make_float2(rowa[(1 + NF + d) * RS], rowb[(1 + NF + d) * RS]);
            a[1 + NF + d] = PINN_FFMA2V(PINN_FMUL2V(s2, zd), zd, PINN_FMUL2V(s1, zdd));
        }
    }
}

// ----------------------------------------------------------------------------------------------
// Forward: one block of NB*4 output units of a linear layer, all jet channels at once.
// Wt is the forward layout [n_in][n_out_p4]; weights are read with 128-bit broadcast loads and
// every loaded weight feeds C FMAs.
// ----------------------------------------------------------------------------------------------
template <int NF, int NS, int NB, bool GEN = true>
PINN_HD void fwd_block_hidden(const float* __restrict__ Wt, int wt_stride, const float* __restrict__ bias,
                              int n_in, const float* __restrict__ in_rows, int RS, const ActC& in_act,
                              float2 (&acc)[NB * 2][1 + NF + NS]) {
    constexpr int C = 1 + NF + NS;
#pragma unroll
    for (int j = 0; j < NB * 2; ++j) {
        acc[j][0] = make_float2(bias[2 * j], bias[2 * j + 1]);
#pragma unroll
        for (int c = 1; c < C; ++c) acc[j][c] = make_float2(0.0f, 0.0f);
    }
    // many-channel problems keep their per-point state in global memory: more iterations in flight overlap
    // the load latency there (measured: cfg5 -10 %), while for the shared-memory-resident narrow problems
    // unrolling only costs instruction-cache reach (cfg2 +7 %)
    constexpr int UNR = (C >= 8) ? PINN_UNR_WIDE : ((C >= 6) ? 2 : 1);
#pragma unroll UNR
    for (int k = 0; k < n_in; ++k) {
        float a[C];
        load_post_jet<NF, NS, GEN>(in_rows + (size_t)k * C * RS, RS, in_act, a);
        const float4* wrow = reinterpret_cast<const float4*>(Wt + (size_t)k * wt_stride);
#pragma unroll
        for (int g = 0; g < NB; ++g) {
            const float4 w = wrow[g];
            const float2 w01 = make_float2(w.x, w.y), w23 = make_float2(w.z, w.w);
#pragma unroll
            for (int c = 0; c < C; ++c) {
                acc[2 * g + 0][c] = PINN_FFMA2(w01, a[c], acc[2 * g + 0][c]);
                acc[2 * g + 1][c] = PINN_FFMA2(w23, a[c], acc[2 * g + 1][c]);
            }
        }
    }
}

// First layer: the input jet is (x_k, v_dir[k], 0): value channel is a dot product with the coordinates,
// first-order channels are the same dot product with the direction vectors, second-order channels vanish.
template <int NF, int NS, int NB>
PINN_HD void fwd_block_input(const float* __restrict__ Wt, int wt_stride, const float* __restrict__ bias,
                             int n_in, const float* __restrict__ coords, int RS, const float* __restrict__ dirv,
                             float2 (&acc)[NB * 2][1 + NF + NS]) {
    constexpr int C = 1 + NF + NS;
#pragma unroll
    for (int j = 0; j < NB * 2; ++j) {
        acc[j][0] = make_float2(bias[2 * j], bias[2 * j + 1]);
#pragma unroll
        for (int c = 1; c < C; ++c) acc[j][c] = make_float2(0.0f, 0.0f);
    }
#pragma unroll 1
    for (int k = 0; k < n_in; ++k) {
        float x = coords[(size_t)k * RS];
        float vd[NF > 0 ? NF : 1];
#pragma unroll
        for (int d = 0; d < NF; ++d) vd[d] = dirv[d * PINN_MAX_DIMS + k];
        const float4* wrow = reinterpret_cast<const float4*>(Wt + (size_t)k * wt_stride);
#pragma unroll
        for (int g = 0; g < NB; ++g) {
            const float4 w = wrow[g];
            const float2 w01 = make_float2(w.x, w.y), w23 = make_float2(w.z, w.w);
            acc[2 * g + 0][0] = PINN_FFMA2(w01, x, acc[2 * g + 0][0]);
            acc[2 * g + 1][0] = PINN_FFMA2(w23, x, acc[2 * g + 1][0]);
#pragma unroll
            for (int d = 0; d < NF; ++d) {
                acc[2 * g + 0][1 + d] = PINN_FFMA2(w01, vd[d], acc[2 * g + 0][1 + d]);
                acc[2 * g + 1][1 + d] = PINN_FFMA2(w23, vd[d], acc[2 * g + 1][1 + d]);
            }
        }
    }
}

// Store a block of freshly computed pre-activation jets: channel 0 goes through act_store().
template <int NF, int NS, int NB, bool GEN = true>
PINN_HD void store_block(float* __restrict__ out_rows, int RS, const ActC& act, int j0, int n_out,
                         const float2 (&acc)[NB * 2][1 + NF + NS]) {
    constexpr int C = 1 + NF + NS;
#pragma unroll
    for (int h = 0; h < NB * 2; ++h) {
        const float2 a = act_store2<GEN>(act, acc[h][0]);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int j = 2 * h + q;
            const bool ok = j0 + j < n_out;
            float* row = out_rows + (size_t)(ok ? j0 + j : j0) * C * RS;
            if (ok) row[0] = q ? a.y : a.x;
#pragma unroll
            for (int c = 1; c < C; ++c)
                if (ok) row[(size_t)c * RS] = q ? acc[h][c].y : acc[h][c].x;
        }
    }
}

// One whole hidden (or input) linear layer, blocked over output units.
template <int NF, int NS, int JF, bool GEN = true>
PINN_HD void fwd_layer(const DevLayer& L, const float* __restrict__ sw, const float* __restrict__ in_rows,
                       bool in_is_coords, int in_act_id, const float* __restrict__ dirv,
                       float* __restrict__ out_rows, int RS) {
    constexpr int NBMAX = JF / 4;
    const float* Wt = sw + L.wt_s;
    const float* bias = sw + L.b_s;
    const ActC in_act = make_actc(in_act_id);
    const ActC out_act = make_actc(L.act);
#pragma unroll 1
    for (int j0 = 0; j0 < L.n_out; j0 += JF) {
        int nb = (L.n_out_p4 - j0) / 4;
        if (nb > NBMAX) nb = NBMAX;
#define PINN_FWD_CASE(NB)                                                                           \
        {                                                                                           \
            float2 acc[NB * 2][1 + NF + NS];                                                        \
            if (in_is_coords)                                                                       \
                fwd_block_input<NF, NS, NB>(Wt + j0, L.n_out_p4, bias + j0, L.n_in, in_rows, RS,    \
                                            dirv, acc);                                             \
            else                                                                                    \
                fwd_block_hidden<NF, NS, NB, GEN>(Wt + j0, L.n_out_p4, bias + j0, L.n_in, in_rows, RS,   \
                                             in_act, acc);                                          \
            store_block<NF, NS, NB, GEN>(out_rows, RS, out_act, j0, L.n_out, acc);                    \
        }
        if (NBMAX >= 4 && nb == 4) PINN_FWD_CASE(4)
        else if (NBMAX >= 3 && nb == 3) PINN_FWD_CASE(3)
        else if (NBMAX >= 2 && nb == 2) PINN_FWD_CASE(2)
        else PINN_FWD_CASE(1)
#undef PINN_FWD_CASE
    }
}

// Where a consumer reads the (activated) output of layer p: a residual layer keeps the sum
// act(z_p) + skip in its post buffer, which reads back like the output of an identity activation;
// any other layer is rebuilt from its stored jet with its own activation.
template <bool GEN = true>
PINN_HD const float* layer_output(const DevPlan& P, int p, const float* __restrict__ units, int C, int RS,
                                  int& act_id) {
    const DevLayer& Lp = P.layer[p];
    if (GEN && Lp.post_base >= 0) { act_id = PINN_ACT_NONE; return units + (size_t)Lp.post_base * C * RS; }
    act_id = Lp.act;
    return units + (size_t)Lp.unit_base * C * RS;
}

// Residual layer l ('… R … fa+'): post buffer <- act-jet(stored jet of l) + output of layer skip_src.
template <int NF, int NS>
PINN_HD void skip_sum_pass(const DevPlan& P, int l, float* __restrict__ units, int RS) {
    constexpr int C = 1 + NF + NS;
    const DevLayer& L = P.layer[l];
    const ActC own = make_actc(L.act);
    int src_act;
    const float* src_rows = layer_output(P, L.skip_src, units, C, RS, src_act);
    const ActC srcc = make_actc(src_act);
    const float* pre_rows = units + (size_t)L.unit_base * C * RS;
    float* post_rows = units + (size_t)L.post_base * C * RS;
#pragma unroll 1
    for (int j = 0; j < L.n_out; ++j) {
        float a[C], b[C];
        load_post_jet<NF, NS>(pre_rows + (size_t)j * C * RS, RS, own, a);
        load_post_jet<NF, NS>(src_rows + (size_t)j * C * RS, RS, srcc, b);
#pragma unroll
        for (int c = 0; c < C; ++c) post_rows[((size_t)j * C + c) * RS] = a[c] + b[c];
    }
}

// Final linear layer (one output unit, no activation): the network jet N lands in registers.
template <int NF, int NS, bool GEN = true>
PINN_HD void fwd_final(const DevLayer& L, const float* __restrict__ sw, const float* __restrict__ in_rows,
                       bool in_is_coords, int in_act_id, const float* __restrict__ dirv, int RS,
                       float (&N)[1 + NF + NS]) {
    constexpr int C = 1 + NF + NS;
    const ActC in_act = make_actc(in_act_id);
    const float* w = sw + L.w_s;            // reverse layout row 0 == the single weight row
    N[0] = sw[L.b_s];
#pragma unroll
    for (int c = 1; c < C; ++c) N[c] = 0.0f;
    if (in_is_coords) {
        for (int k = 0; k < L.n_in; ++k) {
            N[0] = fmaf(w[k], in_rows[(size_t)k * RS], N[0]);
#pragma unroll
            for (int d = 0; d < NF; ++d) N[1 + d] = fmaf(w[k], dirv[d * PINN_MAX_DIMS + k], N[1 + d]);
        }
    } else {
#pragma unroll 1
        for (int k = 0; k < L.n_in; ++k) {
            float a[C];
            load_post_jet<NF, NS, GEN>(in_rows + (size_t)k * C * RS, RS, in_act, a);
            float wk = w[k];
#pragma unroll
            for (int c = 0; c < C; ++c) N[c] = fmaf(wk, a[c], N[c]);
        }
    }
}

// ----------------------------------------------------------------------------------------------
// Expression programs (residual and initial condition).
// ----------------------------------------------------------------------------------------------
PINN_HD float powi_f(float x, int e) {
    bool neg = e < 0;
    unsigned n = neg ? (unsigned)(-e) : (unsigned)e;
    float r = 1.0f, b = x;
    while (n) { if (n & 1u) r *= b; b *= b; n >>= 1; }
    return neg ? 1.0f / r : r;
}

PINN_HD void eval_prog(const PinnInstr* __restrict__ prog, int n, float* __restrict__ scr, int RS,
                       const float* __restrict__ coords, const float* __restrict__ pvals,
                       const int* __restrict__ var_off) {
    for (int i = 0; i < n; ++i) {
        PinnInstr in = prog[i];
        float r;
        switch (in.op) {
            case PINN_OP_CONST: r = in.imm; break;
            case PINN_OP_COORD: r = coords[(size_t)in.a * RS]; break;
            case PINN_OP_VAR:   r = pvals[var_off[in.a]]; break;
            default: {
                float x = scr[(size_t)in.a * RS];
                switch (in.op) {
                    case PINN_OP_ADD:  r = x + scr[(size_t)in.b * RS]; break;
                    case PINN_OP_SUB:  r = x - scr[(size_t)in.b * RS]; break;
                    case PINN_OP_MUL:  r = x * scr[(size_t)in.b * RS]; break;
                    case PINN_OP_DIV:  r = x / scr[(size_t)in.b * RS]; break;
                    case PINN_OP_POW:  r = powf(x, scr[(size_t)in.b * RS]); break;
                    case PINN_OP_NEG:  r = -x; break;
                    case PINN_OP_MULI: r = x * in.imm; break;
                    case PINN_OP_ADDI: r = x + in.imm; break;
                    case PINN_OP_SIN:  r = sinf(x); break;
                    case PINN_OP_COS:  r = cosf(x); break;
                    case PINN_OP_TAN:  r = tanf(x); break;
                    case PINN_OP_EXP:  r = expf(x); break;
                    case PINN_OP_LOG:  r = logf(x); break;
                    case PINN_OP_SQRT: r = sqrtf(x); break;
                    case PINN_OP_TANH: r = tanhf(x); break;
                    case PINN_OP_SIGMOID: r = 1.0f / (1.0f + expf(-x)); break;
                    case PINN_OP_RECIP: r = 1.0f / x; break;
                    case PINN_OP_POWI: r = powi_f(x, (int)in.imm); break;
                    case PINN_OP_ABS:  r = fabsf(x); break;
                    case PINN_OP_SIGN: r = (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f); break;
                    default:           r = 0.0f; break;
                }
            } break;
        }
        scr[(size_t)in.dst * RS] = r;
    }
}

// ----------------------------------------------------------------------------------------------
// Ansatz (model_torch.py:107-128) forward and adjoint, for axis-aligned directions.
// ----------------------------------------------------------------------------------------------
template <int NF, int NS>
struct AnsatzState {
    float G, Gd[NF > 0 ? NF : 1], Gdd[NS > 0 ? NS : 1];      // boundary factor jet
    float S, S1, S2, sig, einv, w;                            // time gate and its t-derivatives
    float v, vd[NF > 0 ? NF : 1], vdd[NS > 0 ? NS : 1];       // BC-transformed value jet
};

template <int NF, int NS, bool GEN = true>
PINN_HD void ansatz_forward(const DevPlan& P, const float* __restrict__ coords, int RS, float log_scale,
                            const float (&N)[1 + NF + NS], const float* __restrict__ icj /* C or null */,
                            AnsatzState<NF, NS>& st, float (&u)[1 + NF + NS]) {
    // boundary factor G = prod_i (x_i-lo_i)(hi_i-x_i)/(hi_i-lo_i)^2 over spatial dims
    st.G = 1.0f;
#pragma unroll
    for (int d = 0; d < NF; ++d) { st.Gd[d] = 0.0f; if (d < NS) st.Gdd[d] = 0.0f; }
    if (P.has_bc) {
        float G = 1.0f;
        for (int i = 0; i < P.nsp; ++i) {
            float x = coords[(size_t)i * RS];
            G *= (x - P.lo[i]) * (P.hi[i] - x) * P.inv_w2[i];
        }
        st.G = G;
#pragma unroll
        for (int d = 0; d < NF; ++d) {
            const int k = P.dir_col[d];
            if (!GEN || k >= 0) {                         // unit vector of column k
                if (k < P.nsp) {
                    float others = 1.0f;
                    for (int i = 0; i < P.nsp; ++i) {
                        if (i != k) {
                            float x = coords[(size_t)i * RS];
                            others *= (x - P.lo[i]) * (P.hi[i] - x) * P.inv_w2[i];
                        }
                    }
                    float xk = coords[(size_t)k * RS];
                    st.Gd[d] = (P.lo[k] + P.hi[k] - 2.0f * xk) * P.inv_w2[k] * others;
                    if (d < NS) st.Gdd[d] = -2.0f * P.inv_w2[k] * others;
                }
            } else {                                      // general direction v: sum_i v_i d_i G, sum_ij v_i v_j d_ij G
                float gd = 0.0f, gdd = 0.0f;
                for (int i = 0; i < P.nsp; ++i) {
                    const float vi = P.dir_vec[d][i];
                    if (vi == 0.0f) continue;
                    const float xi = coords[(size_t)i * RS];
                    const float gpi = (P.lo[i] + P.hi[i] - 2.0f * xi) * P.inv_w2[i];
                    float others = 1.0f;
                    for (int q = 0; q < P.nsp; ++q)
                        if (q != i) { float x = coords[(size_t)q * RS]; others *= (x - P.lo[q]) * (P.hi[q] - x) * P.inv_w2[q]; }
                    gd = fmaf(vi * gpi, others, gd);
                    gdd = fmaf(vi * vi * (-2.0f * P.inv_w2[i]), others, gdd);
                    for (int j = i + 1; j < P.nsp; ++j) {
                        const float vj = P.dir_vec[d][j];
                        if (vj == 0.0f) continue;
                        const float xj = coords[(size_t)j * RS];
                        const float gpj = (P.lo[j] + P.hi[j] - 2.0f * xj) * P.inv_w2[j];
                        float rest = 1.0f;
                        for (int q = 0; q < P.nsp; ++q)
                            if (q != i && q != j) { float x = coords[(size_t)q * RS]; rest *= (x - P.lo[q]) * (P.hi[q] - x) * P.inv_w2[q]; }
                        gdd = fmaf(2.0f * vi * vj * gpi * gpj, rest, gdd);
                    }
                }
                st.Gd[d] = gd;
                if (d < NS) st.Gdd[d] = gdd;
            }
        }
        st.v = fmaf(st.G, N[0], P.bc);
#pragma unroll
        for (int d = 0; d < NF; ++d) {
            st.vd[d] = fmaf(st.Gd[d], N[0], st.G * N[1 + d]);
            if (d < NS)
                st.vdd[d] = fmaf(st.Gdd[d], N[0], fmaf(2.0f * st.Gd[d], N[1 + d], st.G * N[1 + NF + d]));
        }
    } else {
        st.v = N[0];
#pragma unroll
        for (int d = 0; d < NF; ++d) { st.vd[d] = N[1 + d]; if (d < NS) st.vdd[d] = N[1 + NF + d]; }
    }
    if (P.has_ic) {
        float t = coords[(size_t)(P.ndims - 1) * RS];
        st.einv = expf(-log_scale);
        st.w = (t - P.t0) * st.einv;
        st.sig = 1.0f / (1.0f + expf(-st.w));
        st.S = st.sig - 0.5f;
        float sp = st.sig * (1.0f - st.sig);
        st.S1 = sp * st.einv;
        st.S2 = sp * (1.0f - 2.0f * st.sig) * st.einv * st.einv;
        u[0] = fmaf(st.S, st.v, icj[0]);
#pragma unroll
        for (int d = 0; d < NF; ++d) {
            const float vt = P.dir_vec[d][P.ndims - 1];     // t-component of the direction
            float Sd = vt * st.S1;
            u[1 + d] = fmaf(Sd, st.v, fmaf(st.S, st.vd[d], icj[1 + d]));
            if (d < NS) {
                float Sdd = vt * vt * st.S2;
                u[1 + NF + d] = fmaf(Sdd, st.v, fmaf(2.0f * Sd, st.vd[d], fmaf(st.S, st.vdd[d], icj[1 + NF + d])));
            }
        }
    } else {
        u[0] = st.v;
#pragma unroll
        for (int d = 0; d < NF; ++d) { u[1 + d] = st.vd[d]; if (d < NS) u[1 + NF + d] = st.vdd[d]; }
    }
}

// Adjoint of the ansatz: ub (d loss / d u-jet) -> Nb (d loss / d N-jet); returns d loss / d log_scale.
template <int NF, int NS>
PINN_HD float ansatz_adjoint(const DevPlan& P, const AnsatzState<NF, NS>& st,
                             const float (&ub)[1 + NF + NS], float (&Nb)[1 + NF + NS]) {
    float vb, vdb[NF > 0 ? NF : 1], vddb[NS > 0 ? NS : 1];
    float sbar = 0.0f;
    if (P.has_ic) {
        float Sb = ub[0] * st.v, S1b = 0.0f, S2b = 0.0f;
        vb = st.S * ub[0];
#pragma unroll
        for (int d = 0; d < NF; ++d) {
            const float vt = P.dir_vec[d][P.ndims - 1];
            float Sd = vt * st.S1;
            vb = fmaf(Sd, ub[1 + d], vb);
            vdb[d] = st.S * ub[1 + d];
            Sb = fmaf(ub[1 + d], st.vd[d], Sb);
            S1b = fmaf(vt * ub[1 + d], st.v, S1b);
            if (d < NS) {
                float Sdd = vt * vt * st.S2;
                float q = ub[1 + NF + d];
                vb = fmaf(Sdd, q, vb);
                vdb[d] = fmaf(2.0f * Sd, q, vdb[d]);
                vddb[d] = st.S * q;
                Sb = fmaf(q, st.vdd[d], Sb);
                S1b = fmaf(2.0f * vt * q, st.vd[d], S1b);
                S2b = fmaf(vt * vt * q, st.v, S2b);
            }
        }
        // S = sig(w) - 1/2, S1 = sig'(w) e, S2 = sig''(w) e^2, w = (t - t0) e, e = exp(-s), dw/ds = -w
        float sg = st.sig, p1 = sg * (1.0f - sg), p2 = p1 * (1.0f - 2.0f * sg),
              p3 = p1 * fmaf(6.0f * sg, sg - 1.0f, 1.0f);
        float e = st.einv, w = st.w;
        float dS = -p1 * w;
        float dS1 = -e * fmaf(p2, w, p1);
        float dS2 = -e * e * fmaf(p3, w, 2.0f * p2);
        sbar = fmaf(Sb, dS, fmaf(S1b, dS1, S2b * dS2));
    } else {
        vb = ub[0];
#pragma unroll
        for (int d = 0; d < NF; ++d) { vdb[d] = ub[1 + d]; if (d < NS) vddb[d] = ub[1 + NF + d]; }
    }
    if (P.has_bc) {
        float nb0 = st.G * vb;
#pragma unroll
        for (int d = 0; d < NF; ++d) {
            nb0 = fmaf(st.Gd[d], vdb[d], nb0);
            float nd = st.G * vdb[d];
            if (d < NS) {
                nb0 = fmaf(st.Gdd[d], vddb[d], nb0);
                nd = fmaf(2.0f * st.Gd[d], vddb[d], nd);
                Nb[1 + NF + d] = st.G * vddb[d];
            }
            Nb[1 + d] = nd;
        }
        Nb[0] = nb0;
    } else {
        Nb[0] = vb;
#pragma unroll
        for (int d = 0; d < NF; ++d) { Nb[1 + d] = vdb[d]; if (d < NS) Nb[1 + NF + d] = vddb[d]; }
    }
    return sbar;
}

// ----------------------------------------------------------------------------------------------
// Reverse sweep.
// ----------------------------------------------------------------------------------------------
// Adjoint of one activation: post-activation adjoints (ab) + stored pre jet -> pre adjoints (zb).
//   zdd_b = s1*add_b ; zd_b = s1*ad_b + 2 s2 zd add_b ; z_b = s1*a_b + sum s2 zd ad_b + (s3 zd^2 + s2 zdd) add_b
template <int NF, int NS>
PINN_HD void act_adjoint(const ActD& f, const float (&pre)[1 + NF + NS], const float (&ab)[1 + NF + NS],
                         float (&zb)[1 + NF + NS]) {
    float z0 = f.s1 * ab[0];
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        float zd = pre[1 + d];
        float t = f.s2 * zd;
        z0 = fmaf(t, ab[1 + d], z0);
        float zdb = f.s1 * ab[1 + d];
        if (d < NS) {
            float q = ab[1 + NF + d];
            zdb = fmaf(2.0f * t, q, zdb);
            z0 = fmaf(fmaf(f.s3 * zd, zd, f.s2 * pre[1 + NF + d]), q, z0);
            zb[1 + NF + d] = f.s1 * q;
        }
        zb[1 + d] = zdb;
    }
    zb[0] = z0;
}

// The same adjoint for TWO neighbouring units at once (every operation is element-wise, so the pair
// rides on packed FP32x2 instructions): pre/ab/zb hold (unit, unit+1) pairs per channel.
template <int NF, int NS, bool GEN = true>
PINN_HD void act_adjoint2(const ActC& k, const float2 (&pre)[1 + NF + NS], const float2 (&ab)[1 + NF + NS],
                          float2 (&zb)[1 + NF + NS]) {
    const float2 a = pre[0];
    float2 s1 = PINN_FFMA2V(PINN_FFMA2(a, k.c2, make_float2(k.c1, k.c1)), a, make_float2(k.c0, k.c0));
    float2 s2 = PINN_FMUL2V(s1, PINN_FFMA2(a, k.d1, make_float2(k.d0, k.d0)));
    float2 s3 = PINN_FMUL2V(s1, PINN_FFMA2V(PINN_FFMA2(a, k.e2, make_float2(k.e1, k.e1)), a, make_float2(k.e0, k.e0)));
    if (GEN && k.zs) {
        float av;
        act_terms_z(k.zs, a.x, av, s1.x, s2.x, s3.x);
        act_terms_z(k.zs, a.y, av, s1.y, s2.y, s3.y);
    }
    float2 z0 = PINN_FMUL2V(s1, ab[0]);
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        const float2 zd = pre[1 + d];
        const float2 t = PINN_FMUL2V(s2, zd);
        z0 = PINN_FFMA2V(t, ab[1 + d], z0);
        float2 zdb = PINN_FMUL2V(s1, ab[1 + d]);
        if (d < NS) {
            const float2 q = ab[1 + NF + d];
            zdb = PINN_FFMA2V(PINN_FMUL2(t, 2.0f), q, zdb);
            const float2 w = PINN_FFMA2V(PINN_FMUL2V(s3, zd), zd, PINN_FMUL2V(s2, pre[1 + NF + d]));
            z0 = PINN_FFMA2V(w, q, z0);
            zb[1 + NF + d] = PINN_FMUL2V(s1, q);
        }
        zb[1 + d] = zdb;
    }
    zb[0] = z0;
}

#if defined(__CUDA_ARCH__)
// One stage of warp_transpose_reduce at lane distance S.  S is a template parameter so that every index
// into v is a compile-time constant and v stays in registers; the selects pick values, not addresses.
//   S >= NV: every entry is summed with the partner lane's copy of it;
//   S <  NV: the lower half of the lanes keeps entries [0, S), the upper half keeps [S, 2S) and moves them
//            down to [0, S); each sends the other half and adds what the partner sent.
template <int S, int NV>
__device__ __forceinline__ void warp_transpose_stage(float (&v)[NV], int lane) {
    if constexpr (S >= NV) {
#pragma unroll
        for (int i = 0; i < NV; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i], S);
    } else {
        const bool up = (lane & S) != 0;
#pragma unroll
        for (int i = 0; i < S; ++i) {
            const float lo = v[i], hi = v[i + S];
            const float send = up ? lo : hi;
            const float keep = up ? hi : lo;
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, S);
        }
    }
    if constexpr (S > 1) warp_transpose_stage<S / 2, NV>(v, lane);
}

// Sum NV per-lane values over the 32 lanes of a warp with a transposing butterfly: on return the
// lane with (lane % NV) == e holds the total of entry e.  31 shuffles for NV == 32.
template <int NV>
__device__ __forceinline__ float warp_transpose_reduce(float (&v)[NV], int lane) {
    static_assert(NV >= 1 && NV <= 32 && (NV & (NV - 1)) == 0, "NV must be a power of two up to 32");
    warp_transpose_stage<16, NV>(v, lane);
    return v[0];
}
#endif

// Hand NV per-point contributions to the gradient accumulator: on the GPU they are summed over
// the warp first and each entry is added once (by one lane); in the host emulation they are
// added directly.
template <int NV, class AddFn>
PINN_HD void emit_entries(float (&v)[NV], AddFn&& add) {
#if defined(__CUDA_ARCH__)
    int lane = threadIdx.x & 31;
    float t = warp_transpose_reduce<NV>(v, lane);
    if (lane < NV) add(lane, t);
#else
    for (int e = 0; e < NV; ++e) add(e, v[e]);
#endif
}

struct GradSink {
    float* wacc;        // this warp's own accumulator in params layout (+ loss slot): no other warp writes it
    int dump;           // index of a scratch slot of the accumulator that swallows masked-off entries
#if !defined(__CUDACC__)
    bool atomic;        // read by nothing: the host emulation of tests/emul (a plain C++ build) still clears it
#endif
    // add `val` at `idx` when `valid`, branch-free
    PINN_HD void add_if(bool valid, int idx, float val) const {
#if defined(__CUDA_ARCH__)
        const int i = valid ? idx : dump; wacc[i] += val;
#else
        if (valid) wacc[idx] += val;
#endif
    }
    PINN_HD void add(int idx, float val) const { wacc[idx] += val; }
};

// Bias gradients of a layer on their own: for layers whose input width is a multiple of the reduction block
// (the bias column would open a block of its own) and for an input layer with PINN_MAX_DIMS columns.
template <int NF, int NS>
PINN_HD void bias_grad(const DevLayer& L, const float* __restrict__ out_rows, int RS, const GradSink& sink) {
    constexpr int C = 1 + NF + NS;
#pragma unroll 1
    for (int j0 = 0; j0 < L.n_out; j0 += 32) {
        float v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int j = j0 + i < L.n_out ? j0 + i : L.n_out - 1;
            v[i] = out_rows[(size_t)j * C * RS];
        }
        emit_entries<32>(v, [&](int e, float t) {
            sink.add_if(j0 + e < L.n_out, L.b_off + j0 + e, t);
        });
    }
}

// Reverse of linear layer L (its output adjoints zb_L are already stored in out_rows):
//   weight AND bias gradients of L (the bias is normally column n_in of the same reduction batches: its
//   "input jet" is (1, 0, …)) and — fused in the same loop — the adjoints of the layer below, pushed
//   through that layer's activation and written over its stored jet in place.
// JJ = output units per reduction batch (4 normally, 1 for the single-output top layer).
// No guards in the inner loops: rows/columns past the end are read from clamped (valid) addresses,
// meet zero-padded weights, and their reduction entries are dropped at the sink.
template <int NF, int NS, int JJ, bool SKIP, bool GEN = SKIP>
PINN_HD void bwd_layer(const DevLayer& L, int below_act_id, const float* __restrict__ sw,
                       const float* __restrict__ out_rows, float* __restrict__ in_rows, int RS,
                       const GradSink& sink,
                       const float* __restrict__ load_rows, int load_act_id,
                       const float* __restrict__ adj_in /* stashed skip adjoint to add, or null */,
                       float* __restrict__ adj_out /* where to stash the adjoint of a residual layer, or null */,
                       float* __restrict__ dump_rows /* C rows that swallow the stores of masked-off units */) {
    constexpr int C = 1 + NF + NS;
    constexpr int JB = 8;
    const float* W = sw + L.w_s;
    const ActC below = make_actc(below_act_id);
    const ActC load_act = make_actc(SKIP ? load_act_id : below_act_id);
    if (!SKIP) load_rows = in_rows;
    // the bias rides as column n_in of the last block — unless n_in fills its blocks exactly: an extra block for
    // one column would cost 1/8 of a 64-wide layer's reverse work, a separate pass over channel 0 costs ~nothing
    const bool fold_bias = (L.n_in & (JB - 1)) != 0;
    const int n_cols = L.n_in + (fold_bias ? 1 : 0);
#pragma unroll 1
    for (int m0 = 0; m0 < n_cols; m0 += JB) {
        // neighbouring input units are kept as pairs
        float2 post[JB / 2][C];
#pragma unroll
        for (int h = 0; h < JB / 2; ++h) {
            const int ma = m0 + 2 * h, mb = ma + 1;
            const int ca = ma < L.n_in ? ma : L.n_in - 1, cb = mb < L.n_in ? mb : L.n_in - 1;
            load_post_jet2<NF, NS, GEN>(load_rows + (size_t)ca * C * RS, load_rows + (size_t)cb * C * RS, RS, load_act,
                                   post[h]);
            if (ma == L.n_in) {                           // bias column: jet (1, 0, …, 0)
                post[h][0].x = 1.0f;
#pragma unroll
                for (int c = 1; c < C; ++c) post[h][c].x = 0.0f;
            }
            if (mb == L.n_in) {
                post[h][0].y = 1.0f;
#pragma unroll
                for (int c = 1; c < C; ++c) post[h][c].y = 0.0f;
            }
        }
        float2 acc[JB / 2][C];
#pragma unroll
        for (int h = 0; h < JB / 2; ++h)
#pragma unroll
            for (int c = 0; c < C; ++c) acc[h][c] = make_float2(0.0f, 0.0f);
        if (SKIP && adj_in) {                             // the layer below also feeds a skip connection
#pragma unroll
            for (int h = 0; h < JB / 2; ++h) {
                const int ma = m0 + 2 * h < L.n_in ? m0 + 2 * h : L.n_in - 1;
                const int mb = m0 + 2 * h + 1 < L.n_in ? m0 + 2 * h + 1 : L.n_in - 1;
#pragma unroll
                for (int c = 0; c < C; ++c)
                    acc[h][c] = make_float2(adj_in[((size_t)ma * C + c) * RS], adj_in[((size_t)mb * C + c) * RS]);
            }
        }

        constexpr int BUNR = (C >= 8) ? PINN_BWD_UNR_WIDE : 1;
#pragma unroll BUNR
        for (int j0 = 0; j0 < L.n_out; j0 += JJ) {
            float v[JJ * JB];
#pragma unroll
            for (int jj = 0; jj < JJ; ++jj) {
                const int j = j0 + jj;
                const int jc = j < L.n_out ? j : L.n_out - 1;
                const float* row = out_rows + (size_t)jc * C * RS;
                float zb[C];
#pragma unroll
                for (int c = 0; c < C; ++c) zb[c] = row[(size_t)c * RS];
                const float4* wrow = reinterpret_cast<const float4*>(W + (size_t)j * L.n_in_p8 + m0);
                const float4 w0 = wrow[0], w1 = wrow[1];
                const float2 w[JB / 2] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w),
                                          make_float2(w1.x, w1.y), make_float2(w1.z, w1.w)};
#pragma unroll
                for (int h = 0; h < JB / 2; ++h) {
                    float2 e = PINN_FMUL2(post[h][0], zb[0]);
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        acc[h][c] = PINN_FFMA2(w[h], zb[c], acc[h][c]);
                        if (c > 0) e = PINN_FFMA2(post[h][c], zb[c], e);
                    }
                    v[jj * JB + 2 * h] = e.x;
                    v[jj * JB + 2 * h + 1] = e.y;
                }
            }
            emit_entries<JJ * JB>(v, [&](int e, float t) {
                const int j = j0 + e / JB, m = m0 + e % JB;
                sink.add_if(j < L.n_out && m <= L.n_in, m < L.n_in ? L.w_off + j * L.n_in + m : L.b_off + j, t);
            });
        }
        // adjoints of the layer below: through its activation (two units per packed op), stored in place
#pragma unroll
        for (int h = 0; h < JB / 2; ++h) {
            const bool oka = m0 + 2 * h < L.n_in, okb = m0 + 2 * h + 1 < L.n_in;
            const float* rowa = in_rows + (size_t)(oka ? m0 + 2 * h : 0) * C * RS;
            const float* rowb = in_rows + (size_t)(okb ? m0 + 2 * h + 1 : 0) * C * RS;
            float2 pre[C], zb[C];
#pragma unroll
            for (int c = 0; c < C; ++c) pre[c] = make_float2(rowa[(size_t)c * RS], rowb[(size_t)c * RS]);
            act_adjoint2<NF, NS, GEN>(below, pre, acc[h], zb);
            float* wa = oka ? in_rows + (size_t)(m0 + 2 * h) * C * RS : dump_rows;      // masked-off units: dump rows
            float* wb = okb ? in_rows + (size_t)(m0 + 2 * h + 1) * C * RS : dump_rows;
#pragma unroll
            for (int c = 0; c < C; ++c) { wa[(size_t)c * RS] = zb[c].x; wb[(size_t)c * RS] = zb[c].y; }
            if (SKIP && adj_out) {                        // residual layer: its skip source needs this adjoint too
                float* sa = adj_out + (size_t)(oka ? m0 + 2 * h : 0) * C * RS;
                float* sb = adj_out + (size_t)(okb ? m0 + 2 * h + 1 : 0) * C * RS;
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    if (oka) sa[(size_t)c * RS] = acc[h][c].x;
                    if (okb) sb[(size_t)c * RS] = acc[h][c].y;
                }
            }
        }
    }
    if (!fold_bias) bias_grad<NF, NS>(L, out_rows, RS, sink);
}

// Weight (and bias) gradients of the FIRST linear layer: its input jet is (x, e_dir, 0); the bias rides
// in column n_in when n_in < PINN_MAX_DIMS.
template <int NF, int NS>
PINN_HD void wgrad_input_layer(const DevLayer& L, const float* __restrict__ out_rows,
                               const float* __restrict__ coords, int RS, const float* __restrict__ dirv,
                               const GradSink& sink) {
    constexpr int C = 1 + NF + NS;
    float2 x[PINN_MAX_DIMS / 2];
    float2 dv[NF > 0 ? NF : 1][PINN_MAX_DIMS / 2];
#pragma unroll
    for (int h = 0; h < PINN_MAX_DIMS / 2; ++h) {
        const int ma = 2 * h, mb = 2 * h + 1;
        x[h] = make_float2((ma < L.n_in) ? coords[(size_t)ma * RS] : (ma == L.n_in ? 1.0f : 0.0f),
                           (mb < L.n_in) ? coords[(size_t)mb * RS] : (mb == L.n_in ? 1.0f : 0.0f));
#pragma unroll
        for (int d = 0; d < NF; ++d) dv[d][h] = make_float2(dirv[d * PINN_MAX_DIMS + ma], dirv[d * PINN_MAX_DIMS + mb]);
    }
#pragma unroll 1
    for (int j0 = 0; j0 < L.n_out; j0 += 4) {
        float v[4 * PINN_MAX_DIMS];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int j = j0 + jj < L.n_out ? j0 + jj : L.n_out - 1;
            const float* row = out_rows + (size_t)j * C * RS;
            float zb[1 + NF];
#pragma unroll
            for (int c = 0; c < 1 + NF; ++c) zb[c] = row[(size_t)c * RS];
#pragma unroll
            for (int h = 0; h < PINN_MAX_DIMS / 2; ++h) {
                float2 e = PINN_FMUL2(x[h], zb[0]);
#pragma unroll
                for (int d = 0; d < NF; ++d) e = PINN_FFMA2(dv[d][h], zb[1 + d], e);
                v[jj * PINN_MAX_DIMS + 2 * h] = e.x;
                v[jj * PINN_MAX_DIMS + 2 * h + 1] = e.y;
            }
        }
        emit_entries<4 * PINN_MAX_DIMS>(v, [&](int e, float t) {
            const int j = j0 + e / PINN_MAX_DIMS, m = e % PINN_MAX_DIMS;
            sink.add_if(j < L.n_out && m <= L.n_in && m < PINN_MAX_DIMS,
                        m < L.n_in ? L.w_off + j * L.n_in + m : L.b_off + j, t);
        });
    }
    if (L.n_in >= PINN_MAX_DIMS) bias_grad<NF, NS>(L, out_rows, RS, sink);
}

// ----------------------------------------------------------------------------------------------
// The whole step for ONE point.  `st` is the thread's column of per-point storage (row stride RS).
// Returns the residual; accumulates loss / log_scale / V partials into the caller's registers.
// ----------------------------------------------------------------------------------------------
template <int NF, int NS>
struct PointPartials { float loss, sbar, vbar[PINN_MAX_VARS]; };

template <int NF, int NS, int JF, bool GEN = true>
PINN_HD float point_step(const DevPlan& P, const float* __restrict__ sw /* weights */,
                         const float* __restrict__ pvals /* flat params (for log_scale, V) */,
                         float* __restrict__ st, int RS, bool valid, float inv_n,
                         const GradSink& sink, PointPartials<NF, NS>& part) {
    constexpr int C = 1 + NF + NS;
    const int Ln = P.n_layers;
    float* coords = st;
    float* units = st + (size_t)P.row_units * RS;
    float* scr = st + (size_t)P.row_scr * RS;

    // ---- forward through the hidden layers ----
#pragma unroll 1
    for (int l = 0; l + 1 < Ln; ++l) {
        const DevLayer& L = P.layer[l];
        int in_act = PINN_ACT_NONE;
        const float* in_rows = (l == 0) ? coords : layer_output<GEN>(P, l - 1, units, C, RS, in_act);
        fwd_layer<NF, NS, JF, GEN>(L, sw, in_rows, l == 0, in_act, &P.dir_vec[0][0],
                                   units + (size_t)L.unit_base * C * RS, RS);
        if (GEN && L.skip_src >= 0) skip_sum_pass<NF, NS>(P, l, units, RS);
    }
    float N[C];
    {
        const DevLayer& L = P.layer[Ln - 1];
        int in_act = PINN_ACT_NONE;
        const float* in_rows = (Ln == 1) ? coords : layer_output<GEN>(P, Ln - 2, units, C, RS, in_act);
        fwd_final<NF, NS, GEN>(L, sw, in_rows, Ln == 1, in_act, &P.dir_vec[0][0], RS, N);
    }

    // ---- ansatz + residual ----
    float icj[C];
#pragma unroll
    for (int c = 0; c < C; ++c) icj[c] = 0.0f;
    if (P.has_ic) {
        eval_prog(P.ic, P.n_ic, scr, RS, coords, pvals, P.var_off);
#pragma unroll
        for (int c = 0; c < C; ++c) icj[c] = scr[(size_t)P.ic_out[c] * RS];
    }
    float log_scale = pvals[P.log_scale_off];
    AnsatzState<NF, NS> as;
    float u[C];
    ansatz_forward<NF, NS, GEN>(P, coords, RS, log_scale, N, icj, as, u);
#pragma unroll
    for (int c = 0; c < C; ++c) scr[(size_t)c * RS] = u[c];
    eval_prog(P.eq, P.n_eq, scr, RS, coords, pvals, P.var_off);
    float r = scr[(size_t)P.eq_out[0] * RS];
    float rb = valid ? 2.0f * r * inv_n : 0.0f;
    if (valid) part.loss = fmaf(r * inv_n, r, part.loss);
    float ub[C];
#pragma unroll
    for (int c = 0; c < C; ++c) ub[c] = rb * scr[(size_t)P.eq_out[1 + c] * RS];
#pragma unroll
    for (int i = 0; i < PINN_MAX_VARS; ++i)
        if (i < P.n_vars) part.vbar[i] = fmaf(rb, scr[(size_t)P.eq_out[1 + C + i] * RS], part.vbar[i]);
    if (GEN && P.ic_has_vars) {                // u_c = S v_c + ic_c: variables of the initial condition
#pragma unroll
        for (int i = 0; i < PINN_MAX_VARS; ++i) {
            if (i < P.n_vars) {
#pragma unroll
                for (int c = 0; c < C; ++c)
                    part.vbar[i] = fmaf(ub[c], scr[(size_t)P.ic_out[C * (1 + i) + c] * RS], part.vbar[i]);
            }
        }
    }

    float Nb[C];
    part.sbar += ansatz_adjoint<NF, NS>(P, as, ub, Nb);

    // ---- reverse sweep ----
    {
        const DevLayer& L = P.layer[Ln - 1];
        float* out_rows = units + (size_t)L.unit_base * C * RS;
#pragma unroll
        for (int c = 0; c < C; ++c) out_rows[(size_t)c * RS] = Nb[c];
    }
#pragma unroll 1
    for (int l = Ln - 1; l >= 1; --l) {
        const DevLayer& L = P.layer[l];
        float* out_rows = units + (size_t)L.unit_base * C * RS;
        const DevLayer& B = P.layer[l - 1];                 // the layer below
        float* in_rows = units + (size_t)B.unit_base * C * RS;
        int load_act;
        const float* load_rows = layer_output<GEN>(P, l - 1, units, C, RS, load_act);
        const float* adj_in = B.adj_from >= 0 ? units + (size_t)P.layer[B.adj_from].post_base * C * RS : nullptr;
        float* adj_out = B.skip_src >= 0 ? units + (size_t)B.post_base * C * RS : nullptr;
        if (GEN && (B.post_base >= 0 || B.adj_from >= 0)) { // residual wiring around the layer below (rare path)
            if (L.n_out == 1) bwd_layer<NF, NS, 1, true>(L, B.act, sw, out_rows, in_rows, RS, sink, load_rows, load_act, adj_in, adj_out, scr);
            else              bwd_layer<NF, NS, 4, true>(L, B.act, sw, out_rows, in_rows, RS, sink, load_rows, load_act, adj_in, adj_out, scr);
        } else {
            if (L.n_out == 1) bwd_layer<NF, NS, 1, false, GEN>(L, B.act, sw, out_rows, in_rows, RS, sink, in_rows, B.act, nullptr, nullptr, scr);
            else              bwd_layer<NF, NS, 4, false, GEN>(L, B.act, sw, out_rows, in_rows, RS, sink, in_rows, B.act, nullptr, nullptr, scr);
        }
    }
    {
        const DevLayer& L = P.layer[0];
        float* out_rows = units + (size_t)L.unit_base * C * RS;
        wgrad_input_layer<NF, NS>(L, out_rows, coords, RS, &P.dir_vec[0][0], sink);
    }
    return r;
}

// Forward-only value u(x) for one point (predict path): no jets (NF = NS = 0).
template <int JF>
PINN_HD float point_forward(const DevPlan& P, const float* __restrict__ sw, const float* __restrict__ pvals,
                            float* __restrict__ st, int RS, int row_scr_fwd) {
    const int Ln = P.n_layers;
    float* coords = st;
    float* units = st + (size_t)P.row_units * RS;
    float* scr = st + (size_t)row_scr_fwd * RS;
    float dummy_dir[1] = {0.0f};
    for (int l = 0; l + 1 < Ln; ++l) {
        const DevLayer& L = P.layer[l];
        int in_act = PINN_ACT_NONE;
        const float* in_rows = (l == 0) ? coords : layer_output(P, l - 1, units, 1, RS, in_act);
        fwd_layer<0, 0, JF>(L, sw, in_rows, l == 0, in_act, dummy_dir, units + (size_t)L.unit_base * RS, RS);
        if (L.skip_src >= 0) skip_sum_pass<0, 0>(P, l, units, RS);
    }
    float N[1];
    {
        const DevLayer& L = P.layer[Ln - 1];
        int in_act = PINN_ACT_NONE;
        const float* in_rows = (Ln == 1) ? coords : layer_output(P, Ln - 2, units, 1, RS, in_act);
        fwd_final<0, 0>(L, sw, in_rows, Ln == 1, in_act, dummy_dir, RS, N);
    }
    float icj[1] = {0.0f};
    if (P.has_ic) {
        eval_prog(P.ic, P.n_ic, scr, RS, coords, pvals, P.var_off);
        icj[0] = scr[(size_t)P.ic_out[0] * RS];
    }
    AnsatzState<0, 0> as;
    float u[1];
    ansatz_forward<0, 0>(P, coords, RS, pvals[P.log_scale_off], N, icj, as, u);
    return u[0];
}

}  // namespace pinn
