// pinn_device_hi.cuh — per-point math of the fused fit step for derivatives of order 3 and 4 (sm_90a).
//
// The reference's `D` nests arbitrarily (pydens/model_torch.py:174-178): D(D(D(f, x), x), x) is how a user writes
// u_xxx (Korteweg-de Vries), four levels give u_xxxx (beams, Kuramoto-Sivashinsky).  Here every derivative direction
// (an axis of the point matrix) carries its whole univariate Taylor jet up to order K = 3 or 4:
//     channel 0 = value,  channel 1 + d*K + (k-1) = k-th derivative along direction d   (C = 1 + NF*K channels).
// Linear layers act on every channel alike; an activation maps the jet by Faa di Bruno's formula
//     a1 = s1 z1,  a2 = s2 z1^2 + s1 z2,  a3 = s3 z1^3 + 3 s2 z1 z2 + s1 z3,
//     a4 = s4 z1^4 + 6 s3 z1^2 z2 + s2 (3 z2^2 + 4 z1 z3) + s1 z4          (s_k = k-th derivative of the activation)
// and the reverse sweep is its hand-derived adjoint (needs s_{K+1}); for tanh / sigmoid every s_k is a polynomial of
// the stored activation value.  The ansatz (model_torch.py:107-128) is a product of jets (Leibniz), its adjoint the
// transposed product, including d/d log_scale through the time gate.
//
// Written per THREAD like pinn_device.cuh and `__host__ __device__` for the same reason: tests/emul compiles these
// very functions with g++ and checks them against the fp64 oracle.  Scope: dense chains and residual layouts ('R ... +')
// with any of the fused activations; directions are the differentiated arguments plus, per pair of arguments with a
// mixed derivative, the two diagonals e_i +- e_j that carry it by polarisation (u_xxyy = ((d_x+d_y)^4 + (d_x-d_y)^4
// - 2 u_xxxx - 2 u_yyyy) / 12: what the biharmonic operator needs); samplers, variables (in the equation and in the
// initial condition), domains, boundary / initial conditions are as in the main path.  This path favours clarity over
// the last FMA: it exists so that such equations stay on the GPU in one launch instead of falling back to nested
// autograd graphs.
#pragma once

#include "pinn_device.cuh"

namespace pinn {
namespace hi {

template <int NF, int K> struct Jet { static constexpr int C = 1 + NF * K; };

PINN_HD constexpr int chan(int K, int d, int k) { return 1 + d * K + (k - 1); }   // k = 1..K

// s[1..K+1]: derivatives of the activation w.r.t. its argument, from the STORED value a (tanh / sigmoid: the
// activation value itself; identity: anything).
template <int K>
PINN_HD void act_derivs(int act, float a, float (&s)[K + 2]) {
    const float a2 = a * a;
    if (act == PINN_ACT_TANH) {
        const float s1 = 1.0f - a2;
        s[1] = s1;
        s[2] = -2.0f * a * s1;
        s[3] = s1 * fmaf(6.0f, a2, -2.0f);
        s[4] = s1 * a * fmaf(-24.0f, a2, 16.0f);
        if (K + 1 >= 5) s[K + 1 >= 5 ? 5 : 0] = s1 * fmaf(fmaf(120.0f, a2, -120.0f), a2, 16.0f);
    } else if (act == PINN_ACT_SIGMOID) {
        const float s1 = a - a2;
        s[1] = s1;
        s[2] = s1 * fmaf(-2.0f, a, 1.0f);
        s[3] = s1 * fmaf(fmaf(6.0f, a, -6.0f), a, 1.0f);
        s[4] = s1 * fmaf(fmaf(fmaf(-24.0f, a, 36.0f), a, -14.0f), a, 1.0f);
        if (K + 1 >= 5) s[K + 1 >= 5 ? 5 : 0] = s1 * fmaf(fmaf(fmaf(fmaf(120.0f, a, -240.0f), a, 150.0f), a, -30.0f), a, 1.0f);
    } else if (act == PINN_ACT_SIN) {                     // z-stored: `a` is the pre-activation z itself
        float sn, cs;
#if defined(__CUDA_ARCH__)
        sincosf(a, &sn, &cs);
#else
        sn = sinf(a); cs = cosf(a);
#endif
        s[1] = cs; s[2] = -sn; s[3] = -cs; s[4] = sn;
        if (K + 1 >= 5) s[K + 1 >= 5 ? 5 : 0] = cs;
    } else if (act == PINN_ACT_SOFTPLUS || act == PINN_ACT_SILU) {     // z-stored; both are built from the logistic function
        const float z = a;
        const float sg = fmaf(0.5f, tanh_acc(0.5f * z), 0.5f);
        float g[K + 2];                                   // g[n] = n-th derivative of the logistic function at z
        act_derivs<K>(PINN_ACT_SIGMOID, sg, g);
        if (act == PINN_ACT_SOFTPLUS) {                   // softplus' = logistic
            s[1] = sg;
#pragma unroll
            for (int k = 2; k <= K + 1; ++k) s[k] = g[k - 1];
        } else {                                          // SiLU = z logistic(z): s_k = k g_{k-1} + z g_k
            s[1] = fmaf(z, g[1], sg);
#pragma unroll
            for (int k = 2; k <= K + 1; ++k) s[k] = fmaf(z, g[k], (float)k * g[k - 1]);
        }
    } else if (act == PINN_ACT_GELU) {                    // z Phi(z): s_k = k phi^(k-2) + z phi^(k-1), phi^(n) = He_n(-z)... spelled out
        const float z = a, z2 = z * z;
        const float phi = 0.3989422804014327f * expf(-0.5f * z2);
        const float Phi = 0.5f * erfcf(-0.7071067811865476f * z);
        s[1] = fmaf(z, phi, Phi);
        s[2] = phi * (2.0f - z2);
        s[3] = phi * z * (z2 - 4.0f);
        s[4] = phi * fmaf(fmaf(-1.0f, z2, 7.0f), z2, -4.0f);
        if (K + 1 >= 5) s[K + 1 >= 5 ? 5 : 0] = phi * z * fmaf(fmaf(1.0f, z2, -11.0f), z2, 18.0f);
    } else {
        s[1] = 1.0f;
#pragma unroll
        for (int k = 2; k <= K + 1; ++k) s[k] = 0.0f;
    }
}

// value of a hidden unit from what its row stores (tanh / sigmoid / identity store the value, the others store z)
PINN_HD float act_value(int act, float stored) {
    if (act == PINN_ACT_SIN) return sinf(stored);
    if (act == PINN_ACT_SOFTPLUS) return fmaxf(stored, 0.0f) + log1pf(expf(-fabsf(stored)));
    if (act == PINN_ACT_SILU) return stored * fmaf(0.5f, tanh_acc(0.5f * stored), 0.5f);
    if (act == PINN_ACT_GELU) return stored * 0.5f * erfcf(-0.7071067811865476f * stored);
    return stored;
}

// Post-activation jet of one direction from its pre-activation jet z[1..K] (index 0 unused).
template <int K>
PINN_HD void post_dir(const float (&s)[K + 2], const float (&z)[K + 1], float (&p)[K + 1]) {
    const float z1 = z[1], z2 = z[2], z3 = z[3];
    const float z11 = z1 * z1;
    p[1] = s[1] * z1;
    p[2] = fmaf(s[2], z11, s[1] * z2);
    p[3] = fmaf(s[3] * z11, z1, fmaf(3.0f * s[2] * z1, z2, s[1] * z3));
    if (K >= 4) {
        const float z4 = z[K >= 4 ? 4 : 0];
        p[K >= 4 ? 4 : 0] = fmaf(s[4] * z11, z11, fmaf(6.0f * s[3] * z11, z2,
                                 fmaf(s[2], fmaf(3.0f * z2, z2, 4.0f * z1 * z3), s[1] * z4)));
    }
}

// Adjoint of post_dir: post-adjoints pb[1..K] of one direction -> pre-adjoints zb[1..K]; returns the direction's
// contribution to the adjoint of the value channel z0 (through the dependence of every s_k on z0).
template <int K>
PINN_HD float adjoint_dir(const float (&s)[K + 2], const float (&z)[K + 1], const float (&pb)[K + 1], float (&zb)[K + 1]) {
    const float z1 = z[1], z2 = z[2], z3 = z[3];
    const float z11 = z1 * z1;
    const float b1 = pb[1], b2 = pb[2], b3 = pb[3];
    const float b4 = (K >= 4) ? pb[K >= 4 ? 4 : 0] : 0.0f;
    const float z4 = (K >= 4) ? z[K >= 4 ? 4 : 0] : 0.0f;
    const float s5 = (K >= 4) ? s[K >= 4 ? 5 : 0] : 0.0f;
    // d a_k / d z_j
    float zb1 = s[1] * b1;
    zb1 = fmaf(2.0f * s[2] * z1, b2, zb1);
    zb1 = fmaf(fmaf(3.0f * s[3], z11, 3.0f * s[2] * z2), b3, zb1);
    float zb2 = fmaf(3.0f * s[2] * z1, b3, s[1] * b2);
    float zb3 = s[1] * b3;
    if (K >= 4) {
        zb1 = fmaf(fmaf(4.0f * s[4] * z11, z1, fmaf(12.0f * s[3] * z1, z2, 4.0f * s[2] * z3)), b4, zb1);
        zb2 = fmaf(fmaf(6.0f * s[3], z11, 6.0f * s[2] * z2), b4, zb2);
        zb3 = fmaf(4.0f * s[2] * z1, b4, zb3);
        zb[K >= 4 ? 4 : 0] = s[1] * b4;
    }
    zb[1] = zb1; zb[2] = zb2; zb[3] = zb3;
    // d a_k / d z0 = the same formulas with every s_j replaced by s_{j+1}
    float z0 = s[2] * z1 * b1;
    z0 = fmaf(fmaf(s[3], z11, s[2] * z2), b2, z0);
    z0 = fmaf(fmaf(s[4] * z11, z1, fmaf(3.0f * s[3] * z1, z2, s[2] * z3)), b3, z0);
    if (K >= 4)
        z0 = fmaf(fmaf(s5 * z11, z11, fmaf(6.0f * s[4] * z11, z2, fmaf(s[3], fmaf(3.0f * z2, z2, 4.0f * z1 * z3), s[2] * z4))), b4, z0);
    return z0;
}

// Stored rows of one hidden unit (value + pre-activation jets) -> its post-activation jet, all C channels.
template <int NF, int K>
PINN_HD void load_post(const float* __restrict__ row, int RS, int act, float (&p)[1 + NF * K]) {
    const float a = row[0];
    float s[K + 2];
    act_derivs<K>(act, a, s);
    p[0] = act_value(act, a);
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        float z[K + 1], q[K + 1];
#pragma unroll
        for (int k = 1; k <= K; ++k) z[k] = row[(size_t)chan(K, d, k) * RS];
        post_dir<K>(s, z, q);
#pragma unroll
        for (int k = 1; k <= K; ++k) p[chan(K, d, k)] = q[k];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Forward
// ---------------------------------------------------------------------------------------------------------------
// One dense layer, 4 output units at a time: z_j,c = sum_m W[j][m] post_m,c (+ bias on the value channel); the value
// channel is stored through the activation (a hidden unit keeps a, not z), the jets raw.
template <int NF, int K>
PINN_HD void fwd_layer(const DevPlan& P, int l, const float* __restrict__ sw, const float* __restrict__ coords,
                       float* __restrict__ units, int RS) {
    constexpr int C = 1 + NF * K;
    const DevLayer& L = P.layer[l];
    const float* Wt = sw + L.wt_s;                       // [n_in][n_out_p4]
    const float* bias = sw + L.b_s;
    const ActC out_act = make_actc(L.act);
    float* out_rows = units + (size_t)L.unit_base * C * RS;
    int in_act = PINN_ACT_NONE;                          // a residual layer below is read from its post buffer, as identity
    const float* in_rows = l > 0 ? layer_output<true>(P, l - 1, units, C, RS, in_act) : nullptr;
#pragma unroll 1
    for (int j0 = 0; j0 < L.n_out; j0 += 4) {
        float acc[4][C];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            acc[q][0] = bias[j0 + q];
#pragma unroll
            for (int c = 1; c < C; ++c) acc[q][c] = 0.0f;
        }
        if (l == 0) {
            // input jet of coordinate k along direction v: (x_k; v_k at first order; nothing above)
#pragma unroll 1
            for (int k = 0; k < L.n_in; ++k) {
                const float4 w = *reinterpret_cast<const float4*>(Wt + (size_t)k * L.n_out_p4 + j0);
                const float x = coords[(size_t)k * RS];
                const float wq[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    acc[q][0] = fmaf(wq[q], x, acc[q][0]);
#pragma unroll
                    for (int d = 0; d < NF; ++d)
                        acc[q][chan(K, d, 1)] = fmaf(wq[q], P.dir_vec[d][k], acc[q][chan(K, d, 1)]);
                }
            }
        } else {
#pragma unroll 1
            for (int m = 0; m < L.n_in; ++m) {
                float p[C];
                load_post<NF, K>(in_rows + (size_t)m * C * RS, RS, in_act, p);
                const float4 w = *reinterpret_cast<const float4*>(Wt + (size_t)m * L.n_out_p4 + j0);
                const float wq[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int c = 0; c < C; ++c) acc[q][c] = fmaf(wq[q], p[c], acc[q][c]);
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (j0 + q < L.n_out) {
                float* row = out_rows + (size_t)(j0 + q) * C * RS;
                row[0] = act_store<false>(out_act, acc[q][0]);
#pragma unroll
                for (int c = 1; c < C; ++c) row[(size_t)c * RS] = acc[q][c];
            }
        }
    }
}

// Residual layer l ('... R ... fa+', reference Block layout letters): post buffer <- act-jet(stored jet of l) + output of
// layer skip_src (whole jets add channel by channel); consumers read the buffer like the output of an identity activation.
template <int NF, int K>
PINN_HD void skip_sum_jets(const DevPlan& P, int l, float* __restrict__ units, int RS) {
    constexpr int C = 1 + NF * K;
    const DevLayer& L = P.layer[l];
    int src_act;
    const float* src_rows = layer_output<true>(P, L.skip_src, units, C, RS, src_act);
    const float* pre_rows = units + (size_t)L.unit_base * C * RS;
    float* post_rows = units + (size_t)L.post_base * C * RS;
#pragma unroll 1
    for (int j = 0; j < L.n_out; ++j) {
        float a[C], b[C];
        load_post<NF, K>(pre_rows + (size_t)j * C * RS, RS, L.act, a);
        load_post<NF, K>(src_rows + (size_t)j * C * RS, RS, src_act, b);
#pragma unroll
        for (int c = 0; c < C; ++c) post_rows[((size_t)j * C + c) * RS] = a[c] + b[c];
    }
}

// Last layer (one output unit, no activation): the network jet N lands in registers.
template <int NF, int K>
PINN_HD void fwd_final(const DevPlan& P, const float* __restrict__ sw, const float* __restrict__ coords,
                       const float* __restrict__ units, int RS, float (&N)[1 + NF * K]) {
    constexpr int C = 1 + NF * K;
    const int Ln = P.n_layers;
    const DevLayer& L = P.layer[Ln - 1];
    const float* w = sw + L.w_s;                         // reverse layout, row 0 = the single weight row
    N[0] = sw[L.b_s];
#pragma unroll
    for (int c = 1; c < C; ++c) N[c] = 0.0f;
    if (Ln == 1) {
        for (int k = 0; k < L.n_in; ++k) {
            N[0] = fmaf(w[k], coords[(size_t)k * RS], N[0]);
#pragma unroll
            for (int d = 0; d < NF; ++d)
                N[chan(K, d, 1)] = fmaf(w[k], P.dir_vec[d][k], N[chan(K, d, 1)]);
        }
    } else {
        int in_act;
        const float* in_rows = layer_output<true>(P, Ln - 2, units, C, RS, in_act);
#pragma unroll 1
        for (int m = 0; m < L.n_in; ++m) {
            float p[C];
            load_post<NF, K>(in_rows + (size_t)m * C * RS, RS, in_act, p);
            const float wm = w[m];
#pragma unroll
            for (int c = 0; c < C; ++c) N[c] = fmaf(wm, p[c], N[c]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Ansatz (model_torch.py:107-128) as products of jets:  v = bc + G N,  u = S v + ic
//   G = prod_i q_i(x_i), q_i = (x - lo)(hi - x) / w^2 over the spatial dims: along a direction v its jet is the product
//       of the jets (q_i, q_i' v_i, q_i'' v_i^2, 0, 0)
//   S = sigmoid(y) - 1/2, y = (t - t0) / exp(log_scale): along v its jet is sigmoid^(k)(y) (v_t / s)^k
// ---------------------------------------------------------------------------------------------------------------
PINN_HD float binom(int n, int k) {
    const float tab[5][5] = {{1, 0, 0, 0, 0}, {1, 1, 0, 0, 0}, {1, 2, 1, 0, 0}, {1, 3, 3, 1, 0}, {1, 4, 6, 4, 1}};
    return tab[n][k];
}

template <int NF, int K>
struct AnsatzHi {
    float G, Gj[NF][K + 1];            // boundary factor and its jet per direction (Gj[d][0] = G)
    float Sg, Sj[NF][K + 1];           // time gate and its jet per direction
    float dS0, dS[NF][K + 1];          // d/d log_scale of the gate's value and of Sj[d][k], k >= 1
    float v0, vj[NF][K + 1];           // jet of v = bc + G N
};

// c = a * b for jets of derivatives (Leibniz), in place on a
template <int K>
PINN_HD void jet_mul(float (&a)[K + 1], const float (&b)[K + 1]) {
    float c[K + 1];
#pragma unroll
    for (int n = 0; n <= K; ++n) {
        float t = 0.0f;
#pragma unroll
        for (int k = 0; k <= n; ++k) t = fmaf(binom(n, k) * a[k], b[n - k], t);
        c[n] = t;
    }
#pragma unroll
    for (int n = 0; n <= K; ++n) a[n] = c[n];
}

template <int NF, int K>
PINN_HD void ansatz_forward(const DevPlan& P, const float* __restrict__ coords, int RS, float log_scale,
                            const float (&N)[1 + NF * K], const float* __restrict__ icj, AnsatzHi<NF, K>& st,
                            float (&u)[1 + NF * K]) {
    // boundary factor along the line x + tau v: the product over the spatial dims of the quadratics' jets
    // (q, q' v_i, q'' v_i^2, 0, 0) — along an axis this is (G, others q', others q'', 0, 0)
    st.G = 1.0f;
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        float g[K + 1];
        g[0] = 1.0f;
#pragma unroll
        for (int n = 1; n <= K; ++n) g[n] = 0.0f;
        if (P.has_bc) {
            for (int i = 0; i < P.nsp; ++i) {
                const float x = coords[(size_t)i * RS];
                const float vi = P.dir_vec[d][i];
                float q[K + 1];
                q[0] = (x - P.lo[i]) * (P.hi[i] - x) * P.inv_w2[i];
                q[1] = (P.lo[i] + P.hi[i] - 2.0f * x) * P.inv_w2[i] * vi;
                q[2] = -2.0f * P.inv_w2[i] * vi * vi;
#pragma unroll
                for (int n = 3; n <= K; ++n) q[n] = 0.0f;
                jet_mul<K>(g, q);
            }
        }
#pragma unroll
        for (int n = 0; n <= K; ++n) st.Gj[d][n] = g[n];
    }
    if (P.has_bc) {
        float G = 1.0f;
        for (int i = 0; i < P.nsp; ++i) {
            const float x = coords[(size_t)i * RS];
            G *= (x - P.lo[i]) * (P.hi[i] - x) * P.inv_w2[i];
        }
        st.G = G;
    }
#pragma unroll
    for (int d = 0; d < NF; ++d) st.Gj[d][0] = st.G;    // one value for every direction (same product, same order)
    // time gate
    st.Sg = 1.0f; st.dS0 = 0.0f;
    float sg_s[K + 2];
#pragma unroll
    for (int n = 0; n <= K + 1; ++n) sg_s[n] = 0.0f;
    float inv_s = 1.0f, y = 0.0f;
    if (P.has_ic) {
        const float t = coords[(size_t)(P.ndims - 1) * RS];
        inv_s = expf(-log_scale);
        y = (t - P.t0) * inv_s;
        const float sig = 1.0f / (1.0f + expf(-y));
        act_derivs<K>(PINN_ACT_SIGMOID, sig, sg_s);        // sg_s[n] = sigmoid^(n)(y), n = 1..K+1
        st.Sg = sig - 0.5f;
        st.dS0 = -y * sg_s[1];
    }
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        st.Sj[d][0] = st.Sg;
        st.dS[d][0] = st.dS0;
        // along v the gate's argument moves with speed v_t / s:  d^n/dtau^n = sigmoid^(n)(y) (v_t / s)^n, and
        // d/d log_scale of that = -(y sigmoid^(n+1)(y) + n sigmoid^(n)(y)) (v_t / s)^n
        const float rate = P.has_ic ? P.dir_vec[d][P.ndims - 1] * inv_s : 0.0f;
        float pw = 1.0f;
#pragma unroll
        for (int n = 1; n <= K; ++n) {
            pw *= rate;
            st.Sj[d][n] = sg_s[n] * pw;
            st.dS[d][n] = -fmaf(y, sg_s[n + 1], (float)n * sg_s[n]) * pw;
        }
    }
    // v = bc + G N, u = S v + ic
    st.v0 = P.has_bc ? fmaf(st.G, N[0], P.bc) : N[0];
    u[0] = P.has_ic ? fmaf(st.Sg, st.v0, icj[0]) : st.v0;
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        st.vj[d][0] = st.v0;
#pragma unroll
        for (int n = 1; n <= K; ++n) {
            float v = 0.0f;
#pragma unroll
            for (int k = 0; k <= n; ++k) {
                const float Nn = (n - k == 0) ? N[0] : N[chan(K, d, n - k)];
                v = fmaf(binom(n, k) * st.Gj[d][k], Nn, v);
            }
            st.vj[d][n] = v;
        }
#pragma unroll
        for (int n = 1; n <= K; ++n) {
            float w = 0.0f;
#pragma unroll
            for (int k = 0; k <= n; ++k) w = fmaf(binom(n, k) * st.Sj[d][k], st.vj[d][n - k], w);
            u[chan(K, d, n)] = P.has_ic ? w + icj[chan(K, d, n)] : st.vj[d][n];
        }
    }
}

// Adjoint: ub (adjoints of the u-jet) -> Nb (adjoints of the network jet); returns the adjoint of log_scale.
template <int NF, int K>
PINN_HD float ansatz_adjoint(const DevPlan& P, const AnsatzHi<NF, K>& st, const float (&ub)[1 + NF * K],
                             float (&Nb)[1 + NF * K]) {
    constexpr int C = 1 + NF * K;
#pragma unroll
    for (int c = 0; c < C; ++c) Nb[c] = 0.0f;
    float vb0 = P.has_ic ? st.Sg * ub[0] : ub[0];          // adjoint of the value of v
    float sbar = P.has_ic ? st.dS0 * st.v0 * ub[0] : 0.0f;
#pragma unroll
    for (int d = 0; d < NF; ++d) {
        float vb[K + 1];
#pragma unroll
        for (int n = 0; n <= K; ++n) vb[n] = 0.0f;
        if (P.has_ic) {
#pragma unroll
            for (int n = 1; n <= K; ++n) {
                const float un = ub[chan(K, d, n)];
#pragma unroll
                for (int k = 0; k <= n; ++k) {
                    const float c = binom(n, k);
                    vb[n - k] = fmaf(c * st.Sj[d][k], un, vb[n - k]);
                    sbar = fmaf(c * st.dS[d][k] * st.vj[d][n - k], un, sbar);
                }
            }
        } else {
#pragma unroll
            for (int n = 1; n <= K; ++n) vb[n] = ub[chan(K, d, n)];
        }
        vb0 += vb[0];
        // v_n = sum_k C(n,k) Gj[k] N_{n-k}
#pragma unroll
        for (int n = 1; n <= K; ++n) {
#pragma unroll
            for (int k = 0; k <= n; ++k) {
                const float g = P.has_bc ? binom(n, k) * st.Gj[d][k] : (k == 0 ? 1.0f : 0.0f);
                if (n - k == 0) Nb[0] = fmaf(g, vb[n], Nb[0]);
                else Nb[chan(K, d, n - k)] = fmaf(g, vb[n], Nb[chan(K, d, n - k)]);
            }
        }
    }
    Nb[0] = fmaf(P.has_bc ? st.G : 1.0f, vb0, Nb[0]);
    return sbar;
}

// ---------------------------------------------------------------------------------------------------------------
// Reverse sweep
// ---------------------------------------------------------------------------------------------------------------
// Reverse of linear layer l >= 1 (its pre-activation adjoints are stored in its rows): weight gradients of l
// (reduced over the warp, 4 output units x 4 input units per batch) and, fused, the adjoints of the layer below —
// pushed through that layer's activation and written over its stored jet in place.  Rows / columns past the end are
// read from clamped addresses and meet zero-padded weights; their gradient entries are dropped at the sink.
// Residual wiring around the layer below (the bookkeeping of pinn::bwd_layer<..., SKIP = true>): when B closes a
// residual block its output was read from its post buffer, and the adjoint of that output also belongs to the block's
// skip source — it is stashed in the (now dead) post buffer; when B is the source of a skip, the adjoint stashed by the
// closing layer `B.adj_from` is added before B's activation.
template <int NF, int K>
PINN_HD void bwd_layer(const DevPlan& P, int l, const float* __restrict__ sw, float* __restrict__ units, int RS,
                       const GradSink& sink, float* __restrict__ dump_rows) {
    constexpr int C = 1 + NF * K;
    const DevLayer& L = P.layer[l];
    const DevLayer& B = P.layer[l - 1];
    const float* W = sw + L.w_s;                          // [n_out_p4][n_in_p8], zero padded
    const float* out_rows = units + (size_t)L.unit_base * C * RS;
    float* in_rows = units + (size_t)B.unit_base * C * RS;
    int load_act;
    const float* load_rows = layer_output<true>(P, l - 1, units, C, RS, load_act);
    const float* adj_in = B.adj_from >= 0 ? units + (size_t)P.layer[B.adj_from].post_base * C * RS : nullptr;
    float* adj_out = B.skip_src >= 0 ? units + (size_t)B.post_base * C * RS : nullptr;
#pragma unroll 1
    for (int m0 = 0; m0 < L.n_in; m0 += 4) {
        float post[4][C], acc[4][C];
#pragma unroll
        for (int h = 0; h < 4; ++h) {
            const int m = m0 + h < L.n_in ? m0 + h : L.n_in - 1;
            load_post<NF, K>(load_rows + (size_t)m * C * RS, RS, load_act, post[h]);
#pragma unroll
            for (int c = 0; c < C; ++c) acc[h][c] = 0.0f;
        }
#pragma unroll 1
        for (int j0 = 0; j0 < L.n_out; j0 += 4) {
            float v[16];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int j = j0 + jj;                    // < n_out_p4: rows past n_out hold zero weights
                const int jc = j < L.n_out ? j : L.n_out - 1;
                const float* row = out_rows + (size_t)jc * C * RS;
                float zb[C];
#pragma unroll
                for (int c = 0; c < C; ++c) zb[c] = row[(size_t)c * RS];
                const float4 w4 = *reinterpret_cast<const float4*>(W + (size_t)j * L.n_in_p8 + m0);
                const float w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                for (int h = 0; h < 4; ++h) {
                    float e = 0.0f;
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        acc[h][c] = fmaf(w[h], zb[c], acc[h][c]);
                        e = fmaf(post[h][c], zb[c], e);
                    }
                    v[jj * 4 + h] = e;
                }
            }
            emit_entries<16>(v, [&](int e, float t) {
                const int j = j0 + e / 4, m = m0 + e % 4;
                sink.add_if(j < L.n_out && m < L.n_in, L.w_off + j * L.n_in + m, t);
            });
        }
        // adjoints of the layer below through its activation, stored in place
#pragma unroll
        for (int h = 0; h < 4; ++h) {
            const bool ok = m0 + h < L.n_in;
            float* row = in_rows + (size_t)(ok ? m0 + h : 0) * C * RS;
            if (adj_in) {
                const float* ai = adj_in + (size_t)(ok ? m0 + h : 0) * C * RS;
#pragma unroll
                for (int c = 0; c < C; ++c) acc[h][c] += ai[(size_t)c * RS];
            }
            if (adj_out) {
                float* ao = adj_out + (size_t)(ok ? m0 + h : 0) * C * RS;
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    float* dst = ok ? ao + (size_t)c * RS : dump_rows;
                    *dst = acc[h][c];
                }
            }
            float s[K + 2];
            act_derivs<K>(B.act, row[0], s);
            float zb0 = s[1] * acc[h][0];
            float out[C];
#pragma unroll
            for (int d = 0; d < NF; ++d) {
                float z[K + 1], pb[K + 1], zb[K + 1];
#pragma unroll
                for (int k = 1; k <= K; ++k) { z[k] = row[(size_t)chan(K, d, k) * RS]; pb[k] = acc[h][chan(K, d, k)]; }
                zb0 += adjoint_dir<K>(s, z, pb, zb);
#pragma unroll
                for (int k = 1; k <= K; ++k) out[chan(K, d, k)] = zb[k];
            }
            out[0] = zb0;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                float* dst = ok ? row + (size_t)c * RS : dump_rows;      // masked-off units: one dump row
                *dst = out[c];
            }
        }
    }
}

// Bias gradients of layer l: the value-channel adjoints of its output units.
template <int NF, int K>
PINN_HD void bias_grad(const DevPlan& P, int l, const float* __restrict__ units, int RS, const GradSink& sink) {
    constexpr int C = 1 + NF * K;
    const DevLayer& L = P.layer[l];
    const float* out_rows = units + (size_t)L.unit_base * C * RS;
#pragma unroll 1
    for (int j0 = 0; j0 < L.n_out; j0 += 32) {
        float v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int j = j0 + i < L.n_out ? j0 + i : L.n_out - 1;
            v[i] = out_rows[(size_t)j * C * RS];
        }
        emit_entries<32>(v, [&](int e, float t) { sink.add_if(j0 + e < L.n_out, L.b_off + j0 + e, t); });
    }
}

// Weight gradients of the first layer: its input jet is (x_k; 1 along its own axis at first order).
template <int NF, int K>
PINN_HD void wgrad_input_layer(const DevPlan& P, const float* __restrict__ units, const float* __restrict__ coords, int RS,
                               const GradSink& sink) {
    constexpr int C = 1 + NF * K;
    const DevLayer& L = P.layer[0];
    const float* out_rows = units + (size_t)L.unit_base * C * RS;
#pragma unroll 1
    for (int j0 = 0; j0 < L.n_out; j0 += 4) {
        float v[4 * PINN_MAX_DIMS];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int j = j0 + jj < L.n_out ? j0 + jj : L.n_out - 1;
            const float* row = out_rows + (size_t)j * C * RS;
            const float zb0 = row[0];
            float zb1[NF];
#pragma unroll
            for (int d = 0; d < NF; ++d) zb1[d] = row[(size_t)chan(K, d, 1) * RS];
#pragma unroll
            for (int k = 0; k < PINN_MAX_DIMS; ++k) {
                float e = (k < L.n_in) ? zb0 * coords[(size_t)k * RS] : 0.0f;
#pragma unroll
                for (int d = 0; d < NF; ++d)
                    e = fmaf(zb1[d], P.dir_vec[d][k], e);
                v[jj * PINN_MAX_DIMS + k] = e;
            }
        }
        emit_entries<4 * PINN_MAX_DIMS>(v, [&](int e, float t) {
            const int j = j0 + e / PINN_MAX_DIMS, k = e % PINN_MAX_DIMS;
            sink.add_if(j < L.n_out && k < L.n_in, L.w_off + j * L.n_in + k, t);
        });
    }
}

// ---------------------------------------------------------------------------------------------------------------
// The whole step for ONE point (the counterpart of pinn::point_step).
// ---------------------------------------------------------------------------------------------------------------
struct PartialsHi { float loss, sbar, vbar[PINN_MAX_VARS]; };

template <int NF, int K>
PINN_HD float point_step(const DevPlan& P, const float* __restrict__ sw, const float* __restrict__ pvals,
                         float* __restrict__ st, int RS, bool valid, float inv_n, const GradSink& sink, PartialsHi& part) {
    constexpr int C = 1 + NF * K;
    const int Ln = P.n_layers;
    float* coords = st;
    float* units = st + (size_t)P.row_units * RS;
    float* scr = st + (size_t)P.row_scr * RS;

#pragma unroll 1
    for (int l = 0; l + 1 < Ln; ++l) {
        fwd_layer<NF, K>(P, l, sw, coords, units, RS);
        if (P.layer[l].skip_src >= 0) skip_sum_jets<NF, K>(P, l, units, RS);
    }
    float N[C];
    fwd_final<NF, K>(P, sw, coords, units, RS, N);

    float icj[C];
#pragma unroll
    for (int c = 0; c < C; ++c) icj[c] = 0.0f;
    if (P.has_ic) {
        eval_prog(P.ic, P.n_ic, scr, RS, coords, pvals, P.var_off);
#pragma unroll
        for (int c = 0; c < C; ++c) icj[c] = scr[(size_t)P.ic_out[c] * RS];
    }
    const float log_scale = pvals[P.log_scale_off];
    AnsatzHi<NF, K> as;
    float u[C];
    ansatz_forward<NF, K>(P, coords, RS, log_scale, N, icj, as, u);
#pragma unroll
    for (int c = 0; c < C; ++c) scr[(size_t)c * RS] = u[c];
    eval_prog(P.eq, P.n_eq, scr, RS, coords, pvals, P.var_off);
    const float r = scr[(size_t)P.eq_out[0] * RS];
    const float rb = valid ? 2.0f * r * inv_n : 0.0f;
    if (valid) part.loss = fmaf(r * inv_n, r, part.loss);
    float ub[C];
#pragma unroll
    for (int c = 0; c < C; ++c) ub[c] = rb * scr[(size_t)P.eq_out[1 + c] * RS];
#pragma unroll
    for (int i = 0; i < PINN_MAX_VARS; ++i)
        if (i < P.n_vars) part.vbar[i] = fmaf(rb, scr[(size_t)P.eq_out[1 + C + i] * RS], part.vbar[i]);

    if (P.ic_has_vars) {                       // u_c = S v_c + ic_c: variables of the initial condition (README.md:112-118)
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
    part.sbar += ansatz_adjoint<NF, K>(P, as, ub, Nb);

    // reverse sweep: the top layer's row receives the adjoints of the network jet
    {
        const DevLayer& L = P.layer[Ln - 1];
        float* out_rows = units + (size_t)L.unit_base * C * RS;
#pragma unroll
        for (int c = 0; c < C; ++c) out_rows[(size_t)c * RS] = Nb[c];
    }
#pragma unroll 1
    for (int l = Ln - 1; l >= 1; --l) {
        bias_grad<NF, K>(P, l, units, RS, sink);
        bwd_layer<NF, K>(P, l, sw, units, RS, sink, scr);
    }
    bias_grad<NF, K>(P, 0, units, RS, sink);
    wgrad_input_layer<NF, K>(P, units, coords, RS, sink);
    return r;
}

}  // namespace hi
}  // namespace pinn
