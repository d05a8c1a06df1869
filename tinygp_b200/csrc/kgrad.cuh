// Derivatives of a kernel program with respect to its parameters, for one pair of points.  __host__ __device__ like
// kprog.cuh, so that tests/csrc/kgrad_hostcheck.cu runs the same source on the CPU.  Used by the contraction epilogue of
// b200gp_dense_log_probability_grad (grad.cu).
//
// A "slot" is one differentiable scalar of the program:
//   - p0 of every stationary leaf (its scale) and of every CONST (its value);
//   - p1 of ExpSineSquared (gamma) and RationalQuadratic (alpha);
//   - one row-scale sensitivity per row r of each metric m: d k / d lambda at lambda = 1 when row r of M_m is scaled by
//     lambda (what a 0- / 1-D transforms.Linear or transforms.Cholesky needs).
// Slots are numbered in program order: for each instruction, its p0 then its p1; then the metric rows, metric by metric.
//
// kgrad_eval<true> also returns the gradient of k with respect to the coordinate difference delta = x1 - x2 (what
// b200gp_dense_log_probability_grad_x needs; for a stationary kernel it is grad_1 k(x1, x2) = -grad_2 k(x1, x2)).  A
// leaf reads its distance on z = M delta (M = I without a transform), so with f' = d leaf / d distance:
//   L1:  r = |z|_1,   grad = f'(r) M^T sign(z)
//   L2:  r = |z|_2,   grad = f'(r) M^T z / r
//   leaves on the squared distance s (ExpSquared, RationalQuadratic):  grad = 2 f'(s) M^T z  (L1: s = r^2, as above)
// sums and products chain through the leaf adjoints (the normal form's term products, the interpreter's reverse pass).
// At coincident points (z = 0) the gradient is defined as 0: L1 takes sign(0) = 0, and the L2 leaves that are not
// smooth there (Exp, whose f'(0) = -1 / scale gives a direction-dependent limit) contribute 0 instead of NaN.
#pragma once
#include "kprog.cuh"

#define KGRAD_MAX_SLOTS 16
#define KGRAD_MAX_DIM B200GP_METRIC_MAX_DIM     // coordinate gradients: at most this many input dimensions

struct KGrad {
    int nslot;
    int slot0[B200GP_PROG_MAX_INSTR], slot1[B200GP_PROG_MAX_INSTR];   // slot of p0 / p1 of each instruction, -1 if none
    int left[B200GP_PROG_MAX_INSTR], right[B200GP_PROG_MAX_INSTR];    // operands (instruction indices) of ADD / MUL
    int mslot[B200GP_PROG_MAX_METRICS];                               // slot of row 0 of each metric
    // sum-of-products normal form (kprog.cuh KFast) with the derivative of every term coefficient by every CONST slot
    int fast;
    KFast F;
    int fslot0[KFAST_MAX], fslot1[KFAST_MAX];     // slots of the normal form's leaves
    int nconst;
    int cslot[B200GP_PROG_MAX_INSTR];
    double dcoef[KGRAD_MAX_SLOTS][KFAST_MAX];     // d coef[t] / d (CONST value c)
};

// one stationary leaf and its partial derivatives: by p0, p1, and by the two distances it reads (l1, l2sq).  At zero
// distance every derivative is finite; the scale derivative is 0 there.
__host__ __device__ __forceinline__ double kgrad_leaf(const int op, const bool l2, const double p0, const double p1,
                                                     const double l1, const double l2sq, double& d0, double& d1,
                                                     double& dl1, double& dl2sq) {
    d1 = 0.0; dl1 = 0.0; dl2sq = 0.0;
    if (op == B200GP_OP_EXPSQUARED || op == B200GP_OP_RATIONALQUADRATIC) {
        const double sq = l2 ? l2sq : l1 * l1;
        const double r2 = sq / (p0 * p0);
        double v, dsq;   // dsq = dv / d sq
        if (op == B200GP_OP_EXPSQUARED) {
            v = exp(-0.5 * r2);
            d0 = v * r2 / p0;
            dsq = -0.5 * v / (p0 * p0);
        } else {
            const double b = 1.0 + 0.5 * r2 / p1;
            v = pow(b, -p1);
            d0 = v * r2 / (p0 * b);
            d1 = v * (0.5 * r2 / (p1 * b) - log(b));
            dsq = -0.5 * v / (b * p0 * p0);
        }
        if (l2) dl2sq = dsq;
        else dl1 = 2.0 * l1 * dsq;
        return v;
    }
    const double dist = l2 ? ((l2sq == 0.0) ? l1 : sqrt(l2sq)) : l1;
    const double r = dist / p0;
    double v, dr;   // dr = dv / dr
    if (op == B200GP_OP_EXP) {
        v = exp(-r);
        dr = -v;
    } else if (op == B200GP_OP_MATERN32) {
        const double e = exp(-SQRT3 * r);
        v = (1.0 + SQRT3 * r) * e;
        dr = -3.0 * r * e;
    } else if (op == B200GP_OP_MATERN52) {
        const double a = SQRT5 * r, e = exp(-a);
        v = (1.0 + a + a * a / 3.0) * e;
        dr = -SQRT5 * a * (1.0 + a) / 3.0 * e;
    } else if (op == B200GP_OP_COSINE) {
        v = cos(2.0 * PI_D * r);
        dr = -2.0 * PI_D * sin(2.0 * PI_D * r);
    } else {   // EXPSINESQUARED
        const double s = sin(PI_D * r);
        v = exp(-p1 * (s * s));
        dr = -p1 * PI_D * sin(2.0 * PI_D * r) * v;
        d1 = -(s * s) * v;
    }
    d0 = -dr * r / p0;
    const double ddist = dr / p0;
    if (!l2) dl1 = ddist;
    else if (l2sq > 0.0) dl2sq = 0.5 * ddist / dist;   // at l2sq = 0 every row sensitivity carries z_r = 0
    return v;
}

__host__ __device__ __forceinline__ double kgrad_sign(const double z) { return (z > 0.0) ? 1.0 : ((z < 0.0) ? -1.0 : 0.0); }

// host: slot layout and operand indices of a parsed program; false if it has more than KGRAD_MAX_SLOTS slots or an
// opcode without derivatives (the closed forms of quasiseparable kernels)
static inline bool kgrad_prepare(const KProg& P, KGrad& G) {
    G = KGrad{};
    int st[8], sp = 0, ns = 0;
    for (int i = 0; i < P.n; ++i) {
        const int op = P.op[i];
        G.slot0[i] = G.slot1[i] = G.left[i] = G.right[i] = -1;
        if (op == B200GP_OP_ADD || op == B200GP_OP_MUL) {
            G.right[i] = st[--sp];
            G.left[i] = st[sp - 1];
            st[sp - 1] = i;
            continue;
        }
        if (op == B200GP_OP_EXPCOS || op == B200GP_OP_EXPSIN) return false;
        G.slot0[i] = ns++;
        if (op == B200GP_OP_EXPSINESQUARED || op == B200GP_OP_RATIONALQUADRATIC) G.slot1[i] = ns++;
        st[sp++] = i;
    }
    for (int m = 0; m < P.nmetric; ++m) {
        G.mslot[m] = ns;
        ns += P.mrows[m];
    }
    if (ns > KGRAD_MAX_SLOTS) return false;
    G.nslot = ns;
    // normal form: the coefficients are polynomials in the CONST values (each CONST occurs once, so each coefficient is
    // affine in each of them); d coef / d c is the coefficient of the program with c = 1 minus the one with c = 0
    G.fast = kprog_to_fast(P, G.F) ? 1 : 0;
    if (G.fast) {
        int k = 0;
        for (int i = 0; i < P.n; ++i) {
            if (P.op[i] == B200GP_OP_CONST) {
                KProg Q = P;
                KFast F1{}, F0{};
                Q.p0[i] = 1.0;
                kprog_to_fast(Q, F1);
                Q.p0[i] = 0.0;
                kprog_to_fast(Q, F0);
                G.cslot[G.nconst] = G.slot0[i];
                for (int t = 0; t < KFAST_MAX; ++t) G.dcoef[G.nconst][t] = (t < G.F.nterm) ? F1.coef[t] - F0.coef[t] : 0.0;
                ++G.nconst;
            } else if (P.op[i] != B200GP_OP_ADD && P.op[i] != B200GP_OP_MUL) {
                G.fslot0[k] = G.slot0[i];
                G.fslot1[k] = G.slot1[i];
                ++k;
            }
        }
    }
    return true;
}

// k(x1, x2) and dk[s] = d k / d slot s for s < G.nslot (`diff(d)` = x1_d - x2_d as in kprog_eval).  use_fast = false
// forces the interpreter on programs that have a normal form (the CPU check compares the two).  DX: also
// gx[d] = d k / d delta_d for d < ndim (ndim <= KGRAD_MAX_DIM) and 0 for the other KGRAD_MAX_DIM entries; dk is
// computed by the same arithmetic either way.
template <bool DX = false, typename F>
__host__ __device__ __forceinline__ double kgrad_eval(const KProg& P, const KGrad& G, int ndim, F diff, double* dk,
                                                      bool use_fast = true, double* gx = nullptr) {
    for (int s = 0; s < G.nslot; ++s) dk[s] = 0.0;
    // gradient of the identity-metric leaves: a1 * sign(delta) + 2 a2 * delta, with a1 / a2 = d k / d l1 / d l2sq
    auto identity_dx = [&](const double a1, const double a2) {
#pragma unroll
        for (int d = 0; d < KGRAD_MAX_DIM; ++d) {
            gx[d] = 0.0;
            if (d < ndim) {
                const double df = diff(d);
                gx[d] = a1 * kgrad_sign(df) + 2.0 * a2 * df;
            }
        }
    };
    double l1_id = 0.0, l2_id = 0.0;
    for (int d = 0; d < ndim; ++d) {
        const double df = diff(d);
        l1_id += fabs(df);
        l2_id += df * df;
    }
    if (G.fast && use_fast) {
        const KFast& K = G.F;
        double v[KFAST_MAX], d0[KFAST_MAX], d1[KFAST_MAX], gl1[KFAST_MAX], gl2[KFAST_MAX];
        for (int i = 0; i < K.nleaf; ++i)
            v[i] = kgrad_leaf(K.op[i], K.l2[i] != 0, K.p0[i], K.p1[i], l1_id, l2_id, d0[i], d1[i], gl1[i], gl2[i]);
        double k = 0.0, a1 = 0.0, a2 = 0.0;
        for (int t = 0; t < K.nterm; ++t) {
            double prod = 1.0;
            for (int i = 0; i < K.nleaf; ++i)
                if ((K.mask[t] >> i) & 1) prod *= v[i];
            k += K.coef[t] * prod;
            for (int c = 0; c < G.nconst; ++c) dk[G.cslot[c]] += G.dcoef[c][t] * prod;
            for (int i = 0; i < K.nleaf; ++i) {
                if (!((K.mask[t] >> i) & 1)) continue;
                double a = K.coef[t];   // d term / d leaf i (no leaf occurs twice in a term)
                for (int j = 0; j < K.nleaf; ++j)
                    if (j != i && ((K.mask[t] >> j) & 1)) a *= v[j];
                dk[G.fslot0[i]] += a * d0[i];
                if (G.fslot1[i] >= 0) dk[G.fslot1[i]] += a * d1[i];
                if constexpr (DX) {
                    a1 += a * gl1[i];
                    a2 += a * gl2[i];
                }
            }
        }
        if constexpr (DX) identity_dx(a1, a2);
        return k;
    }
    // interpreter: values forward, adjoints backward over the postfix program
    double val[B200GP_PROG_MAX_INSTR], adj[B200GP_PROG_MAX_INSTR];
    double gl1[B200GP_PROG_MAX_INSTR], gl2[B200GP_PROG_MAX_INSTR];
    for (int i = 0; i < P.n; ++i) {
        const int op = P.op[i];
        adj[i] = 0.0;
        gl1[i] = gl2[i] = 0.0;
        if (op == B200GP_OP_ADD) { val[i] = val[G.left[i]] + val[G.right[i]]; continue; }
        if (op == B200GP_OP_MUL) { val[i] = val[G.left[i]] * val[G.right[i]]; continue; }
        if (op == B200GP_OP_CONST) { val[i] = P.p0[i]; continue; }
        double l1 = l1_id, l2sq = l2_id;
        const int m = P.metric[i];
        if (m > 0) {
            l1 = 0.0;
            l2sq = 0.0;
            const double* Mm = P.M[m - 1];
            for (int r = 0; r < P.mrows[m - 1]; ++r) {
                double z = 0.0;
                for (int c = 0; c < ndim; ++c) z += Mm[r * B200GP_METRIC_MAX_DIM + c] * diff(c);
                l1 += fabs(z);
                l2sq += z * z;
            }
        }
        double d0, d1;
        val[i] = kgrad_leaf(op, P.dist[i] == B200GP_DIST_L2, P.p0[i], P.p1[i], l1, l2sq, d0, d1, gl1[i], gl2[i]);
        // keep the parameter partials in dk until the adjoint is known
        dk[G.slot0[i]] = d0;
        if (G.slot1[i] >= 0) dk[G.slot1[i]] = d1;
    }
    adj[P.n - 1] = 1.0;
    for (int i = P.n - 1; i >= 0; --i) {
        const int op = P.op[i];
        const double a = adj[i];
        if (op == B200GP_OP_ADD) {
            adj[G.left[i]] += a;
            adj[G.right[i]] += a;
        } else if (op == B200GP_OP_MUL) {
            adj[G.left[i]] += a * val[G.right[i]];
            adj[G.right[i]] += a * val[G.left[i]];
        } else if (op == B200GP_OP_CONST) {
            dk[G.slot0[i]] = a;
        } else {
            dk[G.slot0[i]] *= a;
            if (G.slot1[i] >= 0) dk[G.slot1[i]] *= a;
        }
    }
    if constexpr (DX) {
        double a1 = 0.0, a2 = 0.0;     // gl1 = gl2 = 0 on ADD / MUL / CONST
        for (int i = 0; i < P.n; ++i)
            if (P.metric[i] == 0) {
                a1 += adj[i] * gl1[i];
                a2 += adj[i] * gl2[i];
            }
        identity_dx(a1, a2);
    }
    // row-scale sensitivities: scaling row r of M_m by lambda moves l2sq by 2 z_r^2 and l1 by |z_r| for every leaf on m
    // (and delta moves z_r by row r of M_m)
    for (int m = 0; m < P.nmetric; ++m) {
        double g1 = 0.0, g2 = 0.0;
        for (int i = 0; i < P.n; ++i)
            if (P.op[i] != B200GP_OP_ADD && P.op[i] != B200GP_OP_MUL && P.op[i] != B200GP_OP_CONST && P.metric[i] == m + 1) {
                g1 += adj[i] * gl1[i];
                g2 += adj[i] * gl2[i];
            }
        const double* Mm = P.M[m];
        for (int r = 0; r < P.mrows[m]; ++r) {
            double z = 0.0;
            for (int c = 0; c < ndim; ++c) z += Mm[r * B200GP_METRIC_MAX_DIM + c] * diff(c);
            dk[G.mslot[m] + r] = 2.0 * z * z * g2 + fabs(z) * g1;
            if constexpr (DX) {
                const double gz = g1 * kgrad_sign(z) + 2.0 * g2 * z;
#pragma unroll
                for (int c = 0; c < KGRAD_MAX_DIM; ++c)
                    if (c < ndim) gx[c] += Mm[r * B200GP_METRIC_MAX_DIM + c] * gz;
            }
        }
    }
    return val[P.n - 1];
}

// element (i, j) of dK / d slot for the Fisher information's derivative build (grad.cu dk_build_kernel), X n x ndim
// row-major: slot < G.nslot is a program slot, slot == G.nslot the scalar noise diagonal (dK / d diag = I); 0 outside the
// n x n matrix, so that the padded rows and columns stay 0 through the products by L^-1
__host__ __device__ __forceinline__ double kgrad_element(const KProg& P, const KGrad& G, int ndim, const double* X,
                                                         int64_t n, int64_t i, int64_t j, int slot) {
    if (i >= n || j >= n) return 0.0;
    if (slot == G.nslot) return (i == j) ? 1.0 : 0.0;
    const double* xa = X + i * ndim;
    const double* xb = X + j * ndim;
    double dk[KGRAD_MAX_SLOTS];
    kgrad_eval(P, G, ndim, [&](int d) { return xa[d] - xb[d]; }, dk);
    double v = 0.0;
#pragma unroll
    for (int s = 0; s < KGRAD_MAX_SLOTS; ++s)
        if (s == slot) v = dk[s];
    return v;
}

// ---- second derivatives (b200gp_dense_log_probability_hessian) ----------------------------------------------------
// d^2 k / d slot_a d slot_b, walked over the program in forward mode with hyper-dual numbers (value, d/da, d/db,
// d^2/dadb) per pair of slots: ADD adds them, MUL applies the product rule, a leaf starts them from its own derivatives
// by (p0, p1, t) below.  So pairs of slots in different terms of a sum come out 0 and pairs in different factors of a
// product come out as products of first derivatives.  The walk always follows the program, also where kgrad_eval takes
// the normal form (its coefficient table stops at first order in the CONST values); both give the same k.
#define KHESS_PAIRS 16      // slot pairs per call (and per pass of the contraction)

// one leaf's value and its derivatives by (p0, p1, t) to second order: d = {v_0, v_1, v_t}, hh = {v_00, v_01, v_11,
// v_0t, v_1t, v_tt}, with t the distance variable the metric's row scales move: l1 on L1; the squared distance for
// ExpSquared / RationalQuadratic on L2; the distance itself for the other leaves on L2 (0 at l2sq = 0).
__host__ __device__ __forceinline__ double khess_leaf(const int op, const bool l2, const double p0, const double p1,
                                                     const double l1, const double l2sq, double* d, double* hh) {
    if (op == B200GP_OP_EXPSQUARED || op == B200GP_OP_RATIONALQUADRATIC) {
        // v = exp(phi(u, p1)), u = sq / p0^2
        const double sq = l2 ? l2sq : l1 * l1;
        const double u = sq / (p0 * p0);
        double v, pu = -0.5, puu = 0.0, pa = 0.0, paa = 0.0, pua = 0.0;
        if (op == B200GP_OP_EXPSQUARED) {
            v = exp(-0.5 * u);
        } else {
            const double a = p1, b = 1.0 + 0.5 * u / a;
            v = pow(b, -a);
            pu = -0.5 / b;
            puu = 0.25 / (a * b * b);
            pa = 0.5 * u / (a * b) - log(b);
            paa = 0.25 * u * u / (a * a * a * b * b);
            pua = -0.25 * u / (a * a * b * b);
        }
        const double u0 = -2.0 * u / p0, us = 1.0 / (p0 * p0), u00 = 6.0 * u / (p0 * p0), u0s = -2.0 / (p0 * p0 * p0);
        const double f0 = pu * u0, fs = pu * us, f1 = pa;
        const double v0 = v * f0, vs = v * fs;
        const double v0s = v * (f0 * fs + puu * u0 * us + pu * u0s), v1s = v * (f1 * fs + pua * us);
        const double vss = v * (fs * fs + puu * us * us);
        d[0] = v0;
        d[1] = v * f1;
        hh[0] = v * (f0 * f0 + puu * u0 * u0 + pu * u00);
        hh[1] = v * (f0 * f1 + pua * u0);
        hh[2] = v * (f1 * f1 + paa);
        if (l2) {
            d[2] = vs; hh[3] = v0s; hh[4] = v1s; hh[5] = vss;
        } else {           // t = l1, sq = t^2
            d[2] = 2.0 * l1 * vs; hh[3] = 2.0 * l1 * v0s; hh[4] = 2.0 * l1 * v1s; hh[5] = 2.0 * vs + 4.0 * l1 * l1 * vss;
        }
        return v;
    }
    const double t = l2 ? ((l2sq == 0.0) ? l1 : sqrt(l2sq)) : l1;
    const double r = t / p0;
    double v, f1, f2, g = 0.0, gg = 0.0, rg = 0.0;   // dv/dr, d2v/dr2, dv/dp1, d2v/dp1^2, d2v/dr dp1
    if (op == B200GP_OP_EXP) {
        v = exp(-r); f1 = -v; f2 = v;
    } else if (op == B200GP_OP_MATERN32) {
        const double e = exp(-SQRT3 * r);
        v = (1.0 + SQRT3 * r) * e; f1 = -3.0 * r * e; f2 = 3.0 * (SQRT3 * r - 1.0) * e;
    } else if (op == B200GP_OP_MATERN52) {
        const double a = SQRT5 * r, e = exp(-a);
        v = (1.0 + a + a * a / 3.0) * e; f1 = -SQRT5 * a * (1.0 + a) / 3.0 * e; f2 = -5.0 / 3.0 * (1.0 + a - a * a) * e;
    } else if (op == B200GP_OP_COSINE) {
        v = cos(2.0 * PI_D * r); f1 = -2.0 * PI_D * sin(2.0 * PI_D * r); f2 = -4.0 * PI_D * PI_D * v;
    } else {   // EXPSINESQUARED
        const double s = sin(PI_D * r), s2 = sin(2.0 * PI_D * r);
        v = exp(-p1 * (s * s));
        f1 = -p1 * PI_D * s2 * v;
        f2 = p1 * PI_D * PI_D * v * (p1 * s2 * s2 - 2.0 * cos(2.0 * PI_D * r));
        g = -(s * s) * v; gg = (s * s) * (s * s) * v; rg = PI_D * s2 * v * (p1 * (s * s) - 1.0);
    }
    const double r0 = -r / p0, rt = 1.0 / p0;
    d[0] = f1 * r0; d[1] = g; d[2] = f1 * rt;
    hh[0] = f2 * r0 * r0 + f1 * 2.0 * r / (p0 * p0);
    hh[1] = rg * r0;
    hh[2] = gg;
    hh[3] = f2 * r0 * rt - f1 / (p0 * p0);
    hh[4] = rg * rt;
    hh[5] = f2 * rt * rt;
    return v;
}

// h[q] = d^2 k / d slot pa[q] d slot pb[q] for q < npair <= KHESS_PAIRS, slots < G.nslot (`diff` as in kgrad_eval).
// A row scale lambda_r of metric m moves a leaf on m through t: dt / dlambda_r = |z_r| on L1, 2 z_r^2 for the squared
// distance, z_r^2 / dist for the distance on L2 (0 at dist = 0, where every z_r is 0), and d^2 t / dlambda_r dlambda_s
// = 0, 2 z_r^2 delta_rs, z_r^2 / dist (delta_rs - z_s^2 / dist^2) in the same three cases.
template <typename F>
__host__ __device__ __forceinline__ void khess_eval(const KProg& P, const KGrad& G, int ndim, F diff, const int* pa,
                                                    const int* pb, int npair, double* h) {
    double l1_id = 0.0, l2_id = 0.0;
    for (int d = 0; d < ndim; ++d) {
        const double df = diff(d);
        l1_id += fabs(df);
        l2_id += df * df;
    }
    double z[B200GP_PROG_MAX_METRICS][B200GP_METRIC_MAX_DIM];
    for (int m = 0; m < P.nmetric; ++m)
        for (int r = 0; r < P.mrows[m]; ++r) {
            double s = 0.0;
            for (int c = 0; c < ndim; ++c) s += P.M[m][r * B200GP_METRIC_MAX_DIM + c] * diff(c);
            z[m][r] = s;
        }
    // every leaf (CONST included) owns a slot, so there are at most KGRAD_MAX_SLOTS of them
    double lv[KGRAD_MAX_SLOTS], ld[KGRAD_MAX_SLOTS][3], lh[KGRAD_MAX_SLOTS][6], lt[KGRAD_MAX_SLOTS];
    int k = 0;
    for (int i = 0; i < P.n; ++i) {
        const int op = P.op[i];
        if (op == B200GP_OP_ADD || op == B200GP_OP_MUL) continue;
        if (op == B200GP_OP_CONST) {
            lv[k++] = P.p0[i];
            continue;
        }
        double l1 = l1_id, l2sq = l2_id;
        const int m = P.metric[i];
        if (m > 0) {
            l1 = 0.0;
            l2sq = 0.0;
            for (int r = 0; r < P.mrows[m - 1]; ++r) {
                l1 += fabs(z[m - 1][r]);
                l2sq += z[m - 1][r] * z[m - 1][r];
            }
        }
        const bool l2 = P.dist[i] == B200GP_DIST_L2;
        lv[k] = khess_leaf(op, l2, P.p0[i], P.p1[i], l1, l2sq, ld[k], lh[k]);
        lt[k] = l2 ? ((l2sq == 0.0) ? l1 : sqrt(l2sq)) : l1;
        ++k;
    }
    for (int q = 0; q < npair; ++q) {
        const int a = pa[q], b = pb[q];
        double sv[8], sa[8], sb[8], sab[8];
        int sp = 0;
        k = 0;
        for (int i = 0; i < P.n; ++i) {
            const int op = P.op[i];
            if (op == B200GP_OP_ADD || op == B200GP_OP_MUL) {
                --sp;
                const double uv = sv[sp - 1], ua = sa[sp - 1], ub = sb[sp - 1], uab = sab[sp - 1];
                const double wv = sv[sp], wa = sa[sp], wb = sb[sp], wab = sab[sp];
                if (op == B200GP_OP_ADD) {
                    sv[sp - 1] = uv + wv; sa[sp - 1] = ua + wa; sb[sp - 1] = ub + wb; sab[sp - 1] = uab + wab;
                } else {
                    sv[sp - 1] = uv * wv;
                    sa[sp - 1] = ua * wv + uv * wa;
                    sb[sp - 1] = ub * wv + uv * wb;
                    sab[sp - 1] = uab * wv + ua * wb + ub * wa + uv * wab;
                }
                continue;
            }
            if (op == B200GP_OP_CONST) {
                sv[sp] = lv[k];
                sa[sp] = (a == G.slot0[i]) ? 1.0 : 0.0;
                sb[sp] = (b == G.slot0[i]) ? 1.0 : 0.0;
                sab[sp] = 0.0;
                ++sp; ++k;
                continue;
            }
            // the directions of slots a and b in (p0, p1, t), and d^2 t / da db
            double ca[3] = {0.0, 0.0, 0.0}, cb[3] = {0.0, 0.0, 0.0}, tab = 0.0;
            ca[0] = (a == G.slot0[i]) ? 1.0 : 0.0; ca[1] = (a == G.slot1[i]) ? 1.0 : 0.0;
            cb[0] = (b == G.slot0[i]) ? 1.0 : 0.0; cb[1] = (b == G.slot1[i]) ? 1.0 : 0.0;
            const int m = P.metric[i];
            if (m > 0) {
                const int ra = a - G.mslot[m - 1], rb = b - G.mslot[m - 1], nr = P.mrows[m - 1];
                const bool l2 = P.dist[i] == B200GP_DIST_L2;
                const bool sql = op == B200GP_OP_EXPSQUARED || op == B200GP_OP_RATIONALQUADRATIC;
                const double dist = lt[k];
                auto dt = [&](int r) {
                    const double zr = z[m - 1][r];
                    if (!l2) return fabs(zr);
                    if (sql) return 2.0 * zr * zr;
                    return (dist > 0.0) ? zr * zr / dist : 0.0;
                };
                if (ra >= 0 && ra < nr) ca[2] = dt(ra);
                if (rb >= 0 && rb < nr) cb[2] = dt(rb);
                if (l2 && ra >= 0 && ra < nr && rb >= 0 && rb < nr) {
                    if (sql) {
                        tab = (ra == rb) ? ca[2] : 0.0;
                    } else if (dist > 0.0) {
                        const double zb = z[m - 1][rb] / dist;
                        tab = ((ra == rb) ? ca[2] : 0.0) - ca[2] * zb * zb;
                    }
                }
            }
            const double* d = ld[k];
            const double* hh = lh[k];
            sv[sp] = lv[k];
            sa[sp] = d[0] * ca[0] + d[1] * ca[1] + d[2] * ca[2];
            sb[sp] = d[0] * cb[0] + d[1] * cb[1] + d[2] * cb[2];
            sab[sp] = ca[0] * (hh[0] * cb[0] + hh[1] * cb[1] + hh[3] * cb[2])
                    + ca[1] * (hh[1] * cb[0] + hh[2] * cb[1] + hh[4] * cb[2])
                    + ca[2] * (hh[3] * cb[0] + hh[4] * cb[1] + hh[5] * cb[2]) + d[2] * tab;
            ++sp; ++k;
        }
        h[q] = sab[0];
    }
}
