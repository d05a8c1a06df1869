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
#pragma once
#include "kprog.cuh"

#define KGRAD_MAX_SLOTS 16

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
// forces the interpreter on programs that have a normal form (the CPU check compares the two).
template <typename F>
__host__ __device__ __forceinline__ double kgrad_eval(const KProg& P, const KGrad& G, int ndim, F diff, double* dk,
                                                      bool use_fast = true) {
    for (int s = 0; s < G.nslot; ++s) dk[s] = 0.0;
    double l1_id = 0.0, l2_id = 0.0;
    for (int d = 0; d < ndim; ++d) {
        const double df = diff(d);
        l1_id += fabs(df);
        l2_id += df * df;
    }
    if (G.fast && use_fast) {
        const KFast& K = G.F;
        double v[KFAST_MAX], d0[KFAST_MAX], d1[KFAST_MAX];
        for (int i = 0; i < K.nleaf; ++i) {
            double dl1, dl2sq;
            v[i] = kgrad_leaf(K.op[i], K.l2[i] != 0, K.p0[i], K.p1[i], l1_id, l2_id, d0[i], d1[i], dl1, dl2sq);
        }
        double k = 0.0;
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
            }
        }
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
    // row-scale sensitivities: scaling row r of M_m by lambda moves l2sq by 2 z_r^2 and l1 by |z_r| for every leaf on m
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
        }
    }
    return val[P.n - 1];
}
