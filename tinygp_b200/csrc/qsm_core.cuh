// Quasiseparable-matrix algebra on generator ARRAYS: the per-chunk bodies of the
// scans behind src/tinygp/solvers/quasisep/core.py and ops.py for matrices whose generators are arbitrary per-point
// arrays (d (n), p, q (n x m), a (n x m x m)) of any order m -- the conditioned covariance of solver.py:124-129 has
// order 4J, its `a` is a dense 16 x 16 block per point at J = 4.
//
// Execution model: ONE WARP per chunk of consecutive points; the m x m (or m x k) scan state and the point's
// generators live in shared memory and the 32 lanes share the entries of every small matrix product.  Every scan is
// chunk composite -> sequential pass over the (few thousand) chunk composites -> replay with the reference's own
// sequential recursion.  The bodies are written against `Lane{lane, nl}` so that tests/csrc (QSM_HOSTCHECK) runs the
// SAME source on the CPU with one lane.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__) && !defined(QSM_HOSTCHECK)
#define QHD __host__ __device__ __forceinline__
#else
#define QHD inline
#endif
#if defined(__CUDA_ARCH__) && !defined(QSM_HOSTCHECK)
#define QSYNC() __syncwarp()
#else
#define QSYNC()
#endif

namespace qsm {

struct Lane { int lane, nl; };

// C (r x c, row stride ldc) = (acc ? C : 0) + alpha * A B with A(i, l) = A[i * ai + l * al], B(l, j) = B[l * bl + j * bj]
// (strides express transposes).  C must not alias A or B.
QHD void mm(Lane L, double* C, int ldc, const double* A, int ai, int al, const double* B, int bl, int bj, int r, int k, int c,
            double alpha, bool acc) {
    for (int e = L.lane; e < r * c; e += L.nl) {
        const int i = e / c, j = e - i * c;
        double s = 0.0;
        for (int l = 0; l < k; ++l) s += A[i * ai + l * al] * B[l * bl + j * bj];
        C[i * ldc + j] = (acc ? C[i * ldc + j] : 0.0) + alpha * s;
    }
    QSYNC();
}
QHD void vcopy(Lane L, double* dst, const double* src, int n) {
    for (int e = L.lane; e < n; e += L.nl) dst[e] = src[e];
}
QHD void vzero(Lane L, double* dst, int n) {
    for (int e = L.lane; e < n; e += L.nl) dst[e] = 0.0;
}
QHD void eye(Lane L, double* dst, int m) {
    for (int e = L.lane; e < m * m; e += L.nl) dst[e] = (e / m == e % m) ? 1.0 : 0.0;
}
// y (r) = A x with A(i, l) = A[i * ai + l * al]
QHD void mv(Lane L, double* y, const double* A, int ai, int al, const double* x, int r, int k) {
    for (int i = L.lane; i < r; i += L.nl) {
        double s = 0.0;
        for (int l = 0; l < k; ++l) s += A[i * ai + l * al] * x[l];
        y[i] = s;
    }
    QSYNC();
}
QHD double dot_all(const double* x, const double* y, int n) {   // every lane computes the same value (n <= 64)
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += x[i] * y[i];
    return s;
}
// Solve M X = B in place (M: m x m destroyed, B: m x c overwritten by X), Gaussian elimination with partial pivoting;
// the pivot search is redundant in every lane (identical results), the row operations are shared.
QHD void solve(Lane L, double* M, double* B, int m, int c) {
    for (int col = 0; col < m; ++col) {
        int piv = col;
        double best = fabs(M[col * m + col]);
        for (int r = col + 1; r < m; ++r) {
            const double v = fabs(M[r * m + col]);
            if (v > best) { best = v; piv = r; }
        }
        QSYNC();
        if (piv != col) {
            for (int e = L.lane; e < m + c; e += L.nl) {
                double* x = (e < m) ? &M[col * m + e] : &B[col * c + (e - m)];
                double* y = (e < m) ? &M[piv * m + e] : &B[piv * c + (e - m)];
                const double t = *x; *x = *y; *y = t;
            }
            QSYNC();
        }
        const double inv = 1.0 / M[col * m + col];
        // eliminate column `col` from every OTHER row (Gauss-Jordan); a lane owns whole rows
        for (int r = L.lane; r < m; r += L.nl) {
            if (r == col) continue;
            const double f = M[r * m + col] * inv;
            for (int k2 = col + 1; k2 < m; ++k2) M[r * m + k2] -= f * M[col * m + k2];
            for (int k2 = 0; k2 < c; ++k2) B[r * c + k2] -= f * B[col * c + k2];
            M[r * m + col] = 0.0;
        }
        QSYNC();
    }
    for (int e = L.lane; e < m * c; e += L.nl) B[e] /= M[(e / c) * m + (e / c)];
    QSYNC();
}

struct Tri { const double* p; const double* q; const double* a; int m; };   // strictly triangular part, n x m / n x m x m

// =====================================================================================================================
// 1. products and solves with dense right-hand sides (ops.py:308-349, 463-512)
//    LMAT:  out_k = p_k . f,              f <- a_k   f + q_k (x) x_k      forward   (ops.py:308-316)
//    UMAT:  out_k = q_k . f,              f <- a_k^T f + p_k (x) x_k      reverse   (ops.py:330-338)
//    LSOL:  y_k = (x_k - p_k . f) / d_k,  f <- a_k   f + q_k (x) y_k      forward   (ops.py:463-472)
//    USOL:  y_k = (x_k - q_k . f) / d_k,  f <- a_k^T f + p_k (x) y_k      reverse   (ops.py:489-498)
//    The chunk composite (f_out = Acal f_in + Ccal) is obtained by running the SAME step on the widened state
//    [I | 0] (m x (m + kc)) with the right-hand side [0 | x_k].
// =====================================================================================================================
enum { LMAT = 0, UMAT = 1, LSOL = 2, USOL = 3 };

struct LowArgs {
    int op; int64_t n; int m, kc; int64_t chunk, nchunks;
    const double* d; Tri t;
    const double* x; int64_t ldx;
    double* out; int64_t ldo; int accumulate;
    double* comp;   // nchunks x m x (m + kc)
    double* fin;    // nchunks x m x kc
};
QHD int low_smem_doubles(int m, int kc) { return 2 * m * (m + kc) + m * m + 2 * m + (m + kc); }

template <bool PHASE1>
QHD void low_step(Lane L, const LowArgs& a, int64_t k, double*& G, double*& T, double* am, double* pv, double* qv, double* xr, int W) {
    const int m = a.m;
    const bool up = (a.op == UMAT || a.op == USOL), sol = (a.op == LSOL || a.op == USOL);
    vcopy(L, am, a.t.a + k * m * m, m * m);
    vcopy(L, pv, (up ? a.t.q : a.t.p) + k * m, m);      // the vector read against the state
    vcopy(L, qv, (up ? a.t.p : a.t.q) + k * m, m);      // the vector that enters the state
    for (int j = L.lane; j < W; j += L.nl) xr[j] = PHASE1 ? (j < m ? 0.0 : a.x[k * a.ldx + (j - m)]) : a.x[k * a.ldx + j];
    QSYNC();
    const double dk = sol ? a.d[k] : 1.0;
    for (int j = L.lane; j < W; j += L.nl) {
        double s = 0.0;
        for (int i = 0; i < m; ++i) s += pv[i] * G[i * W + j];
        const double val = sol ? (xr[j] - s) / dk : s;
        if (!PHASE1) a.out[k * a.ldo + j] = (a.accumulate ? a.out[k * a.ldo + j] : 0.0) + val;
        if (sol) xr[j] = val;
    }
    QSYNC();
    for (int e = L.lane; e < m * W; e += L.nl) {
        const int i = e / W, j = e - i * W;
        double s = qv[i] * xr[j];
        for (int l = 0; l < m; ++l) s += (up ? am[l * m + i] : am[i * m + l]) * G[l * W + j];
        T[e] = s;
    }
    QSYNC();
    double* tmp = G; G = T; T = tmp;
}
QHD void low_range(const LowArgs& a, int64_t c, int64_t& k0, int64_t& k1) {
    k0 = c * a.chunk; k1 = k0 + a.chunk; if (k1 > a.n) k1 = a.n;
}
QHD void low_phase1(Lane L, const LowArgs& a, int64_t c, double* ws) {
    const int m = a.m, W = a.m + a.kc;
    double* G = ws; double* T = G + m * W; double* am = T + m * W; double* pv = am + m * m; double* qv = pv + m; double* xr = qv + m;
    for (int e = L.lane; e < m * W; e += L.nl) G[e] = (e / W == e % W) ? 1.0 : 0.0;
    QSYNC();
    int64_t k0, k1; low_range(a, c, k0, k1);
    const bool rev = (a.op == UMAT || a.op == USOL);
    if (!rev) for (int64_t k = k0; k < k1; ++k) low_step<true>(L, a, k, G, T, am, pv, qv, xr, W);
    else for (int64_t k = k1 - 1; k >= k0; --k) low_step<true>(L, a, k, G, T, am, pv, qv, xr, W);
    vcopy(L, a.comp + c * (int64_t)m * W, G, m * W);
    QSYNC();
}
// one warp: the state entering every chunk
QHD void low_phase2(Lane L, const LowArgs& a, double* ws) {
    const int m = a.m, kc = a.kc, W = m + kc;
    double* F = ws; double* T = F + m * kc;
    vzero(L, F, m * kc);
    QSYNC();
    const bool rev = (a.op == UMAT || a.op == USOL);
    for (int64_t i = 0; i < a.nchunks; ++i) {
        const int64_t c = rev ? a.nchunks - 1 - i : i;
        vcopy(L, a.fin + c * (int64_t)m * kc, F, m * kc);
        const double* G = a.comp + c * (int64_t)m * W;
        for (int e = L.lane; e < m * kc; e += L.nl) {
            const int r = e / kc, j = e - r * kc;
            double s = G[r * W + m + j];
            for (int l = 0; l < m; ++l) s += G[r * W + l] * F[l * kc + j];
            T[e] = s;
        }
        QSYNC();
        double* tmp = F; F = T; T = tmp;
    }
}
QHD void low_phase3(Lane L, const LowArgs& a, int64_t c, double* ws) {
    const int m = a.m, W = a.kc;
    double* G = ws; double* T = G + m * (a.m + a.kc); double* am = T + m * (a.m + a.kc); double* pv = am + m * m; double* qv = pv + m;
    double* xr = qv + m;
    if (a.nchunks > 1) vcopy(L, G, a.fin + c * (int64_t)m * W, m * W);
    else vzero(L, G, m * W);
    QSYNC();
    int64_t k0, k1; low_range(a, c, k0, k1);
    const bool rev = (a.op == UMAT || a.op == USOL);
    if (!rev) for (int64_t k = k0; k < k1; ++k) low_step<false>(L, a, k, G, T, am, pv, qv, xr, W);
    else for (int64_t k = k1 - 1; k >= k0; --k) low_step<false>(L, a, k, G, T, am, pv, qv, xr, W);
}

// =====================================================================================================================
// 2. bilinear scan  F <- L_k F R_k^T + (us_k u_k) (x) v_k  with emissions read from the state BEFORE point k:
//        e1_k = L_k F r1_k  (m1),   e2_k = (l1_k^T F) R_k^T  (m2),   e3_k = l1_k^T F r1_k
//    phi of qsm_mul (ops.py:62-72, 120-123): L = lower_a.a, R = upper_b.a, u = lower_a.q, v = upper_b.q, l1 = lower_a.p,
//    r1 = upper_b.p, forward;  psi (ops.py:77-87, 125-128): L = upper_a.a^T, R = lower_b.a^T, u = upper_a.p, v = lower_b.p,
//    l1 = upper_a.q, r1 = lower_b.q, reverse;  backward pass of symm_inv in its associative form (ops.py:446-449).
// =====================================================================================================================
struct BilArgs {
    int64_t n; int m1, m2; int rev; int64_t chunk, nchunks;
    const double* La; int tL; const double* Ra; int tR;
    const double* u; const double* us; const double* v;
    const double* l1; const double* r1;
    double* e1; int64_t lde1; int acc1;
    double* e2; int64_t lde2; int acc2;
    double* e3; int acc3;
    double* comp;   // nchunks x (m1^2 + m2^2 + m1 m2)
    double* fin;    // nchunks x m1 m2
};
QHD int bil_smem_doubles(int m1, int m2) { return 3 * m1 * m1 + 3 * m2 * m2 + 3 * m1 * m2 + 4 * (m1 + m2); }

struct BilWs { double *Lm, *Rm, *F, *T, *T2, *Ac, *At, *Bc, *Bt, *uv, *vv, *l1, *r1, *g, *h; };
QHD BilWs bil_ws(double* ws, int m1, int m2) {
    BilWs w;
    w.Lm = ws; w.Ac = w.Lm + m1 * m1; w.At = w.Ac + m1 * m1;
    w.Rm = w.At + m1 * m1; w.Bc = w.Rm + m2 * m2; w.Bt = w.Bc + m2 * m2;
    w.F = w.Bt + m2 * m2; w.T = w.F + m1 * m2; w.T2 = w.T + m1 * m2;
    w.uv = w.T2 + m1 * m2; w.l1 = w.uv + m1; w.g = w.l1 + m1; w.vv = w.g + m1; w.r1 = w.vv + m2; w.h = w.r1 + m2;
    return w;   // 3 m1^2 + 3 m2^2 + 3 m1 m2 + 3 m1 + 3 m2
}
QHD void bil_load(Lane L, const BilArgs& a, int64_t k, BilWs& w) {
    const int m1 = a.m1, m2 = a.m2;
    vcopy(L, w.Lm, a.La + k * m1 * m1, m1 * m1);
    vcopy(L, w.Rm, a.Ra + k * m2 * m2, m2 * m2);
    const double s = a.us ? a.us[k] : 1.0;
    for (int e = L.lane; e < m1; e += L.nl) w.uv[e] = s * a.u[k * m1 + e];
    vcopy(L, w.vv, a.v + k * m2, m2);
    QSYNC();
}
// F <- L F R^T + u v^T   (F, T swap)
QHD void bil_update(Lane L, const BilArgs& a, BilWs& w) {
    const int m1 = a.m1, m2 = a.m2;
    mm(L, w.T, m2, w.Lm, a.tL ? 1 : m1, a.tL ? m1 : 1, w.F, m2, 1, m1, m1, m2, 1.0, false);          // T = L F
    for (int e = L.lane; e < m1 * m2; e += L.nl) {
        const int i = e / m2, j = e - i * m2;
        double s = w.uv[i] * w.vv[j];
        for (int l = 0; l < m2; ++l) s += w.T[i * m2 + l] * (a.tR ? w.Rm[l * m2 + j] : w.Rm[j * m2 + l]);   // (T R^T)_ij = sum_l T_il R_jl
        w.T2[e] = s;
    }
    QSYNC();
    double* tmp = w.F; w.F = w.T2; w.T2 = tmp;
}
QHD void bil_phase1(Lane L, const BilArgs& a, int64_t c, double* ws) {
    const int m1 = a.m1, m2 = a.m2;
    BilWs w = bil_ws(ws, m1, m2);
    eye(L, w.Ac, m1); eye(L, w.Bc, m2); vzero(L, w.F, m1 * m2);
    QSYNC();
    int64_t k0 = c * a.chunk, k1 = k0 + a.chunk; if (k1 > a.n) k1 = a.n;
    for (int64_t i = 0; i < k1 - k0; ++i) {
        const int64_t k = a.rev ? k1 - 1 - i : k0 + i;
        bil_load(L, a, k, w);
        bil_update(L, a, w);
        mm(L, w.At, m1, w.Lm, a.tL ? 1 : m1, a.tL ? m1 : 1, w.Ac, m1, 1, m1, m1, m1, 1.0, false);       // Acal <- L Acal
        mm(L, w.Bt, m2, w.Rm, a.tR ? 1 : m2, a.tR ? m2 : 1, w.Bc, m2, 1, m2, m2, m2, 1.0, false);       // Bcal <- R Bcal
        double* t = w.Ac; w.Ac = w.At; w.At = t;
        t = w.Bc; w.Bc = w.Bt; w.Bt = t;
    }
    double* o = a.comp + c * (int64_t)(m1 * m1 + m2 * m2 + m1 * m2);
    vcopy(L, o, w.Ac, m1 * m1); vcopy(L, o + m1 * m1, w.Bc, m2 * m2); vcopy(L, o + m1 * m1 + m2 * m2, w.F, m1 * m2);
    QSYNC();
}
QHD void bil_phase2(Lane L, const BilArgs& a, double* ws) {
    const int m1 = a.m1, m2 = a.m2;
    BilWs w = bil_ws(ws, m1, m2);
    vzero(L, w.F, m1 * m2);
    QSYNC();
    for (int64_t i = 0; i < a.nchunks; ++i) {
        const int64_t c = a.rev ? a.nchunks - 1 - i : i;
        vcopy(L, a.fin + c * (int64_t)m1 * m2, w.F, m1 * m2);
        const double* o = a.comp + c * (int64_t)(m1 * m1 + m2 * m2 + m1 * m2);
        vcopy(L, w.Ac, o, m1 * m1); vcopy(L, w.Bc, o + m1 * m1, m2 * m2);
        QSYNC();
        mm(L, w.T, m2, w.Ac, m1, 1, w.F, m2, 1, m1, m1, m2, 1.0, false);                                 // Acal F
        for (int e = L.lane; e < m1 * m2; e += L.nl) {
            const int r = e / m2, j = e - r * m2;
            double s = o[m1 * m1 + m2 * m2 + e];
            for (int l = 0; l < m2; ++l) s += w.T[r * m2 + l] * w.Bc[j * m2 + l];                          // ... Bcal^T + Ccal
            w.T2[e] = s;
        }
        QSYNC();
        double* tmp = w.F; w.F = w.T2; w.T2 = tmp;
    }
}
QHD void bil_phase3(Lane L, const BilArgs& a, int64_t c, double* ws) {
    const int m1 = a.m1, m2 = a.m2;
    BilWs w = bil_ws(ws, m1, m2);
    if (a.nchunks > 1) vcopy(L, w.F, a.fin + c * (int64_t)m1 * m2, m1 * m2);
    else vzero(L, w.F, m1 * m2);
    QSYNC();
    int64_t k0 = c * a.chunk, k1 = k0 + a.chunk; if (k1 > a.n) k1 = a.n;
    for (int64_t i = 0; i < k1 - k0; ++i) {
        const int64_t k = a.rev ? k1 - 1 - i : k0 + i;
        bil_load(L, a, k, w);
        if (a.l1) vcopy(L, w.l1, a.l1 + k * m1, m1);
        if (a.r1) vcopy(L, w.r1, a.r1 + k * m2, m2);
        QSYNC();
        if (a.r1) mv(L, w.g, w.F, m2, 1, w.r1, m1, m2);               // g = F r1
        if (a.l1) mv(L, w.h, w.F, 1, m2, w.l1, m2, m1);               // h = F^T l1
        if (a.e1) for (int i2 = L.lane; i2 < m1; i2 += L.nl) {        // e1 = L g
            double s = 0.0;
            for (int l = 0; l < m1; ++l) s += (a.tL ? w.Lm[l * m1 + i2] : w.Lm[i2 * m1 + l]) * w.g[l];
            a.e1[k * a.lde1 + i2] = (a.acc1 ? a.e1[k * a.lde1 + i2] : 0.0) + s;
        }
        if (a.e2) for (int j = L.lane; j < m2; j += L.nl) {           // e2 = R h
            double s = 0.0;
            for (int l = 0; l < m2; ++l) s += (a.tR ? w.Rm[l * m2 + j] : w.Rm[j * m2 + l]) * w.h[l];
            a.e2[k * a.lde2 + j] = (a.acc2 ? a.e2[k * a.lde2 + j] : 0.0) + s;
        }
        if (a.e3 && L.lane == 0) a.e3[k] = (a.acc3 ? a.e3[k] : 0.0) + dot_all(w.l1, w.g, m1);
        QSYNC();
        bil_update(L, a, w);
    }
}

// =====================================================================================================================
// 3. Riccati scan: the carry f of the Cholesky factorisation (ops.py:352-365) and of symm_inv's forward pass
//    (ops.py:403-416).  Chunk composite (A, F, G) of ops.py:368-385, folded point by point WITHOUT a linear solve:
//        u = F p, s = d - p.u, v = A^T p, w = q - a u;   F <- a F a^T + w w^T / s,  A <- a A - w v^T / s,  G <- G - v v^T / s
//    entering state of the next chunk: f <- F + A (I + f G)^-1 f A^T;  replay: the reference's sequential recursion.
//    mode 0: emits c, w (Cholesky);  mode 1: emits ig, s, ell (symm_inv forward).
// =====================================================================================================================
struct RicArgs {
    int64_t n; int m; int64_t chunk, nchunks; int mode;
    const double *d, *p, *q, *a;
    double* o_c; double* o_w; double* o_ell;
    double* comp;   // nchunks x 3 m^2
    double* fin;    // nchunks x m^2
    double* fend;   // nchunks x m^2 or null: the state LEAVING each chunk as the replay found it (consistency check)
    long long* info;      // first k (1-based) with a non-positive / non-finite pivot (atomic min); LLONG_MAX = none
};
QHD int ric_smem_doubles(int m) { return 7 * m * m + 6 * m; }

QHD void ric_phase1(Lane L, const RicArgs& a, int64_t c, double* ws) {
    const int m = a.m, mm2 = m * m;
    double* A = ws; double* F = A + mm2; double* G = F + mm2; double* am = G + mm2; double* T = am + mm2; double* T2 = T + mm2;
    double* pv = T2 + mm2 + mm2; double* qv = pv + m; double* u = qv + m; double* v = u + m; double* w = v + m;
    eye(L, A, m); vzero(L, F, mm2); vzero(L, G, mm2);
    QSYNC();
    int64_t k0 = c * a.chunk, k1 = k0 + a.chunk; if (k1 > a.n) k1 = a.n;
    for (int64_t k = k0; k < k1; ++k) {
        vcopy(L, am, a.a + k * mm2, mm2); vcopy(L, pv, a.p + k * m, m); vcopy(L, qv, a.q + k * m, m);
        QSYNC();
        mv(L, u, F, m, 1, pv, m, m);                       // u = F p
        mv(L, v, A, 1, m, pv, m, m);                       // v = A^T p
        const double s = a.d[k] - dot_all(pv, u, m), is = 1.0 / s;
        for (int i = L.lane; i < m; i += L.nl) {           // w = q - a u
            double t = qv[i];
            for (int l = 0; l < m; ++l) t -= am[i * m + l] * u[l];
            w[i] = t;
        }
        QSYNC();
        mm(L, T, m, am, m, 1, F, m, 1, m, m, m, 1.0, false);           // T = a F
        for (int e = L.lane; e < mm2; e += L.nl) {
            const int i = e / m, j = e - i * m;
            double f2 = w[i] * w[j] * is, a2 = -w[i] * v[j] * is;
            for (int l = 0; l < m; ++l) { f2 += T[i * m + l] * am[j * m + l]; a2 += am[i * m + l] * A[l * m + j]; }
            T2[e] = f2; T2[mm2 + e] = a2;
            G[e] -= v[i] * v[j] * is;
        }
        QSYNC();
        vcopy(L, F, T2, mm2); vcopy(L, A, T2 + mm2, mm2);
        QSYNC();
    }
    double* o = a.comp + c * (int64_t)3 * mm2;
    vcopy(L, o, A, mm2); vcopy(L, o + mm2, F, mm2); vcopy(L, o + 2 * mm2, G, mm2);
    QSYNC();
}
QHD void ric_phase2(Lane L, const RicArgs& a, double* ws) {
    const int m = a.m, mm2 = m * m;
    double* f = ws; double* M = f + mm2; double* X = M + mm2; double* T = X + mm2; double* A = T + mm2; double* G = A + mm2;
    vzero(L, f, mm2);
    QSYNC();
    for (int64_t c = 0; c < a.nchunks; ++c) {
        vcopy(L, a.fin + c * (int64_t)mm2, f, mm2);
        const double* o = a.comp + c * (int64_t)3 * mm2;
        vcopy(L, A, o, mm2); vcopy(L, G, o + 2 * mm2, mm2);
        QSYNC();
        mm(L, M, m, f, m, 1, G, m, 1, m, m, m, 1.0, false);            // M = f G
        for (int i = L.lane; i < m; i += L.nl) M[i * m + i] += 1.0;
        vcopy(L, X, f, mm2);
        QSYNC();
        solve(L, M, X, m, m);                                          // X = (I + f G)^-1 f
        mm(L, T, m, A, m, 1, X, m, 1, m, m, m, 1.0, false);            // T = A X
        for (int e = L.lane; e < mm2; e += L.nl) {
            const int i = e / m, j = e - i * m;
            double s = o[mm2 + e];
            for (int l = 0; l < m; ++l) s += T[i * m + l] * A[j * m + l];
            f[e] = s;
        }
        QSYNC();
    }
}
#if defined(__CUDA_ARCH__) && !defined(QSM_HOSTCHECK)
#define QSM_ATOMIC_MIN_LL(ptr, v) atomicMin((long long*)(ptr), (long long)(v))
#else
#define QSM_ATOMIC_MIN_LL(ptr, v) (*(ptr) = (*(ptr) < (v)) ? *(ptr) : (v))
#endif
QHD void ric_phase3(Lane L, const RicArgs& a, int64_t c, double* ws) {
    const int m = a.m, mm2 = m * m;
    double* f = ws; double* am = f + mm2; double* T = am + mm2; double* T2 = T + mm2;
    double* pv = ws + 7 * mm2; double* qv = pv + m; double* u = qv + m; double* w = u + m;
    if (a.nchunks > 1) vcopy(L, f, a.fin + c * (int64_t)mm2, mm2);
    else vzero(L, f, mm2);
    QSYNC();
    int64_t k0 = c * a.chunk, k1 = k0 + a.chunk; if (k1 > a.n) k1 = a.n;
    for (int64_t k = k0; k < k1; ++k) {
        vcopy(L, am, a.a + k * mm2, mm2); vcopy(L, pv, a.p + k * m, m); vcopy(L, qv, a.q + k * m, m);
        QSYNC();
        if (a.mode == 0) {   // ops.py:354-361
            mv(L, u, f, m, 1, pv, m, m);                                // f p
            const double piv = a.d[k] - dot_all(pv, u, m);
            const double ck = sqrt(piv);
            if (!(piv > 0.0) && L.lane == 0) QSM_ATOMIC_MIN_LL(a.info, (long long)(k + 1));
            mm(L, T, m, f, m, 1, am, 1, m, m, m, m, 1.0, false);        // tmp = f a^T
            for (int i = L.lane; i < m; i += L.nl) {                    // w = (q - p tmp) / c
                double t = qv[i];
                for (int l = 0; l < m; ++l) t -= pv[l] * T[l * m + i];
                w[i] = t / ck;
                a.o_w[k * m + i] = w[i];
            }
            if (L.lane == 0) a.o_c[k] = ck;
            QSYNC();
            for (int e = L.lane; e < mm2; e += L.nl) {                  // f <- a tmp + w w^T
                const int i = e / m, j = e - i * m;
                double s = w[i] * w[j];
                for (int l = 0; l < m; ++l) s += am[i * m + l] * T[l * m + j];
                T2[e] = s;
            }
            QSYNC();
            vcopy(L, f, T2, mm2);
            QSYNC();
        } else {             // ops.py:405-413
            mv(L, u, f, m, 1, pv, m, m);                                // fpk = f p
            const double ig = 1.0 / (a.d[k] - dot_all(pv, u, m));
            for (int i = L.lane; i < m; i += L.nl) {                    // left = q - a fpk
                double t = qv[i];
                for (int l = 0; l < m; ++l) t -= am[i * m + l] * u[l];
                w[i] = t;
                a.o_w[k * m + i] = ig * t;                              // s_k
            }
            if (L.lane == 0) a.o_c[k] = ig;
            QSYNC();
            for (int e = L.lane; e < mm2; e += L.nl)                    // ell = a - s p^T
                a.o_ell[k * mm2 + e] = am[e] - ig * w[e / m] * pv[e % m];
            mm(L, T, m, am, m, 1, f, m, 1, m, m, m, 1.0, false);        // a f
            for (int e = L.lane; e < mm2; e += L.nl) {                  // f <- a f a^T + ig left left^T
                const int i = e / m, j = e - i * m;
                double s = ig * w[i] * w[j];
                for (int l = 0; l < m; ++l) s += T[i * m + l] * am[j * m + l];
                T2[e] = s;
            }
            QSYNC();
            vcopy(L, f, T2, mm2);
            QSYNC();
        }
    }
    if (a.fend) vcopy(L, a.fend + c * (int64_t)mm2, f, mm2);
}

// =====================================================================================================================
// 4. SquareQSM.inv (core.py:436-478): a forward pass with a NON-symmetric Riccati carry f (ml x mu) and a backward pass
//    with carry z (mu x ml), both written exactly as the reference's scans and run by ONE warp over the whole series
//    (no chunk decomposition: nothing on the GP path calls it; it completes the class).
//    lower = (p, q, a) of order ml; upper = (h, g, b) = (upper.p, upper.q, upper.a) of order mu.
// =====================================================================================================================
struct SqInvArgs {
    int64_t n; int ml, mu;
    const double *d, *p, *q, *a, *h, *g, *b;
    double *ig, *s, *ell, *v, *del;        // forward outputs: n, n x ml, n x ml x ml, n x mu, n x mu x mu
    double *lam, *t, *u;                   // backward outputs: n, n x ml, n x mu
};
QHD int sqinv_smem_doubles(int ml, int mu) { return 4 * ml * mu + ml * ml + mu * mu + 6 * (ml + mu); }

QHD void sqinv_forward(Lane L, const SqInvArgs& a, double* ws) {
    const int ml = a.ml, mu = a.mu;
    double* f = ws; double* fbk = f + ml * mu; double* T = fbk + ml * mu; double* am = T + 2 * ml * mu; double* bm = am + ml * ml;
    double* pv = bm + mu * mu; double* qv = pv + ml; double* left = qv + ml; double* fhk = left + ml;
    double* hv = fhk + ml; double* gv = hv + mu; double* right = gv + mu;
    vzero(L, f, ml * mu);
    QSYNC();
    for (int64_t k = 0; k < a.n; ++k) {
        vcopy(L, am, a.a + k * ml * ml, ml * ml); vcopy(L, bm, a.b + k * mu * mu, mu * mu);
        vcopy(L, pv, a.p + k * ml, ml); vcopy(L, qv, a.q + k * ml, ml);
        vcopy(L, hv, a.h + k * mu, mu); vcopy(L, gv, a.g + k * mu, mu);
        QSYNC();
        mv(L, fhk, f, mu, 1, hv, ml, mu);                                     // fhk = f h
        mm(L, fbk, mu, f, mu, 1, bm, 1, mu, ml, mu, mu, 1.0, false);          // fbk = f b^T
        const double igk = 1.0 / (a.d[k] - dot_all(pv, fhk, ml));
        for (int i = L.lane; i < ml; i += L.nl) {                             // left = q - a fhk
            double t2 = qv[i];
            for (int l = 0; l < ml; ++l) t2 -= am[i * ml + l] * fhk[l];
            left[i] = t2;
            a.s[k * ml + i] = igk * t2;
        }
        for (int j = L.lane; j < mu; j += L.nl) {                             // right = g - p fbk
            double t2 = gv[j];
            for (int l = 0; l < ml; ++l) t2 -= pv[l] * fbk[l * mu + j];
            right[j] = t2;
            a.v[k * mu + j] = igk * t2;
        }
        if (L.lane == 0) a.ig[k] = igk;
        QSYNC();
        for (int e = L.lane; e < ml * ml; e += L.nl) a.ell[k * ml * ml + e] = am[e] - igk * left[e / ml] * pv[e % ml];
        for (int e = L.lane; e < mu * mu; e += L.nl) a.del[k * mu * mu + e] = bm[e] - igk * right[e / mu] * hv[e % mu];
        for (int e = L.lane; e < ml * mu; e += L.nl) {                        // f <- a fbk + ig left (x) right
            const int i = e / mu, j = e - i * mu;
            double t2 = igk * left[i] * right[j];
            for (int l = 0; l < ml; ++l) t2 += am[i * ml + l] * fbk[l * mu + j];
            T[e] = t2;
        }
        QSYNC();
        vcopy(L, f, T, ml * mu);
        QSYNC();
    }
}
QHD void sqinv_backward(Lane L, const SqInvArgs& a, double* ws) {
    const int ml = a.ml, mu = a.mu;
    double* z = ws; double* zak = z + ml * mu; double* T = zak + ml * mu; double* am = T + 2 * ml * mu; double* bm = am + ml * ml;
    double* pv = bm + mu * mu; double* sv = pv + ml; double* tk = sv + ml; double* spare = tk + ml;
    double* hv = spare + ml; double* vv = hv + mu; double* zsk = vv + mu; double* uk = zsk + mu;
    vzero(L, z, mu * ml);
    QSYNC();
    for (int64_t k = a.n - 1; k >= 0; --k) {
        vcopy(L, am, a.a + k * ml * ml, ml * ml); vcopy(L, bm, a.b + k * mu * mu, mu * mu);
        vcopy(L, pv, a.p + k * ml, ml); vcopy(L, sv, a.s + k * ml, ml);
        vcopy(L, hv, a.h + k * mu, mu); vcopy(L, vv, a.v + k * mu, mu);
        QSYNC();
        mv(L, zsk, z, ml, 1, sv, mu, ml);                                     // zsk = z s      (z: mu x ml)
        mm(L, zak, ml, z, ml, 1, am, ml, 1, mu, ml, ml, 1.0, false);          // zak = z a
        const double lk = a.ig[k] + dot_all(vv, zsk, mu);
        for (int i = L.lane; i < ml; i += L.nl) {                             // t = v zak - l p
            double t2 = -lk * pv[i];
            for (int l = 0; l < mu; ++l) t2 += vv[l] * zak[l * ml + i];
            tk[i] = t2;
            a.t[k * ml + i] = t2;
        }
        for (int j = L.lane; j < mu; j += L.nl) {                             // u = b^T zsk - l h
            double t2 = -lk * hv[j];
            for (int l = 0; l < mu; ++l) t2 += bm[l * mu + j] * zsk[l];
            uk[j] = t2;
            a.u[k * mu + j] = t2;
        }
        if (L.lane == 0) a.lam[k] = lk;
        QSYNC();
        for (int e = L.lane; e < mu * ml; e += L.nl) {                        // z <- b^T zak - (u + l h) (x) p - h (x) t
            const int i = e / ml, j = e - i * ml;
            double t2 = -(uk[i] + lk * hv[i]) * pv[j] - hv[i] * tk[j];
            for (int l = 0; l < mu; ++l) t2 += bm[l * mu + i] * zak[l * ml + j];
            T[e] = t2;
        }
        QSYNC();
        vcopy(L, z, T, mu * ml);
        QSYNC();
    }
}

}  // namespace qsm
