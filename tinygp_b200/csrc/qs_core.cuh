// Shared core of the quasiseparable path: the state-space model, per-point generators, small dense helpers and the
// scan pieces that are written as __host__ __device__ functions so that tests/csrc/qs_hostcheck.cu can run the SAME
// source on the CPU (serially, one "thread" at a time) against the oracle.  Included by quasisep.cu.
#pragma once
#include "common.cuh"
#include <math.h>

#define TREE_R 16
#define QS_THREADS 128

struct QsModel {
    int ncomp, J;   // ncomp = number of LEAVES; a term is a product of 1..3 consecutive leaves (kernels/quasisep.py:298-331)
    int chunk;   // points per thread (runtime tunable, option "qs_chunk")
    int nterm;
    int tfirst[B200GP_QS_MAX_COMP], tn[B200GP_QS_MAX_COMP], toff[B200GP_QS_MAX_COMP], tsize[B200GP_QS_MAX_COMP];
    int kind[B200GP_QS_MAX_COMP];
    int off[B200GP_QS_MAX_COMP];   // state offset of leaf i when every term is a single leaf (the layout-specialised path)
    int mode[B200GP_QS_MAX_COMP];  // SHO: 0 critical, 1 underdamped, 2 overdamped
    double c0[B200GP_QS_MAX_COMP], c1[B200GP_QS_MAX_COMP], c2[B200GP_QS_MAX_COMP];
    double h[B200GP_QS_MAX_J];  // observation model (constant for all supported kernels)
    double q[B200GP_QS_MAX_J];  // h Pinf
    double d0;                  // h Pinf h
};

// ---------------------------------------------------------------------------------------------
// host: lower the component list to a QsModel (constants follow kernels/quasisep.py)
// ---------------------------------------------------------------------------------------------
static inline QsModel build_model(const double* comps, int ncomp) {
    if (ncomp <= 0 || ncomp > B200GP_QS_MAX_COMP) throw GpError("quasisep: bad component count");
    QsModel m{};
    m.ncomp = ncomp;
    int J = 0;
    double Pinf[B200GP_QS_MAX_J][B200GP_QS_MAX_J] = {};
    // per-leaf constants, observation model and stationary covariance
    double lP[B200GP_QS_MAX_COMP][3][3] = {}, lh[B200GP_QS_MAX_COMP][3] = {}, lps[B200GP_QS_MAX_COMP] = {};
    int lsz[B200GP_QS_MAX_COMP] = {}, lmul[B200GP_QS_MAX_COMP] = {};
    for (int i = 0; i < ncomp; ++i) {
        const double* cc = comps + (size_t)i * B200GP_QS_STRIDE;
        const int kind = (int)cc[0];
        const double ps = cc[1], p0 = cc[2], p1 = cc[3], p2 = cc[4], p3 = cc[5];
        lmul[i] = (cc[6] != 0.0) ? 1 : 0;
        lps[i] = ps;
        int sz;
        switch (kind) {
            case B200GP_QS_EXP: sz = 1; break;
            case B200GP_QS_MATERN52: sz = 3; break;
            case B200GP_QS_MATERN32: case B200GP_QS_SHO: case B200GP_QS_CELERITE: case B200GP_QS_COSINE:
            case B200GP_QS_CARMA2: sz = 2; break;
            default: throw GpError("quasisep: unknown component kind");
        }
        lsz[i] = sz;
        m.kind[i] = kind;
        double (&P)[3][3] = lP[i];
        double (&h)[3] = lh[i];
        switch (kind) {
            case B200GP_QS_EXP:  // quasisep.py:491-525; c1 = -1/scale, or minus the decay RATE itself when the host
                                 // gives one in p2 (a real CARMA root, quasisep.py:886-892: exp(-c dt) with no division)
                m.c0[i] = p0; m.c1[i] = (p2 != 0.0) ? -p2 : -1.0 / p0; h[0] = p1; P[0][0] = 1.0; break;
            case B200GP_QS_MATERN32: {  // quasisep.py:528-569
                const double f = sqrt(3.0) / p0;
                m.c0[i] = f; m.c1[i] = f * f; h[0] = p1;
                P[0][0] = 1.0; P[1][1] = 3.0 / (p0 * p0); break;
            }
            case B200GP_QS_MATERN52: {  // quasisep.py:572-633
                const double f = sqrt(5.0) / p0, f2 = f * f, f2o3 = f2 / 3.0;
                m.c0[i] = f; m.c1[i] = f2; h[0] = p1;
                P[0][0] = 1.0; P[0][2] = -f2o3; P[1][1] = f2o3; P[2][0] = -f2o3; P[2][2] = f2 * f2; break;
            }
            case B200GP_QS_SHO: {  // quasisep.py:404-488
                const double w = p0, q = p1;
                m.c0[i] = w; m.c1[i] = q; h[0] = p2;
                P[0][0] = 1.0; P[1][1] = w * w;
                if (fabs(q - 0.5) <= 1e-8 + 1e-5 * 0.5) {  // jnp.allclose(q, 0.5)
                    m.mode[i] = 0;
                } else if (q > 0.5) {
                    m.mode[i] = 1; m.c2[i] = sqrt(fmax(4.0 * (q * q) - 1.0, 0.0));
                } else {
                    m.mode[i] = 2; m.c2[i] = sqrt(fmax(1.0 - 4.0 * (q * q), 0.0));
                }
                break;
            }
            case B200GP_QS_CELERITE: {  // quasisep.py:343-401
                const double a = p0, b = p1, c = p2, d = p3;
                const double c2 = c * c, d2 = d * d, s2 = c2 + d2;
                const double h2_2 = d2 * (a * c - b * d) / (2.0 * c * s2);
                const double h2 = sqrt(h2_2);
                const double h1 = (c * h2 - sqrt(a * d2 - s2 * h2_2)) / d;
                m.c0[i] = c; m.c1[i] = d; h[0] = h1; h[1] = h2;
                P[0][0] = 1.0; P[0][1] = P[1][0] = -c / d; P[1][1] = 1.0 + 2.0 * c2 / d2; break;
            }
            case B200GP_QS_COSINE:  // quasisep.py:636-673
                m.c0[i] = 2.0 * M_PI / p0; h[0] = p1; P[0][0] = P[1][1] = 1.0; break;
            case B200GP_QS_CARMA2: {  // one complex root pair of CARMA (quasisep.py:770-792, 866-900)
                const double c = p0, d = p1, sgn = cc[7];
                m.c0[i] = c; m.c1[i] = d; h[0] = p2; h[1] = p3;
                P[0][0] = sgn; P[0][1] = P[1][0] = -c / d; P[1][1] = sgn + 2.0 * (c / d) * (c / d);
                m.kind[i] = B200GP_QS_CELERITE;   // same transition matrix: the per-point code needs no new case
                break;
            }
        }
    }
    // terms: maximal runs of leaves chained by the mul_next flag; Kronecker structure with the FIRST leaf's index fastest
    // (kernels/quasisep.py:298-331 and _prod_helper :676-687)
    int i = 0;
    while (i < ncomp) {
        int n = 1;
        while (lmul[i + n - 1]) {
            if (i + n >= ncomp) throw GpError("quasisep: a product term runs past the last component");
            ++n;
        }
        if (n > 3) throw GpError("quasisep: a product of more than 3 state-space kernels is not supported");
        int size = 1;
        double ps = 1.0;
        for (int l = 0; l < n; ++l) { size *= lsz[i + l]; ps *= lps[i + l]; }
        if (J + size > B200GP_QS_MAX_J) throw GpError("quasisep: state dimension exceeds 8");
        const int t = m.nterm++;
        m.tfirst[t] = i; m.tn[t] = n; m.toff[t] = J; m.tsize[t] = size;
        for (int l = 0; l < n; ++l) m.off[i + l] = J;   // meaningful for single-leaf terms only
        for (int r = 0; r < size; ++r) {
            double hv = 1.0;
            int rr = r;
            for (int l = 0; l < n; ++l) { hv *= lh[i + l][rr % lsz[i + l]]; rr /= lsz[i + l]; }
            m.h[J + r] = hv;
            for (int c = 0; c < size; ++c) {
                double pv = ps;   // Scale: quasisep.py:334-340
                int r2 = r, c2 = c;
                for (int l = 0; l < n; ++l) {
                    pv *= lP[i + l][r2 % lsz[i + l]][c2 % lsz[i + l]];
                    r2 /= lsz[i + l]; c2 /= lsz[i + l];
                }
                Pinf[J + r][J + c] = pv;
            }
        }
        J += size;
        i += n;
    }
    m.J = J;
    m.d0 = 0.0;
    for (int j = 0; j < J; ++j) {  // q = h Pinf ; d = sum(hP * h)   (quasisep.py:109-111)
        double s = 0.0;
        for (int k = 0; k < J; ++k) s += m.h[k] * Pinf[k][j];
        m.q[j] = s;
    }
    for (int j = 0; j < J; ++j) m.d0 += m.q[j] * m.h[j];
    return m;
}

// ---------------------------------------------------------------------------------------------
// device: per-point generators  a = T(t_{k-1}, t_k)^T,  p = h a      (quasisep.py:102-116)
// ---------------------------------------------------------------------------------------------
// transition_matrix(X1, X2) of ONE leaf as written in the reference (T, not its transpose); returns the leaf's size
__host__ __device__ __forceinline__ int qs_leaf_transition(const QsModel& m, const int ci, const double dt, double (&T)[3][3]) {
    switch (m.kind[ci]) {
        case B200GP_QS_EXP:
            T[0][0] = exp(dt * m.c1[ci]);
            return 1;
        case B200GP_QS_MATERN32: {
            const double f = m.c0[ci], e = exp(-f * dt);
            T[0][0] = e * (1.0 + f * dt); T[0][1] = e * (-m.c1[ci] * dt);
            T[1][0] = e * dt;             T[1][1] = e * (1.0 - f * dt);
            return 2;
        }
        case B200GP_QS_MATERN52: {
            const double f = m.c0[ci], f2 = m.c1[ci], d2 = dt * dt, e = exp(-f * dt);
            T[0][0] = e * (0.5 * f2 * d2 + f * dt + 1.0);
            T[0][1] = e * (-0.5 * f * f2 * d2);
            T[0][2] = e * (0.5 * f2 * f * dt * (f * dt - 2.0));
            T[1][0] = e * (dt * (f * dt + 1.0));
            T[1][1] = e * (-f2 * d2 + f * dt + 1.0);
            T[1][2] = e * (f2 * dt * (f * dt - 3.0));
            T[2][0] = e * (0.5 * d2);
            T[2][1] = e * (0.5 * dt * (2.0 - f * dt));
            T[2][2] = e * (0.5 * f2 * d2 - 2.0 * f * dt + 1.0);
            return 3;
        }
        case B200GP_QS_SHO: {
            const double w = m.c0[ci], q = m.c1[ci];
            if (m.mode[ci] == 0) {
                const double e = exp(-w * dt);
                T[0][0] = e * (1.0 + w * dt); T[0][1] = e * (-(w * w) * dt);
                T[1][0] = e * dt;             T[1][1] = e * (1.0 - w * dt);
            } else {
                const double f = m.c2[ci];
                const double arg = 0.5 * f * w * dt / q;
                const double e = exp(-0.5 * w * dt / q);
                double sn, cs;
                if (m.mode[ci] == 1) {
                    sincos(arg, &sn, &cs);
                } else {
                    sn = sinh(arg);
                    cs = cosh(arg);
                }
                T[0][0] = e * (cs + sn / f);           T[0][1] = e * (-2.0 * q * w * sn / f);
                T[1][0] = e * (2.0 * q * sn / (w * f)); T[1][1] = e * (cs - sn / f);
            }
            return 2;
        }
        case B200GP_QS_CELERITE: {
            double sn, cs;
            sincos(m.c1[ci] * dt, &sn, &cs);
            const double e = exp(-m.c0[ci] * dt);
            // exp(-c dt) * [[cos, -sin], [sin, cos]].T
            T[0][0] = e * cs; T[0][1] = e * sn;
            T[1][0] = e * -sn; T[1][1] = e * cs;
            return 2;
        }
        default: {  // COSINE
            double sn, cs;
            sincos(m.c0[ci] * dt, &sn, &cs);
            T[0][0] = cs; T[0][1] = sn;
            T[1][0] = -sn; T[1][1] = cs;
            return 2;
        }
    }
}

template <int J>
__host__ __device__ __forceinline__ void qs_gen(const QsModel& m, const double dt, double (&a)[J][J], double (&p)[J]) {
    double al[J * J];  // scratch with runtime offsets; copied to registers below
#pragma unroll
    for (int i = 0; i < J * J; ++i) al[i] = 0.0;
    for (int ti = 0; ti < m.nterm; ++ti) {
        const int o = m.toff[ti], f0 = m.tfirst[ti];
        double T[3][3];
        const int sz = qs_leaf_transition(m, f0, dt, T);
        if (m.tn[ti] == 1) {
            for (int r = 0; r < sz; ++r)
                for (int s = 0; s < sz; ++s) al[(o + r) * J + (o + s)] = T[s][r];  // a = T^T
        } else {
            // product term: T = kron-structured product of the leaves' transition matrices, first leaf's index fastest
            double T1[3][3], T2[3][3];
            const int s1 = qs_leaf_transition(m, f0 + 1, dt, T1);
            int s2 = 1;
            T2[0][0] = 1.0;
            if (m.tn[ti] == 3) s2 = qs_leaf_transition(m, f0 + 2, dt, T2);
            const int S = sz * s1 * s2;
            for (int r = 0; r < S; ++r)
                for (int s = 0; s < S; ++s) {
                    const double v = T[s % sz][r % sz] * T1[(s / sz) % s1][(r / sz) % s1] * T2[s / (sz * s1)][r / (sz * s1)];
                    al[(o + r) * J + (o + s)] = v;   // a[r][s] = T_term[s][r]
                }
        }
    }
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = 0; j < J; ++j) a[i][j] = al[i * J + j];
#pragma unroll
    for (int j = 0; j < J; ++j) {  // p = h a
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < J; ++i) s += m.h[i] * a[i][j];
        p[j] = s;
    }
}

// small dense helpers ---------------------------------------------------------------------------
template <int J>
__host__ __device__ __forceinline__ void matmul(const double (&x)[J][J], const double (&y)[J][J], double (&o)[J][J]) {
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = 0; j < J; ++j) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < J; ++k) s += x[i][k] * y[k][j];
            o[i][j] = s;
        }
}
template <int J>
__host__ __device__ __forceinline__ void matmul_nt(const double (&x)[J][J], const double (&y)[J][J], double (&o)[J][J]) {
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = 0; j < J; ++j) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < J; ++k) s += x[i][k] * y[j][k];
            o[i][j] = s;
        }
}
// solve M X = B in place (B overwritten by X); Gaussian elimination with partial pivoting
template <int J>
__host__ __device__ __forceinline__ void solve_inplace(double (&M)[J][J], double (&B)[J][J]) {
#pragma unroll
    for (int c = 0; c < J; ++c) {
        int piv = c;
        double best = fabs(M[c][c]);
#pragma unroll
        for (int r = c + 1; r < J; ++r) {
            const double v = fabs(M[r][c]);
            if (v > best) { best = v; piv = r; }
        }
#pragma unroll
        for (int r = c + 1; r < J; ++r) {
            if (r == piv) {
#pragma unroll
                for (int k = 0; k < J; ++k) {
                    double tmp = M[c][k]; M[c][k] = M[r][k]; M[r][k] = tmp;
                    tmp = B[c][k]; B[c][k] = B[r][k]; B[r][k] = tmp;
                }
            }
        }
        const double inv = 1.0 / M[c][c];
#pragma unroll
        for (int r = c + 1; r < J; ++r) {
            const double f = M[r][c] * inv;
#pragma unroll
            for (int k = 0; k < J; ++k) {
                M[r][k] -= f * M[c][k];
                B[r][k] -= f * B[c][k];
            }
        }
    }
#pragma unroll
    for (int c = J - 1; c >= 0; --c) {
        const double inv = 1.0 / M[c][c];
#pragma unroll
        for (int k = 0; k < J; ++k) {
            double s = B[c][k];
#pragma unroll
            for (int r = c + 1; r < J; ++r) s -= M[c][r] * B[r][k];
            B[c][k] = s * inv;
        }
    }
}

template <int J>
__host__ __device__ __forceinline__ void ldrow(const double* __restrict__ p, int64_t k, double (&v)[J]) {
    if (J == 4 && ((reinterpret_cast<uintptr_t>(p + k * J) & 31) == 0)) {
        const double4 q = *reinterpret_cast<const double4*>(p + k * J);
        v[0] = q.x; v[1 % J] = q.y; v[2 % J] = q.z; v[3 % J] = q.w;
    } else {
#pragma unroll
        for (int j = 0; j < J; ++j) v[j] = p[k * J + j];
    }
}
template <int J>
__host__ __device__ __forceinline__ void strow(double* p, int64_t k, const double (&v)[J]) {
    if (J == 4 && ((reinterpret_cast<uintptr_t>(p + k * J) & 31) == 0)) {
        *reinterpret_cast<double4*>(p + k * J) = make_double4(v[0], v[1 % J], v[2 % J], v[3 % J]);
    } else {
#pragma unroll
        for (int j = 0; j < J; ++j) p[k * J + j] = v[j];
    }
}


#include <limits.h>
#ifdef __CUDA_ARCH__
#define QS_ATOMIC_MIN(ptr, v) atomicMin((ptr), (v))
#else
#define QS_ATOMIC_MIN(ptr, v) (*(ptr) = (*(ptr) < (v)) ? *(ptr) : (v))
#endif

// ---------------------------------------------------------------------------------------------
// 32-byte per-thread vector accesses.  One thread walks `chunk` consecutive points, so neighbouring threads are
// chunk*8 bytes apart and nothing coalesces across the warp; with scalar loads every thread keeps ~5 cache
// lines "hot" and 1024 resident threads thrash L1.  Loading/storing 4 points (one full 32-byte sector) per access makes every sector move
// exactly once.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ void ld4(const double* __restrict__ p, int64_t kb, int64_t k1, double (&v)[4]) {
    if (kb + 3 < k1 && ((reinterpret_cast<uintptr_t>(p + kb) & 31) == 0)) {
        const double4 q = *reinterpret_cast<const double4*>(p + kb);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = (kb + u < k1) ? p[kb + u] : 0.0;
    }
}
__host__ __device__ __forceinline__ void st4(double* p, int64_t kb, int64_t k1, const double (&v)[4]) {
    if (kb + 3 < k1 && ((reinterpret_cast<uintptr_t>(p + kb) & 31) == 0)) {
        *reinterpret_cast<double4*>(p + kb) = make_double4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (kb + u < k1) p[kb + u] = v[u];
    }
}

// ---------------------------------------------------------------------------------------------
// scan monoids.  Storage is structure-of-arrays: element e of item i at buf[e * count + i].
// ---------------------------------------------------------------------------------------------
template <int J>
struct Riccati {
    static constexpr int SIZE = 3 * J * J;   // A, F, G
    static constexpr int STATE = J * J;      // f
    double A[J][J], F[J][J], G[J][J];
    template <class Fn> __host__ __device__ void assign_map(const Riccati& s, Fn fn) {   // element-wise this = fn(s)
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) { A[i][j] = fn(s.A[i][j]); F[i][j] = fn(s.F[i][j]); G[i][j] = fn(s.G[i][j]); }
    }
    __host__ __device__ void identity() {
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) { A[i][j] = (i == j) ? 1.0 : 0.0; F[i][j] = 0.0; G[i][j] = 0.0; }
    }
    __host__ __device__ void load(const double* buf, int64_t count, int64_t i) {
#pragma unroll
        for (int e = 0; e < J * J; ++e) {
            A[e / J][e % J] = buf[(int64_t)e * count + i];
            F[e / J][e % J] = buf[(int64_t)(J * J + e) * count + i];
            G[e / J][e % J] = buf[(int64_t)(2 * J * J + e) * count + i];
        }
    }
    __host__ __device__ void store(double* buf, int64_t count, int64_t i) const {
#pragma unroll
        for (int e = 0; e < J * J; ++e) {
            buf[(int64_t)e * count + i] = A[e / J][e % J];
            buf[(int64_t)(J * J + e) * count + i] = F[e / J][e % J];
            buf[(int64_t)(2 * J * J + e) * count + i] = G[e / J][e % J];
        }
    }
    // this <- this (left) combined with r (right)      (ops.py:376-383)
    // M = I + F_l G_r is inverted ONCE (Gauss-Jordan with partial pivoting through solve_inplace on the identity) and
    // the three solves of the reference become products with M^-1; with G_r symmetric, M^-T G_r = (G_r M^-1)^T.
    __host__ __device__ void combine(const Riccati& r) {
        double M[J][J], Mi[J][J], X[J][J], T1[J][J], T2[J][J];
        matmul<J>(F, r.G, M);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) {
                if (i == j) M[i][j] += 1.0;
                Mi[i][j] = (i == j) ? 1.0 : 0.0;
            }
        solve_inplace<J>(M, Mi);        // Mi = M^-1
        matmul<J>(Mi, A, X);            // M^-1 A_l
        double newA[J][J];
        matmul<J>(r.A, X, newA);        // A_r M^-1 A_l
        matmul<J>(Mi, F, X);            // M^-1 F_l
        matmul<J>(r.A, X, T1);          // A_r M^-1 F_l
        double newF[J][J];
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = i; j < J; ++j) {   // F_r + (A_r M^-1 F_l) A_r^T is symmetric: upper triangle, mirrored
                double acc = r.F[i][j];
#pragma unroll
                for (int k = 0; k < J; ++k) acc += T1[i][k] * r.A[j][k];
                newF[i][j] = acc;
                newF[j][i] = acc;
            }
        matmul<J>(r.G, Mi, X);          // G_r M^-1  = (M^-T G_r)^T
        // T1 = (M^-T G_r) A_l = X^T A_l
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) {
                double acc = 0.0;
#pragma unroll
                for (int k = 0; k < J; ++k) acc += X[k][i] * A[k][j];
                T1[i][j] = acc;
            }
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = i; j < J; ++j) {   // G_l + A_l^T (M^-T G_r A_l): symmetric
                double acc = G[i][j];
#pragma unroll
                for (int k = 0; k < J; ++k) acc += A[k][i] * T1[k][j];
                T2[i][j] = acc;
                T2[j][i] = acc;
            }
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) { G[i][j] = T2[i][j]; A[i][j] = newA[i][j]; F[i][j] = newF[i][j]; }
    }
    // f <- F + A (I + f G)^-1 f A^T
    __host__ __device__ void apply(double (&f)[J][J]) const {
        double M[J][J], X[J][J], T1[J][J];
        matmul<J>(f, G, M);
#pragma unroll
        for (int i = 0; i < J; ++i) M[i][i] += 1.0;
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) X[i][j] = f[i][j];
        solve_inplace<J>(M, X);
        matmul<J>(A, X, T1);
        matmul_nt<J>(T1, A, X);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) f[i][j] = F[i][j] + X[i][j];
    }
};

template <int J>
struct Affine {
    static constexpr int SIZE = J * J + J;  // A, b
    static constexpr int STATE = J;         // g
    double A[J][J], b[J];
    template <class Fn> __host__ __device__ void assign_map(const Affine& s, Fn fn) {
#pragma unroll
        for (int i = 0; i < J; ++i) {
            b[i] = fn(s.b[i]);
#pragma unroll
            for (int j = 0; j < J; ++j) A[i][j] = fn(s.A[i][j]);
        }
    }
    __host__ __device__ void identity() {
#pragma unroll
        for (int i = 0; i < J; ++i) {
            b[i] = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) A[i][j] = (i == j) ? 1.0 : 0.0;
        }
    }
    __host__ __device__ void load(const double* buf, int64_t count, int64_t i) {
#pragma unroll
        for (int e = 0; e < J * J; ++e) A[e / J][e % J] = buf[(int64_t)e * count + i];
#pragma unroll
        for (int e = 0; e < J; ++e) b[e] = buf[(int64_t)(J * J + e) * count + i];
    }
    __host__ __device__ void store(double* buf, int64_t count, int64_t i) const {
#pragma unroll
        for (int e = 0; e < J * J; ++e) buf[(int64_t)e * count + i] = A[e / J][e % J];
#pragma unroll
        for (int e = 0; e < J; ++e) buf[(int64_t)(J * J + e) * count + i] = b[e];
    }
    __host__ __device__ void combine(const Affine& r) {  // (A_r A_l, A_r b_l + b_r)   (ops.py:322-324)
        double nA[J][J], nb[J];
        matmul<J>(r.A, A, nA);
#pragma unroll
        for (int i = 0; i < J; ++i) {
            double s = r.b[i];
#pragma unroll
            for (int k = 0; k < J; ++k) s += r.A[i][k] * b[k];
            nb[i] = s;
        }
#pragma unroll
        for (int i = 0; i < J; ++i) {
            b[i] = nb[i];
#pragma unroll
            for (int j = 0; j < J; ++j) A[i][j] = nA[i][j];
        }
    }
    __host__ __device__ void apply(double (&g)[J]) const {
        double o[J];
#pragma unroll
        for (int i = 0; i < J; ++i) {
            double s = b[i];
#pragma unroll
            for (int k = 0; k < J; ++k) s += A[i][k] * g[k];
            o[i] = s;
        }
#pragma unroll
        for (int i = 0; i < J; ++i) g[i] = o[i];
    }
};

template <int J> __host__ __device__ __forceinline__ void state_load(double (&f)[J][J], const double* buf, int64_t count, int64_t i) {
#pragma unroll
    for (int e = 0; e < J * J; ++e) f[e / J][e % J] = buf[(int64_t)e * count + i];
}
template <int J> __host__ __device__ __forceinline__ void state_store(const double (&f)[J][J], double* buf, int64_t count, int64_t i) {
#pragma unroll
    for (int e = 0; e < J * J; ++e) buf[(int64_t)e * count + i] = f[e / J][e % J];
}
template <int J> __host__ __device__ __forceinline__ void state_load(double (&g)[J], const double* buf, int64_t count, int64_t i) {
#pragma unroll
    for (int e = 0; e < J; ++e) g[e] = buf[(int64_t)e * count + i];
}
template <int J> __host__ __device__ __forceinline__ void state_store(const double (&g)[J], double* buf, int64_t count, int64_t i) {
#pragma unroll
    for (int e = 0; e < J; ++e) buf[(int64_t)e * count + i] = g[e];
}
template <int J> __host__ __device__ __forceinline__ void state_zero(double (&f)[J][J]) {
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = 0; j < J; ++j) f[i][j] = 0.0;
}
template <int J> __host__ __device__ __forceinline__ void state_zero(double (&g)[J]) {
#pragma unroll
    for (int i = 0; i < J; ++i) g[i] = 0.0;
}

template <class Op> struct StateOf;
template <int J> struct StateOf<Riccati<J>> { typedef double type[J][J]; };
template <int J> struct StateOf<Affine<J>> { typedef double type[J]; };


// Backward second-moment recursion  T <- B^T T B + U  (T, U symmetric J x J).  Used for diag((L L^T)^-1): with the
// inverse factor L^-1 = LowerTriQSM(diag = 1/c, lower = (u, v, b)), u = -p/c, v = w/c, b = a - v p^T (core.py:310-317),
//   (Sigma^-1)_ii = sum_{k >= i} (L^-1)_ki^2 = 1/c_i^2 + v_i^T S_i v_i ,   S_{i-1} = u_i u_i^T + b_i^T S_i b_i ,  S_{n-1} = 0
// -- the diagonal of the gram of core.py:424-434 without forming the matrix.
template <int J>
struct GramBack {
    static constexpr int SIZE = 2 * J * J;   // B, U
    static constexpr int STATE = J * J;      // T
    double B[J][J], U[J][J];
    template <class Fn> __host__ __device__ void assign_map(const GramBack& s, Fn fn) {
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) { B[i][j] = fn(s.B[i][j]); U[i][j] = fn(s.U[i][j]); }
    }
    __host__ __device__ void identity() {
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) { B[i][j] = (i == j) ? 1.0 : 0.0; U[i][j] = 0.0; }
    }
    __host__ __device__ void load(const double* buf, int64_t count, int64_t i) {
#pragma unroll
        for (int e = 0; e < J * J; ++e) {
            B[e / J][e % J] = buf[(int64_t)e * count + i];
            U[e / J][e % J] = buf[(int64_t)(J * J + e) * count + i];
        }
    }
    __host__ __device__ void store(double* buf, int64_t count, int64_t i) const {
#pragma unroll
        for (int e = 0; e < J * J; ++e) {
            buf[(int64_t)e * count + i] = B[e / J][e % J];
            buf[(int64_t)(J * J + e) * count + i] = U[e / J][e % J];
        }
    }
    // one point appended on the right of this composite:  U <- b^T U b + u u^T ;  B <- B b
    __host__ __device__ void push(const double (&b)[J][J], const double (&u)[J]) {
        double T1[J][J], nB[J][J];
        matmul<J>(U, b, T1);             // U b
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) {
                double acc = u[i] * u[j];
#pragma unroll
                for (int k = 0; k < J; ++k) acc += b[k][i] * T1[k][j];   // b^T (U b)
                U[i][j] = acc;
            }
        matmul<J>(B, b, nB);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) B[i][j] = nB[i][j];
    }
    // this (applied first) followed by r:  U <- B_r^T U B_r + U_r ;  B <- B B_r
    __host__ __device__ void combine(const GramBack& r) {
        double T1[J][J], nB[J][J];
        matmul<J>(U, r.B, T1);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) {
                double acc = r.U[i][j];
#pragma unroll
                for (int k = 0; k < J; ++k) acc += r.B[k][i] * T1[k][j];
                U[i][j] = acc;
            }
        matmul<J>(B, r.B, nB);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) B[i][j] = nB[i][j];
    }
    __host__ __device__ void apply(double (&T)[J][J]) const {   // T <- B^T T B + U
        double T1[J][J];
        matmul<J>(T, B, T1);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) {
                double acc = U[i][j];
#pragma unroll
                for (int k = 0; k < J; ++k) acc += B[k][i] * T1[k][j];
                T[i][j] = acc;
            }
    }
};


template <int J> struct StateOf<GramBack<J>> { typedef double type[J][J]; };

// ---------------------------------------------------------------------------------------------
// Cholesky: chunk composites and replay
// ---------------------------------------------------------------------------------------------
template <int J>
__host__ __host__ __device__ __forceinline__ void chol_chunk_body(const QsModel& m, const double* __restrict__ t, const double* __restrict__ diag, int64_t n, double* comp, int64_t nchunks, int64_t ch) {
    const int64_t k0 = ch * m.chunk, k1 = ((k0 + m.chunk < n) ? (k0 + m.chunk) : n);
    Riccati<J> R;
    R.identity();
    double tp = (k0 == 0) ? t[0] : t[k0 - 1];
    for (int64_t kb = k0; kb < k1; kb += 4) {
      double t4[4], g4[4];
      ld4(t, kb, k1, t4);
      ld4(diag, kb, k1, g4);
#pragma unroll
      for (int uu = 0; uu < 4; ++uu) {
        if (kb + uu >= k1) break;
        const double tk = t4[uu];
        double a[J][J], p[J];
        qs_gen<J>(m, tk - tp, a, p);
        tp = tk;
        const double d = m.d0 + g4[uu];
        double u[J], v[J], w[J];
        double s = d;
#pragma unroll
        for (int i = 0; i < J; ++i) {
            double x = 0.0, y = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) { x += R.F[i][j] * p[j]; y += R.A[j][i] * p[j]; }
            u[i] = x; v[i] = y;
        }
#pragma unroll
        for (int i = 0; i < J; ++i) s -= p[i] * u[i];
        const double is = 1.0 / s;
#pragma unroll
        for (int i = 0; i < J; ++i) {
            double x = m.q[i];
#pragma unroll
            for (int j = 0; j < J; ++j) x -= a[i][j] * u[j];
            w[i] = x;
        }
        double T1[J][J], T2[J][J];
        matmul<J>(a, R.F, T1);
        matmul_nt<J>(T1, a, T2);
        matmul<J>(a, R.A, T1);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) {
                R.F[i][j] = T2[i][j] + w[i] * w[j] * is;
                R.A[i][j] = T1[i][j] - w[i] * v[j] * is;
                R.G[i][j] -= v[i] * v[j] * is;
            }
      }
    }
    R.store(comp, nchunks, ch);
}

// replay with the sequential recursion of ops.py:354-361; writes c, w, per-chunk sum(log c)
template <int J>
__host__ __host__ __device__ __forceinline__ void chol_replay_body(const QsModel& m, const double* __restrict__ t, const double* __restrict__ diag, int64_t n, const double* fstart, int64_t nchunks, double* c_out, double* w_out, double* logc_part, int* info, const double* __restrict__ x_fuse, double* aff_comp, int64_t ch) {
    const int64_t k0 = ch * m.chunk, k1 = ((k0 + m.chunk < n) ? (k0 + m.chunk) : n);
    double f[J][J];
    state_load<J>(f, fstart, nchunks, ch);
    const bool fuse = (x_fuse != nullptr);
    Affine<J> R;      // forward-solve composite of this chunk (ops.py:475-486 elements), only when fusing
    R.identity();
    double tp = (k0 == 0) ? t[0] : t[k0 - 1];
    double lsum = 0.0;
    for (int64_t kb = k0; kb < k1; kb += 4) {
      double t4[4], g4[4], x4[4], c4[4];
      ld4(t, kb, k1, t4);
      ld4(diag, kb, k1, g4);
      if (fuse) ld4(x_fuse, kb, k1, x4);
#pragma unroll
      for (int uu = 0; uu < 4; ++uu) {
        const int64_t k = kb + uu;
        if (k >= k1) break;
        const double tk = t4[uu];
        double a[J][J], p[J];
        qs_gen<J>(m, tk - tp, a, p);
        tp = tk;
        const double d = m.d0 + g4[uu];
        // ck = sqrt(dk - pk @ fp @ pk)
        double pf[J];
#pragma unroll
        for (int j = 0; j < J; ++j) {
            double s = 0.0;
#pragma unroll
            for (int i = 0; i < J; ++i) s += p[i] * f[i][j];
            pf[j] = s;
        }
        double quad = 0.0;
#pragma unroll
        for (int j = 0; j < J; ++j) quad += pf[j] * p[j];
        const double c2 = d - quad;
        if (!(c2 > 0.0)) QS_ATOMIC_MIN(info, (int)((k < (int64_t)INT_MAX - 1) ? k : ((int64_t)INT_MAX - 1)) + 1);
        const double ck = sqrt(c2);
        // tmp = fp @ ak.T ; wk = (qk - pk @ tmp) / ck ; fk = ak @ tmp + outer(wk, wk)
        double tmp[J][J];
        matmul_nt<J>(f, a, tmp);
        double w[J];
#pragma unroll
        for (int j = 0; j < J; ++j) {
            double s = 0.0;
#pragma unroll
            for (int i = 0; i < J; ++i) s += p[i] * tmp[i][j];
            w[j] = (m.q[j] - s) / ck;
        }
        matmul<J>(a, tmp, f);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) f[i][j] += w[i] * w[j];
        c4[uu] = ck;
        strow<J>(w_out, k, w);
        lsum += log(ck);
        if (fuse) {   // g' = (a - w p^T / c) g + w x / c, folded while c, w, a, p are still in registers
            const double ic = 1.0 / ck, xk = x4[uu];
            double Ak[J][J], nA[J][J], nb[J];
#pragma unroll
            for (int i = 0; i < J; ++i) {
                const double wi = w[i] * ic;
#pragma unroll
                for (int j = 0; j < J; ++j) Ak[i][j] = a[i][j] - wi * p[j];
                double sb = wi * xk;
#pragma unroll
                for (int j = 0; j < J; ++j) sb += Ak[i][j] * R.b[j];
                nb[i] = sb;
            }
            matmul<J>(Ak, R.A, nA);
#pragma unroll
            for (int i = 0; i < J; ++i) {
                R.b[i] = nb[i];
#pragma unroll
                for (int j = 0; j < J; ++j) R.A[i][j] = nA[i][j];
            }
        }
      }
      st4(c_out, kb, k1, c4);
    }
    logc_part[ch] = lsum;
    if (fuse) R.store(aff_comp, nchunks, ch);
}


// ---------------------------------------------------------------------------------------------
// affine scans: triangular solves and products
// ---------------------------------------------------------------------------------------------
// OP_GEN_LOWER / OP_GEN_UPPER: the two state scans of GeneralQSM.matmul (general.py:75-104).  Same recursions as
// the symmetric product, but the replay pass stores the n x J STATES (forward f_k, backward g_k) instead of outputs.
enum { OP_LOWER_SOLVE = 0, OP_UPPER_SOLVE = 1, OP_LOWER_DOT = 2, OP_SYMM_LOWER = 3, OP_SYMM_UPPER = 4,
       OP_GEN_LOWER = 5, OP_GEN_UPPER = 6 };
__host__ __device__ constexpr bool op_reverse(int op) {
    return op == OP_UPPER_SOLVE || op == OP_SYMM_UPPER || op == OP_GEN_UPPER;
}

// logical position i of a reverse scan is physical index n-1-i
template <int J, int OP>
__host__ __host__ __device__ __forceinline__ void affine_chunk_body(const QsModel& m, const double* __restrict__ t, const double* __restrict__ c, const double* __restrict__ w, const double* __restrict__ x, int64_t n, double* comp, int64_t nchunks, int64_t ch) {
    const int64_t l0 = ch * m.chunk, l1 = ((l0 + m.chunk < n) ? (l0 + m.chunk) : n);
    Affine<J> R;
    R.identity();
    double tprev = 0.0;
    if (!op_reverse(OP)) tprev = (l0 == 0) ? t[0] : t[l0 - 1];
    for (int64_t lb = l0; lb < l1; lb += 4) {
      double t4[4], x4[4], c4[4];
      if (!op_reverse(OP)) {   // forward scans: one 32-byte sector per array per 4 points
          ld4(t, lb, l1, t4);
          ld4(x, lb, l1, x4);
          if (OP == OP_LOWER_SOLVE) ld4(c, lb, l1, c4);
      }
#pragma unroll
      for (int uu = 0; uu < 4; ++uu) {
        const int64_t l = lb + uu;
        if (l >= l1) break;
        const int64_t k = op_reverse(OP) ? (n - 1 - l) : l;
        double dt;
        if (!op_reverse(OP)) { dt = t4[uu] - tprev; tprev = t4[uu]; }
        else dt = (k == 0) ? 0.0 : (t[k] - t[k - 1]);
        double a[J][J], p[J];
        qs_gen<J>(m, dt, a, p);
        const double xk = op_reverse(OP) ? x[k] : x4[uu];
        const double ck_in = (OP == OP_LOWER_SOLVE) ? c4[uu] : ((OP == OP_UPPER_SOLVE) ? c[k] : 1.0);
        double wk[J];
        if (OP == OP_LOWER_SOLVE || OP == OP_UPPER_SOLVE || OP == OP_LOWER_DOT) ldrow<J>(w, k, wk);
        double Ak[J][J], bk[J];
        if (OP == OP_LOWER_SOLVE) {  // g' = (a - w p^T / c) g + w x / c
            const double ic = 1.0 / ck_in;
#pragma unroll
            for (int i = 0; i < J; ++i) {
                const double wi = wk[i] * ic;
                bk[i] = wi * xk;
#pragma unroll
                for (int j = 0; j < J; ++j) Ak[i][j] = a[i][j] - wi * p[j];
            }
        } else if (OP == OP_UPPER_SOLVE) {  // g' = (a^T - p w^T / c) g + p x / c
            const double ic = 1.0 / ck_in;
#pragma unroll
            for (int i = 0; i < J; ++i) {
                const double pi = p[i] * ic;
                bk[i] = pi * xk;
#pragma unroll
                for (int j = 0; j < J; ++j) Ak[i][j] = a[j][i] - pi * wk[j];
            }
        } else if (OP == OP_LOWER_DOT) {  // g' = a g + w x
#pragma unroll
            for (int i = 0; i < J; ++i) {
                bk[i] = wk[i] * xk;
#pragma unroll
                for (int j = 0; j < J; ++j) Ak[i][j] = a[i][j];
            }
        } else if (OP == OP_SYMM_LOWER || OP == OP_GEN_LOWER) {  // g' = a g + q x
#pragma unroll
            for (int i = 0; i < J; ++i) {
                bk[i] = m.q[i] * xk;
#pragma unroll
                for (int j = 0; j < J; ++j) Ak[i][j] = a[i][j];
            }
        } else {  // OP_SYMM_UPPER, OP_GEN_UPPER: g' = a^T g + p x
#pragma unroll
            for (int i = 0; i < J; ++i) {
                bk[i] = p[i] * xk;
#pragma unroll
                for (int j = 0; j < J; ++j) Ak[i][j] = a[j][i];
            }
        }
        double nA[J][J], nb[J];
        matmul<J>(Ak, R.A, nA);
#pragma unroll
        for (int i = 0; i < J; ++i) {
            double s = bk[i];
#pragma unroll
            for (int j = 0; j < J; ++j) s += Ak[i][j] * R.b[j];
            nb[i] = s;
        }
#pragma unroll
        for (int i = 0; i < J; ++i) {
            R.b[i] = nb[i];
#pragma unroll
            for (int j = 0; j < J; ++j) R.A[i][j] = nA[i][j];
        }
    }
    }
    R.store(comp, nchunks, ch);
}

// replay; out may alias x only if accumulate == 0 (each thread reads x[k] before writing out[k])
template <int J, int OP>
__host__ __host__ __device__ __forceinline__ void affine_replay_body(const QsModel& m, const double* __restrict__ t, const double* __restrict__ diag, const double* __restrict__ c, const double* __restrict__ w, const double* x, int64_t n, const double* gstart, int64_t nchunks, double* out, double* sq_part, int64_t ch) {
    const int64_t l0 = ch * m.chunk, l1 = ((l0 + m.chunk < n) ? (l0 + m.chunk) : n);
    double g[J];
    state_load<J>(g, gstart, nchunks, ch);
    double ssum = 0.0;
    double tprev = 0.0;
    if (!op_reverse(OP)) tprev = (l0 == 0) ? t[0] : t[l0 - 1];
    for (int64_t lb = l0; lb < l1; lb += 4) {
      double t4[4], x4[4], c4[4], d4[4], o4[4];
      if (!op_reverse(OP)) {   // forward scans: 32-byte vector accesses (see ld4)
          ld4(t, lb, l1, t4);
          ld4(x, lb, l1, x4);
          if (OP == OP_LOWER_SOLVE || OP == OP_LOWER_DOT) ld4(c, lb, l1, c4);
          if (OP == OP_SYMM_LOWER) ld4(diag, lb, l1, d4);
      }
#pragma unroll
      for (int uu = 0; uu < 4; ++uu) {
        const int64_t l = lb + uu;
        if (l >= l1) break;
        const int64_t k = op_reverse(OP) ? (n - 1 - l) : l;
        double dt;
        if (!op_reverse(OP)) { dt = t4[uu] - tprev; tprev = t4[uu]; }
        else dt = (k == 0) ? 0.0 : (t[k] - t[k - 1]);
        double a[J][J], p[J];
        qs_gen<J>(m, dt, a, p);
        const double xk = op_reverse(OP) ? x[k] : x4[uu];
        const double ck_in = op_reverse(OP) ? ((OP == OP_UPPER_SOLVE) ? c[k] : 1.0) : c4[uu];
        const double dk_in = (OP == OP_SYMM_LOWER) ? d4[uu] : 0.0;
        double wk[J];
        if (OP == OP_LOWER_SOLVE || OP == OP_UPPER_SOLVE || OP == OP_LOWER_DOT) ldrow<J>(w, k, wk);
        double y, ng[J];
        if (OP == OP_LOWER_SOLVE) {  // ops.py:465-468: y = (x - p@f)/d ; f = a@f + outer(q, y)
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) s += p[j] * g[j];
            y = (xk - s) / ck_in;
#pragma unroll
            for (int i = 0; i < J; ++i) {
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < J; ++j) v += a[i][j] * g[j];
                ng[i] = v + wk[i] * y;
            }
            o4[uu] = y;
        } else if (OP == OP_UPPER_SOLVE) {  // ops.py:491-494: y = (x - q@f)/d ; f = a.T@f + outer(p, y)
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) s += wk[j] * g[j];
            y = (xk - s) / ck_in;
#pragma unroll
            for (int i = 0; i < J; ++i) {
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < J; ++j) v += a[j][i] * g[j];
                ng[i] = v + p[i] * y;
            }
            out[k] = y;
        } else if (OP == OP_LOWER_DOT) {  // core.py:303-305 + ops.py:310-316: c x + p . f ; f = a f + w x
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) s += p[j] * g[j];
            y = ck_in * xk + s;
#pragma unroll
            for (int i = 0; i < J; ++i) {
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < J; ++j) v += a[i][j] * g[j];
                ng[i] = v + wk[i] * xk;
            }
            o4[uu] = y;
        } else if (OP == OP_SYMM_LOWER) {  // core.py:499-505: d x + lower part
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) s += p[j] * g[j];
            y = (m.d0 + dk_in) * xk + s;
#pragma unroll
            for (int i = 0; i < J; ++i) {
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < J; ++j) v += a[i][j] * g[j];
                ng[i] = v + m.q[i] * xk;
            }
            o4[uu] = y;
        } else if (OP == OP_GEN_LOWER) {  // general.py:77-83: f_k = a_k f_{k-1} + ql_k x_k, every f_k kept
#pragma unroll
            for (int i = 0; i < J; ++i) {
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < J; ++j) v += a[i][j] * g[j];
                ng[i] = v + m.q[i] * xk;
            }
            strow<J>(out, k, ng);
            y = 0.0;
        } else if (OP == OP_GEN_UPPER) {  // general.py:89-101: g_k = a_{k+1}^T g_{k+1} + pu_k x_k, every g_k kept.
            // The carried state here is a_{k+1}^T g_{k+1} (this scan folds a_k^T in when it LEAVES point k).
            double gk[J];
#pragma unroll
            for (int i = 0; i < J; ++i) gk[i] = g[i] + m.h[i] * xk;
            strow<J>(out, k, gk);
#pragma unroll
            for (int i = 0; i < J; ++i) {
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < J; ++j) v += a[j][i] * g[j];
                ng[i] = v + p[i] * xk;
            }
            y = 0.0;
        } else {  // OP_SYMM_UPPER (ops.py:332-338): out += q . f ; f = a^T f + p x
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) s += m.q[j] * g[j];
            y = s;
#pragma unroll
            for (int i = 0; i < J; ++i) {
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < J; ++j) v += a[j][i] * g[j];
                ng[i] = v + p[i] * xk;
            }
            out[k] += y;
        }
#pragma unroll
        for (int i = 0; i < J; ++i) g[i] = ng[i];
        ssum += y * y;
      }
      if (!op_reverse(OP) && OP != OP_GEN_LOWER) st4(out, lb, l1, o4);
    }
    if (sq_part) sq_part[ch] = ssum;
}


// ---------------------------------------------------------------------------------------------
// diag((L L^T)^-1) by a backward scan (see GramBack): logical position l is physical point n-1-l
// ---------------------------------------------------------------------------------------------
template <int J>
__host__ __device__ __forceinline__ void inv_factor_gen(const QsModel& m, const double* __restrict__ t, const double* __restrict__ c,
                                               const double* __restrict__ w, int64_t k, double& g, double (&u)[J],
                                               double (&v)[J], double (&b)[J][J]) {
    const double dt = (k == 0) ? 0.0 : (t[k] - t[k - 1]);
    double a[J][J], p[J], wk[J];
    qs_gen<J>(m, dt, a, p);
    ldrow<J>(w, k, wk);
    g = 1.0 / c[k];
#pragma unroll
    for (int i = 0; i < J; ++i) { u[i] = -g * p[i]; v[i] = g * wk[i]; }
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = 0; j < J; ++j) b[i][j] = a[i][j] - v[i] * p[j];
}

template <int J>
__host__ __device__ __forceinline__ void gram_chunk_body(const QsModel& m, const double* __restrict__ t,
                                                         const double* __restrict__ c, const double* __restrict__ w,
                                                         int64_t n, double* comp, int64_t nchunks, int64_t ch) {
    const int64_t l0 = ch * m.chunk, l1 = (l0 + m.chunk < n) ? (l0 + m.chunk) : n;
    GramBack<J> R;
    R.identity();
    for (int64_t l = l0; l < l1; ++l) {
        double g, u[J], v[J], b[J][J];
        inv_factor_gen<J>(m, t, c, w, n - 1 - l, g, u, v, b);
        R.push(b, u);
    }
    R.store(comp, nchunks, ch);
}

template <int J>
__host__ __device__ __forceinline__ void gram_replay_body(const QsModel& m, const double* __restrict__ t,
                                                          const double* __restrict__ c, const double* __restrict__ w,
                                                          int64_t n, const double* tstart, int64_t nchunks, double* out,
                                                          int64_t ch) {
    const int64_t l0 = ch * m.chunk, l1 = (l0 + m.chunk < n) ? (l0 + m.chunk) : n;
    double T[J][J];
    #pragma unroll
    for (int e = 0; e < J * J; ++e) T[e / J][e % J] = tstart[(int64_t)e * nchunks + ch];
    for (int64_t l = l0; l < l1; ++l) {
        const int64_t k = n - 1 - l;
        double g, u[J], v[J], b[J][J];
        inv_factor_gen<J>(m, t, c, w, k, g, u, v, b);
        double acc = g * g;
#pragma unroll
        for (int i = 0; i < J; ++i) {
            double r = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) r += T[i][j] * v[j];
            acc += v[i] * r;
        }
        out[k] = acc;
        double T1[J][J];
        matmul<J>(T, b, T1);
#pragma unroll
        for (int i = 0; i < J; ++i)
#pragma unroll
            for (int j = 0; j < J; ++j) {
                double r = u[i] * u[j];
#pragma unroll
                for (int kk = 0; kk < J; ++kk) r += b[kk][i] * T1[kk][j];
                T[i][j] = r;
            }
    }
}

