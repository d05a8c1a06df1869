// Structured fast path of the quasiseparable log-probability / factorisation.
//
// Same mathematics as qs_core.cuh (reference: src/tinygp/solvers/quasisep/ops.py:352-399, :463-486 and the state-space
// models of src/tinygp/kernels/quasisep.py:404-673), specialised at COMPILE TIME on the block layout of the model:
// a Sum of state-space kernels has a block-diagonal transition matrix (kernels/quasisep.py:241-295, `Block`), one block
// of size 1 (Exp), 2 (Matern32, SHO, Celerite, Cosine) or 3 (Matern52) per component.  A layout is encoded as base-4
// digits (first block = least significant digit), e.g. SHO + Matern32 -> {2, 2} -> 2 + 2*4 = 10.
//
// What the specialisation buys over the generic J x J code of qs_core.cuh (ALU-bound):
//   * the generators land in registers with compile-time offsets (the generic qs_gen assembles them through a
//     runtime-indexed scratch array = local memory, 176 bytes of stack per thread);
//   * every product with `a` skips the structurally zero blocks (J = 4, {2,2}: 32 instead of 64 FMA per product);
//   * symmetric matrices (f, F, G) are updated on their upper triangle only;
//   * sum(log c) is accumulated as a product with exponent renormalisation (one log per chunk instead of per point);
//   * divisions by model constants are multiplications by constants prepared on the host.
// For log_probability the third pass over the points (forward substitution replay) is gone altogether: with the chunk
// prefix composite (Abar, bbar) that the replay pass maintains anyway, y_k = alpha_k - beta_k . g0 is affine in the
// state g0 at the chunk's left edge, so  sum y_k^2 = s0 - 2 s1.g0 + g0^T S2 g0  with three small accumulators per chunk
// that are evaluated once the (tiny) tree over the chunk composites has produced g0.
#pragma once
#include "qs_core.cuh"

// ---- layout helpers (all usable in constant expressions) --------------------------------------------------------
__host__ __device__ constexpr int lay_nblk(int L) { int n = 0; while (L) { ++n; L >>= 2; } return n; }
__host__ __device__ constexpr int lay_size(int L, int b) { return (L >> (2 * b)) & 3; }
__host__ __device__ constexpr int lay_off(int L, int b) { int o = 0; for (int i = 0; i < b; ++i) o += lay_size(L, i); return o; }
__host__ __device__ constexpr int lay_J(int L) { return lay_off(L, lay_nblk(L)); }
__host__ __device__ constexpr int lay_blk(int L, int i) {
    int b = 0, o = 0;
    while (b < lay_nblk(L) && o + lay_size(L, b) <= i) { o += lay_size(L, b); ++b; }
    return b;
}
__host__ __device__ constexpr bool lay_same(int L, int i, int j) { return lay_blk(L, i) == lay_blk(L, j); }

// layouts compiled in: every composition of J <= 4 plus the common two- and three-component sums up to J = 6
#define QSF_LAYOUTS(X) \
    X(1) X(2) X(3) X(5) X(6) X(9) X(10) X(7) X(13) X(21) X(37) X(25) X(22) X(85) \
    X(42) X(14) X(11) X(15) X(26) X(41) X(38)

// host: layout code of a model, or 0 if a block does not fit the 2-bit encoding (never: sizes are 1..3) / too many blocks
static inline int qsf_layout_of(const QsModel& m) {
    int L = 0;
    if (m.ncomp > 8 || m.nterm != m.ncomp) return 0;   // product terms (Kronecker-structured blocks): generic path only
    for (int i = 0; i < m.ncomp; ++i) {
        const int sz = (m.kind[i] == B200GP_QS_EXP) ? 1 : (m.kind[i] == B200GP_QS_MATERN52 ? 3 : 2);
        L |= sz << (2 * i);
    }
    return L;
}

// constants derived on the host so that the per-point code has no division by a model constant
struct QsFastConst {
    double k0[B200GP_QS_MAX_COMP], k1[B200GP_QS_MAX_COMP], k2[B200GP_QS_MAX_COMP], k3[B200GP_QS_MAX_COMP];
};
static inline QsFastConst qsf_constants(const QsModel& m) {
    QsFastConst c{};
    for (int i = 0; i < m.ncomp; ++i) {
        switch (m.kind[i]) {
            case B200GP_QS_EXP: c.k0[i] = m.c1[i]; break;
            case B200GP_QS_SHO:
                if (m.mode[i] != 0) {
                    const double w = m.c0[i], q = m.c1[i], f = m.c2[i];
                    c.k0[i] = 0.5 * f * w / q;          // arg = k0 dt
                    c.k1[i] = -0.5 * w / q;             // e = exp(k1 dt)
                    c.k2[i] = 1.0 / f;                  // sn / f
                    c.k3[i] = 2.0 * q / (w * f);        // T10 = e * k3 * sn ; T01 = -e * (2 q w / f) sn = -e * k3 w^2 sn
                }
                break;
            default: break;
        }
    }
    return c;
}

// ---- generators: a = blockdiag(T_b^T), p = h a --------------------------------------------------------------------
template <int L, int B, int J>
struct QsfGenBlock {
    __host__ __device__ __forceinline__ static void run(const QsModel& m, const QsFastConst& fc, const double dt, double (&a)[J][J]) {
        constexpr int o = lay_off(L, B), sz = lay_size(L, B);
        if constexpr (sz == 1) {                         // Exp (quasisep.py:491-525)
            a[o][o] = exp(dt * fc.k0[B]);
        } else if constexpr (sz == 3) {                  // Matern52 (quasisep.py:572-633)
            const double f = m.c0[B], f2 = m.c1[B], d2 = dt * dt, e = exp(-f * dt), fd = f * dt;
            // a = T^T
            a[o + 0][o + 0] = e * (0.5 * f2 * d2 + fd + 1.0);
            a[o + 1][o + 0] = e * (-0.5 * f * f2 * d2);
            a[o + 2][o + 0] = e * (0.5 * f2 * f * dt * (fd - 2.0));
            a[o + 0][o + 1] = e * (dt * (fd + 1.0));
            a[o + 1][o + 1] = e * (-f2 * d2 + fd + 1.0);
            a[o + 2][o + 1] = e * (f2 * dt * (fd - 3.0));
            a[o + 0][o + 2] = e * (0.5 * d2);
            a[o + 1][o + 2] = e * (0.5 * dt * (2.0 - fd));
            a[o + 2][o + 2] = e * (0.5 * f2 * d2 - 2.0 * fd + 1.0);
        } else {
            double T00, T01, T10, T11;                   // transition_matrix as written in the reference
            const int kind = m.kind[B];
            if (kind == B200GP_QS_MATERN32) {            // quasisep.py:528-569
                const double f = m.c0[B], e = exp(-f * dt), fd = f * dt;
                T00 = e * (1.0 + fd); T01 = e * (-m.c1[B] * dt);
                T10 = e * dt;         T11 = e * (1.0 - fd);
            } else if (kind == B200GP_QS_SHO) {          // quasisep.py:404-488
                const double w = m.c0[B];
                if (m.mode[B] == 0) {
                    const double e = exp(-w * dt), wd = w * dt;
                    T00 = e * (1.0 + wd); T01 = e * (-(w * w) * dt);
                    T10 = e * dt;         T11 = e * (1.0 - wd);
                } else {
                    const double arg = fc.k0[B] * dt, e = exp(fc.k1[B] * dt);
                    double sn, cs;
                    if (m.mode[B] == 1) {
                        sincos(arg, &sn, &cs);
                    } else {
                        sn = sinh(arg);
                        cs = cosh(arg);
                    }
                    const double sf = sn * fc.k2[B], es = e * sn * fc.k3[B];
                    T00 = e * (cs + sf); T01 = -(w * w) * es;
                    T10 = es;            T11 = e * (cs - sf);
                }
            } else if (kind == B200GP_QS_CELERITE) {     // quasisep.py:343-401
                double sn, cs;
                sincos(m.c1[B] * dt, &sn, &cs);
                const double e = exp(-m.c0[B] * dt);
                T00 = e * cs; T01 = e * sn;
                T10 = -e * sn; T11 = e * cs;
            } else {                                     // Cosine (quasisep.py:636-673)
                double sn, cs;
                sincos(m.c0[B] * dt, &sn, &cs);
                T00 = cs; T01 = sn;
                T10 = -sn; T11 = cs;
            }
            a[o + 0][o + 0] = T00; a[o + 0][o + 1] = T10;
            a[o + 1][o + 0] = T01; a[o + 1][o + 1] = T11;
        }
        if constexpr (B + 1 < lay_nblk(L)) QsfGenBlock<L, B + 1, J>::run(m, fc, dt, a);
    }
};

// a: only the diagonal blocks are written (and read by the helpers below); p = h a
template <int L>
__host__ __device__ __forceinline__ void qsf_gen(const QsModel& m, const QsFastConst& fc, const double dt,
                                                 double (&a)[lay_J(L)][lay_J(L)], double (&p)[lay_J(L)]) {
    constexpr int J = lay_J(L);
    QsfGenBlock<L, 0, J>::run(m, fc, dt, a);
#pragma unroll
    for (int j = 0; j < J; ++j) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < J; ++i)
            if (lay_same(L, i, j)) s += m.h[i] * a[i][j];
        p[j] = s;
    }
}

// out = a X   (a block diagonal)
template <int L, int J>
__host__ __device__ __forceinline__ void qsf_a_times(const double (&a)[J][J], const double (&X)[J][J], double (&o)[J][J]) {
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = 0; j < J; ++j) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < J; ++k)
                if (lay_same(L, i, k)) s += a[i][k] * X[k][j];
            o[i][j] = s;
        }
}
// upper triangle of  T a^T + scale * w w^T  (result symmetric), mirrored into the lower triangle
template <int L, int J>
__host__ __device__ __forceinline__ void qsf_sym_times_aT_plus(const double (&T)[J][J], const double (&a)[J][J],
                                                               const double (&w)[J], const double scale, double (&o)[J][J]) {
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = i; j < J; ++j) {
            double s = (scale * w[i]) * w[j];
#pragma unroll
            for (int k = 0; k < J; ++k)
                if (lay_same(L, j, k)) s += T[i][k] * a[j][k];
            o[i][j] = s;
            o[j][i] = s;
        }
}
// o_i = sum_{k in block(i)} a[i][k] x[k]
template <int L, int J>
__host__ __device__ __forceinline__ void qsf_a_vec(const double (&a)[J][J], const double (&x)[J], double (&o)[J]) {
#pragma unroll
    for (int i = 0; i < J; ++i) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < J; ++k)
            if (lay_same(L, i, k)) s += a[i][k] * x[k];
        o[i] = s;
    }
}

// ---- pass 1: fold a chunk into its Riccati composite (A, F, G) of ops.py:368-385 --------------------------------
template <int L>
__host__ __device__ __forceinline__ void qsf_chunk_body(const QsModel& m, const QsFastConst& fc, const double* __restrict__ t,
                                                        const double* __restrict__ diag, int64_t n, double* comp,
                                                        int64_t nchunks, int64_t ch) {
    constexpr int J = lay_J(L);
    const int64_t k0 = ch * m.chunk, k1 = ((k0 + m.chunk < n) ? (k0 + m.chunk) : n);
    Riccati<J> R;
    R.identity();
    double a[J][J];
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = 0; j < J; ++j) a[i][j] = 0.0;
    double tp = (k0 == 0) ? t[0] : t[k0 - 1];
    for (int64_t kb = k0; kb < k1; kb += 4) {
        double t4[4], g4[4];
        ld4(t, kb, k1, t4);
        ld4(diag, kb, k1, g4);
#pragma unroll
        for (int uu = 0; uu < 4; ++uu) {
            if (kb + uu >= k1) break;
            const double tk = t4[uu];
            double p[J];
            qsf_gen<L>(m, fc, tk - tp, a, p);
            tp = tk;
            double u[J], v[J], w[J], au[J];
            double s = m.d0 + g4[uu];
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
            qsf_a_vec<L, J>(a, u, au);
#pragma unroll
            for (int i = 0; i < J; ++i) w[i] = m.q[i] - au[i];
            double T1[J][J], nF[J][J];
            qsf_a_times<L, J>(a, R.F, T1);
            qsf_sym_times_aT_plus<L, J>(T1, a, w, is, nF);           // F <- a F a^T + w w^T / s
            qsf_a_times<L, J>(a, R.A, T1);                          // A <- a A - w v^T / s
#pragma unroll
            for (int i = 0; i < J; ++i) {
                const double wi = w[i] * is;
#pragma unroll
                for (int j = 0; j < J; ++j) {
                    R.F[i][j] = nF[i][j];
                    R.A[i][j] = T1[i][j] - wi * v[j];
                }
            }
#pragma unroll
            for (int i = 0; i < J; ++i) {                           // G <- G - v v^T / s  (symmetric)
                const double vi = v[i] * is;
#pragma unroll
                for (int j = i; j < J; ++j) {
                    const double gij = R.G[i][j] - vi * v[j];
                    R.G[i][j] = gij;
                    R.G[j][i] = gij;
                }
            }
        }
    }
    R.store(comp, nchunks, ch);
}

// per-chunk accumulators of the fused forward substitution: sum y^2 = s0 - 2 s1.g0 + g0^T S2 g0
template <int J>
struct QsfQuad {
    static constexpr int SIZE = 1 + J + J * (J + 1) / 2;
};

// ---- one point of the fused forward substitution (ops.py:465-468) in composite form ----------------------------------
// With (Abar, bbar) the composite of the chunk's points before k:  g_{k-1} = Abar g0 + bbar, so
//   y_k = (x_k - p.g_{k-1}) / c = alpha - beta . g0 ,   alpha = (x_k - p.bbar) / c ,  beta = p^T Abar / c ,
// then g <- a g + w y :  Abar <- a Abar - w beta ,  bbar <- a bbar + w alpha.   Accumulates sum alpha^2, sum alpha beta,
// sum beta beta^T (upper triangle).
template <int L>
__host__ __device__ __forceinline__ void qsf_fuse_step(const double (&a)[lay_J(L)][lay_J(L)], const double (&p)[lay_J(L)],
                                                       const double (&w)[lay_J(L)], const double ic, const double xk,
                                                       Affine<lay_J(L)>& R, double& s0, double (&s1)[lay_J(L)],
                                                       double (&S2)[lay_J(L)][lay_J(L)]) {
    constexpr int J = lay_J(L);
    double pA[J];
#pragma unroll
    for (int j = 0; j < J; ++j) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < J; ++i) s += p[i] * R.A[i][j];
        pA[j] = s;
    }
    double pb = 0.0;
#pragma unroll
    for (int i = 0; i < J; ++i) pb += p[i] * R.b[i];
    const double alpha = (xk - pb) * ic;
    double beta[J];
#pragma unroll
    for (int j = 0; j < J; ++j) beta[j] = pA[j] * ic;
    s0 = fma(alpha, alpha, s0);
#pragma unroll
    for (int i = 0; i < J; ++i) {
        s1[i] = fma(alpha, beta[i], s1[i]);
#pragma unroll
        for (int j = i; j < J; ++j) S2[i][j] = fma(beta[i], beta[j], S2[i][j]);
    }
    double aA[J][J], ab[J];
    qsf_a_times<L, J>(a, R.A, aA);
    qsf_a_vec<L, J>(a, R.b, ab);
#pragma unroll
    for (int i = 0; i < J; ++i) {
        R.b[i] = fma(w[i], alpha, ab[i]);
#pragma unroll
        for (int j = 0; j < J; ++j) R.A[i][j] = aA[i][j] - w[i] * beta[j];
    }
}

template <int J>
__host__ __device__ __forceinline__ void qsf_quad_store(double* quad, int64_t nchunks, int64_t ch, const double s0,
                                                        const double (&s1)[J], const double (&S2)[J][J]) {
    quad[ch] = s0;
#pragma unroll
    for (int i = 0; i < J; ++i) quad[(int64_t)(1 + i) * nchunks + ch] = s1[i];
    int e = 1 + J;
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = i; j < J; ++j) { quad[(int64_t)e * nchunks + ch] = S2[i][j]; ++e; }
}

// ---- pass 2: replay a chunk from the state f at its left edge (ops.py:354-361); writes c, w, sum(log c), and -- when
// x_fuse != nullptr -- the chunk's forward-substitution composite (ops.py:475-486 elements) plus the QsfQuad sums -----
template <int L>
__host__ __device__ __forceinline__ void qsf_replay_body(const QsModel& m, const QsFastConst& fc, const double* __restrict__ t,
                                                         const double* __restrict__ diag, int64_t n, const double* fstart,
                                                         int64_t nchunks, double* c_out, double* w_out, double* logc_part,
                                                         int* info, const double* __restrict__ x_fuse, double* aff_comp,
                                                         double* quad, int64_t ch) {
    constexpr int J = lay_J(L);
    const int64_t k0 = ch * m.chunk, k1 = ((k0 + m.chunk < n) ? (k0 + m.chunk) : n);
    double f[J][J];
    state_load<J>(f, fstart, nchunks, ch);
    const bool fuse = (x_fuse != nullptr);
    Affine<J> R;
    R.identity();
    double s0 = 0.0, s1[J], S2[J][J];
#pragma unroll
    for (int i = 0; i < J; ++i) {
        s1[i] = 0.0;
#pragma unroll
        for (int j = 0; j < J; ++j) S2[i][j] = 0.0;
    }
    double a[J][J];
#pragma unroll
    for (int i = 0; i < J; ++i)
#pragma unroll
        for (int j = 0; j < J; ++j) a[i][j] = 0.0;
    double tp = (k0 == 0) ? t[0] : t[k0 - 1];
    double lmant = 1.0;      // prod c_k = lmant * 2^lexp, renormalised every 4 points
    int lexp = 0;
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
            double p[J];
            qsf_gen<L>(m, fc, tk - tp, a, p);
            tp = tk;
            const double d = m.d0 + g4[uu];
            double pf[J];
#pragma unroll
            for (int j = 0; j < J; ++j) {
                double s = 0.0;
#pragma unroll
                for (int i = 0; i < J; ++i) s += p[i] * f[i][j];
                pf[j] = s;
            }
            double quadv = 0.0;
#pragma unroll
            for (int j = 0; j < J; ++j) quadv += pf[j] * p[j];
            const double c2 = d - quadv;
            if (!(c2 > 0.0)) QS_ATOMIC_MIN(info, (int)((k < (int64_t)INT_MAX - 1) ? k : ((int64_t)INT_MAX - 1)) + 1);
            const double ck = sqrt(c2);
            const double ic = 1.0 / ck;
            // w = (q - a (f p)) / c   [(p f a^T)_j = sum_k a[j][k] (f p)_k, f symmetric]
            double apf[J], w[J];
            qsf_a_vec<L, J>(a, pf, apf);
#pragma unroll
            for (int j = 0; j < J; ++j) w[j] = (m.q[j] - apf[j]) * ic;
            // f <- a f a^T + w w^T
            double T1[J][J], nf[J][J];
            qsf_a_times<L, J>(a, f, T1);
            qsf_sym_times_aT_plus<L, J>(T1, a, w, 1.0, nf);
#pragma unroll
            for (int i = 0; i < J; ++i)
#pragma unroll
                for (int j = 0; j < J; ++j) f[i][j] = nf[i][j];
            c4[uu] = ck;
            strow<J>(w_out, k, w);
            if (c2 > 0.0) lmant *= ck;         // a failed pivot is reported through info; keep the product finite
            if (fuse) qsf_fuse_step<L>(a, p, w, ic, x4[uu], R, s0, s1, S2);
        }
        {   // renormalise the running product: lmant in [0.5, 1)
            int e;
            lmant = frexp(lmant, &e);
            lexp += e;
        }
        st4(c_out, kb, k1, c4);
    }
    logc_part[ch] = log(lmant) + (double)lexp * 0.6931471805599453094;
    if (fuse) {
        R.store(aff_comp, nchunks, ch);
        qsf_quad_store<J>(quad, nchunks, ch, s0, s1, S2);
    }
}

// ---- |L^-1 x|^2 of an existing factor (c, w): ONE pass over the points (composite + quadratic sums), then the tree over the
// chunk composites and qsf_quad_eval -- gp.py:313-316 without materialising alpha ------------------------------------
template <int L>
__host__ __device__ __forceinline__ void qsf_solvesq_body(const QsModel& m, const QsFastConst& fc, const double* __restrict__ t,
                                                          const double* __restrict__ c, const double* __restrict__ w,
                                                          const double* __restrict__ x, int64_t n, double* aff_comp,
                                                          double* quad, int64_t nchunks, int64_t ch) {
    constexpr int J = lay_J(L);
    const int64_t k0 = ch * m.chunk, k1 = ((k0 + m.chunk < n) ? (k0 + m.chunk) : n);
    Affine<J> R;
    R.identity();
    double s0 = 0.0, s1[J], S2[J][J], a[J][J];
#pragma unroll
    for (int i = 0; i < J; ++i) {
        s1[i] = 0.0;
#pragma unroll
        for (int j = 0; j < J; ++j) { S2[i][j] = 0.0; a[i][j] = 0.0; }
    }
    double tp = (k0 == 0) ? t[0] : t[k0 - 1];
    for (int64_t kb = k0; kb < k1; kb += 4) {
        double t4[4], x4[4], c4[4];
        ld4(t, kb, k1, t4);
        ld4(x, kb, k1, x4);
        ld4(c, kb, k1, c4);
#pragma unroll
        for (int uu = 0; uu < 4; ++uu) {
            const int64_t k = kb + uu;
            if (k >= k1) break;
            double p[J], wk[J];
            qsf_gen<L>(m, fc, t4[uu] - tp, a, p);
            tp = t4[uu];
            ldrow<J>(w, k, wk);
            qsf_fuse_step<L>(a, p, wk, 1.0 / c4[uu], x4[uu], R, s0, s1, S2);
        }
    }
    R.store(aff_comp, nchunks, ch);
    qsf_quad_store<J>(quad, nchunks, ch, s0, s1, S2);
}

// ---- finish: sum over the chunk of y^2 given the state g0 at the chunk's left edge --------------------------------
template <int J>
__host__ __device__ __forceinline__ double qsf_quad_eval(const double* quad, const double* gstart, int64_t nchunks, int64_t ch) {
    double g[J];
    state_load<J>(g, gstart, nchunks, ch);
    double acc = quad[ch];
    int e = 1 + J;
#pragma unroll
    for (int i = 0; i < J; ++i) {
        acc -= 2.0 * quad[(int64_t)(1 + i) * nchunks + ch] * g[i];
#pragma unroll
        for (int j = i; j < J; ++j) {
            const double sij = quad[(int64_t)e * nchunks + ch];
            acc += ((i == j) ? 1.0 : 2.0) * sij * g[i] * g[j];
            ++e;
        }
    }
    return acc;
}
