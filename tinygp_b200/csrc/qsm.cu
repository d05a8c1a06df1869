// Quasiseparable-matrix algebra on the device: the C-ABI `b200gp_qsm_*` behind tinygp_b200/solvers/quasisep/core.py
// and ops.py (reference: src/tinygp/solvers/quasisep/core.py, ops.py; conditioning: solver.py:124-129).
// A b200gp_qsm owns device-resident generator arrays (shared, reference-counted, between a matrix and its parts /
// transposes); every operation is O(n m^3) on the device and returns a new handle -- nothing is densified.
//
// Compiled twice: into libb200gp.so (kernels below, one warp per chunk), and with -DQSM_HOSTCHECK by
// tests/test_qsm_device_code_on_host.py (same bodies, loops instead of launches, malloc instead of cudaMalloc) so that
// the CPU suite exercises this very source against the oracle.
#ifdef QSM_HOSTCHECK
#include <stdexcept>
#include <string>
#include <stdlib.h>
#include <string.h>
struct GpError : std::runtime_error { explicit GpError(const std::string& s) : std::runtime_error(s) {} };
struct b200gp_ctx { std::string err; int64_t qsm_chunk = 0; int64_t launches = 0; int64_t qsm_sequential_redos = 0; };
#define API_BEGIN(ctxptr) b200gp_ctx* _ctx = (ctxptr); if (!_ctx) return 1; try {
#define API_END return 0; } catch (const std::exception& e) { _ctx->err = e.what(); return 2; }
#else
#include "common.cuh"
#endif
#include "qsm_core.cuh"

#include <limits.h>
#include <memory>
#include <vector>

using qsm::Lane;

// ---- memory ----------------------------------------------------------------------------------------------------------
struct QBuf {
    b200gp_ctx* ctx; double* p; size_t bytes;
    QBuf(b200gp_ctx* c, size_t nd) : ctx(c), p(nullptr), bytes(nd * 8) {
#ifdef QSM_HOSTCHECK
        p = (double*)malloc(bytes ? bytes : 8);
#else
        p = (double*)c->alloc(bytes);
#endif
    }
    ~QBuf() {
#ifdef QSM_HOSTCHECK
        free(p);
#else
        ctx->release(p, bytes);
#endif
    }
    QBuf(const QBuf&) = delete;
    QBuf& operator=(const QBuf&) = delete;
};
typedef std::shared_ptr<QBuf> BufP;
static BufP qnew(b200gp_ctx* c, size_t ndoubles) { return std::make_shared<QBuf>(c, ndoubles); }

static void q_h2d(b200gp_ctx* c, double* dst, const double* src, size_t nd) {
#ifdef QSM_HOSTCHECK
    (void)c; memcpy(dst, src, nd * 8);
#else
    CUDA_CHECK(cudaMemcpyAsync(dst, src, nd * 8, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));      // the caller's (pageable) buffer may go away
#endif
}
static void q_d2h(b200gp_ctx* c, double* dst, const double* src, size_t nd) {
#ifdef QSM_HOSTCHECK
    (void)c; memcpy(dst, src, nd * 8);
#else
    CUDA_CHECK(cudaMemcpyAsync(dst, src, nd * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
#endif
}
static void q_zero(b200gp_ctx* c, double* dst, size_t nd) {
#ifdef QSM_HOSTCHECK
    (void)c; memset(dst, 0, nd * 8);
#else
    CUDA_CHECK(cudaMemsetAsync(dst, 0, nd * 8, c->stream));
#endif
}

// ---- launch wrappers ---------------------------------------------------------------------------------------------------
#ifndef QSM_HOSTCHECK
template <class Args, void (*Body)(Lane, const Args&, int64_t, double*)>
__global__ void qsm_chunk_kernel(const Args a, int64_t nchunks, int wsd) {
    extern __shared__ double qsm_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    if (c >= nchunks) return;
    Body(Lane{lane, 32}, a, c, qsm_smem + (size_t)warp * wsd);
}
template <class Args, void (*Body)(Lane, const Args&, double*)>
__global__ void qsm_single_kernel(const Args a) {
    extern __shared__ double qsm_smem[];
    Body(Lane{(int)threadIdx.x, 32}, a, qsm_smem);
}
template <class Args, void (*Fn)(int64_t, const Args&)>
__global__ void qsm_ew_kernel(const Args a, int64_t total) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) Fn(i, a);
}
#endif

template <class Args, void (*Body)(Lane, const Args&, int64_t, double*)>
static void run_chunks(b200gp_ctx* ctx, const Args& a, int64_t nchunks, int wsd) {
#ifdef QSM_HOSTCHECK
    std::vector<double> ws((size_t)wsd + 8);
    for (int64_t c = 0; c < nchunks; ++c) Body(Lane{0, 1}, a, c, ws.data());
    ctx->launches++;
#else
    int wpb = 4;
    while (wpb > 1 && (size_t)wpb * wsd * 8 > (size_t)200 * 1024) wpb >>= 1;
    const size_t smem = (size_t)wpb * wsd * 8;
    if (smem > (size_t)220 * 1024) throw GpError("qsm: generator order too large for the shared-memory scan state");
    if (smem > 48 * 1024)
        CUDA_CHECK(cudaFuncSetAttribute(qsm_chunk_kernel<Args, Body>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t blocks = (nchunks + wpb - 1) / wpb;
    qsm_chunk_kernel<Args, Body><<<(unsigned)blocks, wpb * 32, smem, ctx->stream>>>(a, nchunks, wsd);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
#endif
}
template <class Args, void (*Body)(Lane, const Args&, double*)>
static void run_single(b200gp_ctx* ctx, const Args& a, int wsd) {
#ifdef QSM_HOSTCHECK
    std::vector<double> ws((size_t)wsd + 8);
    Body(Lane{0, 1}, a, ws.data());
    ctx->launches++;
#else
    const size_t smem = (size_t)wsd * 8;
    if (smem > 48 * 1024)
        CUDA_CHECK(cudaFuncSetAttribute(qsm_single_kernel<Args, Body>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    qsm_single_kernel<Args, Body><<<1, 32, smem, ctx->stream>>>(a);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
#endif
}
template <class Args, void (*Fn)(int64_t, const Args&)>
static void run_ew(b200gp_ctx* ctx, const Args& a, int64_t total) {
    if (total <= 0) return;
#ifdef QSM_HOSTCHECK
    for (int64_t i = 0; i < total; ++i) Fn(i, a);
    ctx->launches++;
#else
    int64_t blocks = (total + 255) / 256;
    if (blocks > (int64_t)ctx->num_sms * 32) blocks = (int64_t)ctx->num_sms * 32;
    qsm_ew_kernel<Args, Fn><<<(unsigned)blocks, 256, 0, ctx->stream>>>(a, total);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
#endif
}

// ---- element-wise pieces ---------------------------------------------------------------------------------------------
struct EwBlock {   // dst[k, r0 + i, c0 + j] (rows dR, cols dC) (+)= alpha * (s ? s[k] : 1) * src[k, i, j]  (src R x C, or its transpose)
    double* dst; int dR, dC, r0, c0; const double* src; int R, C; const double* s; double alpha; int acc, transpose, recip;
};
QHD void ew_block(int64_t idx, const EwBlock& a) {
    const int rc = a.R * a.C;
    const int64_t k = idx / rc; const int e = (int)(idx - k * rc); const int i = e / a.C, j = e - i * a.C;
    double v = a.transpose ? a.src[k * rc + j * a.R + i] : a.src[k * rc + e];   // transpose: src is C x R
    double sc = a.alpha;
    if (a.s) sc *= a.recip ? 1.0 / a.s[k] : a.s[k];
    double* d = a.dst + (k * a.dR + a.r0 + i) * a.dC + a.c0 + j;
    *d = (a.acc ? *d : 0.0) + sc * v;
}
struct EwOuter {   // dst[k, r0 + i, c0 + j] (+)= alpha * (s ? s[k] : 1) * u[k, i] * v[k, j]
    double* dst; int dR, dC, r0, c0; const double* u; int R; const double* v; int C; const double* s; double alpha; int acc;
};
QHD void ew_outer(int64_t idx, const EwOuter& a) {
    const int rc = a.R * a.C;
    const int64_t k = idx / rc; const int e = (int)(idx - k * rc); const int i = e / a.C, j = e - i * a.C;
    double* d = a.dst + (k * a.dR + a.r0 + i) * a.dC + a.c0 + j;
    *d = (a.acc ? *d : 0.0) + a.alpha * (a.s ? a.s[k] : 1.0) * a.u[k * a.R + i] * a.v[k * a.C + j];
}
struct EwVec { double* dst; const double* x; const double* y; double alpha, beta; int op; };   // op 0: ax + by, 1: x*y, 2: 1/x
QHD void ew_vec(int64_t i, const EwVec& a) {
    if (a.op == 0) a.dst[i] = a.alpha * a.x[i] + (a.y ? a.beta * a.y[i] : 0.0);
    else if (a.op == 1) a.dst[i] = a.x[i] * a.y[i];
    else a.dst[i] = 1.0 / a.x[i];
}
struct EwKron {    // core.py:218-233: e = j * m1 + i  (i, j = meshgrid(arange(m1), arange(m2)) flattened)
    double* dst; const double* x; const double* y; int m1, m2, matrix;
};
QHD void ew_kron(int64_t idx, const EwKron& a) {
    const int M = a.m1 * a.m2;
    if (!a.matrix) {
        const int64_t k = idx / M; const int e = (int)(idx - k * M);
        a.dst[idx] = a.x[k * a.m1 + e % a.m1] * a.y[k * a.m2 + e / a.m1];
    } else {
        const int64_t k = idx / ((int64_t)M * M); const int ef = (int)(idx - k * (int64_t)M * M); const int e = ef / M, f = ef - e * M;
        a.dst[idx] = a.x[(k * a.m1 + e % a.m1) * a.m1 + f % a.m1] * a.y[(k * a.m2 + e / a.m1) * a.m2 + f / a.m1];
    }
}
struct EwLogSum { const double* x; int64_t n; double* out; };

static void blk(b200gp_ctx* c, int64_t n, double* dst, int dR, int dC, int r0, int c0, const double* src, int R, int C,
                const double* s = nullptr, double alpha = 1.0, bool acc = false, bool transpose = false, bool recip = false) {
    EwBlock a{dst, dR, dC, r0, c0, src, R, C, s, alpha, acc ? 1 : 0, transpose ? 1 : 0, recip ? 1 : 0};
    run_ew<EwBlock, ew_block>(c, a, n * R * C);
}
static void outer(b200gp_ctx* c, int64_t n, double* dst, int dR, int dC, int r0, int c0, const double* u, int R, const double* v, int C,
                  const double* s = nullptr, double alpha = 1.0, bool acc = false) {
    EwOuter a{dst, dR, dC, r0, c0, u, R, v, C, s, alpha, acc ? 1 : 0};
    run_ew<EwOuter, ew_outer>(c, a, n * R * C);
}
static void vec(b200gp_ctx* c, int64_t n, double* dst, const double* x, const double* y, double alpha, double beta, int op) {
    EwVec a{dst, x, y, alpha, beta, op};
    run_ew<EwVec, ew_vec>(c, a, n);
}

#ifdef QSM_HOSTCHECK
enum { B200GP_QSM_DIAG = 0, B200GP_QSM_STRICT_LOWER = 1, B200GP_QSM_STRICT_UPPER = 2, B200GP_QSM_LOWER = 3,
       B200GP_QSM_UPPER = 4, B200GP_QSM_SQUARE = 5, B200GP_QSM_SYMM = 6 };
#endif
// ---- sum of logs: slab i of QSM_LOGSUM_SLABS covers [i * len, (i + 1) * len); one block per slab, fixed reduction tree ----
#define QSM_LOGSUM_SLABS 256
#ifndef QSM_HOSTCHECK
__global__ void __launch_bounds__(256) qsm_logsum_kernel(const double* __restrict__ x, int64_t n, double* __restrict__ part) {
    __shared__ double sh[256];
    const int64_t len = (n + QSM_LOGSUM_SLABS - 1) / QSM_LOGSUM_SLABS;
    const int64_t lo = (int64_t)blockIdx.x * len, hi = (lo + len < n) ? (lo + len) : n;
    double s = 0.0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += 256) s += log(x[i]);
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}
#endif
static void qsm_logsum(b200gp_ctx* ctx, const double* x, int64_t n, double* part) {
#ifdef QSM_HOSTCHECK
    const int64_t len = (n + QSM_LOGSUM_SLABS - 1) / QSM_LOGSUM_SLABS;
    for (int b = 0; b < QSM_LOGSUM_SLABS; ++b) {     // the kernel's summation tree, thread by thread
        double sh[256];
        const int64_t lo = (int64_t)b * len, hi = (lo + len < n) ? (lo + len) : n;
        for (int t = 0; t < 256; ++t) {
            double s = 0.0;
            for (int64_t i = lo + t; i < hi; i += 256) s += log(x[i]);
            sh[t] = s;
        }
        for (int o = 128; o > 0; o >>= 1)
            for (int t = 0; t < o; ++t) sh[t] += sh[t + o];
        part[b] = sh[0];
    }
    ctx->launches++;
#else
    qsm_logsum_kernel<<<QSM_LOGSUM_SLABS, 256, 0, ctx->stream>>>(x, n, part);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
#endif
}

// ---- the object --------------------------------------------------------------------------------------------------------
struct QTri {
    int m = 0; BufP p, q, a;
    bool present() const { return m > 0; }
    qsm::Tri view() const { return qsm::Tri{p->p, q->p, a->p, m}; }
};
struct b200gp_qsm {
    b200gp_ctx* ctx = nullptr;
    int64_t n = 0;
    int symm = 0;
    BufP d;
    QTri lo, up;
    // ops.py `deconstruct` (:217-229): the upper part of a SymmQSM is its lower part read as StrictUpperTriQSM
    const QTri& upper() const { return symm ? lo : up; }
    int kind() const {
        if (symm) return B200GP_QSM_SYMM;
        const bool hd = (bool)d, hl = lo.present(), hu = up.present();
        if (!hl && !hu) return B200GP_QSM_DIAG;
        if (!hd) return hl && !hu ? B200GP_QSM_STRICT_LOWER : (hu && !hl ? B200GP_QSM_STRICT_UPPER : -1);
        if (!hu) return B200GP_QSM_LOWER;
        if (!hl) return B200GP_QSM_UPPER;
        return B200GP_QSM_SQUARE;
    }
};

static b200gp_qsm* q_new(b200gp_ctx* c, int64_t n) {
    b200gp_qsm* r = new b200gp_qsm();
    r->ctx = c; r->n = n;
    return r;
}
// ops.py `construct` (:232-268)
static b200gp_qsm* q_construct(b200gp_ctx* c, int64_t n, BufP d, const QTri& lo, const QTri& up, bool symm) {
    std::unique_ptr<b200gp_qsm> r(q_new(c, n));
    if (!lo.present() && !up.present()) {
        if (!d) throw GpError("qsm: empty result");
        r->d = d;
        return r.release();
    }
    if (symm) {
        if (!d || !lo.present()) throw GpError("qsm: a symmetric result needs a diagonal and a lower part");
        r->d = d; r->lo = lo; r->symm = 1;
        return r.release();
    }
    if (lo.present() && up.present() && !d) throw GpError("qsm: strictly lower + strictly upper has no QSM type (ops.py:262-265)");
    r->d = d; r->lo = lo; r->up = up;
    return r.release();
}

static void chunking(b200gp_ctx* ctx, int64_t n, int64_t& chunk, int64_t& nchunks) {
    int64_t want = ctx->qsm_chunk;
    if (want <= 0) {
        int64_t nch = (n + 7) / 8;                 // at least 8 points per warp, at most 2048 chunks
        if (nch > 2048) nch = 2048;
        if (nch < 1) nch = 1;
        want = (n + nch - 1) / nch;
    }
    chunk = want < 1 ? 1 : want;
    nchunks = (n + chunk - 1) / chunk;
    if (nchunks < 1) nchunks = 1;
}

// ---- scans -------------------------------------------------------------------------------------------------------------
// out (n x nrhs, row stride ld) (+)= op(part) x   for the column tile [j0, j0 + kc)
static void run_low(b200gp_ctx* ctx, int op, int64_t n, const double* d, const QTri& t, const double* x, double* out, int64_t ld,
                    int64_t nrhs, bool accumulate) {
    int64_t chunk, nch;
    chunking(ctx, n, chunk, nch);
    const int m = t.m;
    const int KC = 16;
    BufP comp = qnew(ctx, (size_t)nch * m * (m + KC)), fin = qnew(ctx, (size_t)nch * m * KC);
    for (int64_t j0 = 0; j0 < nrhs; j0 += KC) {
        qsm::LowArgs a{};
        a.op = op; a.n = n; a.m = m; a.kc = (int)((nrhs - j0 < KC) ? (nrhs - j0) : KC); a.chunk = chunk; a.nchunks = nch;
        a.d = d; a.t = t.view(); a.x = x + j0; a.ldx = ld; a.out = out + j0; a.ldo = ld; a.accumulate = accumulate ? 1 : 0;
        a.comp = comp->p; a.fin = fin->p;
        const int wsd = qsm::low_smem_doubles(m, a.kc);
        if (nch > 1) {
            run_chunks<qsm::LowArgs, qsm::low_phase1>(ctx, a, nch, wsd);
            run_single<qsm::LowArgs, qsm::low_phase2>(ctx, a, wsd);
        }
        run_chunks<qsm::LowArgs, qsm::low_phase3>(ctx, a, nch, wsd);
    }
}
static void run_bil(b200gp_ctx* ctx, qsm::BilArgs a) {
    chunking(ctx, a.n, a.chunk, a.nchunks);
    const int csz = a.m1 * a.m1 + a.m2 * a.m2 + a.m1 * a.m2;
    BufP comp = qnew(ctx, (size_t)a.nchunks * csz), fin = qnew(ctx, (size_t)a.nchunks * a.m1 * a.m2);
    a.comp = comp->p; a.fin = fin->p;
    const int wsd = qsm::bil_smem_doubles(a.m1, a.m2);
    if (a.nchunks > 1) {
        run_chunks<qsm::BilArgs, qsm::bil_phase1>(ctx, a, a.nchunks, wsd);
        run_single<qsm::BilArgs, qsm::bil_phase2>(ctx, a, wsd);
    }
    run_chunks<qsm::BilArgs, qsm::bil_phase3>(ctx, a, a.nchunks, wsd);
}
// returns the 1-based index of the first non-positive pivot (mode 0), 0 if none.
// The chunk composites are exact in exact arithmetic but can lose digits when the realisation is far from minimal (the
// order-4J difference M - delta of solver.py:124-129 carries two large, almost cancelling state covariances: the closed-loop
// products have transient gains of several hundred).  The replay is the reference's sequential recursion, so the state it
// LEAVES a chunk with is the accurate continuation of the state it entered with: if that disagrees with the composite-
// derived entering state of the next chunk by more than 1e-10 (relative), the scan is redone as ONE chunk (one warp, the
// plain sequential recursion of ops.py:352-365 / :403-416) -- slower, never less accurate than the reference.
static int64_t run_ric(b200gp_ctx* ctx, qsm::RicArgs a) {
    chunking(ctx, a.n, a.chunk, a.nchunks);
    const int mm2 = a.m * a.m;
    BufP info = qnew(ctx, 1);
    a.info = (long long*)info->p;
    const int wsd = qsm::ric_smem_doubles(a.m);
    for (int attempt = 0; attempt < 2; ++attempt) {
        BufP comp = qnew(ctx, (size_t)a.nchunks * 3 * mm2), fin = qnew(ctx, (size_t)a.nchunks * mm2);
        BufP fend = a.nchunks > 1 ? qnew(ctx, (size_t)a.nchunks * mm2) : BufP();
        a.comp = comp->p; a.fin = fin->p; a.fend = fend ? fend->p : nullptr;
        long long big = LLONG_MAX;
        q_h2d(ctx, info->p, (const double*)&big, 1);
        if (a.nchunks > 1) {
            run_chunks<qsm::RicArgs, qsm::ric_phase1>(ctx, a, a.nchunks, wsd);
            run_single<qsm::RicArgs, qsm::ric_phase2>(ctx, a, wsd);
        }
        run_chunks<qsm::RicArgs, qsm::ric_phase3>(ctx, a, a.nchunks, wsd);
        if (a.nchunks == 1) break;
        std::vector<double> hin((size_t)a.nchunks * mm2), hend((size_t)a.nchunks * mm2);
        q_d2h(ctx, hin.data(), fin->p, hin.size());
        q_d2h(ctx, hend.data(), fend->p, hend.size());
        double worst = 0.0, scale = 0.0;
        for (int64_t c = 0; c + 1 < a.nchunks; ++c)
            for (int e = 0; e < mm2; ++e) {
                const double x = hend[(size_t)c * mm2 + e], y = hin[(size_t)(c + 1) * mm2 + e];
                const double df = fabs(x - y), sc = fabs(x) > fabs(y) ? fabs(x) : fabs(y);
                if (df > worst) worst = df;               // NaN (failed factorisation) compares false: no fallback needed
                if (sc > scale) scale = sc;
            }
        if (!(worst > 1e-10 * (scale > 1.0 ? scale : 1.0))) break;
        a.chunk = a.n; a.nchunks = 1;                     // sequential redo
        ctx->qsm_sequential_redos++;
    }
    long long got = 0;
    q_d2h(ctx, (double*)&got, info->p, 1);
    return got == LLONG_MAX ? 0 : (int64_t)got;
}

// ---- operations ---------------------------------------------------------------------------------------------------------
static QTri tri_new(b200gp_ctx* c, int64_t n, int m) {
    QTri t; t.m = m;
    t.p = qnew(c, (size_t)n * m); t.q = qnew(c, (size_t)n * m); t.a = qnew(c, (size_t)n * m * m);
    return t;
}
// core.py:199-216 (self_add): concatenated p, q; block-diagonal a
static QTri tri_add(b200gp_ctx* c, int64_t n, const QTri& x, const QTri& y) {
    if (!x.present()) return y;
    if (!y.present()) return x;
    const int m = x.m + y.m;
    QTri r = tri_new(c, n, m);
    blk(c, n, r.p->p, 1, m, 0, 0, x.p->p, 1, x.m); blk(c, n, r.p->p, 1, m, 0, x.m, y.p->p, 1, y.m);
    blk(c, n, r.q->p, 1, m, 0, 0, x.q->p, 1, x.m); blk(c, n, r.q->p, 1, m, 0, x.m, y.q->p, 1, y.m);
    q_zero(c, r.a->p, (size_t)n * m * m);
    blk(c, n, r.a->p, m, m, 0, 0, x.a->p, x.m, x.m); blk(c, n, r.a->p, m, m, x.m, x.m, y.a->p, y.m, y.m);
    return r;
}
// core.py:218-233 (self_mul)
static QTri tri_mul(b200gp_ctx* c, int64_t n, const QTri& x, const QTri& y) {
    if (!x.present() || !y.present()) return QTri();
    const int m = x.m * y.m;
    QTri r = tri_new(c, n, m);
    EwKron kp{r.p->p, x.p->p, y.p->p, x.m, y.m, 0}, kq{r.q->p, x.q->p, y.q->p, x.m, y.m, 0}, ka{r.a->p, x.a->p, y.a->p, x.m, y.m, 1};
    run_ew<EwKron, ew_kron>(c, kp, n * m); run_ew<EwKron, ew_kron>(c, kq, n * m); run_ew<EwKron, ew_kron>(c, ka, n * (int64_t)m * m);
    return r;
}
static BufP vec_new(b200gp_ctx* c, int64_t n, const double* x, const double* y, double alpha, double beta, int op) {
    BufP r = qnew(c, (size_t)n);
    vec(c, n, r->p, x, y, alpha, beta, op);
    return r;
}
static bool is_symm_like(const b200gp_qsm* a) { return a->symm || a->kind() == B200GP_QSM_DIAG; }

static b200gp_qsm* op_add(const b200gp_qsm* a, const b200gp_qsm* b) {          // ops.py:24-35
    b200gp_ctx* c = a->ctx; const int64_t n = a->n;
    BufP d = a->d && b->d ? vec_new(c, n, a->d->p, b->d->p, 1.0, 1.0, 0) : (a->d ? a->d : b->d);
    const bool symm = is_symm_like(a) && is_symm_like(b);
    QTri lo = tri_add(c, n, a->lo, b->lo);
    QTri up = symm ? QTri() : tri_add(c, n, a->upper(), b->upper());
    return q_construct(c, n, d, lo, up, symm);
}
static b200gp_qsm* op_emul(const b200gp_qsm* a, const b200gp_qsm* b) {         // ops.py:38-49
    b200gp_ctx* c = a->ctx; const int64_t n = a->n;
    BufP d = a->d && b->d ? vec_new(c, n, a->d->p, b->d->p, 0, 0, 1) : BufP();
    const bool symm = is_symm_like(a) && is_symm_like(b);
    QTri lo = tri_mul(c, n, a->lo, b->lo);
    QTri up = symm ? QTri() : tri_mul(c, n, a->upper(), b->upper());
    return q_construct(c, n, d, lo, up, symm);
}

// ops.py:52-214.  want_upper = false skips the strictly upper part of the result (gram, symmetric x symmetric)
static b200gp_qsm* op_mul(const b200gp_qsm* A, const b200gp_qsm* B, bool force_symm) {
    b200gp_ctx* c = A->ctx; const int64_t n = A->n;
    if (B->n != n) throw GpError("qsm_mul: dimension mismatch");
    const double* da = A->d ? A->d->p : nullptr; const double* db = B->d ? B->d->p : nullptr;
    const QTri& la = A->lo; const QTri& ua = A->upper(); const QTri& lb = B->lo; const QTri& ub = B->upper();
    const bool hla = la.present(), hua = ua.present(), hlb = lb.present(), hub = ub.present();
    if (!hla && !hua && !hlb && !hub) {                                         // ops.py:57-60
        std::unique_ptr<b200gp_qsm> r(q_new(c, n));
        r->d = vec_new(c, n, da, db, 0, 0, 1);
        return r.release();
    }
    const bool symm = force_symm || (is_symm_like(A) && is_symm_like(B));
    const bool phi = hla && hub, psi = hua && hlb;
    const bool h_alpha = (db && hla) || phi, h_beta = (da && hlb) || psi, h_theta = (da && hub) || phi, h_eta = (db && hua) || psi;
    const bool h_lam = (da && db) || phi || psi;
    // widths of the concatenated generators (ops.py:130-141)
    const int ms = (h_alpha ? la.m : 0) + (hlb ? lb.m : 0), mt = (hla ? la.m : 0) + (h_beta ? lb.m : 0);
    const int mv = (hua ? ua.m : 0) + (h_theta ? ub.m : 0), mu = (h_eta ? ua.m : 0) + (hub ? ub.m : 0);
    const bool has_lower = mt > 0 && ms > 0 && (hla || hlb), has_upper = !symm && mu > 0 && mv > 0 && (hua || hub);
    const int mell = (hla ? la.m : 0) + (hlb ? lb.m : 0), mdel = (hua ? ua.m : 0) + (hub ? ub.m : 0);
    if (has_lower && (ms != mell || mt != mell))
        throw GpError("qsm_mul: this operand combination gives generators of unequal widths (a strictly triangular factor without "
                      "a diagonal on the other side); the reference fails on it too (ops.py:130-165)");
    if (has_upper && (mu != mdel || mv != mdel))
        throw GpError("qsm_mul: this operand combination gives generators of unequal widths; the reference fails on it too");
    BufP lam = h_lam ? qnew(c, (size_t)n) : BufP();
    if (h_lam) {
        if (da && db) vec(c, n, lam->p, da, db, 0, 0, 1);
        else q_zero(c, lam->p, (size_t)n);
    }
    QTri lo, up;
    if (has_lower) {
        lo = tri_new(c, n, mell);
        // t = [lower_a.p, beta], s = [alpha, lower_b.q]
        int ot = 0, os = 0;
        if (hla) { blk(c, n, lo.p->p, 1, mell, 0, 0, la.p->p, 1, la.m); ot = la.m; }
        if (h_beta) {
            if (da) blk(c, n, lo.p->p, 1, mell, 0, ot, lb.p->p, 1, lb.m, da);           // beta = d_a * lower_b.p
            else blk(c, n, lo.p->p, 1, mell, 0, ot, lb.p->p, 1, lb.m, nullptr, 0.0);           // zero: psi adds to it
        }
        if (h_alpha) {
            if (db) blk(c, n, lo.q->p, 1, mell, 0, 0, la.q->p, 1, la.m, db);            // alpha = lower_a.q * d_b
            else blk(c, n, lo.q->p, 1, mell, 0, 0, la.q->p, 1, la.m, nullptr, 0.0);
            os = la.m;
        }
        if (hlb) blk(c, n, lo.q->p, 1, mell, 0, os, lb.q->p, 1, lb.m);
        if (hla && hlb) {                                                               // ops.py:143-158
            q_zero(c, lo.a->p, (size_t)n * mell * mell);
            blk(c, n, lo.a->p, mell, mell, 0, 0, la.a->p, la.m, la.m);
            outer(c, n, lo.a->p, mell, mell, 0, la.m, la.q->p, la.m, lb.p->p, lb.m);
            blk(c, n, lo.a->p, mell, mell, la.m, la.m, lb.a->p, lb.m, lb.m);
        } else {
            lo.a = hla ? la.a : lb.a;
        }
    }
    if (has_upper) {
        up = tri_new(c, n, mdel);
        // v = [upper_a.q, theta], u = [eta, upper_b.p]
        int ov = 0, ou = 0;
        if (hua) { blk(c, n, up.q->p, 1, mdel, 0, 0, ua.q->p, 1, ua.m); ov = ua.m; }
        if (h_theta) {
            if (da) blk(c, n, up.q->p, 1, mdel, 0, ov, ub.q->p, 1, ub.m, da);           // theta = d_a * upper_b.q
            else blk(c, n, up.q->p, 1, mdel, 0, ov, ub.q->p, 1, ub.m, nullptr, 0.0);
        }
        if (h_eta) {
            if (db) blk(c, n, up.p->p, 1, mdel, 0, 0, ua.p->p, 1, ua.m, db);            // eta = upper_a.p * d_b
            else blk(c, n, up.p->p, 1, mdel, 0, 0, ua.p->p, 1, ua.m, nullptr, 0.0);
            ou = ua.m;
        }
        if (hub) blk(c, n, up.p->p, 1, mdel, 0, ou, ub.p->p, 1, ub.m);
        if (hua && hub) {                                                               // ops.py:165-181
            q_zero(c, up.a->p, (size_t)n * mdel * mdel);
            blk(c, n, up.a->p, mdel, mdel, 0, 0, ua.a->p, ua.m, ua.m);
            outer(c, n, up.a->p, mdel, mdel, ua.m, 0, ub.q->p, ub.m, ua.p->p, ua.m);
            blk(c, n, up.a->p, mdel, mdel, ua.m, ua.m, ub.a->p, ub.m, ub.m);
        } else {
            up.a = hua ? ua.a : ub.a;
        }
    }
    if (phi) {   // ops.py:62-72, 120-123
        qsm::BilArgs a{};
        a.n = n; a.m1 = la.m; a.m2 = ub.m; a.rev = 0;
        a.La = la.a->p; a.tL = 0; a.Ra = ub.a->p; a.tR = 0;
        a.u = la.q->p; a.us = nullptr; a.v = ub.q->p; a.l1 = la.p->p; a.r1 = ub.p->p;
        if (has_lower) { a.e1 = lo.q->p; a.lde1 = mell; a.acc1 = 1; }                   // alpha += lower_a.a phi upper_b.p
        if (has_upper) { a.e2 = up.q->p + (hua ? ua.m : 0); a.lde2 = mdel; a.acc2 = 1; } // theta += lower_a.p phi upper_b.a^T
        a.e3 = lam->p; a.acc3 = 1;                                                      // lam += lower_a.p phi upper_b.p
        run_bil(c, a);
    }
    if (psi) {   // ops.py:77-87, 125-128
        qsm::BilArgs a{};
        a.n = n; a.m1 = ua.m; a.m2 = lb.m; a.rev = 1;
        a.La = ua.a->p; a.tL = 1; a.Ra = lb.a->p; a.tR = 1;
        a.u = ua.p->p; a.us = nullptr; a.v = lb.p->p; a.l1 = ua.q->p; a.r1 = lb.q->p;
        if (has_upper) { a.e1 = up.p->p; a.lde1 = mdel; a.acc1 = 1; }                   // eta += upper_a.a^T psi lower_b.q
        if (has_lower) { a.e2 = lo.p->p + (hla ? la.m : 0); a.lde2 = mell; a.acc2 = 1; } // beta += upper_a.q psi lower_b.a
        a.e3 = lam->p; a.acc3 = 1;                                                      // lam += upper_a.q psi lower_b.q
        run_bil(c, a);
    }
    return q_construct(c, n, lam, lo, up, symm);
}

static b200gp_qsm* op_transpose(const b200gp_qsm* a) {
    std::unique_ptr<b200gp_qsm> r(q_new(a->ctx, a->n));
    r->d = a->d; r->symm = a->symm;
    if (a->symm) r->lo = a->lo;
    else { r->lo = a->up; r->up = a->lo; }
    return r.release();
}
// core.py:310-317
static b200gp_qsm* op_lower_inv(const b200gp_qsm* L) {
    b200gp_ctx* c = L->ctx; const int64_t n = L->n; const int m = L->lo.m;
    std::unique_ptr<b200gp_qsm> r(q_new(c, n));
    r->d = vec_new(c, n, L->d->p, nullptr, 0, 0, 2);                                     // g = 1 / d
    r->lo = tri_new(c, n, m);
    blk(c, n, r->lo.p->p, 1, m, 0, 0, L->lo.p->p, 1, m, r->d->p, -1.0);                  // u = -g p
    blk(c, n, r->lo.q->p, 1, m, 0, 0, L->lo.q->p, 1, m, r->d->p, 1.0);                   // v = g q
    blk(c, n, r->lo.a->p, m, m, 0, 0, L->lo.a->p, m, m);
    outer(c, n, r->lo.a->p, m, m, 0, 0, r->lo.q->p, m, L->lo.p->p, m, nullptr, -1.0, true);   // b = a - v p^T
    return r.release();
}
// ops.py:403-460 (the forward carry by the Riccati scan, the backward pass in its associative form :446-458)
static b200gp_qsm* op_symm_inv(const b200gp_qsm* S) {
    b200gp_ctx* c = S->ctx; const int64_t n = S->n; const int m = S->lo.m;
    BufP ig = qnew(c, (size_t)n);
    QTri out = tri_new(c, n, m);     // p = t, q = s, a = ell
    qsm::RicArgs ra{};
    ra.n = n; ra.m = m; ra.mode = 1; ra.d = S->d->p; ra.p = S->lo.p->p; ra.q = S->lo.q->p; ra.a = S->lo.a->p;
    ra.o_c = ig->p; ra.o_w = out.q->p; ra.o_ell = out.a->p;
    run_ric(c, ra);
    BufP lam = qnew(c, (size_t)n);
    qsm::BilArgs a{};
    a.n = n; a.m1 = m; a.m2 = m; a.rev = 1;
    a.La = out.a->p; a.tL = 1; a.Ra = out.a->p; a.tR = 1;                                // z <- ell^T z ell + ig p p^T
    a.u = S->lo.p->p; a.us = ig->p; a.v = S->lo.p->p; a.l1 = out.q->p; a.r1 = out.q->p;
    a.e2 = out.p->p; a.lde2 = m; a.acc2 = 0;                                             // s^T z ell  (= s^T z a - (s^T z s) p^T)
    a.e3 = lam->p; a.acc3 = 0;                                                           // s^T z s
    run_bil(c, a);
    blk(c, n, out.p->p, 1, m, 0, 0, S->lo.p->p, 1, m, ig->p, -1.0, true);                // t = s^T z a - lam p = e2 - ig p
    vec(c, n, lam->p, lam->p, ig->p, 1.0, 1.0, 0);                                       // lam = ig + s^T z s
    std::unique_ptr<b200gp_qsm> r(q_new(c, n));
    r->d = lam; r->lo = out; r->symm = 1;
    return r.release();
}

// core.py:436-478 (sequential, one warp)
static b200gp_qsm* op_square_inv(const b200gp_qsm* M) {
    b200gp_ctx* c = M->ctx; const int64_t n = M->n; const int ml = M->lo.m, mu = M->up.m;
    BufP ig = qnew(c, (size_t)n);
    QTri lo = tri_new(c, n, ml), up = tri_new(c, n, mu);          // lower = (t, s, ell), upper = (u, v, del)
    BufP lam = qnew(c, (size_t)n);
    qsm::SqInvArgs a{};
    a.n = n; a.ml = ml; a.mu = mu; a.d = M->d->p;
    a.p = M->lo.p->p; a.q = M->lo.q->p; a.a = M->lo.a->p; a.h = M->up.p->p; a.g = M->up.q->p; a.b = M->up.a->p;
    a.ig = ig->p; a.s = lo.q->p; a.ell = lo.a->p; a.v = up.q->p; a.del = up.a->p;
    a.lam = lam->p; a.t = lo.p->p; a.u = up.p->p;
    const int wsd = qsm::sqinv_smem_doubles(ml, mu);
    run_single<qsm::SqInvArgs, qsm::sqinv_forward>(c, a, wsd);
    run_single<qsm::SqInvArgs, qsm::sqinv_backward>(c, a, wsd);
    std::unique_ptr<b200gp_qsm> r(q_new(c, n));
    r->d = lam; r->lo = lo; r->up = up;
    return r.release();
}

// =========================================================================================================================
extern "C" {

int b200gp_qsm_create(b200gp_ctx* ctx, int64_t n, int kind, int ml, int mu, const double* d, const double* lp, const double* lq,
                      const double* la, const double* up, const double* uq, const double* ua, b200gp_qsm** out) {
    API_BEGIN(ctx)
    if (n <= 0) throw GpError("qsm_create: n must be positive");
    const bool wd = kind == B200GP_QSM_DIAG || kind >= B200GP_QSM_LOWER;
    const bool wl = kind == B200GP_QSM_STRICT_LOWER || kind == B200GP_QSM_LOWER || kind == B200GP_QSM_SQUARE || kind == B200GP_QSM_SYMM;
    const bool wu = kind == B200GP_QSM_STRICT_UPPER || kind == B200GP_QSM_UPPER || kind == B200GP_QSM_SQUARE;
    if (kind < 0 || kind > B200GP_QSM_SYMM) throw GpError("qsm_create: unknown kind");
    if ((wd && !d) || (wl && (!lp || !lq || !la || ml <= 0)) || (wu && (!up || !uq || !ua || mu <= 0)))
        throw GpError("qsm_create: missing generator arrays for this kind");
    std::unique_ptr<b200gp_qsm> r(q_new(_ctx, n));
    if (wd) { r->d = qnew(_ctx, (size_t)n); q_h2d(_ctx, r->d->p, d, (size_t)n); }
    if (wl) {
        r->lo = tri_new(_ctx, n, ml);
        q_h2d(_ctx, r->lo.p->p, lp, (size_t)n * ml); q_h2d(_ctx, r->lo.q->p, lq, (size_t)n * ml); q_h2d(_ctx, r->lo.a->p, la, (size_t)n * ml * ml);
    }
    if (wu) {
        r->up = tri_new(_ctx, n, mu);
        q_h2d(_ctx, r->up.p->p, up, (size_t)n * mu); q_h2d(_ctx, r->up.q->p, uq, (size_t)n * mu); q_h2d(_ctx, r->up.a->p, ua, (size_t)n * mu * mu);
    }
    r->symm = (kind == B200GP_QSM_SYMM);
    *out = r.release();
    API_END
}

int b200gp_qsm_free(b200gp_qsm* q) {
    if (!q) return 0;
    API_BEGIN(q->ctx)
    delete q;
    API_END
}

int b200gp_qsm_info(b200gp_qsm* q, int64_t* n, int* kind, int* ml, int* mu) {
    API_BEGIN(q->ctx)
    if (n) *n = q->n;
    if (kind) *kind = q->kind();
    if (ml) *ml = q->lo.m;
    if (mu) *mu = q->up.m;
    API_END
}

int b200gp_qsm_get(b200gp_qsm* q, double* d, double* lp, double* lq, double* la, double* up, double* uq, double* ua) {
    API_BEGIN(q->ctx)
    const int64_t n = q->n;
    if (d) { if (!q->d) throw GpError("qsm_get: no diagonal"); q_d2h(_ctx, d, q->d->p, (size_t)n); }
    if (lp || lq || la) {
        if (!q->lo.present()) throw GpError("qsm_get: no strictly lower part");
        const int m = q->lo.m;
        if (lp) q_d2h(_ctx, lp, q->lo.p->p, (size_t)n * m);
        if (lq) q_d2h(_ctx, lq, q->lo.q->p, (size_t)n * m);
        if (la) q_d2h(_ctx, la, q->lo.a->p, (size_t)n * m * m);
    }
    if (up || uq || ua) {
        if (!q->up.present()) throw GpError("qsm_get: no strictly upper part");
        const int m = q->up.m;
        if (up) q_d2h(_ctx, up, q->up.p->p, (size_t)n * m);
        if (uq) q_d2h(_ctx, uq, q->up.q->p, (size_t)n * m);
        if (ua) q_d2h(_ctx, ua, q->up.a->p, (size_t)n * m * m);
    }
    API_END
}

// which: 0 diag (DiagQSM), 1 lower (StrictLowerTriQSM), 2 upper (StrictUpperTriQSM); shares the device arrays
int b200gp_qsm_part(b200gp_qsm* q, int which, b200gp_qsm** out) {
    API_BEGIN(q->ctx)
    std::unique_ptr<b200gp_qsm> r(q_new(_ctx, q->n));
    if (which == 0) { if (!q->d) throw GpError("qsm_part: no diagonal"); r->d = q->d; }
    else if (which == 1) { if (!q->lo.present()) throw GpError("qsm_part: no strictly lower part"); r->lo = q->lo; }
    else if (which == 2) { if (!q->upper().present()) throw GpError("qsm_part: no strictly upper part"); r->up = q->upper(); }
    else throw GpError("qsm_part: which must be 0, 1 or 2");
    *out = r.release();
    API_END
}

// LowerTriQSM(diag=, lower=), UpperTriQSM(diag=, upper=), SquareQSM(diag=, lower=, upper=), SymmQSM(diag=, lower=): parts shared
int b200gp_qsm_compose(b200gp_qsm* diag, b200gp_qsm* lower, b200gp_qsm* upper, int symm, b200gp_qsm** out) {
    b200gp_qsm* any = diag ? diag : (lower ? lower : upper);
    if (!any) return 1;
    API_BEGIN(any->ctx)
    std::unique_ptr<b200gp_qsm> r(q_new(_ctx, any->n));
    if (diag) { if (!diag->d || diag->n != r->n) throw GpError("qsm_compose: bad diagonal"); r->d = diag->d; }
    if (lower) { if (!lower->lo.present() || lower->n != r->n) throw GpError("qsm_compose: bad lower part"); r->lo = lower->lo; }
    if (upper) { if (!upper->up.present() || upper->n != r->n) throw GpError("qsm_compose: bad upper part"); r->up = upper->up; }
    if (symm) { if (!diag || !lower || upper) throw GpError("qsm_compose: SymmQSM takes diag and lower"); r->symm = 1; }
    if (r->kind() < 0) throw GpError("qsm_compose: not a QSM type");
    *out = r.release();
    API_END
}

int b200gp_qsm_transpose(b200gp_qsm* q, b200gp_qsm** out) {
    API_BEGIN(q->ctx)
    *out = op_transpose(q);
    API_END
}

// core.py scale(): d * c, lower p * c, upper q * c  (c: one scalar, or n per-row factors when is_vector)
int b200gp_qsm_scale(b200gp_qsm* q, const double* cvals, int is_vector, b200gp_qsm** out) {
    API_BEGIN(q->ctx)
    const int64_t n = q->n;
    BufP s;
    double alpha = 1.0;
    if (is_vector) { s = qnew(_ctx, (size_t)n); q_h2d(_ctx, s->p, cvals, (size_t)n); }
    else alpha = cvals[0];
    std::unique_ptr<b200gp_qsm> r(q_new(_ctx, n));
    r->symm = q->symm;
    if (q->d) { r->d = qnew(_ctx, (size_t)n); blk(_ctx, n, r->d->p, 1, 1, 0, 0, q->d->p, 1, 1, s ? s->p : nullptr, alpha); }
    if (q->lo.present()) {
        r->lo = q->lo; r->lo.p = qnew(_ctx, (size_t)n * q->lo.m);
        blk(_ctx, n, r->lo.p->p, 1, q->lo.m, 0, 0, q->lo.p->p, 1, q->lo.m, s ? s->p : nullptr, alpha);
    }
    if (q->up.present()) {
        r->up = q->up; r->up.q = qnew(_ctx, (size_t)n * q->up.m);
        blk(_ctx, n, r->up.q->p, 1, q->up.m, 0, 0, q->up.q->p, 1, q->up.m, s ? s->p : nullptr, alpha);
    }
    *out = r.release();
    API_END
}

// core.py __neg__: -d, lower -p, upper -p
int b200gp_qsm_neg(b200gp_qsm* q, b200gp_qsm** out) {
    API_BEGIN(q->ctx)
    const int64_t n = q->n;
    std::unique_ptr<b200gp_qsm> r(q_new(_ctx, n));
    r->symm = q->symm;
    if (q->d) r->d = vec_new(_ctx, n, q->d->p, nullptr, -1.0, 0, 0);
    if (q->lo.present()) { r->lo = q->lo; r->lo.p = qnew(_ctx, (size_t)n * q->lo.m); vec(_ctx, n * q->lo.m, r->lo.p->p, q->lo.p->p, nullptr, -1.0, 0, 0); }
    if (q->up.present()) { r->up = q->up; r->up.p = qnew(_ctx, (size_t)n * q->up.m); vec(_ctx, n * q->up.m, r->up.p->p, q->up.p->p, nullptr, -1.0, 0, 0); }
    *out = r.release();
    API_END
}

int b200gp_qsm_add(b200gp_qsm* a, b200gp_qsm* b, b200gp_qsm** out) {
    API_BEGIN(a->ctx)
    if (a->n != b->n) throw GpError("qsm_add: dimension mismatch");
    *out = op_add(a, b);
    API_END
}

int b200gp_qsm_elementwise_mul(b200gp_qsm* a, b200gp_qsm* b, b200gp_qsm** out) {
    API_BEGIN(a->ctx)
    if (a->n != b->n) throw GpError("qsm_elementwise_mul: dimension mismatch");
    *out = op_emul(a, b);
    API_END
}

int b200gp_qsm_mul(b200gp_qsm* a, b200gp_qsm* b, b200gp_qsm** out) {
    API_BEGIN(a->ctx)
    *out = op_mul(a, b, false);
    API_END
}

// core.py:424-434: SymmQSM(diag, lower) of transpose() @ self -- the strictly upper part is never computed
int b200gp_qsm_gram(b200gp_qsm* a, b200gp_qsm** out) {
    API_BEGIN(a->ctx)
    std::unique_ptr<b200gp_qsm> t(op_transpose(a));
    *out = op_mul(t.get(), a, true);
    API_END
}

int b200gp_qsm_inv(b200gp_qsm* a, b200gp_qsm** out) {
    API_BEGIN(a->ctx)
    switch (a->kind()) {
        case B200GP_QSM_LOWER: *out = op_lower_inv(a); break;
        case B200GP_QSM_UPPER: {                                                          // core.py:362-363
            std::unique_ptr<b200gp_qsm> t(op_transpose(a)), ti(op_lower_inv(t.get()));
            *out = op_transpose(ti.get());
        } break;
        case B200GP_QSM_SYMM: *out = op_symm_inv(a); break;
        case B200GP_QSM_DIAG: {
            std::unique_ptr<b200gp_qsm> r(q_new(_ctx, a->n));
            r->d = vec_new(_ctx, a->n, a->d->p, nullptr, 0, 0, 2);
            *out = r.release();
        } break;
        case B200GP_QSM_SQUARE: *out = op_square_inv(a); break;
        default: throw GpError("qsm_inv: a strictly triangular QSM has no inverse");
    }
    API_END
}

// core.py:522-537 -> LowerTriQSM(diag = c, lower = (p, w, a)); *info = 1-based index of the first non-positive pivot, 0 = none
int b200gp_qsm_cholesky(b200gp_qsm* a, b200gp_qsm** out, int64_t* info) {
    API_BEGIN(a->ctx)
    if (!a->symm) throw GpError("qsm_cholesky: needs a SymmQSM");
    const int64_t n = a->n; const int m = a->lo.m;
    std::unique_ptr<b200gp_qsm> r(q_new(_ctx, n));
    r->d = qnew(_ctx, (size_t)n);
    r->lo = a->lo; r->lo.q = qnew(_ctx, (size_t)n * m);
    qsm::RicArgs ra{};
    ra.n = n; ra.m = m; ra.mode = 0; ra.d = a->d->p; ra.p = a->lo.p->p; ra.q = a->lo.q->p; ra.a = a->lo.a->p;
    ra.o_c = r->d->p; ra.o_w = r->lo.q->p;
    const int64_t bad = run_ric(_ctx, ra);
    if (info) *info = bad;
    *out = r.release();
    API_END
}

// Y (n x nrhs, host, in/out) <- A Y    (core.py matmul of every class; ops.py:308-349)
int b200gp_qsm_matmul(b200gp_qsm* a, double* Y, int64_t nrhs) {
    API_BEGIN(a->ctx)
    const int64_t n = a->n;
    if (nrhs <= 0) return 0;
    BufP x = qnew(_ctx, (size_t)n * nrhs), y = qnew(_ctx, (size_t)n * nrhs);
    q_h2d(_ctx, x->p, Y, (size_t)n * nrhs);
    if (a->d) blk(_ctx, n, y->p, 1, (int)nrhs, 0, 0, x->p, 1, (int)nrhs, a->d->p);
    else q_zero(_ctx, y->p, (size_t)n * nrhs);
    if (a->lo.present()) run_low(_ctx, qsm::LMAT, n, nullptr, a->lo, x->p, y->p, nrhs, nrhs, true);
    if (a->upper().present()) run_low(_ctx, qsm::UMAT, n, nullptr, a->upper(), x->p, y->p, nrhs, nrhs, true);
    q_d2h(_ctx, Y, y->p, (size_t)n * nrhs);
    API_END
}

// Y <- A^-1 Y for a LowerTriQSM (forward substitution, ops.py:463-472) or an UpperTriQSM (backward, ops.py:489-498)
int b200gp_qsm_solve(b200gp_qsm* a, double* Y, int64_t nrhs) {
    API_BEGIN(a->ctx)
    const int64_t n = a->n;
    const int k = a->kind();
    if (k != B200GP_QSM_LOWER && k != B200GP_QSM_UPPER) throw GpError("qsm_solve: needs a LowerTriQSM or an UpperTriQSM");
    if (nrhs <= 0) return 0;
    BufP x = qnew(_ctx, (size_t)n * nrhs), y = qnew(_ctx, (size_t)n * nrhs);
    q_h2d(_ctx, x->p, Y, (size_t)n * nrhs);
    if (k == B200GP_QSM_LOWER) run_low(_ctx, qsm::LSOL, n, a->d->p, a->lo, x->p, y->p, nrhs, nrhs, false);
    else run_low(_ctx, qsm::USOL, n, a->d->p, a->up, x->p, y->p, nrhs, nrhs, false);
    q_d2h(_ctx, Y, y->p, (size_t)n * nrhs);
    API_END
}

// sum_k log d_k (solver.py:90-93 on a LowerTriQSM factor): fixed-shape two-stage reduction on the device (deterministic:
// QSM_LOGSUM_SLABS contiguous slabs, each summed by one block's fixed tree; the 256 slab sums are added in index order)
int b200gp_qsm_sum_log_diag(b200gp_qsm* a, double* out) {
    API_BEGIN(a->ctx)
    if (!a->d) throw GpError("qsm_sum_log_diag: no diagonal");
    BufP part = qnew(_ctx, QSM_LOGSUM_SLABS);
    qsm_logsum(_ctx, a->d->p, a->n, part->p);
    double h[QSM_LOGSUM_SLABS];
    q_d2h(_ctx, h, part->p, QSM_LOGSUM_SLABS);
    double s = 0.0;
    for (int i = 0; i < QSM_LOGSUM_SLABS; ++i) s += h[i];
    *out = s;
    API_END
}

#ifdef QSM_HOSTCHECK
int b200gp_create(int, void*, b200gp_ctx** out) { *out = new b200gp_ctx(); return 0; }
int b200gp_destroy(b200gp_ctx* c) { delete c; return 0; }
const char* b200gp_last_error(b200gp_ctx* c) { return c->err.c_str(); }
int b200gp_set_option(b200gp_ctx* c, const char* key, int64_t v) {
    if (!strcmp(key, "qsm_chunk")) { c->qsm_chunk = v; return 0; }
    if (!strcmp(key, "reset")) { c->qsm_chunk = 0; return 0; }
    c->err = "unknown option"; return 2;
}
int b200gp_get_option(b200gp_ctx* c, const char* key, int64_t* v) {
    if (!strcmp(key, "qsm_chunk")) { *v = c->qsm_chunk; return 0; }
    if (!strcmp(key, "qsm_sequential_redos")) { *v = c->qsm_sequential_redos; return 0; }
    c->err = "unknown option"; return 2;
}
#endif

}  // extern "C"

#ifndef QSM_HOSTCHECK
// ---- bridges from the model-based solver (quasisep.cu) ----------------------------------------------------------------
// device buffers of a new SymmQSM (symm = 1) or LowerTriQSM (symm = 0) of order m, for quasisep.cu to fill in place
extern "C" b200gp_qsm* qsm_alloc_for_solver(b200gp_ctx* ctx, int64_t n, int m, int symm, double** d, double** p, double** q, double** a) {
    std::unique_ptr<b200gp_qsm> r(q_new(ctx, n));
    r->d = qnew(ctx, (size_t)n);
    r->lo = tri_new(ctx, n, m);
    r->symm = symm;
    *d = r->d->p; *p = r->lo.p->p; *q = r->lo.q->p; *a = r->lo.a->p;
    return r.release();
}
#endif
