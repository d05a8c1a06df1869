// QuasisepSolver path for sm_90a: the celerite recursions as chunked three-phase scans.
//
// Reference behaviour being replaced: src/tinygp/solvers/quasisep/solver.py:35-139,
// src/tinygp/solvers/quasisep/ops.py:308-365,463-512 (sequential scans; the parallel forms :319-399,
// :475-512 are the algebra the chunk composites come from), src/tinygp/kernels/quasisep.py:102-116
// (generators) and :343-673 (state-space models).
//
// Scheme (every scan): one thread owns a chunk of CHUNK consecutive points and
//   (1) folds its chunk into a composite starting from the identity,
//   (2) a small tree (fan-in TREE_R) combines chunk composites and hands each chunk the state at
//       its left edge,
//   (3) the thread replays its chunk from that state with the *sequential reference recursion*,
//       so emitted values follow ops.py:354-361 / :465-468 operation for operation.
// Generators (a_k, p_k) are recomputed in registers from t[k] - t[k-1]; q and the kernel part of d
// are constants of the model.  Cholesky composites are the (A, F, G) triples of ops.py:368-385; since
// each point is a rank-one element the in-chunk fold needs no linear solve:
//     u = F p, s = d - p.u, v = A^T p, w = q - a u
//     F <- a F a^T + w w^T / s,   A <- a A - w v^T / s,   G <- G - v v^T / s
// HBM traffic per point: read t, diag (and y) ; write c, w  -- 8(3 + 1 + J) bytes for log_probability.
#include "qs_generic.cuh"

QS_FOR_J(extern template, 4)      // quasisep_j4.cu
QS_FOR_J(extern template, 5)      // quasisep_j5.cu
QS_FOR_J(extern template, 6)      // quasisep_j6.cu
QS_FOR_J(extern template, 7)      // quasisep_j7.cu
QS_FOR_J(extern template, 8)      // quasisep_j8.cu

// misc kernels -----------------------------------------------------------------------------------
__global__ void sorted_check_kernel(const double* t, int64_t n, int* flag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i + 1 < n && (t[i + 1] - t[i]) < 0.0) atomicOr(flag, 1);  // np.any(np.diff(X) < 0.0)
}
__global__ void searchsorted_kernel(const double* a, int64_t n, const double* v, int64_t m, int64_t* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const double x = v[i];
    int64_t lo = 0, hi = n;  // first index with a[idx] > x   (side="right")
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] <= x) lo = mid + 1; else hi = mid;
    }
    out[i] = lo - 1;
}
__global__ void add_const_kernel(const double* in, double c0, double* out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i] + c0;
}
__global__ void strided_gather_kernel(const double* src, int64_t stride, int64_t off, double* dst, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i * stride + off];
}
__global__ void strided_scatter_kernel(const double* src, double* dst, int64_t stride, int64_t off, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i * stride + off] = src[i];
}

#define QS_DISPATCH_J(Jv, CALL)                                          \
    switch (Jv) {                                                        \
        case 1: { constexpr int JJ = 1; CALL; } break;                   \
        case 2: { constexpr int JJ = 2; CALL; } break;                   \
        case 3: { constexpr int JJ = 3; CALL; } break;                   \
        case 4: { constexpr int JJ = 4; CALL; } break;                   \
        case 5: { constexpr int JJ = 5; CALL; } break;                   \
        case 6: { constexpr int JJ = 6; CALL; } break;                   \
        case 7: { constexpr int JJ = 7; CALL; } break;                   \
        case 8: { constexpr int JJ = 8; CALL; } break;                   \
        default: throw GpError("quasisep: state dimension > 8 is not compiled in"); \
    }

static void qs_affine(b200gp_qs* s, int op, const double* x, double* out, double* sumsq_dev) {
    ProfTimer tm(s->ctx, &s->ctx->prof.qs_ms);
    s->ctx->prof.qs_launches++;
    s->ctx->prof.qs_bytes += 8.0 * (double)s->n * (3.0 + 2.0 * (1.0 + s->J));  // 2 passes read t,c,w,x ; write out
    switch (op) {
        case OP_LOWER_SOLVE: QS_DISPATCH_J(s->J, (qs_affine_J<JJ, OP_LOWER_SOLVE>(s, x, out, sumsq_dev))) break;
        case OP_UPPER_SOLVE: QS_DISPATCH_J(s->J, (qs_affine_J<JJ, OP_UPPER_SOLVE>(s, x, out, sumsq_dev))) break;
        case OP_LOWER_DOT: QS_DISPATCH_J(s->J, (qs_affine_J<JJ, OP_LOWER_DOT>(s, x, out, sumsq_dev))) break;
        case OP_SYMM_LOWER: QS_DISPATCH_J(s->J, (qs_affine_J<JJ, OP_SYMM_LOWER>(s, x, out, sumsq_dev))) break;
        case OP_SYMM_UPPER: QS_DISPATCH_J(s->J, (qs_affine_J<JJ, OP_SYMM_UPPER>(s, x, out, sumsq_dev))) break;
        case OP_GEN_LOWER: QS_DISPATCH_J(s->J, (qs_affine_J<JJ, OP_GEN_LOWER>(s, x, out, sumsq_dev))) break;
        case OP_GEN_UPPER: QS_DISPATCH_J(s->J, (qs_affine_J<JJ, OP_GEN_UPPER>(s, x, out, sumsq_dev))) break;
        default: throw GpError("quasisep: bad op");
    }
}


static void qs_destroy(b200gp_qs* s) {
    if (!s) return;
    b200gp_ctx* ctx = s->ctx;
    const size_t nb = (size_t)s->n * 8;
    if (s->t && s->owns_inputs) ctx->release(s->t, nb);
    if (s->diag && s->owns_inputs) ctx->release(s->diag, nb);
    if (s->c) ctx->release(s->c, nb);
    if (s->w) ctx->release(s->w, nb * s->J);
    if (s->fused_comp) ctx->release(s->fused_comp, s->fused_comp_bytes);
    delete s;
}

static bool qs_is_unsorted(b200gp_ctx* ctx, const double* t_dev, int64_t n) {
    int* flag = (int*)ctx->alloc(sizeof(int));
    CUDA_CHECK(cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream));
    if (n > 1) {
        sorted_check_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(t_dev, n, flag);
        ctx->launches++;
    }
    int h = 0;
    CUDA_CHECK(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->release(flag, sizeof(int));
    return h != 0;
}

// t / diag may be host or device pointers
static b200gp_qs* qs_create_impl(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t, int64_t n,
                                 const double* diag, int assume_sorted, int* unsorted, const double* x_fuse_dev = nullptr,
                                 bool borrow_device_inputs = false) {
    if (n <= 0) throw GpError("quasisep: n must be positive");
    QsModel model = build_model(comps, ncomp);
    b200gp_qs* s = new b200gp_qs();
    s->ctx = ctx;
    s->n = n;
    s->J = model.J;
    s->model = model;
    s->model.chunk = (int)ctx->qs_chunk;
    if (ctx->qs_chunk == 0) {
        // auto: the scan kernels are chains of dependent fp64 work per thread, so a launch costs (number of waves) x (chunk
        // length); pick the multiple of 4 in [48, qs_chunk_max] that minimises it for 3 resident 128-thread blocks per SM.
        // On ties the LONGER chunk wins: same point-wise time, fewer chunk composites for the scan over them.
        const int64_t per_wave = 3 * (int64_t)ctx->num_sms;
        int best = 64;
        int64_t best_cost = INT64_MAX;
        const int cmax = (int)((ctx->qs_chunk_max >= 48) ? ctx->qs_chunk_max : 128);
        for (int c = 48; c <= cmax; c += 4) {
            const int64_t nblocks = ((n + c - 1) / c + QS_THREADS - 1) / QS_THREADS;
            const int64_t cost = ((nblocks + per_wave - 1) / per_wave) * c;
            if (cost <= best_cost) { best_cost = cost; best = c; }
        }
        s->model.chunk = best;
    }
    try {
        const size_t nb = (size_t)n * 8;
        if (borrow_device_inputs && qs_is_device_ptr(t) && qs_is_device_ptr(diag)) {
            // transient object of the fused log-probability: read the caller's device buffers in place (no 16 B/point copy)
            s->owns_inputs = false;
            s->t = const_cast<double*>(t);
            s->diag = const_cast<double*>(diag);
        } else {
            s->t = (double*)ctx->alloc(nb);
            s->diag = (double*)ctx->alloc(nb);
            CUDA_CHECK(cudaMemcpyAsync(s->t, t, nb, cudaMemcpyDefault, ctx->stream));
            CUDA_CHECK(cudaMemcpyAsync(s->diag, diag, nb, cudaMemcpyDefault, ctx->stream));
        }
        if (unsorted) *unsorted = 0;
        if (!assume_sorted && qs_is_unsorted(ctx, s->t, n)) {
            if (unsorted) *unsorted = 1;
            qs_destroy(s);
            return nullptr;
        }
        s->c = (double*)ctx->alloc(nb);
        s->w = (double*)ctx->alloc(nb * s->J);
        int* info_dev = (int*)ctx->alloc(sizeof(int));
        double* ld_dev = (double*)ctx->alloc(sizeof(double));
        int big = INT_MAX;
        CUDA_CHECK(cudaMemcpyAsync(info_dev, &big, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        {
            ProfTimer tm(ctx, &ctx->prof.qs_ms);
            ctx->prof.qs_launches++;
            ctx->prof.qs_bytes += 8.0 * (double)n * (2.0 * 2.0 + 1.0 + s->J);  // two passes read t,diag ; write c,w
            Scratch ss_dev(ctx, 8);
            bool fast = false;
            if (ctx->qs_kernel != 0 && qsf_supported(s->model))
                fast = qsf_factor(s, s->t, s->diag, info_dev, ld_dev, x_fuse_dev, ss_dev.f64());
            if (fast) {
                if (x_fuse_dev) {
                    s->has_sumsq = true;
                    CUDA_CHECK(cudaMemcpyAsync(&s->sumsq, ss_dev.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
                }
            } else {
                QS_DISPATCH_J(s->J, (qs_factor_J<JJ>(s, info_dev, ld_dev, x_fuse_dev)))
            }
        }
        CUDA_CHECK(cudaMemcpyAsync(&s->info, info_dev, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(&s->logdet_half, ld_dev, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        if (s->info == INT_MAX) s->info = 0;
        ctx->release(info_dev, sizeof(int));
        ctx->release(ld_dev, sizeof(double));
    } catch (...) {
        qs_destroy(s);
        throw;
    }
    return s;
}

// apply `op` column by column to a host matrix Y (n, nrhs)
static void qs_apply_host(b200gp_qs* s, int op, double* Y, int64_t nrhs, int op2 = -1) {
    b200gp_ctx* ctx = s->ctx;
    const int64_t n = s->n;
    if (nrhs <= 0) throw GpError("quasisep: nrhs must be positive");
    Scratch yh_buf(ctx, (size_t)n * nrhs * 8), x_buf(ctx, (size_t)n * 8), o_buf(ctx, (size_t)n * 8);
    double* const yh = yh_buf.f64();
    double* const x = x_buf.f64();
    double* const o = o_buf.f64();
    CUDA_CHECK(cudaMemcpyAsync(yh, Y, (size_t)n * nrhs * 8, cudaMemcpyHostToDevice, ctx->stream));
    for (int64_t r = 0; r < nrhs; ++r) {
        if (nrhs == 1) {
            CUDA_CHECK(cudaMemcpyAsync(x, yh, (size_t)n * 8, cudaMemcpyDeviceToDevice, ctx->stream));
        } else {
            strided_gather_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(yh, nrhs, r, x, n);
            ctx->launches++;
        }
        qs_affine(s, op, x, o, nullptr);
        if (op2 >= 0) qs_affine(s, op2, x, o, nullptr);
        strided_scatter_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(o, yh, nrhs, r, n);
        ctx->launches++;
    }
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(Y, yh, (size_t)n * nrhs * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
}

static double qs_logp_impl(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t, int64_t n,
                           const double* diag, const double* resid, int assume_sorted, int* unsorted) {
    // the right-hand side: used in place when it already lives on the device
    const bool x_borrowed = qs_is_device_ptr(resid);
    double* x = x_borrowed ? const_cast<double*>(resid) : (double*)ctx->alloc((size_t)n * 8);
    auto release_x = [&]() { if (!x_borrowed) ctx->release(x, (size_t)n * 8); };
    if (!x_borrowed) CUDA_CHECK(cudaMemcpyAsync(x, resid, (size_t)n * 8, cudaMemcpyDefault, ctx->stream));
    b200gp_qs* s = nullptr;
    try {
        s = qs_create_impl(ctx, comps, ncomp, t, n, diag, assume_sorted, unsorted, x, /*borrow_device_inputs=*/true);
    } catch (...) {
        release_x();
        throw;
    }
    if (!s) {
        release_x();
        return NAN;
    }
    double logp;
    try {
        double ss = 0.0;
        if (s->has_sumsq) {
            ss = s->sumsq;   // structured path: forward substitution folded into the factorisation passes
        } else {
            double* o = (double*)ctx->alloc((size_t)n * 8);
            double* ss_dev = (double*)ctx->alloc(8);
            {   // tree + replay only: the chunk composites were accumulated inside the Cholesky replay
                ProfTimer tm(ctx, &ctx->prof.qs_ms);
                ctx->prof.qs_launches++;
                ctx->prof.qs_bytes += 8.0 * (double)n * (4.0 + s->J);
                QS_DISPATCH_J(s->J, (qs_affine_J<JJ, OP_LOWER_SOLVE>(s, x, o, ss_dev, s->fused_comp)))
            }
            CUDA_CHECK(cudaMemcpyAsync(&ss, ss_dev, 8, cudaMemcpyDeviceToHost, ctx->stream));
            CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
            ctx->release(o, (size_t)n * 8);
            ctx->release(ss_dev, 8);
        }
        logp = -0.5 * ss - (s->logdet_half + 0.5 * (double)n * log(2.0 * M_PI));  // gp.py:313-316 ; solver.py:90-93
        if (s->info != 0 || !isfinite(logp)) logp = -INFINITY;
        release_x();
    } catch (...) {
        release_x();
        qs_destroy(s);
        throw;
    }
    qs_destroy(s);
    return logp;
}

// =============================================================================================
// C-ABI: quasisep
// =============================================================================================
extern "C" {

int b200gp_qs_check_sorted(b200gp_ctx* ctx, const double* t, int64_t n, int* unsorted) {
    API_BEGIN(ctx)
    if (n <= 0) throw GpError("check_sorted: empty input");
    double* td = (double*)_ctx->alloc((size_t)n * 8);
    CUDA_CHECK(cudaMemcpyAsync(td, t, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
    *unsorted = qs_is_unsorted(_ctx, td, n) ? 1 : 0;
    _ctx->release(td, (size_t)n * 8);
    API_END
}

int b200gp_qs_create(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t, int64_t n, const double* diag,
                     int assume_sorted, b200gp_qs** out, int* unsorted, int* info) {
    API_BEGIN(ctx)
    *out = nullptr;
    b200gp_qs* s = qs_create_impl(_ctx, comps, ncomp, t, n, diag, assume_sorted, unsorted);
    *out = s;
    if (info) *info = s ? s->info : 0;
    API_END
}

int b200gp_qs_create_dev(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t_dev, int64_t n,
                         const double* diag_dev, int assume_sorted, b200gp_qs** out, int* unsorted, int* info) {
    return b200gp_qs_create(ctx, comps, ncomp, t_dev, n, diag_dev, assume_sorted, out, unsorted, info);
}

/* sum of squares of L^-1 y (gp.py:313-316: -0.5 * sum(alpha^2)) without bringing alpha back to the host */
int b200gp_qs_solve_sumsq(b200gp_qs* s, const double* y, double* out) {
    API_BEGIN(s->ctx)
    const int64_t n = s->n;
    Scratch x(_ctx, (size_t)n * 8), ss(_ctx, 8);
    CUDA_CHECK(cudaMemcpyAsync(x.p, y, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
    bool done = false;
    {
        ProfTimer tm(_ctx, &_ctx->prof.qs_ms);
        if (_ctx->qs_kernel != 0) done = qsf_solve_sumsq(s, x.f64(), ss.f64());
    }
    if (!done) {
        Scratch o(_ctx, (size_t)n * 8);
        qs_affine(s, OP_LOWER_SOLVE, x.f64(), o.f64(), ss.f64());
    }
    CUDA_CHECK(cudaMemcpyAsync(out, ss.p, 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

int b200gp_qs_free(b200gp_qs* s) {
    if (!s) return 0;
    API_BEGIN(s->ctx)
    qs_destroy(s);
    API_END
}

int b200gp_qs_state_dim(b200gp_qs* s, int* J) {
    API_BEGIN(s->ctx)
    *J = s->J;
    API_END
}

int b200gp_qs_logdet_half(b200gp_qs* s, double* out) {
    API_BEGIN(s->ctx)
    *out = (s->info != 0) ? NAN : s->logdet_half;
    API_END
}

int b200gp_qs_variance(b200gp_qs* s, double* out) {
    API_BEGIN(s->ctx)
    double* o = (double*)_ctx->alloc((size_t)s->n * 8);
    add_const_kernel<<<nblk(s->n, 256), 256, 0, _ctx->stream>>>(s->diag, s->model.d0, o, s->n);
    _ctx->launches++;
    CUDA_CHECK(cudaMemcpyAsync(out, o, (size_t)s->n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    _ctx->release(o, (size_t)s->n * 8);
    API_END
}

int b200gp_qs_get_factor(b200gp_qs* s, double* c, double* w) {
    API_BEGIN(s->ctx)
    CUDA_CHECK(cudaMemcpyAsync(c, s->c, (size_t)s->n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(w, s->w, (size_t)s->n * s->J * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

int b200gp_qs_get_generators(b200gp_qs* s, double* d, double* p, double* q, double* a) {
    API_BEGIN(s->ctx)
    const int64_t n = s->n;
    const int J = s->J;
    double* dd = (double*)_ctx->alloc((size_t)n * 8);
    double* pd = (double*)_ctx->alloc((size_t)n * J * 8);
    double* qd = (double*)_ctx->alloc((size_t)n * J * 8);
    double* ad = (double*)_ctx->alloc((size_t)n * J * J * 8);
    QS_DISPATCH_J(J, (qs_generators_J<JJ>(_ctx, s->model, s->t, s->diag, n, dd, pd, qd, ad)))
    _ctx->launches++;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(d, dd, (size_t)n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(p, pd, (size_t)n * J * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(q, qd, (size_t)n * J * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(a, ad, (size_t)n * J * J * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    _ctx->release(dd, (size_t)n * 8);
    _ctx->release(pd, (size_t)n * J * 8);
    _ctx->release(qd, (size_t)n * J * 8);
    _ctx->release(ad, (size_t)n * J * J * 8);
    API_END
}

// ---- bridges to the QSM algebra (qsm.cu) ------------------------------------------------------------------------------
b200gp_qsm* qsm_alloc_for_solver(b200gp_ctx* ctx, int64_t n, int m, int symm, double** d, double** p, double** q, double** a);

// Quasisep.to_symm_qsm (kernels/quasisep.py:102-116): the kernel's generators at t, on the device, no noise
int b200gp_qs_kernel_qsm(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t, int64_t n, b200gp_qsm** out) {
    API_BEGIN(ctx)
    if (n <= 0) throw GpError("qs_kernel_qsm: n must be positive");
    const QsModel model = build_model(comps, ncomp);
    const int J = model.J;
    Scratch td(_ctx, (size_t)n * 8);
    CUDA_CHECK(cudaMemcpyAsync(td.p, t, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
    double *d, *p, *q, *a;
    b200gp_qsm* r = qsm_alloc_for_solver(_ctx, n, J, 1, &d, &p, &q, &a);
    try {
        QS_DISPATCH_J(J, (qs_generators_J<JJ>(_ctx, model, td.f64(), nullptr, n, d, p, q, a)))
        _ctx->launches++;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));   // t may be the caller's pageable buffer
    } catch (...) {
        b200gp_qsm_free(r);
        throw;
    }
    *out = r;
    API_END
}

// solver.factor (solver.py:82; core.py:524-539): LowerTriQSM(diag = c, lower = (p, w, a)) with p, a regenerated from t
int b200gp_qs_factor_qsm(b200gp_qs* s, b200gp_qsm** out) {
    API_BEGIN(s->ctx)
    const int64_t n = s->n;
    const int J = s->J;
    double *d, *p, *q, *a;
    b200gp_qsm* r = qsm_alloc_for_solver(_ctx, n, J, 0, &d, &p, &q, &a);
    try {
        QS_DISPATCH_J(J, (qs_generators_J<JJ>(_ctx, s->model, s->t, nullptr, n, d, p, q, a)))
        _ctx->launches++;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(d, s->c, (size_t)n * 8, cudaMemcpyDeviceToDevice, _ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(q, s->w, (size_t)n * J * 8, cudaMemcpyDeviceToDevice, _ctx->stream));
    } catch (...) {
        b200gp_qsm_free(r);
        throw;
    }
    *out = r;
    API_END
}

int b200gp_qs_solve_triangular(b200gp_qs* s, double* Y, int64_t nrhs, int transpose) {
    API_BEGIN(s->ctx)
    qs_apply_host(s, transpose ? OP_UPPER_SOLVE : OP_LOWER_SOLVE, Y, nrhs);
    API_END
}

int b200gp_qs_dot_triangular(b200gp_qs* s, double* Y, int64_t nrhs) {
    API_BEGIN(s->ctx)
    qs_apply_host(s, OP_LOWER_DOT, Y, nrhs);
    API_END
}

int b200gp_qs_matmul(b200gp_qs* s, double* Y, int64_t nrhs) {
    API_BEGIN(s->ctx)
    qs_apply_host(s, OP_SYMM_LOWER, Y, nrhs, OP_SYMM_UPPER);
    API_END
}

int b200gp_qs_log_probability(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t, int64_t n,
                              const double* diag, const double* resid, int assume_sorted, int* unsorted, double* logp) {
    API_BEGIN(ctx)
    *logp = qs_logp_impl(_ctx, comps, ncomp, t, n, diag, resid, assume_sorted, unsorted);
    API_END
}

int b200gp_qs_log_probability_dev(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t_dev, int64_t n,
                                  const double* diag_dev, const double* resid_dev, int assume_sorted, int* unsorted,
                                  double* logp) {
    return b200gp_qs_log_probability(ctx, comps, ncomp, t_dev, n, diag_dev, resid_dev, assume_sorted, unsorted, logp);
}

// kernel.matmul(X1, X2, y) for a quasiseparable kernel in O((n + m) J^2): kernels/quasisep.py:147-163
// (to_general_qsm(X1, X2) @ y).  t_train must be sorted; t_test need not be.
int b200gp_qs_kernel_matmul(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t_test, int64_t m,
                            const double* t_train, int64_t n, const double* Y, int64_t nrhs, double* out) {
    API_BEGIN(ctx)
    if (n <= 0 || m <= 0 || nrhs <= 0) throw GpError("qs_kernel_matmul: empty input");
    b200gp_qs s;   // scan-only view: no factor, no noise diagonal
    s.ctx = _ctx;
    s.n = n;
    s.model = build_model(comps, ncomp);
    s.model.chunk = _ctx->qs_chunk ? (int)_ctx->qs_chunk : 64;
    s.J = s.model.J;
    const size_t nb8 = (size_t)n * 8, mb8 = (size_t)m * 8, sb = (size_t)n * s.J * 8;
    Scratch t2_buf(_ctx, nb8), t1_buf(_ctx, mb8), yh_buf(_ctx, nb8 * nrhs), x_buf(_ctx, nb8), F_buf(_ctx, sb), G_buf(_ctx, sb),
        o_buf(_ctx, mb8 * nrhs);
    double* const t2 = t2_buf.f64();
    double* const t1 = t1_buf.f64();
    double* const yh = yh_buf.f64();
    double* const x = x_buf.f64();
    double* const F = F_buf.f64();
    double* const G = G_buf.f64();
    double* const o = o_buf.f64();
    CUDA_CHECK(cudaMemcpyAsync(t2, t_train, nb8, cudaMemcpyDefault, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(t1, t_test, mb8, cudaMemcpyDefault, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(yh, Y, nb8 * nrhs, cudaMemcpyDefault, _ctx->stream));
    s.t = t2;
    for (int64_t r = 0; r < nrhs; ++r) {
        strided_gather_kernel<<<nblk(n, 256), 256, 0, _ctx->stream>>>(yh, nrhs, r, x, n);
        _ctx->launches++;
        qs_affine(&s, OP_GEN_LOWER, x, F, nullptr);
        qs_affine(&s, OP_GEN_UPPER, x, G, nullptr);
        QS_DISPATCH_J(s.J, (qs_general_gather_J<JJ>(_ctx, s.model, t2, n, t1, m, F, G, o + r, nrhs)))
        _ctx->launches++;
    }
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, o, mb8 * nrhs, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    s.t = nullptr;
    API_END
}

// diag((K + N)^-1) in O(n J^3): the diagonal of (factor.inv()).gram() (core.py:310-317, 424-434) by one backward
// scan, without forming the matrix.  With it the conditioned variance at the inputs (solver.py:124-129 followed by
// solver.py:84-85) is  noise* + N - N^2 diag((K + N)^-1)  -- what gp.predict(y, return_var=True) needs at N = 10^7.
int b200gp_qs_inverse_diagonal(b200gp_qs* s, double* out) {
    API_BEGIN(s->ctx)
    if (s->info != 0) throw GpError("qs_inverse_diagonal: the factorisation failed (matrix not positive definite)");
    const size_t nb = (size_t)s->n * 8;
    Scratch o(_ctx, nb);
    {
        ProfTimer tm(_ctx, &_ctx->prof.qs_ms);
        _ctx->prof.qs_launches++;
        _ctx->prof.qs_bytes += 8.0 * (double)s->n * (2.0 * (2.0 + s->J) + 1.0);  // two passes read t, c, w ; write out
        QS_DISPATCH_J(s->J, (qs_inv_diag_J<JJ>(s, o.f64())))
    }
    CUDA_CHECK(cudaMemcpyAsync(out, o.p, nb, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

__global__ void conditioned_variance_kernel(const double* __restrict__ inv_diag, const double* __restrict__ noise,
                                            const double* __restrict__ noise_pred, int64_t n, double* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = noise_pred[i] + (noise[i] - noise[i] * noise[i] * inv_diag[i]);
}

// Variance of the process conditioned on the data, at the inputs, for the solver's own kernel: the diagonal of
// solver.py:124-129 (`M + noise* - (factor.inv() @ M).gram()`) as read by solver.py:84-85.  With Sigma = K + N and
// M = K = Sigma - N:  K - K Sigma^-1 K = N - N Sigma^-1 N, so the diagonal is  noise* + N - N^2 diag(Sigma^-1)  -- one
// backward scan, O(n J^3), no n x n matrix (what gp.predict(y, return_var=True) needs for a 10^7-point series).
int b200gp_qs_conditioned_variance(b200gp_qs* s, const double* noise_pred, double* out) {
    API_BEGIN(s->ctx)
    if (s->info != 0) throw GpError("qs_conditioned_variance: the factorisation failed (matrix not positive definite)");
    const int64_t n = s->n;
    const size_t nb = (size_t)n * 8;
    Scratch o(_ctx, nb), np_(_ctx, nb);
    CUDA_CHECK(cudaMemcpyAsync(np_.p, noise_pred, nb, cudaMemcpyHostToDevice, _ctx->stream));
    {
        ProfTimer tm(_ctx, &_ctx->prof.qs_ms);
        _ctx->prof.qs_launches++;
        _ctx->prof.qs_bytes += 8.0 * (double)n * (2.0 * (2.0 + s->J) + 4.0);
        QS_DISPATCH_J(s->J, (qs_inv_diag_J<JJ>(s, o.f64())))
        conditioned_variance_kernel<<<nblk(n, 256), 256, 0, _ctx->stream>>>(o.f64(), s->diag, np_.f64(), n, o.f64());
        _ctx->launches++;
        CUDA_CHECK(cudaGetLastError());
    }
    CUDA_CHECK(cudaMemcpyAsync(out, o.p, nb, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

// QuasisepSolver.condition, dense branch (solvers/quasisep/solver.py:131-139):  out = Kss - A^T A with
// A = factor.solve(Ks), Ks = k(X, X*), Kss = k(X*, X*).  The reference adds the predictive noise only in its QSM
// branch (:124-129, X* = X with a quasiseparable kernel) and not in the dense branch: the caller passes
// diag_or_null accordingly (m values added to the diagonal, or NULL).
// Everything runs on the device: Ks^T (rows = test points, each row a contiguous n-vector) from the build kernel,
// one forward-substitution scan per row, then the NT GEMM with the k(X*, X*) generator epilogue shared with
// DirectSolver.condition.  `prog` is the predictive kernel lowered for 1-D coordinates; t_test == NULL means X* = X.
int b200gp_qs_condition(b200gp_qs* s, const double* prog, int n_instr, const double* t_test, int64_t m,
                        const double* diag_or_null, double* out) {
    API_BEGIN(s->ctx)
    KProg P = parse_prog(prog, n_instr, 1);
    const int64_t n = s->n;
    if (t_test == nullptr) m = n;
    else if (m <= 0) throw GpError("qs_condition: empty X_test");
    Scratch xt(_ctx, (size_t)m * 8);
    CUDA_CHECK(cudaMemcpyAsync(xt.p, t_test ? t_test : s->t, (size_t)m * 8, cudaMemcpyDefault, _ctx->stream));
    const int64_t mp = ((m + TILE - 1) / TILE) * TILE, kp = ((n + TILE - 1) / TILE) * TILE;
    const size_t ab = (size_t)mp * kp * 8;
    Scratch Kst(_ctx, ab), At(_ctx, ab), dt(_ctx, (size_t)mp * 8);
    CUDA_CHECK(cudaMemsetAsync(dt.p, 0, (size_t)mp * 8, _ctx->stream));
    if (diag_or_null != nullptr)   // solver.py:124-129 adds the noise; the dense branch :131-139 does not
        CUDA_CHECK(cudaMemcpyAsync(dt.p, diag_or_null, (size_t)m * 8, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemsetAsync(At.p, 0, ab, _ctx->stream));   // pad rows / columns of A^T must be zero for the GEMM
    dense_build_rect(_ctx, P, xt.f64(), m, s->t, n, 1, nullptr, Kst.f64(), kp, mp, kp);
    for (int64_t r = 0; r < m; ++r) qs_affine(s, OP_LOWER_SOLVE, Kst.f64() + r * kp, At.f64() + r * kp, nullptr);
    dense_conditioned_covariance_to_host(_ctx, P, At.f64(), mp, kp, xt.f64(), dt.f64(), 1, m, out);
    API_END
}

int b200gp_searchsorted_right_m1(b200gp_ctx* ctx, const double* sorted, int64_t n, const double* query, int64_t m,
                                 int64_t* out) {
    API_BEGIN(ctx)
    if (n <= 0 || m <= 0) throw GpError("searchsorted: empty input");
    double* a = (double*)_ctx->alloc((size_t)n * 8);
    double* v = (double*)_ctx->alloc((size_t)m * 8);
    int64_t* o = (int64_t*)_ctx->alloc((size_t)m * 8);
    CUDA_CHECK(cudaMemcpyAsync(a, sorted, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(v, query, (size_t)m * 8, cudaMemcpyDefault, _ctx->stream));
    searchsorted_kernel<<<nblk(m, 256), 256, 0, _ctx->stream>>>(a, n, v, m, o);
    _ctx->launches++;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, o, (size_t)m * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    _ctx->release(a, (size_t)n * 8);
    _ctx->release(v, (size_t)m * 8);
    _ctx->release(o, (size_t)m * 8);
    API_END
}

}  // extern "C"
