// Layout-specialised quasiseparable kernels (qs_fast.cuh) and their driver: Cholesky chunk fold -> tree -> replay with the
// fused forward substitution (+ the per-chunk quadratic sums) -> tree -> one small finishing kernel.
// Reference behaviour: src/tinygp/solvers/quasisep/solver.py:73-82 (factor) and src/tinygp/gp.py:313-320 (log-probability).
#include "qs_tree.cuh"
#include "qs_fast.cuh"

// MINB: minimum resident blocks per SM asked of the compiler (register cap 65536 / (128 * MINB)): the fold / replay bodies
// want ~154 / ~222 registers, i.e. 3 / 2 blocks = 12 / 8 warps per SM; MINB = 4 / 3 trades ~100 bytes of spills per thread
// for 16 / 12 warps.
template <int L, int MINB>
__global__ void __launch_bounds__(QS_THREADS, MINB) qsf_chunk_kernel(const __grid_constant__ QsModel m, const __grid_constant__ QsFastConst fc,
                                                               const double* __restrict__ t, const double* __restrict__ diag,
                                                               int64_t n, double* comp, int64_t nchunks) {
    const int64_t ch = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (ch < nchunks) qsf_chunk_body<L>(m, fc, t, diag, n, comp, nchunks, ch);
}
template <int L, int MINB>
__global__ void __launch_bounds__(QS_THREADS, MINB) qsf_replay_kernel(const __grid_constant__ QsModel m, const __grid_constant__ QsFastConst fc,
                                                                const double* __restrict__ t, const double* __restrict__ diag,
                                                                int64_t n, const double* fstart, int64_t nchunks, double* c_out,
                                                                double* w_out, double* logc_part, int* info,
                                                                const double* __restrict__ x_fuse, double* aff_comp, double* quad) {
    const int64_t ch = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (ch < nchunks) qsf_replay_body<L>(m, fc, t, diag, n, fstart, nchunks, c_out, w_out, logc_part, info, x_fuse, aff_comp, quad, ch);
}
template <int L>
__global__ void __launch_bounds__(QS_THREADS) qsf_solvesq_kernel(const __grid_constant__ QsModel m, const __grid_constant__ QsFastConst fc,
                                                                 const double* __restrict__ t, const double* __restrict__ c,
                                                                 const double* __restrict__ w, const double* __restrict__ x,
                                                                 int64_t n, double* aff_comp, double* quad, int64_t nchunks) {
    const int64_t ch = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (ch < nchunks) qsf_solvesq_body<L>(m, fc, t, c, w, x, n, aff_comp, quad, nchunks, ch);
}
template <int J>
__global__ void __launch_bounds__(256) qsf_finish_kernel(const double* quad, const double* gstart, int64_t nchunks, double* part) {
    const int64_t ch = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (ch < nchunks) part[ch] = qsf_quad_eval<J>(quad, gstart, nchunks, ch);
}

// factor (c, w, sum log c, info) and -- with x_fuse -- sum of squares of the forward substitution L^-1 x, all on the stream
template <int L>
void qsf_run(b200gp_qs* s, const double* t, const double* diag, int* info_dev, double* logdet_dev, const double* x_fuse,
             double* sumsq_dev) {
    constexpr int J = lay_J(L);
    b200gp_ctx* ctx = s->ctx;
    const int64_t n = s->n, nch = (n + s->model.chunk - 1) / s->model.chunk;
    const QsFastConst fc = qsf_constants(s->model);
    Scratch comp(ctx, (size_t)Riccati<J>::SIZE * nch * 8), fstart(ctx, (size_t)J * J * nch * 8), part(ctx, (size_t)nch * 8);
    // option "qs_occupancy" = 1 (default): register-capped variants (more resident warps); compiled for the C4 layout only
    const bool capped = (L == 10) && ctx->qs_occupancy != 0;
    if (capped) qsf_chunk_kernel<L, (L == 10) ? 4 : 1><<<nblk(nch, QS_THREADS), QS_THREADS, 0, ctx->stream>>>(s->model, fc, t, diag, n, comp.f64(), nch);
    else qsf_chunk_kernel<L, 1><<<nblk(nch, QS_THREADS), QS_THREADS, 0, ctx->stream>>>(s->model, fc, t, diag, n, comp.f64(), nch);
    ctx->launches++;
    run_tree<Riccati<J>>(ctx, comp.f64(), nch, fstart.f64());
    const bool fuse = (x_fuse != nullptr);
    Scratch acomp(ctx, fuse ? (size_t)Affine<J>::SIZE * nch * 8 : 8), quad(ctx, fuse ? (size_t)QsfQuad<J>::SIZE * nch * 8 : 8);
    if (capped)
        qsf_replay_kernel<L, (L == 10) ? 3 : 1><<<nblk(nch, QS_THREADS), QS_THREADS, 0, ctx->stream>>>(
            s->model, fc, t, diag, n, fstart.f64(), nch, s->c, s->w, part.f64(), info_dev, x_fuse, fuse ? acomp.f64() : nullptr,
            fuse ? quad.f64() : nullptr);
    else
        qsf_replay_kernel<L, 1><<<nblk(nch, QS_THREADS), QS_THREADS, 0, ctx->stream>>>(
            s->model, fc, t, diag, n, fstart.f64(), nch, s->c, s->w, part.f64(), info_dev, x_fuse, fuse ? acomp.f64() : nullptr,
            fuse ? quad.f64() : nullptr);
    ctx->launches++;
    sum_partials(ctx, part.f64(), nch, logdet_dev);
    if (fuse) {
        Scratch gstart(ctx, (size_t)J * nch * 8);
        run_tree<Affine<J>>(ctx, acomp.f64(), nch, gstart.f64());
        qsf_finish_kernel<J><<<nblk(nch, 256), 256, 0, ctx->stream>>>(quad.f64(), gstart.f64(), nch, part.f64());
        ctx->launches++;
        sum_partials(ctx, part.f64(), nch, sumsq_dev);
    }
    CUDA_CHECK(cudaGetLastError());
}

template <int L>
void qsf_solvesq_run(b200gp_qs* s, const double* x, double* sumsq_dev) {
    constexpr int J = lay_J(L);
    b200gp_ctx* ctx = s->ctx;
    const int64_t n = s->n, nch = (n + s->model.chunk - 1) / s->model.chunk;
    const QsFastConst fc = qsf_constants(s->model);
    Scratch acomp(ctx, (size_t)Affine<J>::SIZE * nch * 8), quad(ctx, (size_t)QsfQuad<J>::SIZE * nch * 8);
    Scratch gstart(ctx, (size_t)J * nch * 8), part(ctx, (size_t)nch * 8);
    qsf_solvesq_kernel<L><<<nblk(nch, QS_THREADS), QS_THREADS, 0, ctx->stream>>>(s->model, fc, s->t, s->c, s->w, x, n,
                                                                                 acomp.f64(), quad.f64(), nch);
    ctx->launches++;
    run_tree<Affine<J>>(ctx, acomp.f64(), nch, gstart.f64());
    qsf_finish_kernel<J><<<nblk(nch, 256), 256, 0, ctx->stream>>>(quad.f64(), gstart.f64(), nch, part.f64());
    ctx->launches++;
    sum_partials(ctx, part.f64(), nch, sumsq_dev);
    CUDA_CHECK(cudaGetLastError());
}

#ifdef QSF_PART_LAYOUTS
// an instantiation unit (qs_fast_p*.cu): the kernels of a few layouts, so that the layouts compile in parallel
#define X(code)                                                                                                           \
    template void qsf_run<code>(b200gp_qs*, const double*, const double*, int*, double*, const double*, double*);         \
    template void qsf_solvesq_run<code>(b200gp_qs*, const double*, double*);
QSF_PART_LAYOUTS(X)
#undef X
#else
#define X(code)                                                                                                           \
    extern template void qsf_run<code>(b200gp_qs*, const double*, const double*, int*, double*, const double*, double*);  \
    extern template void qsf_solvesq_run<code>(b200gp_qs*, const double*, double*);
QSF_LAYOUTS(X)
#undef X

// |L^-1 x|^2 for an existing factor; false if the layout is not compiled in
bool qsf_solve_sumsq(b200gp_qs* s, const double* x_dev, double* sumsq_dev) {
    switch (qsf_layout_of(s->model)) {
#define X(code) case code: qsf_solvesq_run<code>(s, x_dev, sumsq_dev); return true;
        QSF_LAYOUTS(X)
#undef X
        default: return false;
    }
}

bool qsf_supported(const QsModel& m) {
    const int L = qsf_layout_of(m);
    switch (L) {
#define X(code) case code: return true;
        QSF_LAYOUTS(X)
#undef X
        default: return false;
    }
}

// returns false if the model's layout has no specialised kernels (the caller falls back to the generic path)
bool qsf_factor(b200gp_qs* s, const double* t, const double* diag, int* info_dev, double* logdet_dev, const double* x_fuse,
                double* sumsq_dev) {
    const int L = qsf_layout_of(s->model);
    switch (L) {
#define X(code) case code: qsf_run<code>(s, t, diag, info_dev, logdet_dev, x_fuse, sumsq_dev); return true;
        QSF_LAYOUTS(X)
#undef X
        default: return false;
    }
}
#endif
