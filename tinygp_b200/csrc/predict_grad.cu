// Gradients of the dense predictive mean and variance with respect to the test inputs (b200gp_dense_predict_grad).
// For the solver's factor L L^T = K, alpha = K^-1 (y - mean) (given by the host), a test point x*_m and
// v_m = K^-1 k(X, x*_m):
//   mu_m  = sum_j k(x*_m, x_j) alpha_j                       d mu_m  / d x*_m = sum_j grad_1 k(x*_m, x_j) alpha_j
//   var_m = k(x*_m, x*_m) + diag*_m - |L^-1 k(X, x*_m)|^2    d var_m / d x*_m = -2 sum_j grad_1 k(x*_m, x_j) v_m,j
// (k(x*, x*) is the same for every x* of a stationary kernel.)
//
// The test points are taken in blocks of at most BLOCK = 4096.  Per block:
// 1. with the variance: At = k(X*, X) (rows = test points, dense_build_rect), At <- At L^-T by the forward substitution
//    of b200gp_dense_condition (same gemm_nt sequence, so the same values), var = k** + diag* - sum_j At_mj^2 per row
//    (one warp per row, fixed order), then Vt = At L^-1 in place by a backward substitution over the block columns of
//    L, from the last to the first:
//        Vt_j <- Vt_j L_jj^-1,   then   Vt_i <- Vt_i - Vt_j L_ji  for every i < j
//    Both are gemm_nt launches; their B operand is the block row j of L (and linv_j in place of its diagonal block)
//    transposed into a 128-wide scratch panel first (row_block_transpose_kernel), an O(np^2) copy in all against the
//    O(np^2 M) flops of the products.
// 2. the contraction (contract_kernel): one thread per test point, one CTA per 128 test points and SLAB = 1024 training
//    points; grad_1 k(x*_m, x_j) comes from kgrad_eval<true> (kgrad.cuh) in registers and is weighted by alpha_j and,
//    with the variance, by Vt_mj in the same pass.  Each CTA writes its per-slab partial sums; reduce_kernel adds them
//    per point and dimension in slab order.  The slabs depend on n only, so a point's outputs do not depend on the
//    other test points of the call, nor on its block.  No floating-point atomics: bitwise reproducible.
#include "common.cuh"
#include "kgrad.cuh"
#include <algorithm>
#include <optional>

namespace pg {
constexpr int THREADS = 128;         // test points per CTA of the contraction
constexpr int CHUNK = 32;            // training points staged in shared memory at a time
constexpr int64_t SLAB = 1024;       // training points per CTA of the contraction (a multiple of CHUNK)
constexpr int64_t BLOCK = 4096;      // test points per block (a multiple of TILE)

struct Args {
    KProg P; KGrad G;
    const double* xt; int64_t m;     // test points of this block, m x ndim
    const double* X; int64_t n;      // training points, n x ndim
    int ndim;
    const double* alpha;             // n
    const double* Vt; int64_t ldv;   // m rows of K^-1 k(X, x*_m), or nullptr (no variance)
    double* part;                    // [slab][mean, var][ndim][mpad]
    int64_t mpad;
};

__global__ void __launch_bounds__(THREADS, 1) contract_kernel(const __grid_constant__ Args g) {
    __shared__ double xs[CHUNK][KGRAD_MAX_DIM], as[CHUNK], vs[THREADS][CHUNK + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t i0 = (int64_t)blockIdx.x * THREADS, i = i0 + tid;
    const int64_t j_begin = (int64_t)blockIdx.y * SLAB, j_end = min(g.n, j_begin + SLAB);
    const int nd = g.ndim;
    const bool with_var = g.Vt != nullptr;
    double xi[KGRAD_MAX_DIM], gm[KGRAD_MAX_DIM], gv[KGRAD_MAX_DIM], gx[KGRAD_MAX_DIM], dk[KGRAD_MAX_SLOTS];
#pragma unroll
    for (int d = 0; d < KGRAD_MAX_DIM; ++d) {
        xi[d] = (i < g.m && d < nd) ? g.xt[i * nd + d] : 0.0;
        gm[d] = gv[d] = 0.0;
    }
    for (int64_t j0 = j_begin; j0 < j_end; j0 += CHUNK) {
        const int cnt = (int)min((int64_t)CHUNK, j_end - j0);
        __syncthreads();
        for (int e = tid; e < CHUNK * nd; e += THREADS) {
            const int jj = e / nd;
            xs[jj][e - jj * nd] = (jj < cnt) ? g.X[(j0 + jj) * nd + e - jj * nd] : 0.0;
        }
        if (tid < CHUNK) as[tid] = (tid < cnt) ? g.alpha[j0 + tid] : 0.0;
        if (with_var)
            for (int r = warp; r < THREADS; r += THREADS / 32)
                vs[r][lane] = (i0 + r < g.m && lane < cnt) ? g.Vt[(i0 + r) * g.ldv + j0 + lane] : 0.0;
        __syncthreads();
        if (i >= g.m) continue;
        for (int jj = 0; jj < cnt; ++jj) {
            kgrad_eval<true>(g.P, g.G, nd, [&](int d) { return xi[d] - xs[jj][d]; }, dk, true, gx);
            const double a = as[jj], v = with_var ? vs[tid][jj] : 0.0;
#pragma unroll
            for (int d = 0; d < KGRAD_MAX_DIM; ++d) {
                gm[d] += a * gx[d];
                gv[d] += v * gx[d];
            }
        }
    }
    if (i >= g.m) return;
    double* p = g.part + (int64_t)blockIdx.y * 2 * nd * g.mpad + i;
#pragma unroll
    for (int d = 0; d < KGRAD_MAX_DIM; ++d)
        if (d < nd) {
            p[(int64_t)d * g.mpad] = gm[d];
            if (with_var) p[(int64_t)(nd + d) * g.mpad] = gv[d];
        }
}

// dmean[i][d] = sum_s partial mean; dvar[i][d] = -2 sum_s partial var (slab order)
__global__ void reduce_kernel(const double* part, int nslab, int nd, int64_t mpad, int64_t m, double* dmean,
                              double* dvar) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * nd) return;
    const int64_t i = e / nd;
    const int d = (int)(e - i * nd);
    double sm = 0.0, sv = 0.0;
    for (int s = 0; s < nslab; ++s) {
        const double* p = part + (int64_t)s * 2 * nd * mpad + i;
        sm += p[(int64_t)d * mpad];
        if (dvar != nullptr) sv += p[(int64_t)(nd + d) * mpad];
    }
    dmean[e] = sm;
    if (dvar != nullptr) dvar[e] = -2.0 * sv;
}

// var[i] = k(x*_i, x*_i) + diag[i] - sum_c At[i][c]^2: one warp per row, lanes over the columns, then a shuffle tree
__global__ void __launch_bounds__(256) variance_kernel(const __grid_constant__ KProg P, const double* At, int64_t ld,
                                                       int nd, const double* diag, int64_t m, double* var) {
    const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= m) return;
    const double* row = At + i * ld;
    double s = 0.0;
    for (int64_t c = lane; c < ld; c += 32) s += row[c] * row[c];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) var[i] = kprog_eval(P, nd, [](int) { return 0.0; }) + diag[i] - s;
}

// R ((j + 1) 128 x 128, row stride TILE): R[c][k] = L[j 128 + k][c] for c < j 128, and linv_j[k][c - j 128] for the
// diagonal block: block row j of L (its diagonal block replaced by its inverse), transposed.  32 x 32 tiles.
__global__ void row_block_transpose_kernel(const double* L, int64_t ld, const double* linv_j, int j, double* R) {
    __shared__ double t[32][33];
    const int64_t c0 = (int64_t)blockIdx.y * 32;      // columns of L = rows of R
    const int k0 = blockIdx.x * 32;                   // rows of block row j = columns of R
    const bool diag = c0 >= (int64_t)j * TILE;
    for (int y = threadIdx.y; y < 32; y += 8) {
        const int k = k0 + y;
        const int64_t c = c0 + threadIdx.x;
        t[y][threadIdx.x] = diag ? linv_j[(int64_t)k * TILE + (c - (int64_t)j * TILE)] : L[((int64_t)j * TILE + k) * ld + c];
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += 8) R[(c0 + y) * TILE + k0 + threadIdx.x] = t[threadIdx.x][y];
}

static inline unsigned nblocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }
}  // namespace pg

extern "C" int b200gp_dense_predict_grad(b200gp_dense* s, const double* prog, int n_instr, const double* Xtest, int64_t m,
                                         const double* alpha, double* dmean, const double* diag_test, double* var,
                                         double* dvar) {
    if (!s) return 1;
    API_BEGIN(s->ctx)
    if (!s->has_prog) throw GpError("predict_grad: solver was built from a precomputed covariance (no coordinates)");
    const int nd = s->ndim;
    if (nd < 1 || nd > KGRAD_MAX_DIM) throw GpError("predict_grad: gradients support 1 to 8 input dimensions");
    if (m <= 0 || Xtest == nullptr || alpha == nullptr || dmean == nullptr) throw GpError("predict_grad: empty X_test or output");
    const bool with_var = diag_test != nullptr;
    if (with_var && (var == nullptr || dvar == nullptr)) throw GpError("predict_grad: variance outputs missing");
    pg::Args g{};
    g.P = parse_prog(prog, n_instr, nd);
    if (!kgrad_prepare(g.P, g.G))
        throw GpError("predict_grad: the kernel program has more than 16 differentiable parameters, or a leaf without "
                      "derivatives (closed forms of quasiseparable kernels)");
    if (s->info > 0) {     // a failed factorisation: NaN, as the factor is from its first bad pivot on
        for (int64_t e = 0; e < m * nd; ++e) dmean[e] = NAN;
        if (with_var)
            for (int64_t e = 0; e < m; ++e) {
                var[e] = NAN;
                for (int d = 0; d < nd; ++d) dvar[e * nd + d] = NAN;
            }
        return 0;
    }
    const int64_t n = s->n, np = s->np;
    const int nblk = (int)(np / TILE);
    const int64_t bmax = std::min(pg::BLOCK, ((m + TILE - 1) / TILE) * TILE);
    const int nslab = (int)((n + pg::SLAB - 1) / pg::SLAB);
    Scratch xt_buf(_ctx, (size_t)m * nd * 8), al_buf(_ctx, (size_t)n * 8);
    Scratch part_buf(_ctx, (size_t)nslab * 2 * nd * bmax * 8);
    Scratch dm_buf(_ctx, (size_t)m * nd * 8);
    std::optional<Scratch> at_buf, r_buf, dt_buf, v_buf, dv_buf;
    if (with_var) {
        at_buf.emplace(_ctx, (size_t)bmax * np * 8);
        r_buf.emplace(_ctx, (size_t)np * TILE * 8);
        dt_buf.emplace(_ctx, (size_t)m * 8);
        v_buf.emplace(_ctx, (size_t)m * 8);
        dv_buf.emplace(_ctx, (size_t)m * nd * 8);
        CUDA_CHECK(cudaMemcpyAsync(dt_buf->p, diag_test, (size_t)m * 8, cudaMemcpyHostToDevice, _ctx->stream));
    }
    CUDA_CHECK(cudaMemcpyAsync(xt_buf.p, Xtest, (size_t)m * nd * 8, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(al_buf.p, alpha, (size_t)n * 8, cudaMemcpyHostToDevice, _ctx->stream));
    g.X = s->X_dev; g.n = n; g.ndim = nd; g.alpha = al_buf.f64(); g.part = part_buf.f64();
    for (int64_t b0 = 0; b0 < m; b0 += pg::BLOCK) {
        const int64_t mb = std::min(pg::BLOCK, m - b0), mp = ((mb + TILE - 1) / TILE) * TILE;
        const int tm = (int)(mp / TILE);
        const double* xb = xt_buf.f64() + b0 * nd;
        double* const At = with_var ? at_buf->f64() : nullptr;
        if (with_var) {
            dense_build_rect(_ctx, g.P, xb, mb, s->X_dev, n, nd, nullptr, At, np, mp, np);
            {   // forward substitution At <- At L^-T: b200gp_dense_condition's sequence
                ProfTimer t(_ctx, &_ctx->prof.solve_ms);
                for (int j = 0; j < nblk; ++j) {
                    double* Aj = At + (int64_t)j * TILE;
                    gemm_nt(_ctx, Aj, np, Aj, np, s->linv + (int64_t)j * TILE * TILE, TILE, tm, 1, TILE, 1.0, 0, 0);
                    if (j + 1 < nblk)
                        gemm_nt(_ctx, Aj + TILE, np, Aj, np, s->mat + (int64_t)(j + 1) * TILE * np + (int64_t)j * TILE, np,
                                tm, nblk - j - 1, TILE, -1.0, 1, 0);
                }
            }
            pg::variance_kernel<<<pg::nblocks(mb, 8), 256, 0, _ctx->stream>>>(g.P, At, np, nd, dt_buf->f64() + b0, mb,
                                                                               v_buf->f64() + b0);
            CUDA_CHECK(cudaGetLastError());
            _ctx->launches++;
            {   // backward substitution Vt = At L^-1 in place
                ProfTimer t(_ctx, &_ctx->prof.bsolve_ms);
                double* const R = r_buf->f64();
                for (int j = nblk - 1; j >= 0; --j) {
                    pg::row_block_transpose_kernel<<<dim3(TILE / 32, (unsigned)((j + 1) * (TILE / 32))), dim3(32, 8), 0,
                                                     _ctx->stream>>>(s->mat, np, s->linv + (int64_t)j * TILE * TILE, j, R);
                    CUDA_CHECK(cudaGetLastError());
                    _ctx->launches++;
                    double* Vj = At + (int64_t)j * TILE;
                    gemm_nt(_ctx, Vj, np, Vj, np, R + (int64_t)j * TILE * TILE, TILE, tm, 1, TILE, 1.0, 0, 0);
                    if (j > 0) gemm_nt(_ctx, At, np, Vj, np, R, TILE, tm, j, TILE, -1.0, 1, 0);
                }
            }
        }
        {
            ProfTimer t(_ctx, &_ctx->prof.contract_ms);
            g.xt = xb; g.m = mb; g.Vt = At; g.ldv = np; g.mpad = mp;
            pg::contract_kernel<<<dim3((unsigned)tm, (unsigned)nslab), pg::THREADS, 0, _ctx->stream>>>(g);
            CUDA_CHECK(cudaGetLastError());
            pg::reduce_kernel<<<pg::nblocks(mb * nd, 256), 256, 0, _ctx->stream>>>(
                g.part, nslab, nd, mp, mb, dm_buf.f64() + b0 * nd, with_var ? dv_buf->f64() + b0 * nd : nullptr);
            CUDA_CHECK(cudaGetLastError());
            _ctx->launches += 2;
        }
    }
    CUDA_CHECK(cudaMemcpyAsync(dmean, dm_buf.p, (size_t)m * nd * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    if (with_var) {
        CUDA_CHECK(cudaMemcpyAsync(var, v_buf->p, (size_t)m * 8, cudaMemcpyDeviceToHost, _ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(dvar, dv_buf->p, (size_t)m * nd * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    }
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}
