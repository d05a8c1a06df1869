// Gradient of the dense log-likelihood with respect to the kernel program's parameters and the noise diagonal
// (b200gp_dense_log_probability_grad).  For r = y - mean, alpha = K^-1 r, W = K^-1:
//   d logp / d theta = 1/2 sum_ij (alpha_i alpha_j - W_ij) dK_ij / d theta,   d logp / d diag_i = 1/2 (alpha_i^2 - W_ii).
//
// 1. factor K = L L^T exactly as b200gp_dense_log_probability does (native fp64 or the int8 update), then alpha by the
//    forward and backward substitutions;
// 2. X = L^-1 in place in the lower triangle, block column by block column from the right, on the DMMA pipe: each tile
//    product runs over the triangular K range only (N^3 / 3 flops);
// 3. U = X^T mirrored into the (unused) upper triangle, so that W_IJ = sum_{K >= I} U_IK U_JK^T is an NT product over
//    row panels of U.  Each lower tile of W lives in one CTA only; its epilogue regenerates dk / d slot for every element
//    (kgrad.cuh), weights it by (alpha_i alpha_j - W_ij) and reduces per-slot partial sums, written per tile.  Partials
//    are then reduced per slot in a fixed-shape tree: no floating-point atomics, bitwise reproducible.
// Extra device memory: O(n) vectors, 128 x np for the transposed diagonal blocks and the block-column operand, and
// tiles x 16 partial sums.  No second np x np buffer.
#include "common.cuh"
#include "dmma.cuh"
#include "kgrad.cuh"
#include <limits.h>

namespace tg {
constexpr int BM = 128, BK = dmma::BK, STAGES = 4, LDS = dmma::LDS, THREADS = 256;
constexpr int STAGE_DOUBLES = 2 * BM * LDS;
constexpr int SMEM_BYTES = STAGES * STAGE_DOUBLES * (int)sizeof(double);   // 163840 (>= the 128 x 128 W tile)
constexpr int CHUNKS = TILE / BK;                                           // K chunks per 128-block

// Tile schedules:
//  PANEL    (inverse, step a): C(0, tj) for tj = j+1 .. T-1, one K block (0)
//  TRMM     (inverse, step b): C(ti, 0) for ti = T-1 .. j+1 (longest K range first), K blocks j+1 .. ti
//  CONTRACT (W tiles):          C(ti, tj) for ti >= tj, ti ascending (longest K range first), K blocks ti .. T-1
enum { PANEL = 0, TRMM = 1, CONTRACT = 2 };

struct Args {
    const double* A; int64_t lda;
    const double* B; int64_t ldb;
    // 128 x 128 blocks that replace A's (B's) block (row block, K block) when the K block equals the row block: the
    // triangular diagonal blocks, stored apart with zeros in their other triangle
    const double* diagA; const double* diagB;
    double* C; int64_t ldc;
    int mode, j, T;
    double alpha;
    // CONTRACT epilogue
    KProg P; KGrad G;
    const double* X; int ndim; int64_t n;
    const double* alphav;   // alpha, padded to np with zeros
    double* wdiag;          // W_ii
    double* partial;        // [tile][KGRAD_MAX_SLOTS]
};

__device__ __forceinline__ void cp_async16(void* smem_ptr, const void* gptr) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_ptr);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gptr));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ const double* block_ptr(const double* base, int64_t ld, const double* diag, int rowblk, int kblk,
                                                   int64_t& ldo) {
    if (diag != nullptr && kblk == rowblk) {
        ldo = TILE;
        return diag + (int64_t)rowblk * TILE * TILE;
    }
    ldo = ld;
    return base + (int64_t)rowblk * TILE * ld + (int64_t)kblk * TILE;
}

// 128 x 128 CTA tile, 8 warps (2 x 4) of 64 x 32, the DMMA warp tile of dmma.cuh (mma.sync.m16n8k16.f64), 4-stage
// cp.async pipeline (the layout of dense.cu's gemm_nt_kernel) over a per-tile K range of 128-blocks
__global__ void __launch_bounds__(THREADS, 1) tri_gemm_kernel(const __grid_constant__ Args g) {
    extern __shared__ __align__(16) double smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp >> 2, wn = warp & 3;
    int ti, tj, klo, khi;
    if (g.mode == PANEL) {
        ti = 0; tj = g.j + 1 + (int)blockIdx.x; klo = khi = 0;
    } else if (g.mode == TRMM) {
        ti = g.T - 1 - (int)blockIdx.x; tj = 0; klo = g.j + 1; khi = ti;
    } else {
        const int b = (int)blockIdx.x;
        ti = (int)((sqrt(8.0 * (double)b + 1.0) - 1.0) * 0.5);
        while ((ti + 1) * (ti + 2) / 2 <= b) ++ti;
        while (ti * (ti + 1) / 2 > b) --ti;
        tj = b - ti * (ti + 1) / 2;
        klo = ti; khi = g.T - 1;
    }
    const int arow = (g.mode == TRMM || g.mode == CONTRACT) ? ti : 0;
    const int brow = (g.mode == TRMM) ? 0 : tj;

    const int lrow = tid >> 3, lc16 = (tid & 7) * 2;
    auto load_stage = [&](int stage, int kc) {     // kc: chunk index from klo * CHUNKS
        double* as = smem + stage * STAGE_DOUBLES;
        double* bs = as + BM * LDS;
        const int kblk = klo + kc / CHUNKS;
        const int koff = (kc % CHUNKS) * BK + lc16;
        int64_t la, lb;
        const double* Ab = block_ptr(g.A, g.lda, g.diagA, arow, kblk, la);
        const double* Bb = block_ptr(g.B, g.ldb, g.diagB, brow, kblk, lb);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = lrow + i * 32;
            cp_async16(as + r * LDS + lc16, Ab + (int64_t)r * la + koff);
            cp_async16(bs + r * LDS + lc16, Bb + (int64_t)r * lb + koff);
        }
    };

    double acc[8][4][2];
#pragma unroll
    for (int mi = 0; mi < 8; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;

    const int KT = (khi - klo + 1) * CHUNKS;
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KT) load_stage(s, s);
        cp_async_commit();
    }
    for (int kc = 0; kc < KT; ++kc) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        const int nk = kc + STAGES - 1;
        if (nk < KT) load_stage(nk % STAGES, nk);
        cp_async_commit();
        const double* as = smem + (kc % STAGES) * STAGE_DOUBLES + wm * dmma::WM * LDS;
        const double* bs = smem + (kc % STAGES) * STAGE_DOUBLES + BM * LDS + wn * dmma::WN * LDS;
        dmma::warp_tile_stage(acc, as, bs, lane);
    }
    cp_async_wait<0>();

    if (g.mode != CONTRACT) {
        const int64_t crow0 = (int64_t)ti * BM + wm * dmma::WM;
        const int64_t ccol0 = (int64_t)tj * BM + wn * dmma::WN;
#pragma unroll
        for (int mi = 0; mi < 8; ++mi) {
            double* crow = g.C + (crow0 + dmma::acc_row(lane, mi)) * g.ldc;
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
                *reinterpret_cast<double2*>(crow + ccol0 + dmma::acc_col(lane, ni, 0)) =
                    make_double2(g.alpha * acc[mi][ni][0], g.alpha * acc[mi][ni][1]);
        }
        return;
    }

    // ---- CONTRACT epilogue: W tile -> shared memory, then the derivative pass over its elements ----
    __syncthreads();                   // every warp is done with the pipeline buffers
    double* Ws = smem;                 // 128 x 128
#pragma unroll
    for (int mi = 0; mi < 8; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
            const int r = wm * dmma::WM + dmma::acc_row(lane, mi), c = wn * dmma::WN + dmma::acc_col(lane, ni, 0);
            Ws[r * BM + c] = acc[mi][ni][0];
            Ws[r * BM + c + 1] = acc[mi][ni][1];
        }
    __syncthreads();
    double gs[KGRAD_MAX_SLOTS];
#pragma unroll
    for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) gs[s] = 0.0;
    const int nd = g.ndim;
    for (int e = tid; e < BM * BM; e += THREADS) {
        const int r = e / BM, c = e % BM;
        const int64_t i = (int64_t)ti * BM + r, j = (int64_t)tj * BM + c;
        if (i >= g.n || j >= g.n || j > i) continue;
        const double w = Ws[e];
        if (i == j) g.wdiag[i] = w;
        const double wt = ((i == j) ? 1.0 : 2.0) * (g.alphav[i] * g.alphav[j] - w);
        const double* xa = g.X + i * nd;
        const double* xb = g.X + j * nd;
        double dk[KGRAD_MAX_SLOTS];
#pragma unroll
        for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) dk[s] = 0.0;
        kgrad_eval(g.P, g.G, nd, [&](int d) { return xa[d] - xb[d]; }, dk);
#pragma unroll
        for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) gs[s] += wt * dk[s];
    }
    __syncthreads();                   // Ws is reused for the block reduction
    double* red = smem;                // THREADS x KGRAD_MAX_SLOTS
#pragma unroll
    for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) red[s * THREADS + tid] = gs[s];
    __syncthreads();
    for (int o = THREADS / 2; o > 0; o >>= 1) {
        if (tid < o)
            for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) red[s * THREADS + tid] += red[s * THREADS + tid + o];
        __syncthreads();
    }
    if (tid < KGRAD_MAX_SLOTS) g.partial[(int64_t)blockIdx.x * KGRAD_MAX_SLOTS + tid] = red[tid * THREADS];
}

// out[s] = 1/2 sum_t partial[t][s]: one block per slot, fixed-shape tree
__global__ void __launch_bounds__(1024) slot_reduce_kernel(const double* partial, int64_t ntiles, double* out) {
    __shared__ double sh[1024];
    const int s = blockIdx.x;
    double a = 0.0;
    for (int64_t t = threadIdx.x; t < ntiles; t += 1024) a += partial[t * KGRAD_MAX_SLOTS + s];
    sh[threadIdx.x] = a;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[s] = 0.5 * sh[0];
}

// each 128 x 128 block b: dst_b = src_b^T
__global__ void block_transpose_kernel(const double* src, double* dst) {
    __shared__ double t[32][33];
    const int64_t b = blockIdx.z;
    src += b * TILE * TILE;
    dst += b * TILE * TILE;
    const int x = blockIdx.x * 32 + threadIdx.x;
    for (int y = blockIdx.y * 32 + threadIdx.y; y < blockIdx.y * 32 + 32; y += 8) t[y - blockIdx.y * 32][threadIdx.x] = src[y * TILE + x];
    __syncthreads();
    const int xo = blockIdx.y * 32 + threadIdx.x;
    for (int y = blockIdx.x * 32 + threadIdx.y; y < blockIdx.x * 32 + 32; y += 8) dst[y * TILE + xo] = t[threadIdx.x][y - blockIdx.x * 32];
}

// upper triangle of the np x np matrix <- transpose of its lower triangle (32 x 32 tiles at or below the diagonal)
__global__ void mirror_lower_kernel(double* M, int64_t ld) {
    __shared__ double t[32][33];
    const int64_t bi = blockIdx.y, bj = blockIdx.x;     // source tile rows bi, columns bj, bj <= bi
    if (bj > bi) return;
    for (int y = threadIdx.y; y < 32; y += 8) t[y][threadIdx.x] = M[(bi * 32 + y) * ld + bj * 32 + threadIdx.x];
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += 8) {
        const int64_t r = bj * 32 + y, c = bi * 32 + threadIdx.x;   // destination (r, c) = source (c, r)
        if (c > r) M[r * ld + c] = t[threadIdx.x][y];
    }
}

__global__ void finish_diag_kernel(const double* alphav, const double* wdiag, int64_t n, double* ddiag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ddiag[i] = 0.5 * (alphav[i] * alphav[i] - wdiag[i]);
}

static void launch(b200gp_ctx* ctx, const Args& g, unsigned nblocks) {
    static bool attr = false;
    if (!attr) {
        CUDA_CHECK(cudaFuncSetAttribute(tri_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr = true;
    }
    if (nblocks == 0) return;
    tri_gemm_kernel<<<nblocks, THREADS, SMEM_BYTES, ctx->stream>>>(g);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
}
}  // namespace tg

extern "C" int b200gp_dense_log_probability_grad(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X,
                                                 int64_t n, int ndim, const double* diag, const double* resid,
                                                 double* logp, double* dprog, double* dmetric, double* ddiag,
                                                 double* alpha) {
    API_BEGIN(ctx)
    const KProg P = parse_prog(prog, n_instr, ndim);
    KGrad G;
    if (!kgrad_prepare(P, G))
        throw GpError("log_probability_grad: the kernel program has more than 16 differentiable parameters, or a leaf "
                      "without derivatives (closed forms of quasiseparable kernels)");
    // the factor of b200gp_dense_log_probability, without its fused forward substitution (alpha needs both solves)
    _ctx->fuse_resid = nullptr;
    b200gp_dense* s = dense_factor_from_prog(_ctx, P, X, n, ndim, diag, true);
    struct Free { b200gp_dense* s; ~Free() { dense_destroy(s); } } free_s{s};
    const int64_t np = s->np, ld = s->np;
    const int T = (int)(np / TILE);
    Scratch y_buf(_ctx, (size_t)np * 8), x_buf(_ctx, (size_t)np * 8), a_buf(_ctx, (size_t)np * 8);
    double* const yv = y_buf.f64();
    double* const xv = x_buf.f64();
    double* const av = a_buf.f64();
    CUDA_CHECK(cudaMemsetAsync(yv, 0, (size_t)np * 8, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(yv, resid, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
    dense_solve_vec_dev(s, yv, xv, false);
    const double ss = dense_sumsq_dev(_ctx, xv, n);
    const double ldh = dense_logdet_half(s);
    double lp = -0.5 * ss - (ldh + 0.5 * (double)n * log(2.0 * M_PI));   // gp.py:313-316, direct.py:61-64
    const int nrows = n_instr;
    for (int i = 0; i < nrows * B200GP_PROG_STRIDE; ++i) dprog[i] = 0.0;
    for (int i = 0; i < B200GP_PROG_MAX_METRICS * B200GP_METRIC_MAX_DIM; ++i) dmetric[i] = 0.0;
    if (s->info != 0 || !isfinite(lp)) {
        *logp = -INFINITY;
        const double nan = NAN;
        const int row0 = nrows - P.n;
        for (int i = 0; i < P.n; ++i)
            for (int q = 2; q < 4; ++q) dprog[(row0 + i) * B200GP_PROG_STRIDE + q] = nan;
        for (int m = 0; m < P.nmetric; ++m)
            for (int r = 0; r < P.mrows[m]; ++r) dmetric[m * B200GP_METRIC_MAX_DIM + r] = nan;
        for (int64_t i = 0; i < n; ++i) ddiag[i] = alpha[i] = nan;
        return 0;
    }
    *logp = lp;
    CUDA_CHECK(cudaMemcpyAsync(yv, xv, (size_t)np * 8, cudaMemcpyDeviceToDevice, _ctx->stream));
    dense_solve_vec_dev(s, yv, av, true);                                  // alpha = L^-T L^-1 r (pad rows: 0)

    const size_t blk_bytes = (size_t)T * TILE * TILE * 8;
    Scratch lt_buf(_ctx, blk_bytes), pt_buf(_ctx, (size_t)TILE * np * 8);
    double* const linvT = lt_buf.f64();
    double* const Pt = pt_buf.f64();
    double* const M = s->mat;
    tg::block_transpose_kernel<<<dim3(TILE / 32, TILE / 32, T), dim3(32, 8), 0, _ctx->stream>>>(s->linv, linvT);
    _ctx->launches++;
    {
        // X = L^-1 in place: for j = T-2 .. 0,  X_ij = sum_{k=j+1..i} X_ik (-L_kj X_jj)  for i > j;  X_jj = linv_j
        ProfTimer t(_ctx, &_ctx->prof.trtri_ms);
        for (int j = T - 2; j >= 0; --j) {
            tg::Args g{};
            // Pt (128 x np, columns k > j) = -(L_kj X_jj)^T = -X_jj^T L_kj^T
            g.mode = tg::PANEL; g.j = j; g.T = T; g.alpha = -1.0;
            g.A = linvT + (int64_t)j * TILE * TILE; g.lda = TILE;
            g.B = M + (int64_t)j * TILE; g.ldb = ld;
            g.C = Pt; g.ldc = np;
            tg::launch(_ctx, g, (unsigned)(T - 1 - j));
            // block column j below the diagonal <- X_{i, j+1..i} Pt^T (diagonal blocks of X from linv)
            g.mode = tg::TRMM; g.alpha = 1.0;
            g.A = M; g.lda = ld; g.diagA = s->linv;
            g.B = Pt; g.ldb = np;
            g.C = M + (int64_t)j * TILE; g.ldc = ld;
            tg::launch(_ctx, g, (unsigned)(T - 1 - j));
        }
    }
    const int64_t ntiles = (int64_t)T * (T + 1) / 2;
    Scratch part_buf(_ctx, (size_t)ntiles * KGRAD_MAX_SLOTS * 8), wd_buf(_ctx, (size_t)np * 8),
        xd_buf(_ctx, (size_t)n * ndim * 8), g_buf(_ctx, KGRAD_MAX_SLOTS * 8), dd_buf(_ctx, (size_t)n * 8);
    {
        ProfTimer t(_ctx, &_ctx->prof.contract_ms);
        tg::mirror_lower_kernel<<<dim3((unsigned)(np / 32), (unsigned)(np / 32)), dim3(32, 8), 0, _ctx->stream>>>(M, ld);
        _ctx->launches++;
        CUDA_CHECK(cudaMemcpyAsync(xd_buf.p, X, (size_t)n * ndim * 8, cudaMemcpyDefault, _ctx->stream));
        tg::Args g{};
        g.mode = tg::CONTRACT; g.T = T; g.alpha = 1.0;
        g.A = M; g.lda = ld; g.diagA = linvT;        // rows of U = X^T; U's diagonal blocks are linv^T
        g.B = M; g.ldb = ld; g.diagB = linvT;
        g.P = P; g.G = G;
        g.X = xd_buf.f64(); g.ndim = ndim; g.n = n;
        g.alphav = av; g.wdiag = wd_buf.f64(); g.partial = part_buf.f64();
        tg::launch(_ctx, g, (unsigned)ntiles);
        tg::slot_reduce_kernel<<<KGRAD_MAX_SLOTS, 1024, 0, _ctx->stream>>>(part_buf.f64(), ntiles, g_buf.f64());
        tg::finish_diag_kernel<<<(unsigned)((n + 255) / 256), 256, 0, _ctx->stream>>>(av, wd_buf.f64(), n, dd_buf.f64());
        _ctx->launches += 2;
        CUDA_CHECK(cudaGetLastError());
    }
    double gh[KGRAD_MAX_SLOTS];
    CUDA_CHECK(cudaMemcpyAsync(gh, g_buf.p, sizeof(gh), cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(ddiag, dd_buf.p, (size_t)n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(alpha, av, (size_t)n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    const int row0 = nrows - P.n;      // metric definitions come first
    for (int i = 0; i < P.n; ++i) {
        if (G.slot0[i] >= 0) dprog[(row0 + i) * B200GP_PROG_STRIDE + 2] = gh[G.slot0[i]];
        if (G.slot1[i] >= 0) dprog[(row0 + i) * B200GP_PROG_STRIDE + 3] = gh[G.slot1[i]];
    }
    for (int m = 0; m < P.nmetric; ++m)
        for (int r = 0; r < P.mrows[m]; ++r) dmetric[m * B200GP_METRIC_MAX_DIM + r] = gh[G.mslot[m] + r];
    API_END
}
