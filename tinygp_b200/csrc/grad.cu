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
//
// b200gp_dense_log_probability_grad_x adds the gradient with respect to the coordinates, from the same epilogue:
//   d logp / d x_i = sum_{j != i} (alpha_i alpha_j - W_ij) grad_1 k(x_i, x_j)
// (K_ij and K_ji both depend on x_i, and grad_2 k(x_j, x_i) = grad_1 k(x_i, x_j) for a stationary k).  Each element
// i > j of a W tile adds w_ij g_ij (g_ij = d k / d delta at delta = x_i - x_j, kgrad.cuh) to row i and subtracts it from
// row j.  The tile reduces these into per-tile row sums (a warp-shuffle tree per row, then its four warps in order) and
// column sums (per thread in registers, then the two threads of a column in order) and writes both; dx_reduce_kernel
// then adds, per point, the row sums of tiles (I, 0..I) and subtracts the column sums of tiles (I..T-1, I) in that
// order.  No floating-point atomics: bitwise reproducible.  The partials take tiles x 2 x 128 x ndim doubles, about
// n^2 ndim / 16 bytes: 805 MB at n = 65536, ndim = 3 (2.1 GB at the cap, ndim = 8).  The plain gradient instantiates the
// tile kernel with DX = false, where none of this is compiled.
//
// b200gp_dense_fisher: the expected Fisher information F_ab = 1/2 tr(W dK_a W dK_b) = 1/2 <dK_a, C_b>, C_b = X^T X dK_b
// X^T X, from the same factor and X = L^-1 (steps 1 and 2, then U = X^T mirrored as in step 3).  For each slot b, in one
// np x np work buffer:
//   dK_b (dk_build_kernel; the identity for the noise slot)  -> . X^T -> transpose -> . X^T  = X dK_b X^T = E_b
//   E_b                                                       -> . X   -> transpose -> . X    = X^T E_b X   = C_b
// Each ". X^T" / ". X" is an in-place product by a triangular factor on the DMMA mainloop (RMUL_XT / RMUL_X): one launch
// per output column block, descending (ascending), each CTA owning one row block, so a launch writes exactly the column
// block that no later launch reads.  Then the contraction tiles (FISHER) read the lower tiles of C_b from memory into the
// CONTRACT epilogue with weight c_ij in place of alpha_i alpha_j - W_ij; the noise slot's entry is 1/2 tr(C_b) from the
// C_b diagonal the epilogue writes.  Same fixed-shape reductions as the gradient: bitwise reproducible.
#include "common.cuh"
#include "dmma.cuh"
#include "kgrad.cuh"
#include <limits.h>
#include <optional>

namespace tg {
using dmma::BM; using dmma::SK; using dmma::THREADS; using dmma::SMEM_BYTES;   // SMEM_BYTES >= the 128 x 128 W tile
constexpr int CHUNKS = TILE / SK;                                               // K chunks per 128-block
// the CONTRACT epilogue's W tile and row sums stay in the operand ring, clear of its mbarriers
static_assert((BM * BM + 4 * KGRAD_MAX_DIM * BM) * (int)sizeof(double) <= dmma::RING_BYTES, "epilogue fits the ring");

// Tile schedules (A's row block ti, B's row block tj):
//  TRMM     (inverse): C(ti, 0) for ti = T-1 .. j+1 (longest K range first), K blocks j+1 .. ti
//  CONTRACT (W tiles): C(ti, tj) for ti >= tj, ti ascending (longest K range first), K blocks ti .. T-1
//  RMUL_XT  (C = A X^T in place, B = X with diagB = linv):    C(ti, j) for every ti, K blocks 0 .. j
//  RMUL_X   (C = A X in place, B = U = X^T with diagB = linvT): C(ti, j) for every ti, K blocks j .. T-1
//  FISHER   (Fisher contraction): the tiles of CONTRACT, weight tile read from A, no mainloop
enum { TRMM, CONTRACT, RMUL_XT, RMUL_X, FISHER };

struct Args {
    const double* A; int64_t lda;
    const double* B; int64_t ldb;
    // 128 x 128 blocks that replace A's (B's) block (row block, K block) when the K block equals the row block: the
    // triangular diagonal blocks, stored apart with zeros in their other triangle
    const double* diagA; const double* diagB;
    double* C; int64_t ldc;
    int mode, j, T;
    // CONTRACT epilogue
    KProg P; KGrad G;
    const double* X; int ndim; int64_t n;
    const double* alphav;   // alpha, padded to np with zeros
    double* wdiag;          // W_ii
    double* partial;        // [tile][KGRAD_MAX_SLOTS]
    double* dxpart;         // DX: [tile][row sums, column sums][ndim][BM]
};

__device__ __forceinline__ const double* block_ptr(const double* base, int64_t ld, const double* diag, int rowblk, int kblk,
                                                   int64_t& ldo) {
    if (diag != nullptr && kblk == rowblk) {
        ldo = TILE;
        return diag + (int64_t)rowblk * TILE * TILE;
    }
    ldo = ld;
    return base + (int64_t)rowblk * TILE * ld + (int64_t)kblk * TILE;
}

// The 128 x 128 CTA tile of dmma.cuh's cta_tile_nt over a per-tile K range of 128-blocks, A's and B's diagonal blocks
// substituted.  DX: the CONTRACT epilogue also writes the tile's coordinate-gradient partials.
template <bool DX>
__global__ void __launch_bounds__(THREADS, 1) tri_gemm_kernel(const __grid_constant__ Args g) {
    extern __shared__ __align__(16) double smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp >> 2, wn = warp & 3;
    int ti, tj, klo, khi;
    if (g.mode == TRMM) {
        ti = g.T - 1 - (int)blockIdx.x; tj = 0; klo = g.j + 1; khi = ti;
    } else if (g.mode == RMUL_XT || g.mode == RMUL_X) {
        ti = (int)blockIdx.x; tj = g.j;
        klo = (g.mode == RMUL_XT) ? 0 : g.j;
        khi = (g.mode == RMUL_XT) ? g.j : g.T - 1;
    } else {
        const int b = (int)blockIdx.x;
        ti = (int)((sqrt(8.0 * (double)b + 1.0) - 1.0) * 0.5);
        while ((ti + 1) * (ti + 2) / 2 <= b) ++ti;
        while (ti * (ti + 1) / 2 > b) --ti;
        tj = b - ti * (ti + 1) / 2;
        klo = ti; khi = g.T - 1;
    }

    double acc[8][4][2];
    if (g.mode != FISHER)
        dmma::cta_tile_nt(
            acc, smem, (khi - klo + 1) * CHUNKS,
            [&](int kc) {
                const int kblk = klo + kc / CHUNKS, k0 = (kc % CHUNKS) * SK;
                dmma::Operands o;
                o.a = block_ptr(g.A, g.lda, g.diagA, ti, kblk, o.lda);
                o.b = block_ptr(g.B, g.ldb, g.diagB, tj, kblk, o.ldb);
                o.k = k0;
                return o;
            },
            [](int) {});

    if (g.mode != CONTRACT && g.mode != FISHER) {
        const int64_t crow0 = (int64_t)ti * BM + wm * dmma::WM;
        const int64_t ccol0 = (int64_t)tj * BM + wn * dmma::WN;
#pragma unroll
        for (int mi = 0; mi < 8; ++mi) {
            double* crow = g.C + (crow0 + dmma::acc_row(lane, mi)) * g.ldc;
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
                *reinterpret_cast<double2*>(crow + ccol0 + dmma::acc_col(lane, ni, 0)) =
                    make_double2(acc[mi][ni][0], acc[mi][ni][1]);
        }
        return;
    }

    // ---- CONTRACT epilogue: W tile -> shared memory, then the derivative pass over its elements ----
    // (FISHER: the tile of C_b from A instead, and the weight c_ij in place of alpha_i alpha_j - W_ij)
    double* Ws = smem;                 // 128 x 128
    if (g.mode == FISHER) {
        const double* src = g.A + (int64_t)ti * BM * g.lda + (int64_t)tj * BM;
        for (int e = tid; e < BM * BM; e += THREADS) Ws[e] = src[(int64_t)(e / BM) * g.lda + e % BM];
    } else {
        __syncthreads();               // every warp is done with the pipeline buffers
#pragma unroll
        for (int mi = 0; mi < 8; ++mi)
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) {
                const int r = wm * dmma::WM + dmma::acc_row(lane, mi), c = wn * dmma::WN + dmma::acc_col(lane, ni, 0);
                Ws[r * BM + c] = acc[mi][ni][0];
                Ws[r * BM + c + 1] = acc[mi][ni][1];
            }
    }
    __syncthreads();
    double gs[KGRAD_MAX_SLOTS];
#pragma unroll
    for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) gs[s] = 0.0;
    const int nd = g.ndim;
    if constexpr (DX) {
        // thread tid visits column tid % BM and rows tid / BM + 2k: its column sum stays in registers; the 32 lanes of
        // a warp share the row, reduced by shuffles into rowp[warp % 4][d][row]
        double* rowp = smem + BM * BM;     // 4 x KGRAD_MAX_DIM x BM doubles past the W tile
        double gcol[KGRAD_MAX_DIM];
#pragma unroll
        for (int d = 0; d < KGRAD_MAX_DIM; ++d) gcol[d] = 0.0;
        for (int e = tid; e < BM * BM; e += THREADS) {
            const int r = e / BM, c = e % BM;
            const int64_t i = (int64_t)ti * BM + r, j = (int64_t)tj * BM + c;
            double gx[KGRAD_MAX_DIM];
#pragma unroll
            for (int d = 0; d < KGRAD_MAX_DIM; ++d) gx[d] = 0.0;
            if (i < g.n && j < g.n && j <= i) {
                const double w = Ws[e];
                if (i == j) g.wdiag[i] = w;
                const double wt = ((i == j) ? 1.0 : 2.0) * (g.alphav[i] * g.alphav[j] - w);
                const double* xa = g.X + i * nd;
                const double* xb = g.X + j * nd;
                double dk[KGRAD_MAX_SLOTS];
#pragma unroll
                for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) dk[s] = 0.0;
                kgrad_eval<true>(g.P, g.G, nd, [&](int d) { return xa[d] - xb[d]; }, dk, true, gx);
#pragma unroll
                for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) gs[s] += wt * dk[s];
                const double om = (i > j) ? g.alphav[i] * g.alphav[j] - w : 0.0;
#pragma unroll
                for (int d = 0; d < KGRAD_MAX_DIM; ++d) gx[d] *= om;
            }
#pragma unroll
            for (int d = 0; d < KGRAD_MAX_DIM; ++d) {
                if (d < nd) {
                    gcol[d] += gx[d];
                    double v = gx[d];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                    if (lane == 0) rowp[((warp & 3) * KGRAD_MAX_DIM + d) * BM + r] = v;
                }
            }
        }
        __syncthreads();
        double* colp = smem + 2 * THREADS * KGRAD_MAX_SLOTS;   // past the slot reduction's buffer below
        if (tid >= BM)
#pragma unroll
            for (int d = 0; d < KGRAD_MAX_DIM; ++d)
                if (d < nd) colp[d * BM + tid - BM] = gcol[d];
        __syncthreads();
        if (tid < BM) {
            double* out = g.dxpart + (int64_t)blockIdx.x * 2 * nd * BM;
#pragma unroll
            for (int d = 0; d < KGRAD_MAX_DIM; ++d)
                if (d < nd) {
                    double rs = rowp[d * BM + tid];
#pragma unroll
                    for (int q = 1; q < 4; ++q) rs += rowp[(q * KGRAD_MAX_DIM + d) * BM + tid];
                    out[d * BM + tid] = rs;
                    out[(nd + d) * BM + tid] = gcol[d] + colp[d * BM + tid];
                }
        }
    } else {
        for (int e = tid; e < BM * BM; e += THREADS) {
            const int r = e / BM, c = e % BM;
            const int64_t i = (int64_t)ti * BM + r, j = (int64_t)tj * BM + c;
            if (i >= g.n || j >= g.n || j > i) continue;
            const double w = Ws[e];
            if (i == j) g.wdiag[i] = w;
            const double wt = ((i == j) ? 1.0 : 2.0) * ((g.mode == FISHER) ? w : g.alphav[i] * g.alphav[j] - w);
            const double* xa = g.X + i * nd;
            const double* xb = g.X + j * nd;
            double dk[KGRAD_MAX_SLOTS];
#pragma unroll
            for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) dk[s] = 0.0;
            kgrad_eval(g.P, g.G, nd, [&](int d) { return xa[d] - xb[d]; }, dk);
#pragma unroll
            for (int s = 0; s < KGRAD_MAX_SLOTS; ++s) gs[s] += wt * dk[s];
        }
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

// out[s] = 1/2 sum_t partial[t * stride + s]: one block per slot, fixed-shape tree
__global__ void __launch_bounds__(1024) slot_reduce_kernel(const double* partial, int64_t ntiles, int64_t stride,
                                                           double* out) {
    __shared__ double sh[1024];
    const int s = blockIdx.x;
    double a = 0.0;
    for (int64_t t = threadIdx.x; t < ntiles; t += 1024) a += partial[t * stride + s];
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

// dX[i][d] = sum_{J <= I} row sums of tile (I, J) - sum_{I' >= I} column sums of tile (I', I), I = i / BM, in this order
__global__ void __launch_bounds__(BM) dx_reduce_kernel(const double* dxpart, int T, int nd, int64_t n, double* dX) {
    const int I = blockIdx.x, d = blockIdx.y, r = threadIdx.x;
    const int64_t stride = 2 * (int64_t)nd * BM;
    double s = 0.0;
    const double* p = dxpart + ((int64_t)I * (I + 1) / 2) * stride + d * BM + r;
#pragma unroll 4
    for (int J = 0; J <= I; ++J) s += p[J * stride];
#pragma unroll 4
    for (int I2 = I; I2 < T; ++I2) s -= dxpart[((int64_t)I2 * (I2 + 1) / 2 + I) * stride + (nd + d) * BM + r];
    const int64_t i = (int64_t)I * BM + r;
    if (i < n) dX[i * nd + d] = s;
}

__global__ void finish_diag_kernel(const double* alphav, const double* wdiag, int64_t n, double* ddiag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ddiag[i] = 0.5 * (alphav[i] * alphav[i] - wdiag[i]);
}

// D (np x np) = dK / d slot (kgrad_element): 32 x 8 threads per 32 x 32 tile, 4 rows each
__global__ void __launch_bounds__(256) dk_build_kernel(const KProg P, const KGrad G, const double* X, int ndim, int64_t n,
                                                       int64_t np, int slot, double* D) {
    const int64_t j = (int64_t)blockIdx.x * 32 + threadIdx.x;
    for (int64_t i = (int64_t)blockIdx.y * 32 + threadIdx.y; i < (int64_t)blockIdx.y * 32 + 32; i += 8)
        D[i * np + j] = kgrad_element(P, G, ndim, X, n, i, j, slot);
}

// M (np x np) <- M^T in place: the block at (by, bx), bx <= by, swaps with its mirror (32 x 32 tiles)
__global__ void transpose_inplace_kernel(double* M, int64_t ld) {
    __shared__ double a[32][33], b[32][33];
    const int64_t bi = blockIdx.y, bj = blockIdx.x;
    if (bj > bi) return;
    for (int y = threadIdx.y; y < 32; y += 8) {
        a[y][threadIdx.x] = M[(bi * 32 + y) * ld + bj * 32 + threadIdx.x];
        b[y][threadIdx.x] = M[(bj * 32 + y) * ld + bi * 32 + threadIdx.x];
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += 8) {
        M[(bj * 32 + y) * ld + bi * 32 + threadIdx.x] = a[threadIdx.x][y];
        M[(bi * 32 + y) * ld + bj * 32 + threadIdx.x] = b[threadIdx.x][y];
    }
}

template <bool DX = false>
static void launch(b200gp_ctx* ctx, const Args& g, unsigned nblocks) {
    static bool attr = false;
    if (!attr) {
        CUDA_CHECK(cudaFuncSetAttribute(tri_gemm_kernel<DX>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr = true;
    }
    if (nblocks == 0) return;
    tri_gemm_kernel<DX><<<nblocks, THREADS, SMEM_BYTES, ctx->stream>>>(g);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
}

// step 2's launch for block column j < T - 1: C_ij = sum_{k=j+1..i} A_ik B_k^T for i > j, A's diagonal blocks from
// diagA, B 128 rows; every matrix np = 128 T columns wide
static void trmm(b200gp_ctx* ctx, int T, int j, const double* A, const double* diagA, const double* B, double* C) {
    Args g{};
    g.mode = TRMM; g.j = j; g.T = T;
    g.A = A; g.lda = (int64_t)T * TILE; g.diagA = diagA;
    g.B = B; g.ldb = (int64_t)T * TILE;
    g.C = C + (int64_t)j * TILE; g.ldc = (int64_t)T * TILE;
    launch(ctx, g, (unsigned)(T - 1 - j));
}

// step 3's launch: the lower tiles of W = U U^T, U = A (np x np, np = 128 T) with its diagonal blocks from diagA, and
// the CONTRACT epilogue over them.  dxpart != nullptr: the coordinate gradient too (tri_gemm_kernel<true>), reduced per
// point into dX.
static void contract(b200gp_ctx* ctx, int T, const double* A, const double* diagA, const KProg& P, const KGrad& G,
                     const double* X, int ndim, int64_t n, const double* alphav, double* wdiag, double* partial,
                     double* dxpart, double* dX) {
    Args g{};
    g.mode = CONTRACT; g.T = T;
    g.A = A; g.lda = (int64_t)T * TILE; g.diagA = diagA;
    g.B = A; g.ldb = (int64_t)T * TILE; g.diagB = diagA;
    g.P = P; g.G = G;
    g.X = X; g.ndim = ndim; g.n = n;
    g.alphav = alphav; g.wdiag = wdiag; g.partial = partial;
    const unsigned ntiles = (unsigned)((int64_t)T * (T + 1) / 2);
    if (dxpart == nullptr) {
        launch(ctx, g, ntiles);
        return;
    }
    g.dxpart = dxpart;
    launch<true>(ctx, g, ntiles);
    dx_reduce_kernel<<<dim3((unsigned)T, (unsigned)ndim), BM, 0, ctx->stream>>>(dxpart, T, ndim, n, dX);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
}
}  // namespace tg

// the kernel program and its slot layout for kgrad_eval; a program without device derivatives is refused, the message
// prefixed by `who`
static void parse_for_grad(const char* who, const double* prog, int n_instr, int ndim, KProg& P, KGrad& G) {
    P = parse_prog(prog, n_instr, ndim);
    if (!kgrad_prepare(P, G))
        throw GpError(std::string(who) + ": the kernel program has more than 16 differentiable parameters, or a leaf "
                      "without derivatives (closed forms of quasiseparable kernels)");
}

// step 1 of the gradient and the Fisher information: the program parsed for kgrad_eval, and the factor of
// b200gp_dense_log_probability without its fused forward substitution (alpha needs both solves), freed with this object
struct GradFactor {
    KProg P;
    KGrad G;
    b200gp_dense* s;
    GradFactor(b200gp_ctx* ctx, const char* who, const double* prog, int n_instr, const double* X, int64_t n, int ndim,
               const double* diag) {
        parse_for_grad(who, prog, n_instr, ndim, P, G);
        ctx->fuse_resid = nullptr;
        s = dense_factor_from_prog(ctx, P, X, n, ndim, diag, true);
    }
    ~GradFactor() { dense_destroy(s); }
    GradFactor(const GradFactor&) = delete;
    GradFactor& operator=(const GradFactor&) = delete;
};

// what slot q of kgrad_prepare's layout differentiates, as o[0..2]: {0, program row, column 2 (p0) or 3 (p1)} for an
// instruction's parameter, {1, metric m, row r} for a row scale of a metric (n_rows: program rows, metric definitions
// first)
static void slot_origin(const KProg& P, const KGrad& G, int n_rows, int q, int* o) {
    for (int i = 0; i < P.n; ++i)
        if (G.slot0[i] == q || G.slot1[i] == q) {
            o[0] = 0; o[1] = n_rows - P.n + i; o[2] = (G.slot0[i] == q) ? 2 : 3;
            return;
        }
    for (int m = 0; m < P.nmetric; ++m)
        if (q >= G.mslot[m] && q < G.mslot[m] + P.mrows[m]) {
            o[0] = 1; o[1] = m; o[2] = q - G.mslot[m];
            return;
        }
}

// steps 2 and 3's operands: X = L^-1 in place in the lower block triangle of s->mat (its diagonal blocks stay in
// s->linv), linvT <- the diagonal blocks transposed (T x 128 x 128), U = X^T mirrored into the upper triangle, and xd <-
// the n x ndim coordinates X (host or device).  The mirror and the upload count toward the profile field `prof`
// (nullptr: toward none).
static void invert_factor(b200gp_ctx* _ctx, b200gp_dense* s, double* linvT, const double* X, int64_t n, int ndim,
                          double* xd, double* prof) {
    const int64_t np = s->np, ld = s->np;
    const int T = (int)(np / TILE);
    double* const M = s->mat;
    {
        Scratch pt_buf(_ctx, (size_t)TILE * np * 8);
        double* const Pt = pt_buf.f64();
        tg::block_transpose_kernel<<<dim3(TILE / 32, TILE / 32, T), dim3(32, 8), 0, _ctx->stream>>>(s->linv, linvT);
        _ctx->launches++;
        // X = L^-1 in place: for j = T-2 .. 0,  X_ij = sum_{k=j+1..i} X_ik (-L_kj X_jj)  for i > j;  X_jj = linv_j
        ProfTimer t(_ctx, &_ctx->prof.trtri_ms);
        for (int j = T - 2; j >= 0; --j) {
            // Pt (128 x np, column blocks k > j) = -(L_kj X_jj)^T = -X_jj^T L_kj^T
            gemm_nt(_ctx, Pt + (int64_t)(j + 1) * TILE, np, linvT + (int64_t)j * TILE * TILE, TILE,
                    M + (int64_t)(j + 1) * TILE * ld + (int64_t)j * TILE, ld, 1, T - 1 - j, TILE, -1.0, 0, 0);
            // block column j below the diagonal <- X_{i, j+1..i} Pt^T (diagonal blocks of X from linv)
            tg::trmm(_ctx, T, j, M, s->linv, Pt, M);
        }
    }
    std::optional<ProfTimer> t;
    if (prof != nullptr) t.emplace(_ctx, prof);
    tg::mirror_lower_kernel<<<dim3((unsigned)(np / 32), (unsigned)(np / 32)), dim3(32, 8), 0, _ctx->stream>>>(M, ld);
    _ctx->launches++;
    CUDA_CHECK(cudaMemcpyAsync(xd, X, (size_t)n * ndim * 8, cudaMemcpyDefault, _ctx->stream));
}

// both entry points; dX == nullptr: the plain gradient (tri_gemm_kernel<false>)
static int dense_log_probability_grad(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n,
                                      int ndim, const double* diag, const double* resid, double* logp, double* dprog,
                                      double* dmetric, double* ddiag, double* alpha, double* dX) {
    API_BEGIN(ctx)
    if (dX != nullptr && (ndim < 1 || ndim > KGRAD_MAX_DIM))
        throw GpError("log_probability_grad_x: coordinate gradients support 1 to 8 input dimensions");
    const GradFactor f(_ctx, "log_probability_grad", prog, n_instr, X, n, ndim, diag);
    const KProg& P = f.P;
    const KGrad& G = f.G;
    b200gp_dense* const s = f.s;
    const int64_t np = s->np;
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
    for (int i = 0; i < n_instr * B200GP_PROG_STRIDE; ++i) dprog[i] = 0.0;
    for (int i = 0; i < B200GP_PROG_MAX_METRICS * B200GP_METRIC_MAX_DIM; ++i) dmetric[i] = 0.0;
    if (s->info != 0 || !isfinite(lp)) {
        *logp = -INFINITY;
        const double nan = NAN;
        const int row0 = n_instr - P.n;    // metric definitions come first
        for (int i = 0; i < P.n; ++i)
            for (int q = 2; q < 4; ++q) dprog[(row0 + i) * B200GP_PROG_STRIDE + q] = nan;
        for (int m = 0; m < P.nmetric; ++m)
            for (int r = 0; r < P.mrows[m]; ++r) dmetric[m * B200GP_METRIC_MAX_DIM + r] = nan;
        for (int64_t i = 0; i < n; ++i) ddiag[i] = alpha[i] = nan;
        if (dX != nullptr)
            for (int64_t i = 0; i < n * ndim; ++i) dX[i] = nan;
        return 0;
    }
    *logp = lp;
    CUDA_CHECK(cudaMemcpyAsync(yv, xv, (size_t)np * 8, cudaMemcpyDeviceToDevice, _ctx->stream));
    dense_solve_vec_dev(s, yv, av, true);                                  // alpha = L^-T L^-1 r (pad rows: 0)

    Scratch lt_buf(_ctx, (size_t)T * TILE * TILE * 8), xd_buf(_ctx, (size_t)n * ndim * 8);
    invert_factor(_ctx, s, lt_buf.f64(), X, n, ndim, xd_buf.f64(), &_ctx->prof.contract_ms);
    const int64_t ntiles = (int64_t)T * (T + 1) / 2;
    Scratch part_buf(_ctx, (size_t)ntiles * KGRAD_MAX_SLOTS * 8), wd_buf(_ctx, (size_t)np * 8),
        g_buf(_ctx, KGRAD_MAX_SLOTS * 8), dd_buf(_ctx, (size_t)n * 8);
    const bool want_dx = dX != nullptr;
    std::optional<Scratch> dxp_buf, dx_buf;
    if (want_dx) {
        dxp_buf.emplace(_ctx, (size_t)ntiles * 2 * ndim * TILE * 8);
        dx_buf.emplace(_ctx, (size_t)n * ndim * 8);
    }
    {
        ProfTimer t(_ctx, &_ctx->prof.contract_ms);
        // rows of U = X^T; U's diagonal blocks are linv^T
        tg::contract(_ctx, T, s->mat, lt_buf.f64(), P, G, xd_buf.f64(), ndim, n, av, wd_buf.f64(), part_buf.f64(),
                     want_dx ? dxp_buf->f64() : nullptr, want_dx ? dx_buf->f64() : nullptr);
        tg::slot_reduce_kernel<<<KGRAD_MAX_SLOTS, 1024, 0, _ctx->stream>>>(part_buf.f64(), ntiles, KGRAD_MAX_SLOTS,
                                                                          g_buf.f64());
        tg::finish_diag_kernel<<<(unsigned)((n + 255) / 256), 256, 0, _ctx->stream>>>(av, wd_buf.f64(), n, dd_buf.f64());
        _ctx->launches += 2;
        CUDA_CHECK(cudaGetLastError());
    }
    double gh[KGRAD_MAX_SLOTS];
    CUDA_CHECK(cudaMemcpyAsync(gh, g_buf.p, sizeof(gh), cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(ddiag, dd_buf.p, (size_t)n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(alpha, av, (size_t)n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    if (want_dx) CUDA_CHECK(cudaMemcpyAsync(dX, dx_buf->p, (size_t)n * ndim * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    for (int q = 0; q < G.nslot; ++q) {
        int o[3];
        slot_origin(P, G, n_instr, q, o);
        (o[0] == 0 ? dprog[o[1] * B200GP_PROG_STRIDE + o[2]] : dmetric[o[1] * B200GP_METRIC_MAX_DIM + o[2]]) = gh[q];
    }
    API_END
}

extern "C" int b200gp_dense_log_probability_grad(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X,
                                                 int64_t n, int ndim, const double* diag, const double* resid,
                                                 double* logp, double* dprog, double* dmetric, double* ddiag,
                                                 double* alpha) {
    return dense_log_probability_grad(ctx, prog, n_instr, X, n, ndim, diag, resid, logp, dprog, dmetric, ddiag, alpha,
                                      nullptr);
}

extern "C" int b200gp_dense_log_probability_grad_x(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X,
                                                   int64_t n, int ndim, const double* diag, const double* resid,
                                                   double* logp, double* dprog, double* dmetric, double* ddiag,
                                                   double* alpha, double* dX) {
    if (dX == nullptr) {
        if (ctx) ctx->err = "log_probability_grad_x: dX is NULL";
        return ctx ? 2 : 1;
    }
    return dense_log_probability_grad(ctx, prog, n_instr, X, n, ndim, diag, resid, logp, dprog, dmetric, ddiag, alpha,
                                      dX);
}

extern "C" int b200gp_dense_fisher(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n,
                                   int ndim, const double* diag, int with_diag, int* nslot, int* slots, double* fisher) {
    API_BEGIN(ctx)
    if (with_diag != 0 && with_diag != 1) throw GpError("fisher: with_diag is 0 or 1");
    if (nslot == nullptr || slots == nullptr || fisher == nullptr) throw GpError("fisher: nslot, slots and fisher are required");
    const GradFactor f(_ctx, "fisher", prog, n_instr, X, n, ndim, diag);
    const KProg& P = f.P;
    const KGrad& G = f.G;
    b200gp_dense* const s = f.s;
    const int S = G.nslot, NP = S + with_diag;
    *nslot = S;
    for (int q = 0; q < S; ++q) slot_origin(P, G, n_instr, q, slots + 3 * q);
    if (s->info != 0 || !isfinite(dense_logdet_half(s))) {
        for (int i = 0; i < NP * NP; ++i) fisher[i] = NAN;
        return 0;
    }
    const int64_t np = s->np, ld = s->np;
    const int T = (int)(np / TILE);
    Scratch lt_buf(_ctx, (size_t)T * TILE * TILE * 8), xd_buf(_ctx, (size_t)n * ndim * 8);
    double* const linvT = lt_buf.f64();
    double* const M = s->mat;
    invert_factor(_ctx, s, linvT, X, n, ndim, xd_buf.f64(), nullptr);
    std::optional<Scratch> wk_buf;
    try {
        wk_buf.emplace(_ctx, (size_t)np * np * 8);
    } catch (const GpError& e) {
        char buf[384];
        snprintf(buf, sizeof(buf), "fisher: the %lld x %lld fp64 work buffer (%.2f GB) does not fit next to the factor: %s",
                 (long long)np, (long long)np, (double)np * (double)np * 8e-9, e.what());
        throw GpError(buf);
    }
    double* const Wk = wk_buf->f64();
    const int64_t ntiles = (int64_t)T * (T + 1) / 2;
    Scratch part_buf(_ctx, (size_t)ntiles * KGRAD_MAX_SLOTS * 8), wd_buf(_ctx, (size_t)np * 8),
        f_buf(_ctx, (size_t)NP * NP * 8);
    const dim3 sq_grid((unsigned)(np / 32), (unsigned)(np / 32)), sq_block(32, 8);
    // Wk <- Wk X^T (RMUL_XT, column blocks descending) or Wk X (RMUL_X, ascending), in place
    auto rmul = [&](int mode) {
        for (int jj = 0; jj < T; ++jj) {
            tg::Args g{};
            g.mode = mode; g.T = T; g.j = (mode == tg::RMUL_XT) ? T - 1 - jj : jj;
            g.A = Wk; g.lda = np;
            g.B = M; g.ldb = ld; g.diagB = (mode == tg::RMUL_XT) ? s->linv : linvT;
            g.C = Wk; g.ldc = np;
            tg::launch(_ctx, g, (unsigned)T);
        }
    };
    auto transpose = [&]() {
        tg::transpose_inplace_kernel<<<sq_grid, sq_block, 0, _ctx->stream>>>(Wk, np);
        _ctx->launches++;
    };
    for (int b = 0; b < NP; ++b) {
        tg::dk_build_kernel<<<sq_grid, sq_block, 0, _ctx->stream>>>(P, G, xd_buf.f64(), ndim, n, np, b, Wk);
        _ctx->launches++;
        rmul(tg::RMUL_XT);
        transpose();
        rmul(tg::RMUL_XT);     // E_b = X dK_b X^T
        rmul(tg::RMUL_X);
        transpose();
        rmul(tg::RMUL_X);      // C_b = X^T E_b X
        tg::Args g{};
        g.mode = tg::FISHER; g.T = T;
        g.A = Wk; g.lda = np;
        g.P = P; g.G = G;
        g.X = xd_buf.f64(); g.ndim = ndim; g.n = n;
        g.wdiag = wd_buf.f64(); g.partial = part_buf.f64();
        tg::launch(_ctx, g, (unsigned)ntiles);
        double* const row = f_buf.f64() + (int64_t)b * NP;
        if (S > 0) {
            tg::slot_reduce_kernel<<<S, 1024, 0, _ctx->stream>>>(part_buf.f64(), ntiles, KGRAD_MAX_SLOTS, row);
            _ctx->launches++;
        }
        if (with_diag) {
            tg::slot_reduce_kernel<<<1, 1024, 0, _ctx->stream>>>(wd_buf.f64(), n, 1, row + S);   // 1/2 tr(C_b)
            _ctx->launches++;
        }
        CUDA_CHECK(cudaGetLastError());
    }
    std::vector<double> fr((size_t)NP * NP);
    CUDA_CHECK(cudaMemcpyAsync(fr.data(), f_buf.p, fr.size() * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    // row b holds 1/2 <dK_a, C_b>: both triangles from the mean, so the matrix is symmetric bit for bit
    for (int a = 0; a < NP; ++a)
        for (int b = 0; b < NP; ++b) fisher[a * NP + b] = 0.5 * (fr[(size_t)a * NP + b] + fr[(size_t)b * NP + a]);
    API_END
}

// ---- diagnostics entry point: one launch of tri_gemm_kernel on host operands through the launchers of
// dense_log_probability_grad (tg::trmm, tg::contract; include/b200gp.h).  Every size is checked before anything is
// allocated, so that the kernels read and write only the buffers allocated here.
extern "C" int b200gp_grad_tiles_test(b200gp_ctx* ctx, int mode, int T, int j, const double* A, const double* diagA,
                                      const double* B, double* C, const double* prog, int n_instr, const double* X,
                                      int64_t n, int ndim, const double* alpha, double* wdiag, double* partial,
                                      double* dxpart, double* dX) {
    API_BEGIN(ctx)
    if (T < 1 || (int64_t)T * (T + 1) > INT_MAX) throw GpError("grad tiles test: 1 <= T, T (T + 1) <= INT_MAX");
    if (A == nullptr || diagA == nullptr) throw GpError("grad tiles test: A and diagA are required");
    const int64_t np = (int64_t)T * TILE;
    const size_t sq_bytes = (size_t)np * np * 8, blk_bytes = (size_t)T * TILE * TILE * 8;
    if (mode == tg::TRMM) {
        if (j < 0 || j > T - 2) throw GpError("grad tiles test: TRMM needs 0 <= j <= T - 2");
        if (B == nullptr || C == nullptr) throw GpError("grad tiles test: TRMM needs B and C");
        const size_t b_bytes = (size_t)TILE * np * 8;
        Scratch a_buf(_ctx, sq_bytes), d_buf(_ctx, blk_bytes), b_buf(_ctx, b_bytes), c_buf(_ctx, sq_bytes);
        CUDA_CHECK(cudaMemcpyAsync(a_buf.p, A, sq_bytes, cudaMemcpyHostToDevice, _ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(d_buf.p, diagA, blk_bytes, cudaMemcpyHostToDevice, _ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(b_buf.p, B, b_bytes, cudaMemcpyHostToDevice, _ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(c_buf.p, C, sq_bytes, cudaMemcpyHostToDevice, _ctx->stream));
        tg::trmm(_ctx, T, j, a_buf.f64(), d_buf.f64(), b_buf.f64(), c_buf.f64());
        CUDA_CHECK(cudaMemcpyAsync(C, c_buf.p, sq_bytes, cudaMemcpyDeviceToHost, _ctx->stream));
        CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
        return 0;
    }
    if (mode != tg::CONTRACT) throw GpError("grad tiles test: mode is 0 (TRMM) or 1 (CONTRACT)");
    if (n < 1 || n > np) throw GpError("grad tiles test: CONTRACT needs 1 <= n <= 128 T");
    if (ndim < 1 || ndim > KGRAD_MAX_DIM) throw GpError("grad tiles test: CONTRACT needs 1 <= ndim <= 8");
    if (prog == nullptr || X == nullptr || alpha == nullptr || wdiag == nullptr || partial == nullptr)
        throw GpError("grad tiles test: CONTRACT needs prog, X, alpha, wdiag and partial");
    if ((dxpart == nullptr) != (dX == nullptr)) throw GpError("grad tiles test: dxpart and dX go together");
    KProg P;
    KGrad G;
    parse_for_grad("grad tiles test", prog, n_instr, ndim, P, G);
    const bool want_dx = dX != nullptr;
    const int64_t ntiles = (int64_t)T * (T + 1) / 2;
    const size_t part_bytes = (size_t)ntiles * KGRAD_MAX_SLOTS * 8, dxp_bytes = (size_t)ntiles * 2 * ndim * TILE * 8,
                 x_bytes = (size_t)n * ndim * 8;
    Scratch a_buf(_ctx, sq_bytes), d_buf(_ctx, blk_bytes), x_buf(_ctx, x_bytes), al_buf(_ctx, (size_t)np * 8),
        wd_buf(_ctx, (size_t)np * 8), part_buf(_ctx, part_bytes);
    std::optional<Scratch> dxp_buf, dx_buf;
    if (want_dx) {
        dxp_buf.emplace(_ctx, dxp_bytes);
        dx_buf.emplace(_ctx, x_bytes);
    }
    CUDA_CHECK(cudaMemcpyAsync(a_buf.p, A, sq_bytes, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(d_buf.p, diagA, blk_bytes, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(x_buf.p, X, x_bytes, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemsetAsync(al_buf.p, 0, (size_t)np * 8, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(al_buf.p, alpha, (size_t)n * 8, cudaMemcpyHostToDevice, _ctx->stream));
    tg::contract(_ctx, T, a_buf.f64(), d_buf.f64(), P, G, x_buf.f64(), ndim, n, al_buf.f64(), wd_buf.f64(),
                 part_buf.f64(), want_dx ? dxp_buf->f64() : nullptr, want_dx ? dx_buf->f64() : nullptr);
    if (want_dx) {
        CUDA_CHECK(cudaMemcpyAsync(dxpart, dxp_buf->p, dxp_bytes, cudaMemcpyDeviceToHost, _ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(dX, dx_buf->p, x_bytes, cudaMemcpyDeviceToHost, _ctx->stream));
    }
    CUDA_CHECK(cudaMemcpyAsync(wdiag, wd_buf.p, (size_t)n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(partial, part_buf.p, part_bytes, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}
