// Dense DirectSolver path for sm_90a: pairwise kernel build (K1), blocked right-looking Cholesky
// whose panel/trailing updates run on the fp64 tensor pipe (DMMA, mma.sync.m16n8k16.f64, dmma.cuh) (K2),
// triangular solves + reductions behind log_probability (K3), L@z (K4).
//
// Reference behaviour being replaced: src/tinygp/solvers/direct.py:30-95 (DirectSolver),
// src/tinygp/kernels/base.py:84-103 (Kernel.__call__), src/tinygp/kernels/stationary.py:76-235,
// src/tinygp/kernels/distance.py:41-59, src/tinygp/noise.py:77-78.
//
// Data layout in HBM: one np x np row-major fp64 matrix (np = n rounded up to 128; the pad is an
// identity block so it contributes log 1 = 0 to the determinant), lower triangle significant.
// Row-major makes BOTH operands of every update  C_ij -= P_i P_j^T  K-contiguous (a panel row is
// a contiguous run of doubles), which is exactly the row.col operand form of mma.m16n8k16.f64.
#include "common.cuh"
#include "dmma.cuh"
#include <limits.h>
#include <optional>

// =============================================================================================
// kernel-program evaluation (device)
// =============================================================================================
#include "kprog.cuh"

KProg parse_prog(const double* prog, int n_rows, int ndim) { return parse_prog_impl(prog, n_rows, ndim); }

// =============================================================================================
// K1: pairwise kernel build.  out[(i)*ld + j] for i < rows_pad, j < cols_pad.
// =============================================================================================
struct BuildArgs {
    const double* X1;   // n1 x ndim
    const double* X2;   // n2 x ndim
    const double* diag; // indexed by global row, or null
    double* out;
    int64_t ld;
    int64_t n1, n2;          // valid extents (in units of out rows / cols, relative to row_off/col_off)
    int64_t rows_pad, cols_pad;
    int64_t row_off, col_off;  // global indices of out(0,0), used for the diagonal / identity pad
    int ndim;
    int pad_identity;  // padded entries: (grow==gcol) ? 1 : 0 instead of 0
    // batched build (blockIdx.z = problem): one program per problem, outputs batch_stride apart
    const KProg* progs;
    int64_t batch_stride;
    // batched single-leaf build: per-problem (coef, c0, c1) of build_rect_kernel_single (3 doubles per problem, device), the
    // common leaf's opcode and metric; lower_only: skip the tiles strictly right of the row's 128-wide diagonal tile column
    // (a factorisation reads the lower triangle only)
    const double* batch_consts;
    int batch_op, batch_l2;
    int lower_only;
};

#define BUILD_ROWS 32
#define BUILD_COLS 128
// FAST: the program in sum-of-products normal form (kprog.cuh KFast) -- no interpreter loop, no stack in local memory.
// The interpreted version keeps its 8-entry value stack in local memory.
template <bool FAST>
__global__ void __launch_bounds__(256, 3) build_rect_kernel_t(const __grid_constant__ KProg P0, const __grid_constant__ KFast F0,
                                                             const BuildArgs a) {
    __shared__ double x1s[BUILD_ROWS * MAX_NDIM];
    __shared__ double x2s[BUILD_COLS * MAX_NDIM];
    __shared__ KProg Pb;
    const int tid = threadIdx.x;
    if (a.progs != nullptr) {
        const int* src = reinterpret_cast<const int*>(a.progs + blockIdx.z);
        int* dst = reinterpret_cast<int*>(&Pb);
        for (int i = tid; i < (int)(sizeof(KProg) / sizeof(int)); i += 256) dst[i] = src[i];
    }
    const KProg& P = (a.progs != nullptr) ? Pb : P0;
    double* const outb = a.out + (int64_t)blockIdx.z * a.batch_stride;
    const int64_t r0 = (int64_t)blockIdx.y * BUILD_ROWS;
    const int64_t c0 = (int64_t)blockIdx.x * BUILD_COLS;
    if (a.lower_only && (c0 + a.col_off) / TILE > (r0 + a.row_off) / TILE) return;   // block-uniform
    const int nd = a.ndim;
    for (int i = tid; i < BUILD_ROWS * nd; i += 256) {
        const int64_t r = r0 + i / nd;
        x1s[i] = (r < a.n1) ? a.X1[r * nd + (i % nd)] : 0.0;
    }
    for (int i = tid; i < BUILD_COLS * nd; i += 256) {
        const int64_t c = c0 + i / nd;
        x2s[i] = (c < a.n2) ? a.X2[c * nd + (i % nd)] : 0.0;
    }
    __syncthreads();
    const int cl = (tid & 63) * 2;  // two consecutive columns per thread -> 16-byte stores, 512 B per warp
    const int rl0 = tid >> 6;       // 0..3
#pragma unroll 2
    for (int rr = 0; rr < BUILD_ROWS / 4; ++rr) {
        const int rl = rl0 + rr * 4;
        const int64_t r = r0 + rl;
        if (r >= a.rows_pad) break;
        double v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int64_t c = c0 + cl + e;
            const int64_t gr = r + a.row_off, gc = c + a.col_off;
            if (r < a.n1 && c < a.n2) {
                const double* xa = x1s + rl * nd;
                const double* xb = x2s + (cl + e) * nd;
                double k;
                if (FAST) k = kfast_eval(F0, nd, [&](int d) { return xa[d] - xb[d]; });
                else k = kprog_eval(P, nd, [&](int d) { return xa[d] - xb[d]; });
                if (a.diag != nullptr && gr == gc) k += a.diag[gr];
                v[e] = k;
            } else {
                v[e] = (a.pad_identity && gr == gc) ? 1.0 : 0.0;
            }
        }
        const int64_t c = c0 + cl;
        double* dst = outb + r * a.ld + c;
        if (c + 1 < a.cols_pad && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
            *reinterpret_cast<double2*>(dst) = make_double2(v[0], v[1]);
        } else {
            if (c < a.cols_pad) dst[0] = v[0];
            if (c + 1 < a.cols_pad) dst[1] = v[1];
        }
    }
}

// SINGLE: coef * one stationary leaf, identity metric, 1-3 dimensions, everything about the program a template parameter --
// the shape of the benchmark workloads (`amp * ExpSquared(scale)`) and of most hyper-parameter searches.  The normal-form
// kernel above spends most of its instructions on loop / predicate / runtime-dispatch overhead around one fp64 exp.  Here a thread keeps its two columns'
// coordinates in registers, the row coordinates come from shared memory as broadcasts, model constants are folded on the
// host (1 / scale^2: one rounding in the argument, within the 1e-13 parity tolerance), and tiles that touch neither the
// diagonal nor the padding run without a single predicate.  Boundary / diagonal tiles take the general element path.
template <int OP, bool L2, int ND>
__device__ __forceinline__ double single_leaf(const double (&xa)[ND], const double (&xb)[ND], const double c0, const double c1) {
    double l1 = 0.0, l2sq = 0.0;
#pragma unroll
    for (int d = 0; d < ND; ++d) {
        const double df = xa[d] - xb[d];
        if (L2) l2sq = fma(df, df, l2sq);
        else l1 += fabs(df);
    }
    if (OP == B200GP_OP_EXPSQUARED) return exp((L2 ? l2sq : l1 * l1) * c0);            // c0 = -0.5 / scale^2
    const double dist = L2 ? sqrt(l2sq) : l1;                                          // sqrt(0) = 0 = the reference's guard value
    const double r = dist * c0;                                                        // c0 = sqrt3|sqrt5|1 / scale
    if (OP == B200GP_OP_EXP) return exp(-r);
    if (OP == B200GP_OP_MATERN32) return (1.0 + r) * exp(-r);
    return (1.0 + r + r * r * c1) * exp(-r);                                           // MATERN52, c1 = 1/3
}

template <int OP, bool L2, int ND>
__global__ void __launch_bounds__(256, 3) build_rect_kernel_single(const BuildArgs a_in, const double coef_in, const double c0_in,
                                                                   const double c1_in) {
    __shared__ double x1s[BUILD_ROWS * ND];
    const int tid = threadIdx.x;
    const int64_t r0 = (int64_t)blockIdx.y * BUILD_ROWS;
    const int64_t c0g = (int64_t)blockIdx.x * BUILD_COLS;
    BuildArgs a = a_in;
    if (a.lower_only && (c0g + a.col_off) / TILE > (r0 + a.row_off) / TILE) return;   // block-uniform
    double coef = coef_in, c0 = c0_in, c1 = c1_in;
    if (a.batch_consts != nullptr) {     // blockIdx.z = problem: its own amplitude / scale, its own output matrix
        const double* bc = a.batch_consts + 3 * (int64_t)blockIdx.z;
        coef = bc[0]; c0 = bc[1]; c1 = bc[2];
        a.out += (int64_t)blockIdx.z * a.batch_stride;
    }
    for (int i = tid; i < BUILD_ROWS * ND; i += 256) {
        const int64_t r = r0 + i / ND;
        x1s[i] = (r < a.n1) ? a.X1[r * ND + (i % ND)] : 0.0;
    }
    const int cl = (tid & 63) * 2;  // two consecutive columns per thread -> 16-byte stores, 512 B per warp
    const int rl0 = tid >> 6;       // 0..3
    double xb[2][ND];
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int d = 0; d < ND; ++d) {
            const int64_t c = c0g + cl + e;
            xb[e][d] = (c < a.n2) ? a.X2[c * ND + d] : 0.0;
        }
    __syncthreads();
    // interior tile: all rows / columns valid, not on the diagonal of the global matrix, 16-byte aligned rows
    const int64_t gr0 = r0 + a.row_off, gc0 = c0g + a.col_off;
    const bool interior = (r0 + BUILD_ROWS <= a.n1) && (c0g + BUILD_COLS <= a.n2) && (r0 + BUILD_ROWS <= a.rows_pad) &&
                          (c0g + BUILD_COLS <= a.cols_pad) && (gr0 + BUILD_ROWS <= gc0 || gc0 + BUILD_COLS <= gr0) &&
                          ((reinterpret_cast<uintptr_t>(a.out + r0 * a.ld + c0g) | (uintptr_t)(a.ld * 8)) & 15) == 0;
    if (interior) {
        double* dst = a.out + (r0 + rl0) * a.ld + c0g + cl;
        const int64_t step = 4 * a.ld;
#pragma unroll 4
        for (int rr = 0; rr < BUILD_ROWS / 4; ++rr) {
            double xa[ND];
#pragma unroll
            for (int d = 0; d < ND; ++d) xa[d] = x1s[(rl0 + rr * 4) * ND + d];
            const double v0 = coef * single_leaf<OP, L2, ND>(xa, xb[0], c0, c1);
            const double v1 = coef * single_leaf<OP, L2, ND>(xa, xb[1], c0, c1);
            *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
            dst += step;
        }
        return;
    }
    for (int rr = 0; rr < BUILD_ROWS / 4; ++rr) {
        const int rl = rl0 + rr * 4;
        const int64_t r = r0 + rl;
        if (r >= a.rows_pad) break;
        double xa[ND];
#pragma unroll
        for (int d = 0; d < ND; ++d) xa[d] = x1s[rl * ND + d];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int64_t c = c0g + cl + e;
            if (c >= a.cols_pad) continue;
            const int64_t gr = r + a.row_off, gc = c + a.col_off;
            double v;
            if (r < a.n1 && c < a.n2) {
                v = coef * single_leaf<OP, L2, ND>(xa, xb[e], c0, c1);
                if (a.diag != nullptr && gr == gc) v += a.diag[gr];
            } else {
                v = (a.pad_identity && gr == gc) ? 1.0 : 0.0;
            }
            a.out[r * a.ld + c] = v;
        }
    }
}

template <int OP, bool L2>
static void launch_single_nd(cudaStream_t st, dim3 grid, const BuildArgs& a, double coef, double c0, double c1) {
    switch (a.ndim) {
        case 1: build_rect_kernel_single<OP, L2, 1><<<grid, 256, 0, st>>>(a, coef, c0, c1); break;
        case 2: build_rect_kernel_single<OP, L2, 2><<<grid, 256, 0, st>>>(a, coef, c0, c1); break;
        default: build_rect_kernel_single<OP, L2, 3><<<grid, 256, 0, st>>>(a, coef, c0, c1); break;
    }
}
// (coef, c0, c1) of build_rect_kernel_single for a single-leaf normal form; false if the leaf has no compiled kernel
static bool single_constants(const KFast& F, double* out3) {
    if (F.nleaf != 1 || F.nterm != 1 || F.mask[0] != 1) return false;
    const double p0 = F.p0[0];
    out3[0] = F.coef[0]; out3[2] = 0.0;
    switch (F.op[0]) {
        case B200GP_OP_EXPSQUARED: out3[1] = -0.5 / (p0 * p0); return true;
        case B200GP_OP_EXP: out3[1] = 1.0 / p0; return true;
        case B200GP_OP_MATERN32: out3[1] = SQRT3 / p0; return true;
        case B200GP_OP_MATERN52: out3[1] = SQRT5 / p0; out3[2] = 1.0 / 3.0; return true;
        default: return false;
    }
}

// true if the program is coef * (one stationary leaf) of a kind compiled above and the launch was made
static bool launch_build_single(b200gp_ctx* ctx, dim3 grid, const KFast& F, const BuildArgs& a) {
    if (ctx->build_fast < 2 || F.nleaf != 1 || F.nterm != 1 || F.mask[0] != 1 || a.ndim < 1 || a.ndim > 3) return false;
    if (grid.z != 1 && a.batch_consts == nullptr) return false;
    const double coef = F.coef[0], p0 = F.p0[0];
    const bool l2 = F.l2[0] != 0;
    cudaStream_t st = ctx->stream;
#define SINGLE(OPv, C0, C1) \
    do { if (l2) launch_single_nd<OPv, true>(st, grid, a, coef, (C0), (C1)); else launch_single_nd<OPv, false>(st, grid, a, coef, (C0), (C1)); return true; } while (0)
    switch (F.op[0]) {
        case B200GP_OP_EXPSQUARED: SINGLE(B200GP_OP_EXPSQUARED, -0.5 / (p0 * p0), 0.0);
        case B200GP_OP_EXP: SINGLE(B200GP_OP_EXP, 1.0 / p0, 0.0);
        case B200GP_OP_MATERN32: SINGLE(B200GP_OP_MATERN32, SQRT3 / p0, 0.0);
        case B200GP_OP_MATERN52: SINGLE(B200GP_OP_MATERN52, SQRT5 / p0, 1.0 / 3.0);
        default: return false;
    }
#undef SINGLE
}

// single-leaf specialisation (option "build_fast" = 2, default), else the normal form when the program has one
// ("build_fast" >= 1), else the interpreter (also for batched programs)
static void launch_build_rect(b200gp_ctx* ctx, dim3 grid, const KProg& prog, const BuildArgs& a) {
    KFast F{};
    if (a.progs != nullptr && a.batch_consts != nullptr) {   // batched hyper-parameter grid of one single-leaf kernel
        F.nleaf = F.nterm = 1; F.mask[0] = 1; F.op[0] = a.batch_op; F.l2[0] = a.batch_l2; F.p0[0] = 1.0; F.coef[0] = 1.0;
        if (launch_build_single(ctx, grid, F, a)) return;
    }
    if (a.progs == nullptr && ctx->build_fast != 0 && kprog_to_fast(prog, F)) {
        if (launch_build_single(ctx, grid, F, a)) return;
        build_rect_kernel_t<true><<<grid, 256, 0, ctx->stream>>>(prog, F, a);
    } else {
        build_rect_kernel_t<false><<<grid, 256, 0, ctx->stream>>>(prog, F, a);
    }
}

// diag: out[i] = k(x_i, x_i)
__global__ void build_diag_kernel(const __grid_constant__ KProg P, int64_t n, double* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = kprog_eval_zero(P);
}

// out[i] = sum_j k(X1_i, X2_j) y_j   (Kernel.matmul, base.py:68-82) -- one warp per row
__global__ void __launch_bounds__(256) kernel_matvec_kernel(const __grid_constant__ KProg P, const double* X1, int64_t n1,
                                                            const double* X2, int64_t n2, int ndim,
                                                            const double* y, double* out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * 8 + warp;
    if (i >= n1) return;
    double xi[MAX_NDIM];
    for (int d = 0; d < ndim; ++d) xi[d] = X1[i * ndim + d];
    double acc = 0.0;
    for (int64_t j = lane; j < n2; j += 32) {
        const double* xj = X2 + j * ndim;
        acc += kprog_eval(P, ndim, [&](int d) { return xi[d] - xj[d]; }) * y[j];
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) out[i] = acc;
}

void dense_build_rect(b200gp_ctx* ctx, const KProg& prog, const double* X1, int64_t n1,
                      const double* X2, int64_t n2, int ndim, const double* diag_or_null,
                      double* out, int64_t ld, int64_t rows_pad, int64_t cols_pad) {
    BuildArgs a{};
    a.X1 = X1; a.X2 = X2; a.diag = diag_or_null; a.out = out; a.ld = ld;
    a.n1 = n1; a.n2 = n2; a.rows_pad = rows_pad; a.cols_pad = cols_pad;
    a.row_off = 0; a.col_off = 0; a.ndim = ndim; a.pad_identity = (diag_or_null != nullptr);
    dim3 grid((unsigned)((cols_pad + BUILD_COLS - 1) / BUILD_COLS), (unsigned)((rows_pad + BUILD_ROWS - 1) / BUILD_ROWS));
    ProfTimer t(ctx, &ctx->prof.build_ms);
    launch_build_rect(ctx, grid, prog, a);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
    ctx->prof.build_bytes += 8.0 * (double)rows_pad * (double)cols_pad;
}

// =============================================================================================
// K2 core: NT GEMM on the fp64 tensor pipe.   C (op)= alpha * A(MxK) * B(NxK)^T
// The 128 x 128 CTA tile's mainloop is dmma.cuh's cta_tile_nt (DMMA m16n8k16, 3-slot cp.async ring), which grad.cu's
// tile kernel runs too; this kernel adds the tile schedules and the beta_mode epilogues.
// =============================================================================================
namespace gemm {
using dmma::BM; using dmma::SK; using dmma::THREADS; using dmma::SMEM_BYTES;
constexpr int BAND = 16;  // tile rows per rasterisation band (L2 reuse of the panel operands)
constexpr int C_PREFETCH = 2;   // stages (64 of K) before the end of K at which a beta_mode 1 tile of C is prefetched into L2

struct Args {
    const double* A; int64_t lda;
    const double* B; int64_t ldb;
    double* C; int64_t ldc;
    int tiles_m, tiles_n, K;
    double alpha;
    int beta_mode;  // 0: C = alpha AB ; 1: C += alpha AB ; 2: C = generator + alpha AB
    int lower;      // 1: square C, only tiles with tj <= ti are computed
    // generator (beta_mode 2): C(i,j) = k(x_{row0+i}, x_{col0+j}) + [row==col] diag
    const double* X; const double* diag; int ndim; int64_t n_valid; int64_t row0, col0;
    // batched launch (blockIdx.y = problem): element strides between problems
    int batch; int64_t strideA, strideB, strideC;
};

// linear CTA index -> lower-triangular tile (ti, tj), banded so that concurrently resident CTAs
// share 16 A row-panels and a handful of B row-panels (both stay in L2).
__device__ __forceinline__ void lower_tile(int b, int T, int& ti, int& tj) {
    int R = 0;
    for (;;) {
        const int h = min(BAND, T - R * BAND);
        const int cnt = R * BAND * h + h * (h + 1) / 2;
        if (b < cnt) {
            const int full = R * BAND * h;
            if (b < full) {
                tj = b / h;
                ti = R * BAND + b % h;
            } else {
                b -= full;
                int r = 0;
                while (b >= r + 1) { b -= r + 1; ++r; }
                ti = R * BAND + r;
                tj = R * BAND + b;
            }
            return;
        }
        b -= cnt;
        ++R;
    }
}

// LOWER = true is the trailing SYRK update (the N^3/3 kernel); false = panel / rectangular GEMMs.  Two
// instantiations so that profilers list them separately.
template <bool LOWER>
__global__ void __launch_bounds__(THREADS, 1) gemm_nt_kernel(const __grid_constant__ KProg P, const Args g) {
    extern __shared__ __align__(16) double smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp >> 2, wn = warp & 3;

    int ti, tj;
    if (LOWER) {
        lower_tile((int)blockIdx.x, g.tiles_m, ti, tj);
    } else {
        ti = (int)blockIdx.x % g.tiles_m;
        tj = (int)blockIdx.x / g.tiles_m;
    }
    const int64_t bz = blockIdx.y;
    const double* Ag = g.A + bz * g.strideA + (int64_t)ti * BM * g.lda;
    const double* Bg = g.B + bz * g.strideB + (int64_t)tj * BM * g.ldb;

    double acc[8][4][2];
    const int KT = g.K / SK;
    dmma::cta_tile_nt(
        acc, smem, KT,
        [&](int kc) { return dmma::Operands{Ag, g.lda, Bg, g.ldb, (int64_t)kc * SK}; },
        [&](int kc) {
            if (g.beta_mode == 1 && kc == (KT > C_PREFETCH ? KT - C_PREFETCH : 0)) {
                // the C tile (128 rows x 8 lines of 128 B) into L2, so that the epilogue's reads do not wait on HBM
#pragma unroll
                for (int i = 0; i < BM * BM / 16 / THREADS; ++i) {
                    const int line = tid + i * THREADS;
                    const double* p = g.C + bz * g.strideC + ((int64_t)ti * BM + (line >> 3)) * g.ldc +
                                      (int64_t)tj * BM + (line & 7) * 16;
                    asm volatile("prefetch.global.L2 [%0];\n" ::"l"(p));
                }
            }
        });

    // epilogue: acc[mi][ni][q] is C(row0 + acc_row(mi), col0 + acc_col(ni, q)); q = 0, 1 are adjacent columns
    const int64_t crow0 = (int64_t)ti * BM + wm * dmma::WM;
    const int64_t ccol0 = (int64_t)tj * BM + wn * dmma::WN;
    if (g.beta_mode == 1) {
        // C += alpha AB.  Two accumulator rows' reads are issued before any of their writes: one read-write round trip
        // per element would serialise 32 memory latencies per thread (the compiler cannot move a read of C above a
        // write to C).
#pragma unroll
        for (int mi = 0; mi < 8; mi += 2) {
            double* crow[2];
            double2 v[2][4];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                crow[h] = g.C + bz * g.strideC + (crow0 + dmma::acc_row(lane, mi + h)) * g.ldc;
#pragma unroll
                for (int ni = 0; ni < 4; ++ni)
                    v[h][ni] = *reinterpret_cast<const double2*>(crow[h] + ccol0 + dmma::acc_col(lane, ni, 0));
            }
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    v[h][ni].x += g.alpha * acc[mi + h][ni][0];
                    v[h][ni].y += g.alpha * acc[mi + h][ni][1];
                    *reinterpret_cast<double2*>(crow[h] + ccol0 + dmma::acc_col(lane, ni, 0)) = v[h][ni];
                }
        }
        return;
    }
#pragma unroll
    for (int mi = 0; mi < 8; ++mi) {
        const int64_t r = crow0 + dmma::acc_row(lane, mi);
        double* crow = g.C + bz * g.strideC + r * g.ldc;
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
            const int64_t c = ccol0 + dmma::acc_col(lane, ni, 0);
            double2 v;
            if (g.beta_mode == 2) {
                const int64_t gr = g.row0 + r;
                double e[2];
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int64_t gc = g.col0 + c + q;
                    if (gr < g.n_valid && gc < g.n_valid) {
                        const double* xa = g.X + gr * g.ndim;
                        const double* xb = g.X + gc * g.ndim;
                        e[q] = kprog_eval(P, g.ndim, [&](int d) { return xa[d] - xb[d]; });
                        if (gr == gc) e[q] += g.diag[gr];
                    } else {
                        e[q] = (gr == gc) ? 1.0 : 0.0;
                    }
                }
                v = make_double2(e[0], e[1]);
            } else {
                v = make_double2(0.0, 0.0);
            }
            v.x += g.alpha * acc[mi][ni][0];
            v.y += g.alpha * acc[mi][ni][1];
            *reinterpret_cast<double2*>(crow + c) = v;
        }
    }
}

static bool g_attr_set = false;
static void launch(b200gp_ctx* ctx, const KProg& P, const Args& g) {
    if (!g_attr_set) {
        CUDA_CHECK(cudaFuncSetAttribute(gemm_nt_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        CUDA_CHECK(cudaFuncSetAttribute(gemm_nt_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        g_attr_set = true;
    }
    int64_t ntiles;
    if (g.lower)
        ntiles = (int64_t)g.tiles_m * (g.tiles_m + 1) / 2;
    else
        ntiles = (int64_t)g.tiles_m * g.tiles_n;
    if (ntiles <= 0) return;
    dim3 grid((unsigned)ntiles, (unsigned)(g.batch > 0 ? g.batch : 1));
    if (g.lower)
        gemm_nt_kernel<true><<<grid, THREADS, SMEM_BYTES, ctx->stream>>>(P, g);
    else
        gemm_nt_kernel<false><<<grid, THREADS, SMEM_BYTES, ctx->stream>>>(P, g);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
}
}  // namespace gemm

static const KProg& empty_prog() {
    static KProg p{};
    return p;
}

void gemm_nt(b200gp_ctx* ctx, double* C, int64_t ldc, const double* A, int64_t lda, const double* B, int64_t ldb,
             int tiles_m, int tiles_n, int K, double alpha, int beta_mode, int lower, int batch, int64_t strideA,
             int64_t strideB, int64_t strideC) {
    gemm::Args g{};
    g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.C = C; g.ldc = ldc;
    g.tiles_m = tiles_m; g.tiles_n = tiles_n; g.K = K; g.alpha = alpha;
    g.beta_mode = beta_mode; g.lower = lower;
    g.batch = batch; g.strideA = strideA; g.strideB = strideB; g.strideC = strideC;
    gemm::launch(ctx, empty_prog(), g);
}

// =============================================================================================
// diagonal block: Cholesky of a 128 x 128 block and its triangular inverse, in shared memory (row stride 129 doubles),
// one CTA of 512 threads per block (a batched launch: one CTA per problem).
// The Cholesky is right-looking in steps of 8 columns: every thread that owns a row of the 8-column panel factors the
// panel's 8 x 8 diagonal block redundantly in registers (no barrier inside) and solves its own row against it; the rank-8
// update of the trailing triangle then runs on 4 x 4 register tiles (2 FMAs per shared-memory load).  The inverse is
// built in place 8 columns at a time from the right; thread (part = tid / 128, i = tid % 128) sums a quarter of row i's
// dot products.  The first bad pivot (NaN or <= 0) goes to *info as global_off + its column + 1 (atomicMin).
// =============================================================================================
#define PF_LD 129
#define PF_THREADS 512
constexpr int PF_SMEM = (TILE * PF_LD + TILE * 8 + 4 * TILE * 8) * (int)sizeof(double);

__global__ void __launch_bounds__(PF_THREADS, 1) potf2_trtri_kernel(double* A, int64_t lda, double* linv, int* info,
                                                                    int global_off, int64_t strideA,
                                                                    int64_t stride_linv) {
    extern __shared__ __align__(16) double sm[];
    A += (int64_t)blockIdx.x * strideA;
    linv += (int64_t)blockIdx.x * stride_linv;
    info += blockIdx.x;
    double* S = sm;                       // TILE x PF_LD
    double* T = sm + TILE * PF_LD;        // TILE x 8 : column block of L being inverted
    double* red = T + TILE * 8;           // 4 x TILE x 8 partial sums
    const int tid = threadIdx.x;
    const int i = tid & (TILE - 1);
    const int part = tid >> 7;

    for (int e = tid; e < TILE * TILE; e += PF_THREADS) {
        const int r = e >> 7, c = e & (TILE - 1);
        S[r * PF_LD + c] = (c <= r) ? A[(int64_t)r * lda + c] : 0.0;
    }
    __syncthreads();

    // ---------------- phase 1: Cholesky ----------------
    for (int jb = 0; jb < TILE / 8; ++jb) {
        const int j0 = jb * 8;
        // load phase (diagonal block + own row), then a barrier: the stores below overwrite what others read here
        const bool owner = (tid < TILE && tid >= j0);
        double D[8][8], arow[8];
        if (owner) {
#pragma unroll
            for (int a = 0; a < 8; ++a)
#pragma unroll
                for (int b = 0; b <= a; ++b) D[a][b] = S[(j0 + a) * PF_LD + j0 + b];
#pragma unroll
            for (int c = 0; c < 8; ++c) arow[c] = S[tid * PF_LD + j0 + c];
        }
        __syncthreads();
        if (owner) {
            const int r = tid;
            int firstbad = -1;
            double invd[8];     // 1 / L_cc: the column is scaled by the reciprocal (as LAPACK's dpotf2 does with DSCAL), which
                                // takes the 36 fp64 divisions per 8 x 8 block out of the serial chain
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                double v = D[c][c];
#pragma unroll
                for (int k = 0; k < c; ++k) v -= D[c][k] * D[c][k];
                if (!(v > 0.0) && firstbad < 0) firstbad = c;
                const double sq = sqrt(v);
                const double isq = 1.0 / sq;
                D[c][c] = sq;
                invd[c] = isq;
#pragma unroll
                for (int a = c + 1; a < 8; ++a) {
                    double w = D[a][c];
#pragma unroll
                    for (int k = 0; k < c; ++k) w -= D[a][k] * D[c][k];
                    D[a][c] = w * isq;
                }
            }
            if (r == j0 && firstbad >= 0) atomicMin(info, global_off + j0 + firstbad + 1);
            if (r < j0 + 8) {
                // every owner of a diagonal-block row holds the same factored block: one of them stores it all
                // (static register indices; a per-row select would push D into local memory)
                if (r == j0) {
#pragma unroll
                    for (int a = 0; a < 8; ++a)
#pragma unroll
                        for (int b = 0; b <= a; ++b) S[(j0 + a) * PF_LD + j0 + b] = D[a][b];
                }
            } else {
                double x[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    double w = arow[c];
#pragma unroll
                    for (int k = 0; k < c; ++k) w -= x[k] * D[c][k];
                    x[c] = w * invd[c];
                }
#pragma unroll
                for (int c = 0; c < 8; ++c) S[r * PF_LD + j0 + c] = x[c];
            }
        }
        __syncthreads();
        const int m = TILE - j0 - 8;
        if (m > 0) {
            const int nt = m >> 2, ntiles = nt * (nt + 1) / 2;
            for (int e = tid; e < ntiles; e += PF_THREADS) {
                int ti = (int)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);
                while ((ti + 1) * (ti + 2) / 2 <= e) ++ti;
                while (ti * (ti + 1) / 2 > e) --ti;
                const int tj = e - ti * (ti + 1) / 2;
                const int i0 = j0 + 8 + 4 * ti, c0 = j0 + 8 + 4 * tj;
                double acc[4][4];
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
#pragma unroll
                for (int k = 0; k < 8; ++k) {   // 8 loads feed 16 FMAs; no big register arrays
                    double lr[4], lc[4];
#pragma unroll
                    for (int a = 0; a < 4; ++a) {
                        lr[a] = S[(i0 + a) * PF_LD + j0 + k];
                        lc[a] = S[(c0 + a) * PF_LD + j0 + k];
                    }
#pragma unroll
                    for (int a = 0; a < 4; ++a)
#pragma unroll
                        for (int b = 0; b < 4; ++b) acc[a][b] += lr[a] * lc[b];
                }
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b)
                        if (c0 + b <= i0 + a) S[(i0 + a) * PF_LD + c0 + b] -= acc[a][b];
            }
        }
        __syncthreads();
    }

    for (int e = tid; e < TILE * TILE; e += PF_THREADS) {
        const int r = e >> 7, c = e & (TILE - 1);
        if (c <= r) A[(int64_t)r * lda + c] = S[r * PF_LD + c];
    }
    __syncthreads();

    // ---------------- phase 2: X = L^-1 in place, 8 columns at a time from the right ----------------
    //   X[i, jb] = -( sum_{k > jb-block, k <= i} X[i,k] L[k, jb] ) inv(L[jb,jb]) ,   X[jb,jb] = inv(L[jb,jb])
    for (int jb = TILE / 8 - 1; jb >= 0; --jb) {
        const int j0 = jb * 8;
        for (int e = tid; e < TILE * 8; e += PF_THREADS) {
            const int k = e >> 3, c = e & 7;
            T[e] = (k >= j0) ? S[k * PF_LD + j0 + c] : 0.0;
        }
        __syncthreads();
        double acc[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] = 0.0;
        if (i >= j0 + 8) {
            const double* ri = S + i * PF_LD;
            for (int k = j0 + 8 + part; k <= i; k += 4) {
                const double xik = ri[k];
#pragma unroll
                for (int c = 0; c < 8; ++c) acc[c] += xik * T[k * 8 + c];
            }
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) red[(part * TILE + i) * 8 + c] = acc[c];
        __syncthreads();
        if (part == 0 && i >= j0) {
            // inverse of the 8x8 lower diagonal block (rows j0..j0+7 of T), in registers
            double Di[8][8], rd[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) rd[c] = 1.0 / T[(j0 + c) * 8 + c];     // 8 independent reciprocals, then only FMAs
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                Di[c][c] = rd[c];
#pragma unroll
                for (int a = c + 1; a < 8; ++a) {
                    double w = 0.0;
#pragma unroll
                    for (int k = c; k < a; ++k) w += T[(j0 + a) * 8 + k] * Di[k][c];
                    Di[a][c] = -w * rd[a];
                }
            }
            if (i < j0 + 8) {
                if (i == j0) {
#pragma unroll
                    for (int a = 0; a < 8; ++a)
#pragma unroll
                        for (int c = 0; c <= a; ++c) S[(j0 + a) * PF_LD + j0 + c] = Di[a][c];
                }
            } else {
                double v[8];
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    v[c] = red[i * 8 + c] + red[(TILE + i) * 8 + c] + red[(2 * TILE + i) * 8 + c] + red[(3 * TILE + i) * 8 + c];
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    double w = 0.0;
#pragma unroll
                    for (int cp = c; cp < 8; ++cp) w += v[cp] * Di[cp][c];
                    S[i * PF_LD + j0 + c] = -w;
                }
            }
        }
        __syncthreads();
    }
    for (int e = tid; e < TILE * TILE; e += PF_THREADS) {
        const int r = e >> 7, c = e & (TILE - 1);
        linv[e] = (c <= r) ? S[r * PF_LD + c] : 0.0;
    }
}

static void potf2(b200gp_ctx* ctx, double* A, int64_t lda, double* linv, int* info, int global_off, int batch = 1,
                  int64_t strideA = 0, int64_t stride_linv = 0) {
    static bool attr = false;
    if (!attr) {
        CUDA_CHECK(cudaFuncSetAttribute(potf2_trtri_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PF_SMEM));
        attr = true;
    }
    potf2_trtri_kernel<<<batch, PF_THREADS, PF_SMEM, ctx->stream>>>(A, lda, linv, info, global_off, strideA, stride_linv);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
}

// =============================================================================================
// blocked right-looking Cholesky driver (outer panel nb, 128-wide tile columns inside a panel)
// =============================================================================================
__global__ void set_int_kernel(int* p, int v) { *p = v; }

// Panel factorisation of the columns [k0, k0+kb), one 128-wide tile column at a time.  The kb x kb DIAGONAL BLOCK is
// factored by a chain of small kernels whose length is set by the serial 128 x 128 potf2 steps, while the rows BELOW the
// block are updated / solved on the caller's stream, tile column by tile column, as soon as the potf2 of that column has
// produced inv(L_jj).  The wide GEMMs do not wait for the next potf2 and vice versa, so per panel the time is
// ~max(potf2 chain, wide GEMMs) instead of their sum.
// Inside the diagonal block the order is right-looking: after a tile column is solved, the remaining (blk - 1) x (blk - 1)
// lower tiles of the block are updated with K = 128 (up to 28 tiles in parallel) instead of each tile column being updated
// just before its potf2 with K = j0 (1-7 tiles, a single CTA running the longest K).  The rows below are updated
// left-looking: tile column c0 of them with K = j0 (all earlier columns of the panel) just before its solve.
// [r0, r1): the rows below the block this call solves.  The sharded path passes its rank's chunk (every rank factors the
// diagonal block redundantly); the tiles and their arithmetic do not depend on the range, so the rows a rank produces are
// bit-identical to the unsharded run.
void dense_panel_factor_rows(b200gp_dense* s, int64_t k0, int64_t kb, int64_t r0, int64_t r1) {
    b200gp_ctx* ctx = s->ctx;
    const int64_t np = s->np, ld = s->ld;
    double* M = s->mat;
    const int64_t bend = k0 + kb;
    const int64_t lo = (r0 > bend) ? r0 : bend, hi = (r1 < np) ? r1 : np;
    if (lo % TILE || hi % TILE) throw GpError("panel_factor_rows: row range must be 128-aligned");
    const int own = (hi > lo) ? (int)((hi - lo) / TILE) : 0;
    cudaStream_t wide = ctx->stream;            // the caller's stream keeps the wide GEMMs (and the ProfTimer events)
    // The chain of small kernels runs on a HIGH-PRIORITY stream: when an SM frees up, the block scheduler then places the
    // chain's CTA before the pending CTAs of the wide GEMM grid.  (First attempt, chain on the default-priority stream and
    // GEMMs on a side stream: no overlap at all -- the potf2 CTA queued behind every pending GEMM CTA.)
    if (!ctx->stream_hi) {
        int lo = 0, hi = 0;
        CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        CUDA_CHECK(cudaStreamCreateWithPriority(&ctx->stream_hi, cudaStreamNonBlocking, hi));
    }
    cudaStream_t chain = ctx->stream_hi;
    cudaEvent_t ev = ctx->get_event();
    struct Restore { b200gp_ctx* c; cudaStream_t st; ~Restore() { c->stream = st; } } restore{ctx, wide};
    CUDA_CHECK(cudaEventRecord(ev, wide));      // the chain must see the block column as the caller left it
    CUDA_CHECK(cudaStreamWaitEvent(chain, ev, 0));
    for (int64_t j0 = 0; j0 < kb; j0 += TILE) {
        const int64_t c0 = k0 + j0;
        const int blk = (int)((bend - c0) / TILE);
        const double* li = s->linv + (c0 / TILE) * TILE * TILE;
        ctx->stream = chain;
        potf2(ctx, M + c0 * ld + c0, ld, s->linv + (c0 / TILE) * TILE * TILE, s->info_dev, (int)c0);
        if (own) CUDA_CHECK(cudaEventRecord(ev, chain));            // L[c0 rows, k0..c0) and inv(L_jj) are final here
        if (blk > 1) {
            gemm_nt(ctx, M + (c0 + TILE) * ld + c0, ld, M + (c0 + TILE) * ld + c0, ld, li, TILE, blk - 1, 1, TILE, 1.0, 0, 0);
            // trailing tiles of the diagonal block: C -= X X^T, X = the tile column just solved
            gemm_nt(ctx, M + (c0 + TILE) * ld + (c0 + TILE), ld, M + (c0 + TILE) * ld + c0, ld, M + (c0 + TILE) * ld + c0, ld,
                    blk - 1, blk - 1, TILE, -1.0, 1, 1);
        }
        if (own) {
            CUDA_CHECK(cudaStreamWaitEvent(wide, ev, 0));
            ctx->stream = wide;
            if (j0 > 0) gemm_nt(ctx, M + lo * ld + c0, ld, M + lo * ld + k0, ld, M + c0 * ld + k0, ld, own, 1, (int)j0, -1.0, 1, 0);
            gemm_nt(ctx, M + lo * ld + c0, ld, M + lo * ld + c0, ld, li, TILE, own, 1, TILE, 1.0, 0, 0);
        }
    }
    ctx->stream = wide;
    CUDA_CHECK(cudaEventRecord(ev, chain));     // join: the last block-row solve
    CUDA_CHECK(cudaStreamWaitEvent(wide, ev, 0));
    ctx->event_pool.push_back(ev);
}

// the whole panel: every row below the diagonal block
void dense_panel_factor(b200gp_dense* s, int64_t k0, int64_t kb) { dense_panel_factor_rows(s, k0, kb, k0 + kb, s->np); }

// generate K (+ diag, identity pad) for rows [r0, np), columns [c0, c0+ncols) straight into the matrix
void dense_build_region(b200gp_dense* s, int64_t r0, int64_t c0, int64_t ncols) {
    b200gp_ctx* ctx = s->ctx;
    const int64_t np = s->np, ld = s->np;
    BuildArgs a{};
    a.X1 = s->X_dev + r0 * s->ndim;
    a.X2 = s->X_dev + c0 * s->ndim;
    a.diag = s->diag_dev; a.out = s->mat + r0 * ld + c0; a.ld = ld;
    a.n1 = (s->n > r0) ? (s->n - r0) : 0;
    a.n2 = (s->n > c0) ? ((s->n - c0 < ncols) ? (s->n - c0) : ncols) : 0;
    a.rows_pad = np - r0; a.cols_pad = ncols;
    a.row_off = r0; a.col_off = c0; a.ndim = s->ndim; a.pad_identity = 1;
    dim3 grid((unsigned)((ncols + BUILD_COLS - 1) / BUILD_COLS), (unsigned)((np - r0 + BUILD_ROWS - 1) / BUILD_ROWS));
    ProfTimer t(ctx, &ctx->prof.build_ms);
    launch_build_rect(ctx, grid, s->prog, a);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
    ctx->prof.build_bytes += 8.0 * (double)(np - r0) * (double)ncols;
}

double dense_kernel_diag_value(const KProg& P) { return kprog_eval_zero(P); }

// rows [r0, r1) x columns [c0, c0+ncols) only (multi-GPU row sharding)
struct BuildRegionArgs { int64_t r0, r1, c0, ncols; };
void dense_build_rows(b200gp_dense* s, const BuildRegionArgs& q) {
    b200gp_ctx* ctx = s->ctx;
    const int64_t ld = s->ld;
    BuildArgs a{};
    a.X1 = s->X_dev + q.r0 * s->ndim;
    a.X2 = s->X_dev + q.c0 * s->ndim;
    a.diag = s->diag_dev; a.out = s->mat + q.r0 * ld + q.c0; a.ld = ld;
    a.n1 = (s->n > q.r0) ? ((s->n - q.r0 < q.r1 - q.r0) ? (s->n - q.r0) : (q.r1 - q.r0)) : 0;
    a.n2 = (s->n > q.c0) ? ((s->n - q.c0 < q.ncols) ? (s->n - q.c0) : q.ncols) : 0;
    a.rows_pad = q.r1 - q.r0; a.cols_pad = q.ncols;
    a.row_off = q.r0; a.col_off = q.c0; a.ndim = s->ndim; a.pad_identity = 1;
    dim3 grid((unsigned)((q.ncols + BUILD_COLS - 1) / BUILD_COLS), (unsigned)((q.r1 - q.r0 + BUILD_ROWS - 1) / BUILD_ROWS));
    ProfTimer t(ctx, &ctx->prof.build_ms);
    launch_build_rect(ctx, grid, s->prog, a);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
    ctx->prof.build_bytes += 8.0 * (double)(q.r1 - q.r0) * (double)q.ncols;
}

void dense_factor_ozaki(b200gp_dense* s, int S);  // ozaki.cu

void dense_factor_inplace(b200gp_dense* s, bool generate) {
    b200gp_ctx* ctx = s->ctx;
    const int64_t np = s->np, ld = s->np;
    int64_t NB = ctx->nb;
    if (NB < TILE) NB = TILE;
    NB = (NB / TILE) * TILE;
    double* M = s->mat;

    if (generate && ctx->oz_slices > 0 && np >= ctx->oz_min_n) {
        dense_factor_ozaki(s, (int)ctx->oz_slices);
        return;
    }

    set_int_kernel<<<1, 1, 0, ctx->stream>>>(s->info_dev, INT_MAX);
    ctx->launches++;

    if (generate) {
        // panel 0 (all rows, first NB columns) is the only part of K ever written by a stand-alone
        // build; every other tile is generated inside the first trailing update's epilogue.
        dense_build_region(s, 0, 0, (NB < np) ? NB : np);
    }

    for (int64_t k0 = 0; k0 < np; k0 += NB) {
        const int64_t kb = (NB < np - k0) ? NB : (np - k0);
        {
            ProfTimer t(ctx, &ctx->prof.panel_ms);
            dense_panel_factor(s, k0, kb);
        }
        const int64_t r0 = k0 + kb;
        if (r0 < np) {
            gemm::Args g{};
            g.A = M + r0 * ld + k0; g.lda = ld;
            g.B = M + r0 * ld + k0; g.ldb = ld;
            g.C = M + r0 * ld + r0; g.ldc = ld;
            g.tiles_m = g.tiles_n = (int)((np - r0) / TILE);
            g.K = (int)kb; g.alpha = -1.0; g.lower = 1;
            g.beta_mode = (generate && k0 == 0) ? 2 : 1;
            g.X = s->X_dev; g.diag = s->diag_dev; g.ndim = s->ndim; g.n_valid = s->n;
            g.row0 = r0; g.col0 = r0;
            ProfTimer t(ctx, &ctx->prof.syrk_ms);
            gemm::launch(ctx, (g.beta_mode == 2) ? s->prog : empty_prog(), g);
            const double T = (double)g.tiles_m;
            ctx->prof.syrk_flop += T * (T + 1.0) / 2.0 * 2.0 * TILE * TILE * (double)kb;
            ctx->prof.syrk_launches++;
        }
    }
    CUDA_CHECK(cudaMemcpyAsync(&s->info, s->info_dev, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (s->info == INT_MAX) s->info = 0;
    if (s->info > s->n) s->info = 0;  // cannot happen (pad is identity), defensive
}

// =============================================================================================
// reductions
// =============================================================================================
// out[0] = sum_{i<n} f(v[i*stride]) with f = log (mode 0) or square (mode 1); single block,
// fixed-shape tree so the result is deterministic.
__global__ void __launch_bounds__(1024) reduce_kernel(const double* v, int64_t stride, int64_t n, int mode, double* out,
                                                      int64_t batch_stride) {
    __shared__ double sh[1024];
    v += (int64_t)blockIdx.x * batch_stride;
    out += blockIdx.x;
    double acc = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += 1024) {
        const double x = v[i * stride];
        acc += (mode == 0) ? log(x) : x * x;
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = sh[0];
}

static double reduce_to_host(b200gp_ctx* ctx, const double* v, int64_t stride, int64_t n, int mode) {
    double* d = (double*)ctx->alloc(sizeof(double));
    reduce_kernel<<<1, 1024, 0, ctx->stream>>>(v, stride, n, mode, d, 0);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
    double h = 0.0;
    CUDA_CHECK(cudaMemcpyAsync(&h, d, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->release(d, sizeof(double));
    return h;
}

double dense_logdet_half(b200gp_dense* s) { return reduce_to_host(s->ctx, s->mat, s->np + 1, s->n, 0); }
double dense_sumsq_dev(b200gp_ctx* ctx, const double* x_dev, int64_t n) { return reduce_to_host(ctx, x_dev, 1, n, 1); }

// =============================================================================================
// K3: triangular solves with a vector right-hand side, one launch per 128-block.
// forward  (L x = y): every CTA recomputes x_j = inv(L_jj) y_j, then updates its rows below.
// backward (L^T x = y): x_j = inv(L_jj)^T y_j, then y[c] -= sum_r L[jr][c] x_j[r] for columns left.
// =============================================================================================
__global__ void __launch_bounds__(256) trsv_fwd_step(const double* __restrict__ mat, int64_t ld,
                                                      const double* __restrict__ linv_j, double* y, double* x,
                                                      int j, int64_t np, int64_t stride_mat, int64_t stride_linv) {
    __shared__ __align__(32) double ys[TILE];
    __shared__ __align__(32) double xs[TILE];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    mat += (int64_t)blockIdx.y * stride_mat;      // batched launch
    linv_j += (int64_t)blockIdx.y * stride_linv;
    y += (int64_t)blockIdx.y * np;
    x += (int64_t)blockIdx.y * np;
    if (tid < TILE) ys[tid] = y[(int64_t)j * TILE + tid];
    __syncthreads();
    for (int r = warp; r < TILE; r += 8) {
        const double* row = linv_j + r * TILE;
        double s = 0.0;
        for (int c = lane; c <= r; c += 32) s += row[c] * ys[c];
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) xs[r] = s;
    }
    __syncthreads();
    if (blockIdx.x == 0 && tid < TILE) x[(int64_t)j * TILE + tid] = xs[tid];
    const int64_t rbase = (int64_t)(j + 1) * TILE + (int64_t)blockIdx.x * 64 + warp * 8;
    const double4 xv = *reinterpret_cast<const double4*>(xs + lane * 4);
#pragma unroll
    for (int rr = 0; rr < 8; ++rr) {
        const int64_t r = rbase + rr;
        if (r >= np) break;
        const double4 lv = *reinterpret_cast<const double4*>(mat + r * ld + (int64_t)j * TILE + lane * 4);
        double s = lv.x * xv.x + lv.y * xv.y + lv.z * xv.z + lv.w * xv.w;
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) y[r] -= s;
    }
}

__global__ void __launch_bounds__(256) trsv_bwd_step(const double* __restrict__ mat, int64_t ld,
                                                      const double* __restrict__ linv_j, double* y, double* x, int j) {
    __shared__ double ys[TILE];
    __shared__ double xs[TILE];
    __shared__ double part[TILE];
    const int tid = threadIdx.x;
    if (tid < TILE) ys[tid] = y[(int64_t)j * TILE + tid];
    __syncthreads();
    {
        // x[c] = sum_{r >= c} linv[r][c] y[r] ; two half-ranges of r per column
        const int c = tid & (TILE - 1), half = tid >> 7;
        double s = 0.0;
        const int rbeg = half ? 64 : 0, rend = half ? TILE : 64;
        for (int r = max(rbeg, c); r < rend; ++r) s += linv_j[r * TILE + c] * ys[r];
        if (half) part[c] = s;
        __syncthreads();
        if (!half) xs[c] = s + part[c];
    }
    __syncthreads();
    if (blockIdx.x == 0 && tid < TILE) x[(int64_t)j * TILE + tid] = xs[tid];
    const int64_t c = (int64_t)blockIdx.x * 256 + tid;
    if (c < (int64_t)j * TILE) {
        const double* base = mat + (int64_t)j * TILE * ld + c;
        double s0 = 0.0, s1 = 0.0;
#pragma unroll 8
        for (int r = 0; r < TILE; r += 2) {
            s0 += base[(int64_t)r * ld] * xs[r];
            s1 += base[(int64_t)(r + 1) * ld] * xs[r + 1];
        }
        y[c] -= s0 + s1;
    }
}

void dense_solve_vec_dev(b200gp_dense* s, double* y_dev, double* x_dev, bool transpose) {
    b200gp_ctx* ctx = s->ctx;
    const int nblk = (int)(s->np / TILE);
    ProfTimer t(ctx, &ctx->prof.solve_ms);
    if (!transpose) {
        for (int j = 0; j < nblk; ++j) {
            const int64_t rows_below = s->np - (int64_t)(j + 1) * TILE;
            const unsigned grid = (unsigned)((rows_below + 63) / 64);
            trsv_fwd_step<<<grid ? grid : 1, 256, 0, ctx->stream>>>(s->mat, s->np, s->linv + (int64_t)j * TILE * TILE,
                                                                    y_dev, x_dev, j, s->np, 0, 0);
            ctx->launches++;
        }
    } else {
        for (int j = nblk - 1; j >= 0; --j) {
            const unsigned grid = (unsigned)(((int64_t)j * TILE + 255) / 256);
            trsv_bwd_step<<<grid ? grid : 1, 256, 0, ctx->stream>>>(s->mat, s->np, s->linv + (int64_t)j * TILE * TILE,
                                                                    y_dev, x_dev, j);
            ctx->launches++;
        }
    }
    CUDA_CHECK(cudaGetLastError());
}

// streaming helpers (multi-GPU / large-N fused log_probability): forward-substitution steps for the 128-blocks
// of ONE block column right after it has been factored, and that column's contribution to sum(log L_ii)
void dense_trsv_fwd_blocks(b200gp_dense* s, double* y_dev, double* x_dev, int j_begin, int j_end) {
    b200gp_ctx* ctx = s->ctx;
    ProfTimer t(ctx, &ctx->prof.solve_ms);
    for (int j = j_begin; j < j_end; ++j) {
        const int64_t rows_below = s->np - (int64_t)(j + 1) * TILE;
        const unsigned grid = (unsigned)((rows_below + 63) / 64);
        trsv_fwd_step<<<grid ? grid : 1, 256, 0, ctx->stream>>>(s->mat, s->ld, s->linv + (int64_t)j * TILE * TILE, y_dev,
                                                                x_dev, j, s->np, 0, 0);
        ctx->launches++;
    }
    CUDA_CHECK(cudaGetLastError());
}
void dense_logdiag_partial(b200gp_dense* s, int64_t c0, int64_t count, double* out_dev) {
    if (count <= 0) return;
    reduce_kernel<<<1, 1024, 0, s->ctx->stream>>>(s->mat + c0 * s->ld + c0, s->ld + 1, count, 0, out_dev, 0);
    s->ctx->launches++;
}

// =============================================================================================
// K4: out = L z  (direct.py:72-73), one warp per row
// =============================================================================================
__global__ void __launch_bounds__(256) trmv_lower_kernel(const double* __restrict__ mat, int64_t ld, int64_t n,
                                                          const double* __restrict__ z, double* out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * 8 + warp;
    if (i >= n) return;
    const double* row = mat + i * ld;
    double s = 0.0;
    for (int64_t c = lane; c <= i; c += 32) s += row[c] * z[c];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[i] = s;
}

// small layout helpers -----------------------------------------------------------------------
// dst (rows_dst x ld_dst) <- transpose of src (n x m, row-major), zero padded
__global__ void transpose_pad_kernel(const double* src, int64_t n, int64_t m, double* dst, int64_t rows_dst, int64_t ld_dst) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows_dst * ld_dst) return;
    const int64_t r = idx / ld_dst, c = idx % ld_dst;  // dst[r][c] = src[c][r]
    dst[idx] = (r < m && c < n) ? src[c * m + r] : 0.0;
}
__global__ void transpose_unpad_kernel(const double* src, int64_t ld_src, double* dst, int64_t n, int64_t m) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * m) return;
    const int64_t i = idx / m, r = idx % m;  // dst[i][r] = src[r][i]
    dst[idx] = src[r * ld_src + i];
}
__global__ void copy_pad_kernel(const double* src, int64_t n, double* dst, int64_t np) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < np) dst[i] = (i < n) ? src[i] : 0.0;
}
// load an n x n host-layout matrix into the padded np x np buffer with an identity pad
__global__ void pad_cov_kernel(const double* src, int64_t n, double* dst, int64_t np) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= np * np) return;
    const int64_t r = idx / np, c = idx % np;
    dst[idx] = (r < n && c < n) ? src[r * n + c] : ((r == c) ? 1.0 : 0.0);
}
__global__ void extract_lower_kernel(const double* src, int64_t ld, double* dst, int64_t n) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * n) return;
    const int64_t r = idx / n, c = idx % n;
    dst[idx] = (c <= r) ? src[r * ld + c] : 0.0;
}
__global__ void extract_rect_kernel(const double* src, int64_t ld, double* dst, int64_t n, int64_t m) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * m) return;
    dst[idx] = src[(idx / m) * ld + (idx % m)];
}

static inline unsigned nblocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// =============================================================================================
// object lifecycle
// =============================================================================================
static b200gp_dense* dense_alloc(b200gp_ctx* ctx, int64_t n);
static b200gp_dense* dense_alloc(b200gp_ctx* ctx, int64_t n) {
    if (n <= 0) throw GpError("dense: n must be positive");
    b200gp_dense* s = new b200gp_dense();
    s->ctx = ctx;
    s->n = n;
    s->np = ((n + TILE - 1) / TILE) * TILE;
    s->ld = s->np;
    try {
        s->mat_bytes = (size_t)s->np * s->np * sizeof(double);
        s->mat_alloc = (double*)ctx->alloc(s->mat_bytes);
        s->mat = s->mat_alloc;
        s->linv = (double*)ctx->alloc((size_t)(s->np / TILE) * TILE * TILE * sizeof(double));
        s->info_dev = (int*)ctx->alloc(sizeof(int));
    } catch (...) {
        dense_destroy(s);
        throw;
    }
    return s;
}

void dense_destroy(b200gp_dense* s) {
    if (!s) return;
    b200gp_ctx* ctx = s->ctx;
    if (s->mat_alloc) ctx->release(s->mat_alloc, s->mat_bytes);
    if (s->linv) ctx->release(s->linv, (size_t)(s->np / TILE) * TILE * TILE * sizeof(double));
    if (s->info_dev) ctx->release(s->info_dev, sizeof(int));
    if (s->owns_inputs) {
        if (s->X_dev) ctx->release(s->X_dev, (size_t)s->n * s->ndim * sizeof(double));
        if (s->diag_dev) ctx->release(s->diag_dev, (size_t)s->n * sizeof(double));
    }
    delete s;
}

// allocate the dense object and copy X / diag to the device, WITHOUT factoring (multi-GPU step API)
b200gp_dense* dense_alloc_for_prog(b200gp_ctx* ctx, const KProg& prog, const double* X, int64_t n, int ndim,
                                   const double* diag) {
    if (ndim < 1 || ndim > MAX_NDIM) throw GpError("dense: ndim must be in [1, 16]");
    b200gp_dense* s = dense_alloc(ctx, n);
    try {
        s->has_prog = true;
        s->prog = prog;
        s->ndim = ndim;
        s->owns_inputs = true;
        s->X_dev = (double*)ctx->alloc((size_t)n * ndim * sizeof(double));
        s->diag_dev = (double*)ctx->alloc((size_t)n * sizeof(double));
        CUDA_CHECK(cudaMemcpyAsync(s->X_dev, X, (size_t)n * ndim * sizeof(double), cudaMemcpyDefault, ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(s->diag_dev, diag, (size_t)n * sizeof(double), cudaMemcpyDefault, ctx->stream));
    } catch (...) {
        dense_destroy(s);
        throw;
    }
    return s;
}

b200gp_dense* dense_factor_from_prog(b200gp_ctx* ctx, const KProg& prog, const double* X_dev, int64_t n,
                                     int ndim, const double* diag_dev, bool copy_inputs) {
    if (ndim < 1 || ndim > MAX_NDIM) throw GpError("dense: ndim must be in [1, 16]");
    b200gp_dense* s = dense_alloc(ctx, n);
    try {
        s->has_prog = true;
        s->prog = prog;
        s->ndim = ndim;
        if (copy_inputs) {
            s->owns_inputs = true;
            s->X_dev = (double*)ctx->alloc((size_t)n * ndim * sizeof(double));
            s->diag_dev = (double*)ctx->alloc((size_t)n * sizeof(double));
            CUDA_CHECK(cudaMemcpyAsync(s->X_dev, X_dev, (size_t)n * ndim * sizeof(double), cudaMemcpyDefault, ctx->stream));
            CUDA_CHECK(cudaMemcpyAsync(s->diag_dev, diag_dev, (size_t)n * sizeof(double), cudaMemcpyDefault, ctx->stream));
        } else {
            s->X_dev = const_cast<double*>(X_dev);
            s->diag_dev = const_cast<double*>(diag_dev);
        }
        dense_factor_inplace(s, true);
    } catch (...) {
        dense_destroy(s);
        throw;
    }
    return s;
}

// out_host (m x m) = k(X*, X*) + diag* - At At^T for At (mp x kp row-major, zero padded, rows = test points):
// one NT GEMM on the tensor pipe with K = kp whose C tile is generated in the epilogue (beta_mode 2).  Shared by
// DirectSolver.condition (direct.py:88-95) and QuasisepSolver.condition's dense branch (solvers/quasisep/solver.py:131-139).
void dense_conditioned_covariance_to_host(b200gp_ctx* ctx, const KProg& P, const double* At, int64_t mp, int64_t kp,
                                          const double* xt_dev, const double* dt_dev, int nd, int64_t m,
                                          double* out_host) {
    if (mp % TILE != 0 || kp % TILE != 0) throw GpError("conditioned covariance: operands must be padded to 128");
    const int tm = (int)(mp / TILE);
    Scratch C(ctx, (size_t)mp * mp * 8), o(ctx, (size_t)m * m * 8);
    {
        gemm::Args g{};
        g.A = At; g.lda = kp; g.B = At; g.ldb = kp; g.C = C.f64(); g.ldc = mp;
        g.tiles_m = g.tiles_n = tm; g.K = (int)kp; g.alpha = -1.0; g.beta_mode = 2; g.lower = 0;
        g.X = xt_dev; g.diag = dt_dev; g.ndim = nd; g.n_valid = m; g.row0 = 0; g.col0 = 0;
        gemm::launch(ctx, P, g);
    }
    extract_rect_kernel<<<nblocks(m * m, 256), 256, 0, ctx->stream>>>(C.f64(), mp, o.f64(), m, m);
    ctx->launches++;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out_host, o.p, (size_t)m * m * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
}

// =============================================================================================
// C-ABI: dense
// =============================================================================================
extern "C" {

int b200gp_kernel_matrix(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X1, int64_t n1,
                         const double* X2, int64_t n2, int ndim, double* out) {
    API_BEGIN(ctx)
    if (ndim < 1 || ndim > MAX_NDIM) throw GpError("kernel_matrix: ndim must be in [1, 16]");
    if (n1 <= 0 || n2 <= 0) throw GpError("kernel_matrix: empty input");
    KProg P = parse_prog(prog, n_instr, ndim);
    Scratch x1_buf(_ctx, (size_t)n1 * ndim * 8);
    double* const x1 = x1_buf.f64();
    Scratch x2_buf(_ctx, (size_t)n2 * ndim * 8);
    double* const x2 = x2_buf.f64();
    Scratch o_buf(_ctx, (size_t)n1 * n2 * 8);
    double* const o = o_buf.f64();
    CUDA_CHECK(cudaMemcpyAsync(x1, X1, (size_t)n1 * ndim * 8, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(x2, X2, (size_t)n2 * ndim * 8, cudaMemcpyHostToDevice, _ctx->stream));
    dense_build_rect(_ctx, P, x1, n1, x2, n2, ndim, nullptr, o, n2, n1, n2);
    CUDA_CHECK(cudaMemcpyAsync(out, o, (size_t)n1 * n2 * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

int b200gp_kernel_diag(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n, int ndim,
                       double* out) {
    API_BEGIN(ctx)
    (void)X;  // stationary kernels: k(x, x) does not depend on x (nor on a linear input transform)
    if (n <= 0) throw GpError("kernel_diag: empty input");
    KProg P = parse_prog(prog, n_instr, ndim);
    Scratch o_buf(_ctx, (size_t)n * 8);
    double* const o = o_buf.f64();
    build_diag_kernel<<<nblocks(n, 256), 256, 0, _ctx->stream>>>(P, n, o);
    CUDA_CHECK(cudaGetLastError());
    _ctx->launches++;
    CUDA_CHECK(cudaMemcpyAsync(out, o, (size_t)n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

int b200gp_kernel_matvec(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X1, int64_t n1,
                         const double* X2, int64_t n2, int ndim, const double* y, double* out) {
    API_BEGIN(ctx)
    if (ndim < 1 || ndim > MAX_NDIM) throw GpError("kernel_matvec: ndim must be in [1, 16]");
    if (n1 <= 0 || n2 <= 0) throw GpError("kernel_matvec: empty input");
    KProg P = parse_prog(prog, n_instr, ndim);
    Scratch x1_buf(_ctx, (size_t)n1 * ndim * 8);
    double* const x1 = x1_buf.f64();
    Scratch x2_buf(_ctx, (size_t)n2 * ndim * 8);
    double* const x2 = x2_buf.f64();
    Scratch yd_buf(_ctx, (size_t)n2 * 8);
    double* const yd = yd_buf.f64();
    Scratch o_buf(_ctx, (size_t)n1 * 8);
    double* const o = o_buf.f64();
    CUDA_CHECK(cudaMemcpyAsync(x1, X1, (size_t)n1 * ndim * 8, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(x2, X2, (size_t)n2 * ndim * 8, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(yd, y, (size_t)n2 * 8, cudaMemcpyHostToDevice, _ctx->stream));
    kernel_matvec_kernel<<<nblocks(n1, 8), 256, 0, _ctx->stream>>>(P, x1, n1, x2, n2, ndim, yd, o);
    CUDA_CHECK(cudaGetLastError());
    _ctx->launches++;
    CUDA_CHECK(cudaMemcpyAsync(out, o, (size_t)n1 * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

int b200gp_dense_create(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n, int ndim,
                        const double* diag, b200gp_dense** out, int* info) {
    API_BEGIN(ctx)
    KProg P = parse_prog(prog, n_instr, ndim);
    b200gp_dense* s = dense_factor_from_prog(_ctx, P, X, n, ndim, diag, true);
    *out = s;
    if (info) *info = s->info;
    API_END
}

// DirectSolver.__init__ (direct.py:30-53) and, in the same pass, sum((L^-1 resid)^2) -- the data term of
// gp.py:313-316: the int8 factorisation substitutes panel by panel on a side stream under the update of the next block
// column (option "solve_overlap"), so `GaussianProcess(...).log_probability(y)` pays no separate triangular solve.
int b200gp_dense_create_with_resid(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n, int ndim,
                                   const double* diag, const double* resid, b200gp_dense** out, int* info, double* sumsq) {
    API_BEGIN(ctx)
    KProg P = parse_prog(prog, n_instr, ndim);
    _ctx->fuse_resid = (_ctx->solve_overlap != 0) ? resid : nullptr;
    _ctx->fuse_n = n;
    _ctx->fuse_y = _ctx->fuse_x = nullptr;
    b200gp_dense* s = nullptr;
    try {
        s = dense_factor_from_prog(_ctx, P, X, n, ndim, diag, true);
    } catch (...) {
        _ctx->fuse_resid = nullptr;
        throw;
    }
    _ctx->fuse_resid = nullptr;
    try {
        const int64_t np = s->np;
        double* y = _ctx->fuse_y;
        double* x = _ctx->fuse_x;
        _ctx->fuse_y = _ctx->fuse_x = nullptr;
        if (x == nullptr) {
            y = (double*)_ctx->alloc((size_t)np * 8);
            x = (double*)_ctx->alloc((size_t)np * 8);
            CUDA_CHECK(cudaMemsetAsync(y, 0, (size_t)np * 8, _ctx->stream));
            CUDA_CHECK(cudaMemcpyAsync(y, resid, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
            dense_solve_vec_dev(s, y, x, false);
        }
        *sumsq = dense_sumsq_dev(_ctx, x, n);
        _ctx->release(y, (size_t)np * 8);
        _ctx->release(x, (size_t)np * 8);
    } catch (...) {
        dense_destroy(s);
        throw;
    }
    *out = s;
    if (info) *info = s->info;
    API_END
}

int b200gp_dense_create_dev(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X_dev, int64_t n,
                            int ndim, const double* diag_dev, b200gp_dense** out, int* info) {
    return b200gp_dense_create(ctx, prog, n_instr, X_dev, n, ndim, diag_dev, out, info);  // cudaMemcpyDefault
}

int b200gp_dense_create_from_cov(b200gp_ctx* ctx, const double* cov, int64_t n, b200gp_dense** out, int* info) {
    API_BEGIN(ctx)
    b200gp_dense* s = dense_alloc(_ctx, n);
    try {
        double* tmp = (double*)_ctx->alloc((size_t)n * n * 8);
        CUDA_CHECK(cudaMemcpyAsync(tmp, cov, (size_t)n * n * 8, cudaMemcpyDefault, _ctx->stream));
        pad_cov_kernel<<<nblocks(s->np * s->np, 256), 256, 0, _ctx->stream>>>(tmp, n, s->mat, s->np);
        CUDA_CHECK(cudaGetLastError());
        _ctx->launches++;
        dense_factor_inplace(s, false);
        _ctx->release(tmp, (size_t)n * n * 8);
    } catch (...) {
        dense_destroy(s);
        throw;
    }
    *out = s;
    if (info) *info = s->info;
    API_END
}

int b200gp_dense_free(b200gp_dense* s) {
    if (!s) return 0;
    API_BEGIN(s->ctx)
    dense_destroy(s);
    API_END
}

int b200gp_dense_logdet_half(b200gp_dense* s, double* out) {
    API_BEGIN(s->ctx)
    *out = dense_logdet_half(s);
    API_END
}

int b200gp_dense_solve_triangular(b200gp_dense* s, double* Y, int64_t nrhs, int transpose) {
    API_BEGIN(s->ctx)
    if (nrhs <= 0) throw GpError("solve_triangular: nrhs must be positive");
    const int64_t n = s->n, np = s->np;
    Scratch yh_buf(_ctx, (size_t)n * nrhs * 8);
    double* const yh = yh_buf.f64();
    Scratch yt_buf(_ctx, (size_t)nrhs * np * 8);
    double* const yt = yt_buf.f64();
    Scratch xt_buf(_ctx, (size_t)nrhs * np * 8);
    double* const xt = xt_buf.f64();
    CUDA_CHECK(cudaMemcpyAsync(yh, Y, (size_t)n * nrhs * 8, cudaMemcpyHostToDevice, _ctx->stream));
    transpose_pad_kernel<<<nblocks(nrhs * np, 256), 256, 0, _ctx->stream>>>(yh, n, nrhs, yt, nrhs, np);
    _ctx->launches++;
    for (int64_t r = 0; r < nrhs; ++r) dense_solve_vec_dev(s, yt + r * np, xt + r * np, transpose != 0);
    transpose_unpad_kernel<<<nblocks(n * nrhs, 256), 256, 0, _ctx->stream>>>(xt, np, yh, n, nrhs);
    _ctx->launches++;
    CUDA_CHECK(cudaMemcpyAsync(Y, yh, (size_t)n * nrhs * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

int b200gp_dense_dot_triangular(b200gp_dense* s, double* Y, int64_t nrhs) {
    API_BEGIN(s->ctx)
    if (nrhs <= 0) throw GpError("dot_triangular: nrhs must be positive");
    const int64_t n = s->n, np = s->np;
    Scratch yh_buf(_ctx, (size_t)n * nrhs * 8);
    double* const yh = yh_buf.f64();
    Scratch yt_buf(_ctx, (size_t)nrhs * np * 8);
    double* const yt = yt_buf.f64();
    Scratch xt_buf(_ctx, (size_t)nrhs * np * 8);
    double* const xt = xt_buf.f64();
    CUDA_CHECK(cudaMemcpyAsync(yh, Y, (size_t)n * nrhs * 8, cudaMemcpyHostToDevice, _ctx->stream));
    transpose_pad_kernel<<<nblocks(nrhs * np, 256), 256, 0, _ctx->stream>>>(yh, n, nrhs, yt, nrhs, np);
    _ctx->launches++;
    for (int64_t r = 0; r < nrhs; ++r) {
        trmv_lower_kernel<<<nblocks(np, 8), 256, 0, _ctx->stream>>>(s->mat, np, np, yt + r * np, xt + r * np);
        _ctx->launches++;
    }
    transpose_unpad_kernel<<<nblocks(n * nrhs, 256), 256, 0, _ctx->stream>>>(xt, np, yh, n, nrhs);
    _ctx->launches++;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(Y, yh, (size_t)n * nrhs * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

// condition (direct.py:75-95), all on the tensor pipe:  with rows = test points,
//   At (mp x np) = Ks^T = k(X*, X);  forward substitution block by block on At (NT GEMMs);
//   out = Kss + diag* - At At^T  (NT GEMM with K = np, C generated in the epilogue).
int b200gp_dense_condition(b200gp_dense* s, const double* prog, int n_instr, const double* Xtest, int64_t m,
                           const double* diag_test, double* out) {
    API_BEGIN(s->ctx)
    if (!s->has_prog) throw GpError("condition: solver was built from a precomputed covariance (no coordinates)");
    KProg P = parse_prog(prog, n_instr, s->ndim);
    const int64_t n = s->n, np = s->np;
    const int nd = s->ndim;
    double* xt_dev;
    bool own_xt = false;
    if (Xtest == nullptr) {
        m = n;
        xt_dev = s->X_dev;
    } else {
        if (m <= 0) throw GpError("condition: empty X_test");
        xt_dev = (double*)_ctx->alloc((size_t)m * nd * 8);
        own_xt = true;
        CUDA_CHECK(cudaMemcpyAsync(xt_dev, Xtest, (size_t)m * nd * 8, cudaMemcpyHostToDevice, _ctx->stream));
    }
    const int64_t mp = ((m + TILE - 1) / TILE) * TILE;
    double* dt = (double*)_ctx->alloc((size_t)mp * 8);
    CUDA_CHECK(cudaMemsetAsync(dt, 0, (size_t)mp * 8, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(dt, diag_test, (size_t)m * 8, cudaMemcpyHostToDevice, _ctx->stream));
    double* At = (double*)_ctx->alloc((size_t)mp * np * 8);
    // Ks^T, zero padded
    dense_build_rect(_ctx, P, xt_dev, m, s->X_dev, n, nd, nullptr, At, np, mp, np);
    const int nblk = (int)(np / TILE), tm = (int)(mp / TILE);
    {
        ProfTimer t(_ctx, &_ctx->prof.solve_ms);
        for (int j = 0; j < nblk; ++j) {
            double* Aj = At + (int64_t)j * TILE;
            gemm_nt(_ctx, Aj, np, Aj, np, s->linv + (int64_t)j * TILE * TILE, TILE, tm, 1, TILE, 1.0, 0, 0);
            if (j + 1 < nblk)
                gemm_nt(_ctx, Aj + TILE, np, Aj, np, s->mat + (int64_t)(j + 1) * TILE * np + (int64_t)j * TILE, np,
                        tm, nblk - j - 1, TILE, -1.0, 1, 0);
        }
    }
    dense_conditioned_covariance_to_host(_ctx, P, At, mp, np, xt_dev, dt, nd, m, out);
    _ctx->release(At, (size_t)mp * np * 8);
    _ctx->release(dt, (size_t)mp * 8);
    if (own_xt) _ctx->release(xt_dev, (size_t)m * nd * 8);
    API_END
}

// C (m, m) <- C - At At^T for host operands, At (m, k) row-major: the Kss - A^T A of direct.py:93-95 / quasisep solver.py:131-139
// for solvers that have no kernel program on the device (a factor of a precomputed covariance, i.e. noise.Dense / noise.Banded,
// or of generator arrays): the host passes A^T = (L^-1 Ks)^T from its own triangular solve.  fp64 DMMA GEMM, operands zero
// padded to the 128-tile.
int b200gp_gram_downdate(b200gp_ctx* ctx, const double* At, int64_t m, int64_t k, double* C) {
    API_BEGIN(ctx)
    if (m <= 0 || k <= 0) throw GpError("gram_downdate: empty operand");
    const int64_t mp = ((m + TILE - 1) / TILE) * TILE, kp = ((k + TILE - 1) / TILE) * TILE;
    Scratch a_buf(_ctx, (size_t)mp * kp * 8), c_buf(_ctx, (size_t)mp * mp * 8);
    double* const a = a_buf.f64();
    double* const c = c_buf.f64();
    CUDA_CHECK(cudaMemsetAsync(a, 0, (size_t)mp * kp * 8, _ctx->stream));
    CUDA_CHECK(cudaMemsetAsync(c, 0, (size_t)mp * mp * 8, _ctx->stream));
    CUDA_CHECK(cudaMemcpy2DAsync(a, (size_t)kp * 8, At, (size_t)k * 8, (size_t)k * 8, (size_t)m, cudaMemcpyHostToDevice,
                                 _ctx->stream));
    CUDA_CHECK(cudaMemcpy2DAsync(c, (size_t)mp * 8, C, (size_t)m * 8, (size_t)m * 8, (size_t)m, cudaMemcpyHostToDevice,
                                 _ctx->stream));
    gemm_nt(_ctx, c, mp, a, kp, a, kp, (int)(mp / TILE), (int)(mp / TILE), (int)kp, -1.0, 1, 0);
    CUDA_CHECK(cudaMemcpy2DAsync(C, (size_t)m * 8, c, (size_t)mp * 8, (size_t)m * 8, (size_t)m, cudaMemcpyDeviceToHost,
                                 _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

int b200gp_dense_covariance(b200gp_dense* s, double* out) {
    API_BEGIN(s->ctx)
    if (!s->has_prog) throw GpError("covariance: solver was built from a precomputed covariance; the host keeps it");
    const int64_t n = s->n;
    Scratch o_buf(_ctx, (size_t)n * n * 8);
    double* const o = o_buf.f64();
    BuildArgs a{};
    a.X1 = s->X_dev; a.X2 = s->X_dev; a.diag = s->diag_dev; a.out = o; a.ld = n;
    a.n1 = n; a.n2 = n; a.rows_pad = n; a.cols_pad = n; a.ndim = s->ndim; a.pad_identity = 0;
    dim3 grid((unsigned)((n + BUILD_COLS - 1) / BUILD_COLS), (unsigned)((n + BUILD_ROWS - 1) / BUILD_ROWS));
    {
        ProfTimer t(_ctx, &_ctx->prof.build_ms);
        launch_build_rect(_ctx, grid, s->prog, a);
        CUDA_CHECK(cudaGetLastError());
        _ctx->launches++;
        _ctx->prof.build_bytes += 8.0 * (double)n * (double)n;
    }
    CUDA_CHECK(cudaMemcpyAsync(out, o, (size_t)n * n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

int b200gp_dense_get_factor(b200gp_dense* s, double* out) {
    API_BEGIN(s->ctx)
    const int64_t n = s->n;
    Scratch o_buf(_ctx, (size_t)n * n * 8);
    double* const o = o_buf.f64();
    extract_lower_kernel<<<nblocks(n * n, 256), 256, 0, _ctx->stream>>>(s->mat, s->np, o, n);
    CUDA_CHECK(cudaGetLastError());
    _ctx->launches++;
    CUDA_CHECK(cudaMemcpyAsync(out, o, (size_t)n * n * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

extern "C++" double ozaki_logp_streaming(b200gp_ctx* ctx, const KProg& P, const double* X, int64_t n, int ndim,
                                         const double* diag, const double* resid, int S);   // ozaki.cu

static double dense_logp_impl(b200gp_ctx* ctx, const KProg& P, const double* X, int64_t n, int ndim,
                              const double* diag, const double* resid) {
    // X / diag / resid may be host or device pointers (cudaMemcpyDefault resolves them)
    {
        // no factor is retained by this entry point, so very large problems stream their block columns (no N x N
        // fp64 matrix: only the digit planes stay resident).  Smaller ones keep the matrix: the rolling column
        // buffer competes with the operand planes for L2.
        const int64_t npad = ((n + TILE - 1) / TILE) * TILE;
        const double need = (double)npad * (double)npad * (8.0 + (double)ctx->oz_slices);
        if (ctx->oz_slices > 0 && npad >= ctx->oz_min_n && need > 70e9)     // 80 GB of HBM3
            return ozaki_logp_streaming(ctx, P, X, n, ndim, diag, resid, (int)ctx->oz_slices);
    }
    // the int8 factorisation runs the forward substitution itself, panel by panel on a side stream under the update of
    // the next block column (option "solve_overlap"); it leaves L^-1 resid in ctx->fuse_x
    ctx->fuse_resid = (ctx->solve_overlap != 0) ? resid : nullptr;
    ctx->fuse_n = n;
    ctx->fuse_y = ctx->fuse_x = nullptr;
    b200gp_dense* s = nullptr;
    try {
        s = dense_factor_from_prog(ctx, P, X, n, ndim, diag, true);
    } catch (...) {
        ctx->fuse_resid = nullptr;
        throw;
    }
    ctx->fuse_resid = nullptr;
    double logp;
    try {
        const int64_t np = s->np;
        double* y = ctx->fuse_y;
        double* x = ctx->fuse_x;
        ctx->fuse_y = ctx->fuse_x = nullptr;
        if (x == nullptr) {     // native fp64 path (or the overlap is off): substitute now
            y = (double*)ctx->alloc((size_t)np * 8);
            x = (double*)ctx->alloc((size_t)np * 8);
            CUDA_CHECK(cudaMemsetAsync(y, 0, (size_t)np * 8, ctx->stream));
            CUDA_CHECK(cudaMemcpyAsync(y, resid, (size_t)n * 8, cudaMemcpyDefault, ctx->stream));
            dense_solve_vec_dev(s, y, x, false);
        }
        const double ss = dense_sumsq_dev(ctx, x, n);
        const double ld = dense_logdet_half(s);
        logp = -0.5 * ss - (ld + 0.5 * (double)n * log(2.0 * M_PI));   // gp.py:313-316, direct.py:61-64
        if (s->info != 0 || !isfinite(logp)) logp = -INFINITY;
        ctx->release(y, (size_t)np * 8);
        ctx->release(x, (size_t)np * 8);
    } catch (...) {
        dense_destroy(s);
        throw;
    }
    dense_destroy(s);
    return logp;
}

int b200gp_dense_log_probability(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n,
                                 int ndim, const double* diag, const double* resid, double* logp) {
    API_BEGIN(ctx)
    KProg P = parse_prog(prog, n_instr, ndim);
    *logp = dense_logp_impl(_ctx, P, X, n, ndim, diag, resid);
    API_END
}

int b200gp_dense_log_probability_dev(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X_dev,
                                     int64_t n, int ndim, const double* diag_dev, const double* resid_dev,
                                     double* logp) {
    return b200gp_dense_log_probability(ctx, prog, n_instr, X_dev, n, ndim, diag_dev, resid_dev, logp);
}

}  // extern "C"

// =============================================================================================
// batched log_probability over a hyper-parameter grid (BASELINE config 5): B problems share X, diag, y and
// differ in their kernel program.  Every kernel of the blocked factorisation is launched once for the
// whole batch (grid.y / grid.x = problem), so the launch chain is paid once per batch, not per problem.
// =============================================================================================
__global__ void finish_logp_kernel(const double* ld_half, const double* sumsq, const int* info, int64_t n, int64_t nb,
                                   double* logp) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    double lp = -0.5 * sumsq[b] - (ld_half[b] + 0.5 * (double)n * log(2.0 * M_PI));   // gp.py:313-316
    if (info[b] != INT_MAX || !isfinite(lp)) lp = -INFINITY;
    logp[b] = lp;
}
__global__ void fill_int_kernel(int* p, int v, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
__global__ void replicate_pad_kernel(const double* src, int64_t n, double* dst, int64_t np, int64_t nbatch) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= np * nbatch) return;
    const int64_t i = idx % np;
    dst[idx] = (i < n) ? src[i] : 0.0;
}

static void dense_logp_batched_chunk(b200gp_ctx* ctx, const KProg* progs_dev, int64_t B, const double* X_dev, int64_t n,
                                     int ndim, const double* diag_dev, const double* resid_dev, double* logp_dev,
                                     const double* consts_dev, int batch_op, int batch_l2) {
    const int64_t np = ((n + TILE - 1) / TILE) * TILE, ld = np;
    const int nblk = (int)(np / TILE);
    const int64_t smat = np * np, slinv = (int64_t)nblk * TILE * TILE;
    double* M = (double*)ctx->alloc((size_t)B * smat * 8);
    double* linv = (double*)ctx->alloc((size_t)B * slinv * 8);
    int* info = (int*)ctx->alloc((size_t)B * sizeof(int));
    double* y = (double*)ctx->alloc((size_t)B * np * 8);
    double* x = (double*)ctx->alloc((size_t)B * np * 8);
    double* red = (double*)ctx->alloc((size_t)2 * B * 8);
    fill_int_kernel<<<nblocks(B, 256), 256, 0, ctx->stream>>>(info, INT_MAX, B);
    ctx->launches++;
    {   // K_b = k_b(X, X) + diag for every problem (lower triangle is what the factorisation reads)
        BuildArgs a{};
        a.X1 = X_dev; a.X2 = X_dev; a.diag = diag_dev; a.out = M; a.ld = ld;
        a.n1 = n; a.n2 = n; a.rows_pad = np; a.cols_pad = np; a.ndim = ndim; a.pad_identity = 1;
        a.progs = progs_dev; a.batch_stride = smat;
        a.batch_consts = consts_dev; a.batch_op = batch_op; a.batch_l2 = batch_l2;
        a.lower_only = 1;      // the blocked factorisation below reads (and writes) lower-triangle 128-tiles only
        dim3 grid((unsigned)((np + BUILD_COLS - 1) / BUILD_COLS), (unsigned)((np + BUILD_ROWS - 1) / BUILD_ROWS), (unsigned)B);
        ProfTimer t(ctx, &ctx->prof.build_ms);
        launch_build_rect(ctx, grid, empty_prog(), a);
        CUDA_CHECK(cudaGetLastError());
        ctx->launches++;
        ctx->prof.build_bytes += 8.0 * (double)B * (double)np * (double)np;
    }
    int64_t NB = ctx->nb_batched;
    for (int64_t k0 = 0; k0 < np; k0 += NB) {
        const int64_t kb = (NB < np - k0) ? NB : (np - k0);
        {
            ProfTimer t(ctx, &ctx->prof.panel_ms);
            for (int64_t j0 = 0; j0 < kb; j0 += TILE) {
                const int64_t c0 = k0 + j0;
                if (j0 > 0)
                    gemm_nt(ctx, M + c0 * ld + c0, ld, M + c0 * ld + k0, ld, M + c0 * ld + k0, ld, (int)((np - c0) / TILE), 1,
                            (int)j0, -1.0, 1, 0, (int)B, smat, smat, smat);
                potf2(ctx, M + c0 * ld + c0, ld, linv + (c0 / TILE) * TILE * TILE, info, (int)c0, (int)B, smat, slinv);
                if (c0 + TILE < np)
                    gemm_nt(ctx, M + (c0 + TILE) * ld + c0, ld, M + (c0 + TILE) * ld + c0, ld, linv + (c0 / TILE) * TILE * TILE,
                            TILE, (int)((np - c0 - TILE) / TILE), 1, TILE, 1.0, 0, 0, (int)B, smat, slinv, smat);
            }
        }
        const int64_t r0 = k0 + kb;
        if (r0 < np) {
            const int T = (int)((np - r0) / TILE);
            ProfTimer t(ctx, &ctx->prof.syrk_ms);
            gemm_nt(ctx, M + r0 * ld + r0, ld, M + r0 * ld + k0, ld, M + r0 * ld + k0, ld, T, T, (int)kb, -1.0, 1, 1, (int)B,
                    smat, smat, smat);
            ctx->prof.syrk_flop += (double)B * T * (T + 1.0) / 2.0 * 2.0 * TILE * TILE * (double)kb;
            ctx->prof.syrk_launches++;
        }
    }
    // forward solves for all problems at once
    replicate_pad_kernel<<<nblocks(B * np, 256), 256, 0, ctx->stream>>>(resid_dev, n, y, np, B);
    ctx->launches++;
    {
        ProfTimer t(ctx, &ctx->prof.solve_ms);
        for (int j = 0; j < nblk; ++j) {
            const int64_t rows_below = np - (int64_t)(j + 1) * TILE;
            const unsigned gx = (unsigned)((rows_below + 63) / 64);
            dim3 grid(gx ? gx : 1, (unsigned)B);
            trsv_fwd_step<<<grid, 256, 0, ctx->stream>>>(M, np, linv + (int64_t)j * TILE * TILE, y, x, j, np, smat, slinv);
            ctx->launches++;
        }
    }
    reduce_kernel<<<(unsigned)B, 1024, 0, ctx->stream>>>(M, np + 1, n, 0, red, smat);       // sum log L_ii
    reduce_kernel<<<(unsigned)B, 1024, 0, ctx->stream>>>(x, 1, n, 1, red + B, np);          // |alpha|^2
    finish_logp_kernel<<<nblocks(B, 256), 256, 0, ctx->stream>>>(red, red + B, info, n, B, logp_dev);
    ctx->launches += 3;
    CUDA_CHECK(cudaGetLastError());
    ctx->release(M, (size_t)B * smat * 8);
    ctx->release(linv, (size_t)B * slinv * 8);
    ctx->release(info, (size_t)B * sizeof(int));
    ctx->release(y, (size_t)B * np * 8);
    ctx->release(x, (size_t)B * np * 8);
    ctx->release(red, (size_t)2 * B * 8);
}

extern "C" int b200gp_dense_log_probability_batched(b200gp_ctx* ctx, const double* progs, int n_instr, int64_t nbatch,
                                                    const double* X, int64_t n, int ndim, const double* diag,
                                                    const double* resid, double* logp) {
    API_BEGIN(ctx)
    if (nbatch <= 0 || n <= 0) throw GpError("batched log_probability: empty batch");
    if (ndim < 1 || ndim > MAX_NDIM) throw GpError("batched log_probability: ndim must be in [1, 16]");
    std::vector<KProg> hp((size_t)nbatch);
    for (int64_t b = 0; b < nbatch; ++b) hp[b] = parse_prog(progs + (size_t)b * n_instr * B200GP_PROG_STRIDE, n_instr, ndim);
    // a hyper-parameter grid of ONE single-leaf kernel (amp * ExpSquared(scale), ...: BASELINE config 5) runs the build in the
    // compile-time specialised kernel with per-problem constants instead of the interpreter
    std::vector<double> hc((size_t)nbatch * 3);
    int batch_op = -1, batch_l2 = 0;
    bool single = (_ctx->build_fast >= 2 && ndim <= 3);
    for (int64_t b = 0; b < nbatch && single; ++b) {
        KFast F{};
        if (!kprog_to_fast(hp[b], F) || !single_constants(F, &hc[(size_t)b * 3])) { single = false; break; }
        if (b == 0) { batch_op = F.op[0]; batch_l2 = F.l2[0]; }
        else if (F.op[0] != batch_op || F.l2[0] != batch_l2) single = false;
    }
    double* dc = single ? (double*)_ctx->alloc((size_t)nbatch * 3 * 8) : nullptr;
    if (dc) CUDA_CHECK(cudaMemcpyAsync(dc, hc.data(), (size_t)nbatch * 3 * 8, cudaMemcpyHostToDevice, _ctx->stream));
    KProg* dp = (KProg*)_ctx->alloc((size_t)nbatch * sizeof(KProg));
    double* dX = (double*)_ctx->alloc((size_t)n * ndim * 8);
    double* dd = (double*)_ctx->alloc((size_t)n * 8);
    double* dr = (double*)_ctx->alloc((size_t)n * 8);
    double* dl = (double*)_ctx->alloc((size_t)nbatch * 8);
    CUDA_CHECK(cudaMemcpyAsync(dp, hp.data(), (size_t)nbatch * sizeof(KProg), cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(dX, X, (size_t)n * ndim * 8, cudaMemcpyDefault, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(dd, diag, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(dr, resid, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));  // hp is host-stack memory
    const int64_t np = ((n + TILE - 1) / TILE) * TILE;
    int64_t chunk = (int64_t)(((size_t)40 << 30) / ((size_t)np * np * 8));   // <= 40 GiB of matrices per chunk
    if (chunk < 1) chunk = 1;
    if (chunk > 4096) chunk = 4096;
    for (int64_t b0 = 0; b0 < nbatch; b0 += chunk) {
        const int64_t B = (chunk < nbatch - b0) ? chunk : (nbatch - b0);
        dense_logp_batched_chunk(_ctx, dp + b0, B, dX, n, ndim, dd, dr, dl + b0, dc ? dc + 3 * b0 : nullptr, batch_op, batch_l2);
    }
    CUDA_CHECK(cudaMemcpyAsync(logp, dl, (size_t)nbatch * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    _ctx->release(dp, (size_t)nbatch * sizeof(KProg));
    if (dc) _ctx->release(dc, (size_t)nbatch * 3 * 8);
    _ctx->release(dX, (size_t)n * ndim * 8);
    _ctx->release(dd, (size_t)n * 8);
    _ctx->release(dr, (size_t)n * 8);
    _ctx->release(dl, (size_t)nbatch * 8);
    API_END
}

// =============================================================================================
// diagnostics entry points (include/b200gp.h): one launch of the GEMM or of the diagonal-block kernel on device copies
// of host buffers.  Every size is checked before anything is allocated, so that the kernels read and write only the
// buffers allocated here; the whole output buffers come back, so that a write outside the intended elements shows.
// =============================================================================================
extern "C" int b200gp_gemm_nt_test(b200gp_ctx* ctx, const double* A, int64_t a_elems, int64_t lda, int64_t strideA,
                                   const double* B, int64_t b_elems, int64_t ldb, int64_t strideB, double* C,
                                   int64_t c_elems, int64_t ldc, int64_t strideC, int batch, int tiles_m, int tiles_n,
                                   int K, double alpha, int beta_mode, int lower, const double* prog, int n_instr,
                                   const double* X, int ndim, const double* diag, int64_t n_valid, int64_t row0,
                                   int64_t col0) {
    API_BEGIN(ctx)
    using gemm::BM;
    if (A == nullptr || B == nullptr || C == nullptr) throw GpError("gemm test: A, B and C are required");
    if (batch < 1 || batch > 65535) throw GpError("gemm test: 1 <= batch <= 65535");
    if (tiles_m < 1 || tiles_n < 1) throw GpError("gemm test: tiles_m, tiles_n >= 1");
    if (lower && tiles_n != tiles_m) throw GpError("gemm test: the lower schedule needs tiles_n == tiles_m");
    const int64_t ntiles = lower ? (int64_t)tiles_m * (tiles_m + 1) / 2 : (int64_t)tiles_m * tiles_n;
    if (ntiles > INT_MAX) throw GpError("gemm test: too many tiles");
    if (K < BM || K % BM != 0) throw GpError("gemm test: K is a positive multiple of 128");
    if (beta_mode < 0 || beta_mode > 2) throw GpError("gemm test: beta_mode is 0, 1 or 2");
    // 16-byte cp.async operand rows and double2 stores of C: even row strides and problem strides
    if (lda < K || ldb < K || ldc < (int64_t)tiles_n * BM || ((lda | ldb | ldc) & 1))
        throw GpError("gemm test: lda, ldb >= K, ldc >= 128 tiles_n, all even");
    if (strideA < 0 || strideB < 0 || strideC < 0 || ((strideA | strideB | strideC) & 1))
        throw GpError("gemm test: problem strides are even and >= 0");
    // footprints in double: exact below 2^53, and no int64 overflow for any argument
    const double rows_a = (double)tiles_m * BM, rows_b = (double)tiles_n * BM, nb1 = batch - 1;
    if (a_elems > ((int64_t)1 << 50) || b_elems > ((int64_t)1 << 50) || c_elems > ((int64_t)1 << 50))
        throw GpError("gemm test: buffers of at most 2^50 elements");
    if (nb1 * strideA + (rows_a - 1) * lda + K > (double)a_elems) throw GpError("gemm test: A is too small");
    if (nb1 * strideB + (rows_b - 1) * ldb + K > (double)b_elems) throw GpError("gemm test: B is too small");
    if (nb1 * strideC + (rows_a - 1) * ldc + rows_b > (double)c_elems) throw GpError("gemm test: C is too small");
    KProg P{};
    if (beta_mode == 2) {
        if (prog == nullptr || X == nullptr || diag == nullptr) throw GpError("gemm test: beta_mode 2 needs prog, X, diag");
        if (ndim < 1 || ndim > MAX_NDIM) throw GpError("gemm test: ndim must be in [1, 16]");
        if (n_valid < 1 || row0 < 0 || col0 < 0) throw GpError("gemm test: n_valid >= 1, row0, col0 >= 0");
        P = parse_prog(prog, n_instr, ndim);
    }
    Scratch a_buf(_ctx, (size_t)a_elems * 8), b_buf(_ctx, (size_t)b_elems * 8), c_buf(_ctx, (size_t)c_elems * 8);
    std::optional<Scratch> x_buf, d_buf;
    CUDA_CHECK(cudaMemcpyAsync(a_buf.p, A, (size_t)a_elems * 8, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(b_buf.p, B, (size_t)b_elems * 8, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(c_buf.p, C, (size_t)c_elems * 8, cudaMemcpyHostToDevice, _ctx->stream));
    gemm::Args g{};
    g.A = a_buf.f64(); g.lda = lda; g.B = b_buf.f64(); g.ldb = ldb; g.C = c_buf.f64(); g.ldc = ldc;
    g.tiles_m = tiles_m; g.tiles_n = tiles_n; g.K = K; g.alpha = alpha; g.beta_mode = beta_mode; g.lower = lower;
    g.batch = batch; g.strideA = strideA; g.strideB = strideB; g.strideC = strideC;
    if (beta_mode == 2) {
        x_buf.emplace(_ctx, (size_t)n_valid * ndim * 8);
        d_buf.emplace(_ctx, (size_t)n_valid * 8);
        CUDA_CHECK(cudaMemcpyAsync(x_buf->p, X, (size_t)n_valid * ndim * 8, cudaMemcpyHostToDevice, _ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(d_buf->p, diag, (size_t)n_valid * 8, cudaMemcpyHostToDevice, _ctx->stream));
        g.X = x_buf->f64(); g.diag = d_buf->f64(); g.ndim = ndim; g.n_valid = n_valid; g.row0 = row0; g.col0 = col0;
    }
    gemm::launch(_ctx, (beta_mode == 2) ? P : empty_prog(), g);
    CUDA_CHECK(cudaMemcpyAsync(C, c_buf.p, (size_t)c_elems * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    API_END
}

extern "C" int b200gp_potf2_test(b200gp_ctx* ctx, double* A, int64_t a_elems, int64_t lda, int64_t strideA, int batch,
                                 int global_off, double* linv, int* info) {
    API_BEGIN(ctx)
    if (A == nullptr || linv == nullptr || info == nullptr) throw GpError("potf2 test: A, linv and info are required");
    if (batch < 1 || batch > 65535) throw GpError("potf2 test: 1 <= batch <= 65535");
    if (lda < TILE || strideA < 0) throw GpError("potf2 test: lda >= 128, strideA >= 0");
    if (global_off < 0 || global_off > INT_MAX - TILE) throw GpError("potf2 test: 0 <= global_off <= INT_MAX - 128");
    if (a_elems > ((int64_t)1 << 50) || (double)(batch - 1) * strideA + (double)(TILE - 1) * lda + TILE > (double)a_elems)
        throw GpError("potf2 test: A is too small");
    const size_t linv_bytes = (size_t)batch * TILE * TILE * 8;
    Scratch a_buf(_ctx, (size_t)a_elems * 8), l_buf(_ctx, linv_bytes), i_buf(_ctx, (size_t)batch * sizeof(int));
    CUDA_CHECK(cudaMemcpyAsync(a_buf.p, A, (size_t)a_elems * 8, cudaMemcpyHostToDevice, _ctx->stream));
    fill_int_kernel<<<nblocks(batch, 256), 256, 0, _ctx->stream>>>((int*)i_buf.p, INT_MAX, batch);
    CUDA_CHECK(cudaGetLastError());
    _ctx->launches++;
    potf2(_ctx, a_buf.f64(), lda, l_buf.f64(), (int*)i_buf.p, global_off, batch, strideA, (int64_t)TILE * TILE);
    CUDA_CHECK(cudaMemcpyAsync(A, a_buf.p, (size_t)a_elems * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(linv, l_buf.p, linv_bytes, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(info, i_buf.p, (size_t)batch * sizeof(int), cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    for (int b = 0; b < batch; ++b)
        if (info[b] == INT_MAX) info[b] = 0;
    API_END
}
