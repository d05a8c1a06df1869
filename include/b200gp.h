/* b200gp.h -- C-ABI of the B200-native solver backend for tinygp-style Gaussian processes.
 *
 * The reference (dfm/tinygp @ 5302d5a) has no FFI: its boundary is the Python `Solver`
 * protocol (src/tinygp/solvers/solver.py:15-82) that `GaussianProcess.__init__` calls as a
 * constructor (src/tinygp/gp.py:106-112).  The host package `tinygp_b200` re-declares that
 * protocol and binds every method to one of the entry points below through ctypes.  Each
 * entry point names the reference call it replaces.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; b200gp_last_error(ctx) gives
 *     the message.  No exception crosses the ABI.
 *   - all matrices are row-major fp64.  Pointers are HOST pointers unless the name ends in
 *     `_dev` (then they are device pointers on the context's device).
 *   - a context owns one device, one stream and a cache of device buffers; objects created
 *     from a context (`b200gp_dense`, `b200gp_qs`) own their device-resident factor until freed.
 *   - calls are host-synchronous (equivalent to jax's .block_until_ready()); a context is
 *     single-threaded.  ctypes releases the GIL for the duration of a call.
 *   - non positive-definite input never fails a call: `info` > 0 is the 1-based index of the
 *     first bad pivot and the factor holds NaNs, which the host maps to log_probability = -inf
 *     (src/tinygp/gp.py:316).
 */
#ifndef B200GP_H
#define B200GP_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200gp_ctx b200gp_ctx;
typedef struct b200gp_dense b200gp_dense;
typedef struct b200gp_qs b200gp_qs;

/* ---- kernel programs -------------------------------------------------------------------
 * A stationary kernel expression (kernels/base.py:170-209 Sum/Product/Constant over the leaves
 * of kernels/stationary.py:76-235) is lowered by the host to a postfix program of
 * B200GP_PROG_STRIDE doubles per instruction: {opcode, distance, p0, p1}.
 */
#define B200GP_PROG_STRIDE 4
#define B200GP_PROG_MAX_INSTR 32
/* Input transforms (transforms.py:23-161 Transform/Linear/Cholesky/Subspace).  Linear, Cholesky and
 * Subspace are linear maps z = M x, and a stationary leaf only sees differences, so a transformed
 * leaf evaluates its distance on M (x1 - x2).  A program may start with up to B200GP_PROG_MAX_METRICS
 * metric definitions: one header row {B200GP_OP_METRIC, id (1-based), rows, cols} followed by
 * ceil(rows*cols/4) rows holding M row-major (zero padded); rows, cols <= B200GP_METRIC_MAX_DIM and
 * cols must equal ndim of the call.  A leaf selects metric `id` by adding 2*id to its distance code
 * (id 0 = untransformed coordinates).  Metric rows count towards n_instr (<= B200GP_PROG_MAX_ROWS) but
 * not towards B200GP_PROG_MAX_INSTR. */
#define B200GP_PROG_MAX_METRICS 3
#define B200GP_METRIC_MAX_DIM 8
#define B200GP_PROG_MAX_ROWS (B200GP_PROG_MAX_INSTR + B200GP_PROG_MAX_METRICS * 17)
enum {
    B200GP_OP_CONST = 0,          /* p0 = value                      base.py:190-209        */
    B200GP_OP_EXP = 1,            /* p0 = scale                      stationary.py:76-82    */
    B200GP_OP_EXPSQUARED = 2,     /* p0 = scale                      stationary.py:104-106  */
    B200GP_OP_MATERN32 = 3,       /* p0 = scale                      stationary.py:126-129  */
    B200GP_OP_MATERN52 = 4,       /* p0 = scale                      stationary.py:150-153  */
    B200GP_OP_COSINE = 5,         /* p0 = scale                      stationary.py:173-175  */
    B200GP_OP_EXPSINESQUARED = 6, /* p0 = scale, p1 = gamma          stationary.py:202-205  */
    B200GP_OP_RATIONALQUADRATIC = 7, /* p0 = scale, p1 = alpha       stationary.py:232-235  */
    /* closed forms k(tau) of the quasiseparable kernels, used when one is evaluated densely
     * (kernels/quasisep.py:118-163 evaluate / condition at test points); r = distance (unscaled) */
    B200GP_OP_EXPCOS = 8,         /* exp(-p0 r) cos(p1 r)            quasisep.py:343-488    */
    B200GP_OP_EXPSIN = 9,         /* exp(-p0 r) sin(p1 r)            quasisep.py:343-488    */
    B200GP_OP_ADD = 16,           /* pops two, pushes sum            base.py:170-177        */
    B200GP_OP_MUL = 17,           /* pops two, pushes product        base.py:180-187        */
    B200GP_OP_METRIC = 32         /* metric definition header (see above)  transforms.py:57-161 */
};
enum { B200GP_DIST_L1 = 0, B200GP_DIST_L2 = 1 }; /* kernels/distance.py:41-59 */

/* ---- context ---------------------------------------------------------------------------- */
int b200gp_version(void);
/* stream: a cudaStream_t to launch on (e.g. torch's current stream) or NULL for a private one. */
int b200gp_create(int device, void* stream, b200gp_ctx** out);
int b200gp_destroy(b200gp_ctx* ctx);
const char* b200gp_last_error(b200gp_ctx* ctx);
/* number of kernel launches issued by this context since creation (bench "gpu_launches"). */
int64_t b200gp_launch_count(b200gp_ctx* ctx);
/* tunables: "nb" (outer panel width, multiple of 128), "profile" (0/1: per-kernel CUDA-event timers),
 * "build_ahead" (0/1: generate block column J+1 on a side stream under the int8 update of column J),
 * "qs_chunk" (points per thread in the quasiseparable scans), "qs_tree" (0: thread-sequential fan-in-16 tree over the
 * chunk composites, 1: warp-shuffle scan kernels, fan-in 32) */
int b200gp_set_option(b200gp_ctx* ctx, const char* key, int64_t value);
/* read an option back (tests restore what they change); key "reset" of b200gp_set_option restores every default */
int b200gp_get_option(b200gp_ctx* ctx, const char* key, int64_t* value);

/* per-kernel device timings accumulated while option "profile"=1 (ms, CUDA events on ctx stream) */
typedef struct {
    double syrk_ms;     /* trailing-update DMMA GEMM launches             */
    double syrk_flop;   /* useful flop issued by those launches (2*M*N*K over computed tiles) */
    int64_t syrk_launches;
    double panel_ms;    /* potf2 + panel GEMMs                            */
    double build_ms;    /* stand-alone kernel-matrix build launches       */
    double build_bytes; /* bytes written by those launches                */
    double solve_ms;    /* triangular solves                              */
    double qs_ms;       /* quasiseparable scan kernels                    */
    double qs_bytes;    /* algorithmic bytes moved by them                */
    int64_t qs_launches;
    double i8_ops;      /* int8 tensor ops (2 x MAC) issued by the fixed-point update launches (time: syrk_ms) */
    double trtri_ms;    /* b200gp_dense_log_probability_grad: in-place triangular inverse L^-1 */
    double contract_ms; /* b200gp_dense_log_probability_grad: mirror + W tiles + derivative epilogue + reductions */
} b200gp_profile;
int b200gp_get_profile(b200gp_ctx* ctx, b200gp_profile* out, int reset);

/* fp64 tensor (DMMA) peak micro-benchmark on this device: returns achieved TFLOP/s of a register-resident loop, on
 * all SMs, of the mma shape the fp64 GEMM mainloops issue (mma.sync.m16n8k16.f64), and of a DFMA loop.
 * The loop length is the option "peak_iters", in units of 16 m8n8k4 instructions per warp (equal flops for every shape). */
int b200gp_measure_fp64_peak(b200gp_ctx* ctx, double* dmma_tflops, double* dfma_tflops);
/* the same DMMA loop for one fp64 mma shape (m, n, k): (8, 8, 4), (16, 8, 4), (16, 8, 8) or (16, 8, 16); TFLOP/s
 * counting 2 m n k flop per instruction.  For measurement only (tools/dmma_shapes.py). */
int b200gp_measure_dmma_shape(b200gp_ctx* ctx, int m, int n, int k, double* tflops);
/* int8 tensor peak micro-benchmark: wgmma.m64n128k32.s32.s8.s8 issued back to back by two warpgroups on every SM
 * from resident shared-memory operands (no TMA traffic); returns TOP/s (2 x MAC). */
int b200gp_measure_i8_peak(b200gp_ctx* ctx, double* tops);

/* diagnostics for the int8 fixed-point tensor-core update (wgmma s8 x s8 -> s32, ozaki.cu):
 * C (rows x rows, host, in/out) -= sum_{s+t<S} 2^-(12+7(s+t)) rs_i rs_j Q_s Q_t^T with Q_s the S int8 digit planes
 * (each rows x K, row-major, host).  rows % 256 == 0, K % 128 == 0.  Used by the parity tests only. */
int b200gp_i8_update_test(b200gp_ctx* ctx, const int8_t* planes, int S, int64_t rows, int64_t K,
                          const double* rs, double* C);
/* timing diagnostic of ONE update-launch shape: (rows x cols) fp64 block, K int8 columns, S planes filled on the device;
 * mean milliseconds over `reps` launches and (optional, 16 slots) the in-kernel cycle counters of one more launch.
 * ldq / ldc: row strides of the digit planes / of C (0 = compact), to reproduce the strides of a large factorisation.
 * The kernel variant follows the context options (ozaki_cluster / ozaki_pairing / ozaki_layout / ...). */
int b200gp_i8_update_bench(b200gp_ctx* ctx, int64_t rows, int64_t cols, int64_t K, int S, int reps,
                           int64_t ldq, int64_t ldc, double* ms_out, unsigned long long* dbg_out);
/* diagnostics for the gradient's triangular tile kernel (grad.cu): one launch with the arguments and grid that
 * b200gp_dense_log_probability_grad uses, on host operands; T 128-blocks, np = 128 T, matrices row-major, diagA the T
 * 128 x 128 blocks that replace A's diagonal blocks.  Used by the kernel-level tests only.
 * mode 0 (inverse step, 0 <= j <= T-2): A (np x np), B (128 x np), C (np x np, in/out); tile rows ti = j+1..T-1 of
 *   block column j of C <- sum_{k=j+1..ti} A_ti,k B_k^T, every other element of C is left as it is.
 * mode 1 (W tiles, 1 <= n <= np, 1 <= ndim <= 8): U = A with diagonal blocks diagA; for ti >= tj, W_ti,tj =
 *   sum_{k=ti..T-1} U_ti,k U_tj,k^T weighted as in the gradient with the kernel program (prog, n_instr), X (n x ndim)
 *   and alpha (n); out: wdiag (n), partial (T (T+1) / 2 x 16 per-tile slot partials) and, with dxpart and dX both
 *   non-NULL (the coordinate-gradient instantiation), dxpart (per tile [row sums, column sums][ndim][128]) and the
 *   reduced dX (n x ndim).  B and C are unused. */
int b200gp_grad_tiles_test(b200gp_ctx* ctx, int mode, int T, int j, const double* A, const double* diagA,
                           const double* B, double* C, const double* prog, int n_instr, const double* X, int64_t n,
                           int ndim, const double* alpha, double* wdiag, double* partial, double* dxpart, double* dX);
/* diagnostics for the fp64 tensor-core GEMM of the dense factorisation (dense.cu gemm_nt_kernel): one launch with
 * exactly these arguments on device copies of the host buffers A (a_elems doubles), B (b_elems) and C (c_elems, in/out:
 * the whole buffer comes back).  For problem p < batch and each computed 128 x 128 tile (ti, tj) -- every tj <= ti < tiles_m
 * with lower != 0 (then tiles_n == tiles_m), else every ti < tiles_m, tj < tiles_n --
 *   C_p(ti, tj) = G + alpha sum_{k < K} A_p(ti, k) B_p(tj, k)^T   (A_p = A + p strideA, row r at A_p + r lda; B, C alike),
 * with G = 0 (beta_mode 0), the tile's previous value (1), or the generator (2): k(x_{row0+i}, x_{col0+j}) from the
 * kernel program (prog, n_instr) on X (n_valid x ndim), plus diag[row0+i] where row0 + i == col0 + j; 1 on that diagonal
 * and 0 elsewhere once row0 + i or col0 + j >= n_valid.  K is a positive multiple of 128, the row strides and the
 * problem strides are even.  Every other element of C is left as it is.  Used by the kernel-level tests only. */
int b200gp_gemm_nt_test(b200gp_ctx* ctx, const double* A, int64_t a_elems, int64_t lda, int64_t strideA,
                        const double* B, int64_t b_elems, int64_t ldb, int64_t strideB, double* C, int64_t c_elems,
                        int64_t ldc, int64_t strideC, int batch, int tiles_m, int tiles_n, int K, double alpha,
                        int beta_mode, int lower, const double* prog, int n_instr, const double* X, int ndim,
                        const double* diag, int64_t n_valid, int64_t row0, int64_t col0);
/* diagnostics for the diagonal-block kernel of the dense factorisation (dense.cu potf2_trtri_kernel): one launch on
 * device copies of A (a_elems doubles, in/out: the whole buffer comes back), which holds `batch` 128 x 128 blocks at
 * A + p strideA with row stride lda.  Each block's lower triangle is replaced by its Cholesky factor L (the strict upper
 * triangle is neither read nor written); linv (batch x 128 x 128) receives L^-1 with zeros above the diagonal; info[p]
 * = global_off + the 1-based column of the block's first pivot that is not > 0 (NaN included), or 0.  Used by the
 * kernel-level tests only. */
int b200gp_potf2_test(b200gp_ctx* ctx, double* A, int64_t a_elems, int64_t lda, int64_t strideA, int batch,
                      int global_off, double* linv, int* info);
/* option keys for b200gp_set_option: "nb", "profile", "peak_iters", "trim",
 * "ozaki_slices" (0 = native fp64 DMMA trailing update; 2..8 = int8 digit planes), "ozaki_min_n". */

/* ---- kernels.Kernel.__call__  (kernels/base.py:84-103) ---------------------------------- */
/* out[n1*n2] = k(X1_i, X2_j);  X1 (n1, ndim), X2 (n2, ndim) row-major. */
int b200gp_kernel_matrix(b200gp_ctx* ctx, const double* prog, int n_instr,
                         const double* X1, int64_t n1, const double* X2, int64_t n2, int ndim,
                         double* out);
/* out[n] = k(X_i, X_i)  (evaluate_diag, base.py:59-66) */
int b200gp_kernel_diag(b200gp_ctx* ctx, const double* prog, int n_instr,
                       const double* X, int64_t n, int ndim, double* out);
/* out[n1] = k(X1, X2) @ y  (Kernel.matmul, base.py:68-82) without materialising K on the host */
int b200gp_kernel_matvec(b200gp_ctx* ctx, const double* prog, int n_instr,
                         const double* X1, int64_t n1, const double* X2, int64_t n2, int ndim,
                         const double* y, double* out);

/* ---- solvers.DirectSolver  (solvers/direct.py:17-95) ------------------------------------ */
/* __init__ (direct.py:30-53): K = k(X,X) + diag generated tile-by-tile on the device and
 * factored in place, L L^T = K.  `info` as described above. */
int b200gp_dense_create(b200gp_ctx* ctx, const double* prog, int n_instr,
                        const double* X, int64_t n, int ndim, const double* diag,
                        b200gp_dense** out, int* info);
/* same with X/diag already resident on the device (bench `value` leg) */
int b200gp_dense_create_dev(b200gp_ctx* ctx, const double* prog, int n_instr,
                            const double* X_dev, int64_t n, int ndim, const double* diag_dev,
                            b200gp_dense** out, int* info);
/* __init__ with covariance= given (direct.py:50-53): factor a host n x n matrix. */
/* DirectSolver.__init__ fused with the data term of log_probability (gp.py:313-316): *sumsq = sum((L^-1 resid)^2); the
 * forward substitution runs panel by panel under the factorisation (resid: n values, host or device) */
int b200gp_dense_create_with_resid(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n, int ndim,
                                   const double* diag, const double* resid, b200gp_dense** out, int* info, double* sumsq);
int b200gp_dense_create_from_cov(b200gp_ctx* ctx, const double* cov, int64_t n,
                                 b200gp_dense** out, int* info);
int b200gp_dense_free(b200gp_dense* s);
/* normalization() - n/2 log(2 pi) = sum_i log L_ii   (direct.py:61-64) */
int b200gp_dense_logdet_half(b200gp_dense* s, double* out);
/* solve_triangular (direct.py:66-70): Y (n, nrhs) row-major, in place. */
int b200gp_dense_solve_triangular(b200gp_dense* s, double* Y, int64_t nrhs, int transpose);
/* dot_triangular (direct.py:72-73): Y <- L @ Y, Y (n, nrhs). */
int b200gp_dense_dot_triangular(b200gp_dense* s, double* Y, int64_t nrhs);
/* condition (direct.py:75-95): out (m, m) = Kss - A^T A, A = L^-1 Ks; Xtest NULL => X. */
int b200gp_dense_condition(b200gp_dense* s, const double* prog, int n_instr,
                           const double* Xtest, int64_t m, const double* diag_test, double* out);
/* C (m, m) <- C - At At^T, At (m, k) row-major, host operands: "Kss - A.T @ A" (direct.py:93-95; quasisep solver.py:137-139)
 * for solvers without a kernel program on the device (a factor of a precomputed covariance -- noise.Dense / noise.Banded,
 * noise.py:98-240 -- or of generator arrays); the host passes A^T from its own solve_triangular call. */
int b200gp_gram_downdate(b200gp_ctx* ctx, const double* At, int64_t m, int64_t k, double* C);
/* covariance() (direct.py:58-59): regenerated by the build kernel; only valid for objects
 * created from a program.  out (n, n). */
int b200gp_dense_covariance(b200gp_dense* s, double* out);
/* scale_tril (direct.py:28): lower factor, zeros above the diagonal.  out (n, n). */
int b200gp_dense_get_factor(b200gp_dense* s, double* out);
/* GaussianProcess.log_probability (gp.py:126-138,313-320) for a fresh factor, fused:
 * logp = -0.5 |L^-1 r|^2 - sum log L_ii - n/2 log 2pi ; non-finite -> -inf.  r = y - mean. */
int b200gp_dense_log_probability(b200gp_ctx* ctx, const double* prog, int n_instr,
                                 const double* X, int64_t n, int ndim, const double* diag,
                                 const double* resid, double* logp);
int b200gp_dense_log_probability_dev(b200gp_ctx* ctx, const double* prog, int n_instr,
                                     const double* X_dev, int64_t n, int ndim,
                                     const double* diag_dev, const double* resid_dev, double* logp);
/* log_probability (gp.py:313-320, as b200gp_dense_log_probability) and its gradient, for a fresh factor that this call
 * builds and frees.  With r = resid, alpha = K^-1 r and W = K^-1:
 *   d logp / d theta = 1/2 sum_ij (alpha_i alpha_j - W_ij) dK_ij / d theta,   d logp / d diag_i = 1/2 (alpha_i^2 - W_ii).
 * Outputs (host):
 *   dprog   n_instr x 4, the program's shape: for each instruction row, column 2 = d logp / d p0 (leaf scale or CONST
 *           value) and column 3 = d logp / d p1 (ExpSineSquared gamma, RationalQuadratic alpha); 0 everywhere else,
 *           metric-definition rows included;
 *   dmetric B200GP_PROG_MAX_METRICS x B200GP_METRIC_MAX_DIM: entry (m, r) = d logp / d lambda at lambda = 1 when row r
 *           of metric m + 1 is scaled by lambda (0 for rows / metrics the program does not have);
 *   ddiag   n;  alpha  n (= d logp / d mean = -d logp / d y).
 * At most 16 differentiable scalars per program (one per leaf scale, CONST, gamma / alpha, metric row); programs with
 * more, or with the closed forms of quasiseparable kernels (B200GP_OP_EXPCOS / EXPSIN), are refused.  L^-1 is formed
 * in place and W is never stored: peak memory is that of b200gp_dense_log_probability plus O(n) per-row buffers.
 * Deterministic: no floating-point atomics.  Non positive-definite input does not fail: logp = -inf and every gradient
 * output is NaN. */
int b200gp_dense_log_probability_grad(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n,
                                      int ndim, const double* diag, const double* resid, double* logp, double* dprog,
                                      double* dmetric, double* ddiag, double* alpha);
/* b200gp_dense_log_probability_grad plus the gradient with respect to the coordinates, from the same contraction:
 *   dX  n x ndim, row-major (host): d logp / d x_i = sum_{j != i} (alpha_i alpha_j - W_ij) grad_1 k(x_i, x_j).
 * The kernel is stationary, so grad_1 k(x_i, x_j) depends on x_i - x_j only; at coincident points (x_i = x_j, i != j)
 * it is taken as 0 (the L1 distance and the L2 Exp leaf have no derivative there).  ndim <= B200GP_METRIC_MAX_DIM.
 * The other outputs are bitwise equal to b200gp_dense_log_probability_grad's.  The per-tile partials of dX add about
 * n^2 ndim / 16 bytes of device memory (805 MB at n = 65536, ndim = 3).  Non positive-definite input: logp = -inf and
 * every output, dX included, is NaN. */
int b200gp_dense_log_probability_grad_x(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n,
                                        int ndim, const double* diag, const double* resid, double* logp, double* dprog,
                                        double* dmetric, double* ddiag, double* alpha, double* dX);
/* batched hyper-parameter grid (BASELINE config 5): nbatch programs of equal length over one X;
 * diag (n) and resid (n) shared.  logp[nbatch]. */
int b200gp_dense_log_probability_batched(b200gp_ctx* ctx, const double* progs, int n_instr,
                                         int64_t nbatch, const double* X, int64_t n, int ndim,
                                         const double* diag, const double* resid, double* logp);

/* ---- one dense log_probability sharded over several GPUs (one process per GPU) ---------------------------
 * Step API driven by the host (tinygp_b200/multigpu.py) with ONE all-gather per block column in between
 * (torch.distributed / NCCL): for J in 0..ncol-1: update_rows(J, my rows) -> pack -> [all_gather] -> unpack ->
 * panel(J); then finish().  Every rank ends up with the complete factor. */
typedef struct b200gp_mg b200gp_mg;
/* streaming != 0: keep no np x np fp64 matrix (rolling np x nb column buffer; the forward solve and log-det
 * are folded into each panel step) -- only the int8 digit planes stay resident (S N^2 bytes per GPU). */
int b200gp_mg_create(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n, int ndim,
                     const double* diag, const double* resid, int slices, int streaming, b200gp_mg** out);
int b200gp_mg_free(b200gp_mg* m);
/* the panel step in two halves (sharded triangular solve): factor the diagonal block (its rows must be valid on every
 * rank: the host broadcasts them) and solve this rank's rows [r0, r1) below it; after the host has all-gathered the
 * finished column, _finish cuts the digits of all rows (and, streaming, folds the forward substitution / log-det). */
int b200gp_mg_panel_factor(b200gp_mg* m, int J, int64_t r0, int64_t r1);
int b200gp_mg_panel_finish(b200gp_mg* m, int J);
/* streaming mode only: make a caller-owned contiguous device buffer (rows x nb doubles, rows >= np) the rolling block
 * column, so that rank chunks are contiguous and the column can be all-gathered in place by NCCL (no pack / unpack) */
int b200gp_mg_use_colbuf(b200gp_mg* m, double* buf_dev, int64_t rows);
int b200gp_mg_geometry(b200gp_mg* m, int64_t* np, int64_t* nb, int* ncol);
int b200gp_mg_update_rows(b200gp_mg* m, int J, int64_t r0, int64_t r1);
int b200gp_mg_pack(b200gp_mg* m, int J, int64_t r0, int64_t r1, double* buf_dev);
int b200gp_mg_unpack(b200gp_mg* m, int J, int64_t r0, int64_t r1, const double* buf_dev);
int b200gp_mg_panel(b200gp_mg* m, int J);
int b200gp_mg_finish(b200gp_mg* m, double* logp);

/* ---- solvers.QuasisepSolver  (solvers/quasisep/solver.py:19-139) ------------------------- */
/* Quasiseparable kernels (kernels/quasisep.py) are lowered to a list of `ncomp` components
 * (a Sum is block-diagonal, quasisep.py:241-295), each B200GP_QS_STRIDE doubles:
 * {kind, sigma_scale, p0, p1, p2, p3, mul_next, 0}.  sigma_scale multiplies Pinf (Scale, :334-340).  mul_next = 1
 * chains the component with the next one into a Product term (quasisep.py:298-331: Kronecker-structured state, the
 * first factor's index fastest as in _prod_helper :676-687; up to 3 factors, term size <= 6). */
#define B200GP_QS_STRIDE 8
#define B200GP_QS_MAX_COMP 8
#define B200GP_QS_MAX_J 8
enum {
    B200GP_QS_EXP = 0,      /* p0 = scale, p1 = sigma [, p2 = decay rate used instead of 1/scale]   quasisep.py:491-525 */
    B200GP_QS_MATERN32 = 1, /* p0 = scale, p1 = sigma                 quasisep.py:528-569 */
    B200GP_QS_MATERN52 = 2, /* p0 = scale, p1 = sigma                 quasisep.py:572-633 */
    B200GP_QS_SHO = 3,      /* p0 = omega, p1 = quality, p2 = sigma   quasisep.py:404-488 */
    B200GP_QS_CELERITE = 4, /* p0..p3 = a, b, c, d                    quasisep.py:343-401 */
    B200GP_QS_COSINE = 5,   /* p0 = scale, p1 = sigma                 quasisep.py:636-673 */
    /* one complex-conjugate root pair -c -+ i d of a CARMA process (quasisep.py:690-900): p0 = c, p1 = d, p2, p3 = the two
     * entries of its observation model (:770-792), slot 7 = sign of Re(acf) (:870); transition exp(-c dt) [[cos, sin],
     * [-sin, cos]](d dt) (:886-900), Pinf = [[s, -c/d], [-c/d, s + 2 c^2/d^2]] (:866-882).  The real roots of a CARMA process
     * are B200GP_QS_EXP components with sigma_scale = sign of Re(acf). */
    B200GP_QS_CARMA2 = 6
};
/* _check_sorted (solver.py:142-146): *unsorted = any(diff(t) < 0), bit-exact boolean. */
int b200gp_qs_check_sorted(b200gp_ctx* ctx, const double* t, int64_t n, int* unsorted);
/* __init__ (solver.py:35-82): generators (quasisep.py:102-116) + noise + Cholesky (ops.py:352-365).
 * `unsorted` is set (and nothing factored, rc=0) if assume_sorted==0 and t is not sorted. */
int b200gp_qs_create(b200gp_ctx* ctx, const double* comps, int ncomp,
                     const double* t, int64_t n, const double* diag, int assume_sorted,
                     b200gp_qs** out, int* unsorted, int* info);
int b200gp_qs_create_dev(b200gp_ctx* ctx, const double* comps, int ncomp,
                         const double* t_dev, int64_t n, const double* diag_dev, int assume_sorted,
                         b200gp_qs** out, int* unsorted, int* info);
int b200gp_qs_free(b200gp_qs* s);
int b200gp_qs_state_dim(b200gp_qs* s, int* J);
int b200gp_qs_logdet_half(b200gp_qs* s, double* out);     /* sum log c   (solver.py:90-93) */
int b200gp_qs_variance(b200gp_qs* s, double* out);        /* d (n)       (solver.py:84-85) */
/* factor generators: c (n), w (n, J)  (LowerTriQSM(diag=c, lower=(p, w, a)), core.py:524-539) */
int b200gp_qs_get_factor(b200gp_qs* s, double* c, double* w);
/* symmetric generators d (n), p (n,J), q (n,J), a (n,J,J)  (quasisep.py:102-116) */
int b200gp_qs_get_generators(b200gp_qs* s, double* d, double* p, double* q, double* a);
/* sum_k (L^-1 y)_k^2 -- the data term of gp.py:313-316 (`-0.5 * jnp.sum(jnp.square(alpha))`) reduced on the device, so
 * log_probability never brings the N-vector alpha back to the host (y: host or device, n doubles). */
int b200gp_qs_solve_sumsq(b200gp_qs* s, const double* y, double* out);
/* solve_triangular (solver.py:95-99; ops.py:463-472 / 489-498): Y (n, nrhs) in place */
int b200gp_qs_solve_triangular(b200gp_qs* s, double* Y, int64_t nrhs, int transpose);
/* dot_triangular (solver.py:101-102; core.py:303-305, ops.py:308-316) */
int b200gp_qs_dot_triangular(b200gp_qs* s, double* Y, int64_t nrhs);
/* SymmQSM @ y (core.py:499-505): Y <- K Y with K the covariance incl. noise */
int b200gp_qs_matmul(b200gp_qs* s, double* Y, int64_t nrhs);
/* fused log_probability for a fresh factor (gp.py:313-320 through solver.py:73-99) */
int b200gp_qs_log_probability(b200gp_ctx* ctx, const double* comps, int ncomp,
                              const double* t, int64_t n, const double* diag, const double* resid,
                              int assume_sorted, int* unsorted, double* logp);
int b200gp_qs_log_probability_dev(b200gp_ctx* ctx, const double* comps, int ncomp,
                                  const double* t_dev, int64_t n, const double* diag_dev,
                                  const double* resid_dev, int assume_sorted, int* unsorted,
                                  double* logp);
/* Quasisep.matmul(X1, X2, y) = to_general_qsm(X1, X2) @ y  (kernels/quasisep.py:118-163, solvers/quasisep/
 * general.py:66-106) in O((n + m) J^2): a forward and a backward state scan over the n sorted training
 * coordinates, then one searchsorted + two transition matrices per test point.  Host buffers; Y is n x nrhs and
 * out is m x nrhs, row-major.  This is the predictive mean at arbitrary test points (gp.py:357). */
int b200gp_qs_kernel_matmul(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t_test,
                            int64_t m, const double* t_train, int64_t n, const double* Y, int64_t nrhs,
                            double* out);
/* diag((K + N)^-1), n values (host): the diagonal of `factor.inv().gram()` (solvers/quasisep/core.py:310-317,
 * 424-434) by one backward scan in O(n J^3), without forming the matrix.  The conditioned variance at the inputs
 * (solver.py:124-129 then :84-85) is  noise* + N - N^2 diag((K + N)^-1). */
int b200gp_qs_inverse_diagonal(b200gp_qs* s, double* out);
/* variance of the conditioned process at the inputs for the solver's own kernel = diagonal of solver.py:124-129 as
 * read by solver.py:84-85:  out_i = noise_pred_i + N_i - N_i^2 diag((K + N)^-1)_i  (n values in, n out, host). */
int b200gp_qs_conditioned_variance(b200gp_qs* s, const double* noise_pred, double* out);
/* QuasisepSolver.condition (solvers/quasisep/solver.py:104-139): out (m x m, host, row-major) =
 * k(X*, X*) [+ diag] - A^T A with A = factor.solve(k(X, X*)).  The reference adds the predictive noise in its QSM
 * branch (:124-129: X* = X and a quasiseparable kernel; returned here densified) and NOT in the dense branch
 * (:131-139), so `diag_or_null` (m values) is passed only for the former.  `prog` is the predictive kernel's
 * program for 1-D coordinates; t_test == NULL means X* = X (m is ignored, out is n x n).  Build kernel -> one
 * forward-substitution scan per test point -> NT GEMM with the generator epilogue; no host arithmetic. */
int b200gp_qs_condition(b200gp_qs* s, const double* prog, int n_instr, const double* t_test, int64_t m,
                        const double* diag_or_null, double* out);
/* jnp.searchsorted(X2, X1, side="right") - 1  (kernels/quasisep.py:121): bit-exact indices */
int b200gp_searchsorted_right_m1(b200gp_ctx* ctx, const double* sorted, int64_t n,
                                 const double* query, int64_t m, int64_t* out);

/* ---- quasiseparable-matrix algebra on generator arrays  (solvers/quasisep/core.py, ops.py) ---------------- */
/* A b200gp_qsm holds DEVICE-resident generators of one of core.py's seven classes: d (n); strictly lower and / or
 * strictly upper parts (p, q: n x m, a: n x m x m, row-major) of orders ml, mu.  StrictLowerTriQSM (core.py:168-236):
 * M[i, j] = p_i . a_{i-1} ... a_{j+1} . q_j (i > j); StrictUpperTriQSM with the same (p, q, a) is its transpose
 * (core.py:239-292).  Handles returned by the operations are new objects; parts and transposes share device arrays.
 * Every operation is a chunked scan in O(n m^3) -- one warp per chunk, matrix state in shared memory -- nothing is
 * densified.  This is what QuasisepSolver.condition's QSM branch (solver.py:124-129) is made of. */
typedef struct b200gp_qsm b200gp_qsm;
enum {
    B200GP_QSM_DIAG = 0,         /* DiagQSM           core.py:134-165 */
    B200GP_QSM_STRICT_LOWER = 1, /* StrictLowerTriQSM core.py:168-236 */
    B200GP_QSM_STRICT_UPPER = 2, /* StrictUpperTriQSM core.py:239-292 */
    B200GP_QSM_LOWER = 3,        /* LowerTriQSM       core.py:295-345 */
    B200GP_QSM_UPPER = 4,        /* UpperTriQSM       core.py:348-393 */
    B200GP_QSM_SQUARE = 5,       /* SquareQSM         core.py:396-481 */
    B200GP_QSM_SYMM = 6          /* SymmQSM           core.py:484-540 */
};
/* constructors of core.py from host arrays (NULL for the parts the kind does not have; SYMM takes d + lower) */
int b200gp_qsm_create(b200gp_ctx* ctx, int64_t n, int kind, int ml, int mu, const double* d, const double* lp,
                      const double* lq, const double* la, const double* up, const double* uq, const double* ua,
                      b200gp_qsm** out);
int b200gp_qsm_free(b200gp_qsm* q);
int b200gp_qsm_info(b200gp_qsm* q, int64_t* n, int* kind, int* ml, int* mu);
/* download generator arrays (NULL = skip) */
int b200gp_qsm_get(b200gp_qsm* q, double* d, double* lp, double* lq, double* la, double* up, double* uq, double* ua);
/* `.diag` (which = 0), `.lower` (1), `.upper` (2) of the dataclasses of core.py, sharing the device arrays */
int b200gp_qsm_part(b200gp_qsm* q, int which, b200gp_qsm** out);
/* LowerTriQSM(diag=, lower=) / UpperTriQSM(diag=, upper=) / SquareQSM(diag=, lower=, upper=) / SymmQSM(diag=, lower=) */
int b200gp_qsm_compose(b200gp_qsm* diag, b200gp_qsm* lower, b200gp_qsm* upper, int symm, b200gp_qsm** out);
int b200gp_qsm_transpose(b200gp_qsm* q, b200gp_qsm** out);                       /* core.py transpose() */
/* scale() of core.py:155-156, 196-197, 272-273: c is one scalar, or n per-row factors if is_vector */
int b200gp_qsm_scale(b200gp_qsm* q, const double* c, int is_vector, b200gp_qsm** out);
int b200gp_qsm_neg(b200gp_qsm* q, b200gp_qsm** out);                             /* __neg__ */
int b200gp_qsm_add(b200gp_qsm* a, b200gp_qsm* b, b200gp_qsm** out);              /* elementwise_add  ops.py:24-35 */
int b200gp_qsm_elementwise_mul(b200gp_qsm* a, b200gp_qsm* b, b200gp_qsm** out);  /* elementwise_mul  ops.py:38-49 */
/* qsm_mul (ops.py:52-214): the phi / psi scans (:62-87) and the per-point assembly (:92-203).  Operand pairs for which
 * the reference builds generators of unequal widths (it then fails) are refused with a message. */
int b200gp_qsm_mul(b200gp_qsm* a, b200gp_qsm* b, b200gp_qsm** out);
int b200gp_qsm_gram(b200gp_qsm* a, b200gp_qsm** out);                            /* SquareQSM.gram  core.py:424-434 */
/* LowerTriQSM.inv (core.py:310-317), UpperTriQSM.inv (:362-363), SymmQSM.inv = symm_inv (ops.py:403-460);
 * SquareQSM.inv (core.py:436-478: sequential, one warp) */
int b200gp_qsm_inv(b200gp_qsm* a, b200gp_qsm** out);
/* SymmQSM.cholesky (core.py:522-537, ops.py:352-365).  *info = 1-based index of the first non-positive pivot (the
 * generators are NaN from there on, like the reference's), 0 if none */
int b200gp_qsm_cholesky(b200gp_qsm* a, b200gp_qsm** out, int64_t* info);
/* matmul of every class (ops.py:308-349): Y (n x nrhs, host, row-major) <- A Y */
int b200gp_qsm_matmul(b200gp_qsm* a, double* Y, int64_t nrhs);
/* LowerTriQSM.solve / UpperTriQSM.solve (core.py:319-336, 366-383; ops.py:463-512): Y <- A^-1 Y */
int b200gp_qsm_solve(b200gp_qsm* a, double* Y, int64_t nrhs);
int b200gp_qsm_sum_log_diag(b200gp_qsm* a, double* out);                         /* solver.py:90-93 on a factor */
/* Quasisep.to_symm_qsm(t) (kernels/quasisep.py:102-116) as a device SymmQSM, no noise; t: n sorted host values */
int b200gp_qs_kernel_qsm(b200gp_ctx* ctx, const double* comps, int ncomp, const double* t, int64_t n, b200gp_qsm** out);
/* `solver.factor` (solver.py:82): LowerTriQSM(diag = c, lower = (p, w, a)) of a model-based solver */
int b200gp_qs_factor_qsm(b200gp_qs* s, b200gp_qsm** out);

#ifdef __cplusplus
}
#endif
#endif /* B200GP_H */
