// Shared internals of libb200gp: context, error handling, device buffer cache, kernel programs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>
#include <string>
#include <vector>
#include <stdexcept>
#include "../../include/b200gp.h"

#define TILE 128  // diagonal-block / tile edge used throughout the dense path

struct GpError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

#define CUDA_CHECK(expr)                                                                   \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess) {                                                           \
            char _buf[512];                                                                \
            snprintf(_buf, sizeof(_buf), "%s failed at %s:%d: %s", #expr, __FILE__,        \
                     __LINE__, cudaGetErrorString(_e));                                    \
            throw GpError(_buf);                                                           \
        }                                                                                  \
    } while (0)

// ---- kernel program (device-side copy passed by value as a kernel parameter) -------------
struct KProg {
    int n;
    int op[B200GP_PROG_MAX_INSTR];
    int dist[B200GP_PROG_MAX_INSTR];
    double p0[B200GP_PROG_MAX_INSTR];
    double p1[B200GP_PROG_MAX_INSTR];
    // linear input transforms (transforms.py): metric[i] = 0 (identity) or 1-based index into M
    int metric[B200GP_PROG_MAX_INSTR];
    int nmetric;
    int mcols;  // = ndim of the coordinates every metric applies to (0 if no metrics)
    int mrows[B200GP_PROG_MAX_METRICS];
    double M[B200GP_PROG_MAX_METRICS][B200GP_METRIC_MAX_DIM * B200GP_METRIC_MAX_DIM];
};

KProg parse_prog(const double* prog, int n_rows, int ndim);

struct CachedBuf {
    void* ptr;
    size_t bytes;
};

struct b200gp_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;
    int64_t launches = 0;
    int64_t nb = 1024;  // outer panel width of the blocked Cholesky
    bool profile = false;
    b200gp_profile prof{};
    std::vector<CachedBuf> cache;  // freed big buffers kept for reuse
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    int num_sms = 132;
    int64_t peak_iters = 4096;  // loop length of the fp64 peak micro-benchmarks
    int64_t qs_chunk_max = 256; // upper end of the automatic chunk-length search of the quasiseparable scans
    int64_t qs_chunk = 0;       // points per thread in the quasiseparable scans (0 = chosen per problem size, see qs_create_impl)
    int64_t qsm_chunk = 0;      // points per warp in the QSM-algebra scans (qsm.cu); 0 = chosen per problem size
    int64_t qsm_sequential_redos = 0;   // read-only counter: Riccati scans redone sequentially after the consistency check (qsm.cu run_ric)
    int64_t qs_tree = 1;        // 1: warp-shuffle scan over the chunk composites (fan-in 32; default), 0: thread-sequential fan-in-16 tree
    int64_t qs_kernel = 1;      // quasiseparable factorisation: 1 = layout-specialised kernels (qs_fast.cuh) when the model's block
                                // layout is compiled in, 0 = always the generic J x J kernels of qs_core.cuh
    int64_t qs_occupancy = 1;   // structured quasisep kernels: 1 = register-capped variants (16 / 12 resident warps per SM), 0 = natural
    int64_t build_fast = 2;     // kernel-matrix build: 2 = + compile-time single-leaf kernels (coef * one stationary leaf, <= 3-D),
                                // 1 = sum-of-products normal form when the program has one, 0 = interpreter
    int64_t oz_splitk = 1024;   // int8 update (default launch shape): > 0 = split K over idle SM pairs, value = fixed cost of a tile in K
                                // columns for the policy (ozaki.cu choose_splitk); 0 = one K range per tile
    int64_t mg_splitk = 0;       // sharded path: 0 (default) = one K range per tile: bit-identical results for every rank count;
                                 // 1 = tail split-K on every rank's rows too (the summation order then depends on the rank count)
    int64_t oz_splitk_force = 0; // > 1: that many K segments in every default-shape launch (tests)
    int64_t nb_batched = 4096;  // outer panel width of the batched small-N driver: 4096 = N of config 5, i.e. one left-looking sweep (reads C
                                // once per 128-column block)
    // > 0: int8 fixed-point trailing update with this many digit planes (ozaki.cu) once N >= oz_min_n; 0 = DMMA.  7 planes =
    // 48 bits under the row scale, 8 = 55 bits (ozaki_slices).
    int64_t oz_slices = 7;
    int64_t oz_lookahead = 0;   // overlap the fp64 panel factorisation with the int8 update on a second stream
    cudaStream_t stream2 = nullptr;
    int64_t build_ahead = 0;    // 1: generate block column J+1 on a side stream under the int8 update of column J
    // fused log_probability: residual whose forward substitution dense_factor_ozaki runs panel by panel on a side stream,
    // under the int8 update of the NEXT block column (set by dense_logp_impl, consumed by the factorisation)
    const double* fuse_resid = nullptr;   // n values, host or device
    int64_t fuse_n = 0;
    double* fuse_y = nullptr;             // np, owned by the caller of the factorisation afterwards (ctx->alloc)
    double* fuse_x = nullptr;             // np: L^-1 resid once the factorisation has returned
    int64_t solve_overlap = 1;            // option: 1 = hide the forward substitution of log_probability under the factorisation
    cudaStream_t stream_solve = nullptr;
    cudaStream_t stream_hi = nullptr;   // high-priority stream of the panel factorisation's diagonal-block chain
    int64_t oz_prefetch = 0;    // L2 prefetch distance (K-chunks of 128) of the int8 update's TMA producer
    int64_t oz_pairing = 1;    // int8 update: 1 = accumulate two digit groups at once (default: 16 instead of 28 operand-stage loads
                               // per K chunk at 7 planes), 0 = one group per pass, 2 = diagnostic (paired loop order, single groups)
    int64_t oz_layout = 0;     // digit planes: 0 plane-major, 1 chunk-major (all planes of a K chunk adjacent)
    int64_t oz_cluster = 2;     // int8 update kernel: 2 = 2 x 1 cluster with tail split-K (default: B slices multicast to the CTA below),
                                // 1 = wide 256-row CTA tile, CM*10 + CN = cluster shapes of 128 x 128 CTA tiles (ozaki.cu)
    int64_t oz_subpanel = 0;    // two-level blocking of the int8 factorisation: fp64 panel width inside a block column (0 = off:
                                // default)
    int64_t oz_l2promo = 3;     // TMA L2 promotion of the digit-plane maps: 0 none, 1 64 B, 2 128 B, 3 256 B
    // from this size on the int8 fixed-point update is used (with oz_slices > 0); below it the native DMMA path.  Default:
    // never -- on an H100 (400 W) the DMMA factorisation is the faster one at N = 65536 (4.45 against 5.84 s per
    // log_probability, 7 planes) and 40x closer to the LAPACK value; ozaki_min_n = 0 forces the int8 path.  The comparison
    // is against an untuned int8 kernel (ozaki.cu): at 9 warps per CTA ptxas caps it at 168 registers, so the paired and
    // wide variants spill, and each consumer warpgroup waits for its MMAs after every stage instead of keeping one wgmma
    // group in flight; it reached 23 % of the resident-operand wgmma rate.
    int64_t oz_min_n = (int64_t)1 << 40;
    // deferred (non-blocking) kernel timers: event pairs resolved at the next flush_timers()
    struct Pending { cudaEvent_t a, b; double* acc; };
    std::vector<Pending> pending;
    std::vector<cudaEvent_t> event_pool;
    cudaEvent_t get_event();
    void flush_timers();  // synchronises the stream

    void* alloc(size_t bytes);
    void release(void* p, size_t bytes);  // return to cache
    void trim();                          // cudaFree everything cached
};

// RAII device scratch buffer from the context's cache: returned to it on scope exit, also when an error is thrown.
struct Scratch {
    b200gp_ctx* c;
    size_t bytes;
    void* p;
    Scratch(b200gp_ctx* ctx, size_t nbytes) : c(ctx), bytes(nbytes), p(ctx->alloc(nbytes)) {}
    ~Scratch() { c->release(p, bytes); }
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    double* f64() const { return static_cast<double*>(p); }
};

// RAII timer that accumulates into a profile field when ctx->profile is on.  It only records two
// events on the stream (no host synchronisation); elapsed times are resolved by flush_timers().
struct ProfTimer {
    b200gp_ctx* c;
    double* acc;
    cudaEvent_t a = nullptr;
    ProfTimer(b200gp_ctx* ctx, double* field) : c(ctx), acc(field) {
        if (c->profile) {
            a = c->get_event();
            cudaEventRecord(a, c->stream);
        }
    }
    ~ProfTimer() {
        if (c->profile) {
            cudaEvent_t b = c->get_event();
            cudaEventRecord(b, c->stream);
            c->pending.push_back({a, b, acc});
        }
    }
};

#define API_BEGIN(ctxptr)            \
    b200gp_ctx* _ctx = (ctxptr);     \
    if (!_ctx) return 1;             \
    try {                            \
        CUDA_CHECK(cudaSetDevice(_ctx->device));
#define API_END                      \
        return 0;                    \
    } catch (const std::exception& e) { \
        _ctx->err = e.what();        \
        return 2;                    \
    }

// ---- dense path (dense.cu) -----------------------------------------------------------------
struct b200gp_dense {
    b200gp_ctx* ctx = nullptr;
    int64_t n = 0;    // logical size
    int64_t np = 0;   // padded to a multiple of TILE
    int64_t ld = 0;   // leading dimension of `mat` (= np, or the panel width in streaming mode)
    size_t mat_bytes = 0;    // bytes owned behind mat_alloc (0: not owned)
    double* mat_alloc = nullptr;
    double* mat = nullptr;   // row-major; element (r, c) at mat[r * ld + c]; lower triangle holds L after factorisation.
                             // In streaming mode this is a VIRTUAL base (column buffer minus the block-column offset).
    double* linv = nullptr;  // np/TILE inverses of the diagonal blocks, each TILE x TILE
    int* info_dev = nullptr;
    int info = 0;
    // what is needed to regenerate covariance() / run condition()
    bool has_prog = false;
    KProg prog{};
    int ndim = 0;
    double* X_dev = nullptr;     // n x ndim
    double* diag_dev = nullptr;  // n
    bool owns_inputs = false;
};

void dense_build_rect(b200gp_ctx* ctx, const KProg& prog, const double* X1, int64_t n1,
                      const double* X2, int64_t n2, int ndim, const double* diag_or_null,
                      double* out, int64_t ld, int64_t rows_pad, int64_t cols_pad);
void dense_conditioned_covariance_to_host(b200gp_ctx* ctx, const KProg& P, const double* At, int64_t mp, int64_t kp,
                                          const double* xt_dev, const double* dt_dev, int nd, int64_t m,
                                          double* out_host);
b200gp_dense* dense_factor_from_prog(b200gp_ctx* ctx, const KProg& prog, const double* X_dev,
                                     int64_t n, int ndim, const double* diag_dev, bool copy_inputs);
void dense_factor_inplace(b200gp_dense* s, bool generate);
void dense_destroy(b200gp_dense* s);
double dense_logdet_half(b200gp_dense* s);
void dense_solve_vec_dev(b200gp_dense* s, double* y_dev /* np, destroyed */, double* x_dev /* np */,
                         bool transpose);
double dense_sumsq_dev(b200gp_ctx* ctx, const double* x_dev, int64_t n);
// C (op)= alpha A B^T on the fp64 tensor pipe, over tiles_m x tiles_n tiles of 128 x 128 (lower: only the tiles of a square
// C's lower triangle), K a multiple of 16; A's rows start every lda doubles, B's every ldb, both K-contiguous.  beta_mode
// 0: C = alpha AB, 1: C += alpha AB.  batch > 1: that many problems, strideA / B / C elements apart.
void gemm_nt(b200gp_ctx* ctx, double* C, int64_t ldc, const double* A, int64_t lda, const double* B, int64_t ldb,
             int tiles_m, int tiles_n, int K, double alpha, int beta_mode, int lower, int batch = 1, int64_t strideA = 0,
             int64_t strideB = 0, int64_t strideC = 0);
