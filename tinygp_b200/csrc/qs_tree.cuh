// Shared pieces of the quasiseparable path's translation units (quasisep.cu, qs_fast.cu): the solver object, the tree
// over chunk composites (thread-sequential fan-in-16 or warp-shuffle scan) and the partial-sum reduction.
#pragma once
#include "common.cuh"
#include <limits.h>
#include "qs_core.cuh"

#define QS_CHUNK 64

struct b200gp_qs {
    b200gp_ctx* ctx = nullptr;
    int64_t n = 0;
    int J = 0;
    QsModel model{};
    double* t = nullptr;     // n
    double* diag = nullptr;  // n
    double* c = nullptr;     // n
    double* w = nullptr;     // n x J
    int info = 0;
    double logdet_half = 0.0;
    // fused log_probability: forward-solve chunk composites accumulated inside the Cholesky replay pass
    double* fused_comp = nullptr;
    size_t fused_comp_bytes = 0;
    // structured fast path (qs_fast.cu): sum of squares of L^-1 x already reduced inside the factorisation
    bool has_sumsq = false;
    double sumsq = 0.0;
    bool owns_inputs = true;   // false: t / diag are the caller's device buffers (transient log-probability object)
};

static inline bool qs_is_device_ptr(const void* p) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeDevice;
}
// qs_fast.cu
bool qsf_supported(const QsModel& m);
bool qsf_solve_sumsq(b200gp_qs* s, const double* x_dev, double* sumsq_dev);
bool qsf_factor(b200gp_qs* s, const double* t, const double* diag, int* info_dev, double* logdet_dev, const double* x_fuse,
                double* sumsq_dev);

// up-sweep: parent[i] = fold of child[i*R .. i*R+R-1]
template <class Op>
__global__ void __launch_bounds__(QS_THREADS) tree_up_kernel(const double* child, int64_t nchild, double* parent, int64_t nparent) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nparent) return;
    Op acc, e;
    const int64_t b = i * TREE_R;
    acc.load(child, nchild, b);
    for (int64_t j = b + 1; j < b + TREE_R && j < nchild; ++j) {
        e.load(child, nchild, j);
        acc.combine(e);
    }
    acc.store(parent, nparent, i);
}
// top: a single thread walks the (<= TREE_R) top items and emits the state at each item's left edge
template <class Op>
__global__ void tree_top_kernel(const double* items, int64_t n, double* start) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    typename StateOf<Op>::type s;
    state_zero(s);
    Op e;
    for (int64_t i = 0; i < n; ++i) {
        state_store(s, start, n, i);
        e.load(items, n, i);
        e.apply(s);
    }
}
// down-sweep: child start states from the parent's start state
template <class Op>
__global__ void __launch_bounds__(QS_THREADS) tree_down_kernel(const double* child, int64_t nchild, const double* pstart,
                                                               int64_t nparent, double* cstart) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nparent) return;
    typename StateOf<Op>::type s;
    state_load(s, pstart, nparent, i);
    Op e;
    const int64_t b = i * TREE_R;
    for (int64_t j = b; j < b + TREE_R && j < nchild; ++j) {
        state_store(s, cstart, nchild, j);
        if (j + 1 < b + TREE_R && j + 1 < nchild) {
            e.load(child, nchild, j);
            e.apply(s);
        }
    }
}

static __global__ void sum_partials_kernel(const double* part, int64_t n, double* out) {
    __shared__ double sh[1024];
    double acc = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += 1024) acc += part[i];
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = sh[0];
}
static inline unsigned nblk(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// fixed-shape (deterministic) sum of n per-chunk partials: one block per slab of 8192 values, then one block over the
// slab sums (a single block over all chunks of a long series is a serial tail)
static __global__ void sum_slabs_kernel(const double* part, int64_t n, double* slab_sums) {
    __shared__ double sh[256];
    const int64_t lo = (int64_t)blockIdx.x * 8192, hi = (lo + 8192 < n) ? lo + 8192 : n;
    double acc = 0.0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += 256) acc += part[i];
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) slab_sums[blockIdx.x] = sh[0];
}
static void sum_partials(b200gp_ctx* ctx, const double* part, int64_t n, double* out) {
    if (n <= 16384) {
        sum_partials_kernel<<<1, 1024, 0, ctx->stream>>>(part, n, out);
        ctx->launches++;
        return;
    }
    const int64_t nslab = (n + 8191) / 8192;
    Scratch slabs(ctx, (size_t)nslab * 8);
    sum_slabs_kernel<<<(unsigned)nslab, 256, 0, ctx->stream>>>(part, n, slabs.f64());
    sum_partials_kernel<<<1, 1024, 0, ctx->stream>>>(slabs.f64(), nslab, out);
    ctx->launches += 2;
}

// ---------------------------------------------------------------------------------------------
// warp-shuffle scan over the chunk composites (option "qs_tree" = 1): the alternative to the thread-sequential
// fan-in-16 tree above.  One warp scans 32 consecutive composites with a Hillis-Steele inclusive scan
// (5 x __shfl_up of the composite + combine), stores every item's EXCLUSIVE in-warp prefix and the warp total; the
// totals are scanned the same way (fan-in 32: 156250 chunks -> 4883 -> 153 -> 5), and one fully parallel pass per level
// turns "state at the left edge of my warp" + "my exclusive prefix" into "state at my left edge".  Critical path per
// level: 5 combines + 1 apply instead of 15 combines + 16 applies.  The composites are SoA, so the warp's loads and
// stores of one element are coalesced.
// ---------------------------------------------------------------------------------------------
template <class Op>
__global__ void __launch_bounds__(QS_THREADS) warp_scan_kernel(const double* items, int64_t n, double* pre, double* totals,
                                                               int64_t ntot) {
    const int lane = threadIdx.x & 31;
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= ntot) return;                                  // whole warps only: ntot = ceil(n / 32)
    const int64_t i = w * 32 + lane;
    Op cur;
    if (i < n) cur.load(items, n, i);
    else cur.identity();
    Op left;                                                // one temporary: two composites live (register budget)
#pragma unroll 1
    for (int d = 1; d < 32; d <<= 1) {
        left.assign_map(cur, [d](double v) { return __shfl_up_sync(0xffffffffu, v, d); });
        if (lane >= d) {                                    // prefix[i] = prefix[i - d] (applied first) then prefix-part[i]
            left.combine(cur);
            cur = left;
        }
    }
    left.assign_map(cur, [](double v) { return __shfl_up_sync(0xffffffffu, v, 1); });   // exclusive prefix
    if (lane == 0) left.identity();
    if (i < n) left.store(pre, n, i);
    const int64_t last = ((n - w * 32) < 32 ? (n - w * 32) : 32) - 1;     // last valid lane of this warp
    if (totals != nullptr && lane == last) cur.store(totals, ntot, w);
}

// start[i] = pre[i] applied to the state at the left edge of i's warp (zero at the top level)
template <class Op>
__global__ void __launch_bounds__(QS_THREADS) warp_propagate_kernel(const double* pre, int64_t n, const double* pstart,
                                                                    int64_t nparent, double* start) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    typename StateOf<Op>::type s;
    if (pstart != nullptr) state_load(s, pstart, nparent, i >> 5);
    else state_zero(s);
    Op e;
    e.load(pre, n, i);
    e.apply(s);
    state_store(s, start, n, i);
}

// ---------------------------------------------------------------------------------------------
// host-side tree driver: chunk composites -> start state per chunk
// ---------------------------------------------------------------------------------------------
template <class Op>
static void run_tree_warp(b200gp_ctx* ctx, double* comp0, int64_t n0, double* start0) {
    std::vector<int64_t> counts{n0};
    while (counts.back() > 32) counts.push_back((counts.back() + 31) / 32);
    const int L = (int)counts.size();
    std::vector<double*> items(L, nullptr), pre(L, nullptr), starts(L, nullptr);
    items[0] = comp0;
    starts[0] = start0;
    for (int l = 0; l < L; ++l) {
        pre[l] = (double*)ctx->alloc((size_t)Op::SIZE * counts[l] * 8);
        if (l > 0) {
            items[l] = (double*)ctx->alloc((size_t)Op::SIZE * counts[l] * 8);
            starts[l] = (double*)ctx->alloc((size_t)Op::STATE * counts[l] * 8);
        }
    }
    for (int l = 0; l < L; ++l) {                      // up: scan every level, totals feed the next one
        const int64_t nw = (counts[l] + 31) / 32;
        warp_scan_kernel<Op><<<nblk(nw * 32, QS_THREADS), QS_THREADS, 0, ctx->stream>>>(
            items[l], counts[l], pre[l], (l + 1 < L) ? items[l + 1] : nullptr, nw);
        ctx->launches++;
    }
    for (int l = L - 1; l >= 0; --l) {                 // down: one parallel pass per level
        warp_propagate_kernel<Op><<<nblk(counts[l], QS_THREADS), QS_THREADS, 0, ctx->stream>>>(
            pre[l], counts[l], (l + 1 < L) ? starts[l + 1] : nullptr, (l + 1 < L) ? counts[l + 1] : 0, starts[l]);
        ctx->launches++;
    }
    CUDA_CHECK(cudaGetLastError());
    for (int l = 0; l < L; ++l) {
        ctx->release(pre[l], (size_t)Op::SIZE * counts[l] * 8);
        if (l > 0) {
            ctx->release(items[l], (size_t)Op::SIZE * counts[l] * 8);
            ctx->release(starts[l], (size_t)Op::STATE * counts[l] * 8);
        }
    }
}

template <class Op>
static void run_tree(b200gp_ctx* ctx, double* comp0, int64_t n0, double* start0) {
    if (ctx->qs_tree == 1) {
        run_tree_warp<Op>(ctx, comp0, n0, start0);
        return;
    }
    std::vector<double*> comps{comp0};
    std::vector<int64_t> counts{n0};
    std::vector<size_t> bytes{0};
    while (counts.back() > TREE_R) {
        const int64_t nc = counts.back(), np_ = (nc + TREE_R - 1) / TREE_R;
        const size_t b = (size_t)Op::SIZE * np_ * 8;
        double* parent = (double*)ctx->alloc(b);
        tree_up_kernel<Op><<<nblk(np_, QS_THREADS), QS_THREADS, 0, ctx->stream>>>(comps.back(), nc, parent, np_);
        ctx->launches++;
        comps.push_back(parent);
        counts.push_back(np_);
        bytes.push_back(b);
    }
    const int L = (int)counts.size();
    std::vector<double*> starts(L, nullptr);
    std::vector<size_t> sbytes(L, 0);
    for (int l = 0; l < L; ++l) {
        if (l == 0) {
            starts[l] = start0;
        } else {
            sbytes[l] = (size_t)Op::STATE * counts[l] * 8;
            starts[l] = (double*)ctx->alloc(sbytes[l]);
        }
    }
    tree_top_kernel<Op><<<1, 32, 0, ctx->stream>>>(comps[L - 1], counts[L - 1], starts[L - 1]);
    ctx->launches++;
    for (int l = L - 2; l >= 0; --l) {
        tree_down_kernel<Op><<<nblk(counts[l + 1], QS_THREADS), QS_THREADS, 0, ctx->stream>>>(
            comps[l], counts[l], starts[l + 1], counts[l + 1], starts[l]);
        ctx->launches++;
    }
    CUDA_CHECK(cudaGetLastError());
    for (int l = 1; l < L; ++l) {
        ctx->release(comps[l], bytes[l]);
        ctx->release(starts[l], sbytes[l]);
    }
}

