// Context, device-buffer cache, options, profile counters and the fp64 peak micro-benchmarks.
#include "common.cuh"
#include "dmma.cuh"
#include <string.h>
#include <algorithm>

void* b200gp_ctx::alloc(size_t bytes) {
    if (bytes == 0) bytes = 8;
    // best fit from the cache: smallest cached buffer that is large enough and not > 1.25x
    int best = -1;
    for (int i = 0; i < (int)cache.size(); ++i) {
        if (cache[i].bytes >= bytes && (double)cache[i].bytes <= 1.25 * (double)bytes + 4096.0) {
            if (best < 0 || cache[i].bytes < cache[best].bytes) best = i;
        }
    }
    if (best >= 0) {
        void* p = cache[best].ptr;
        cache.erase(cache.begin() + best);
        return p;
    }
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        trim();  // drop cached buffers and retry once
        e = cudaMalloc(&p, bytes);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        char buf[256];
        snprintf(buf, sizeof(buf), "cudaMalloc of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
        throw GpError(buf);
    }
    return p;
}

void b200gp_ctx::release(void* p, size_t bytes) {
    if (!p) return;
    if (bytes == 0) bytes = 8;
    // the stream may still be using p: all frees go through the cache, and a cached buffer is only
    // ever handed to work enqueued later on the same stream, so ordering is preserved.
    cache.push_back({p, bytes});
    size_t total = 0;
    for (auto& c : cache) total += c.bytes;
    // keep at most ~110 GiB or 64 entries cached (N = 65536: 34 GB matrix + up to 34 GB of int8 digit planes)
    while (cache.size() > 64 || total > ((size_t)110 << 30)) {
        cudaStreamSynchronize(stream);
        total -= cache.front().bytes;
        cudaFree(cache.front().ptr);
        cache.erase(cache.begin());
    }
}

cudaEvent_t b200gp_ctx::get_event() {
    if (!event_pool.empty()) {
        cudaEvent_t e = event_pool.back();
        event_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}

void b200gp_ctx::flush_timers() {
    if (pending.empty()) return;
    cudaStreamSynchronize(stream);
    for (auto& p : pending) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) *p.acc += ms;
        event_pool.push_back(p.a);
        event_pool.push_back(p.b);
    }
    pending.clear();
    cudaGetLastError();
}

void b200gp_ctx::trim() {
    cudaStreamSynchronize(stream);
    for (auto& c : cache) cudaFree(c.ptr);
    cache.clear();
}

// ---- fp64 peak micro-benchmarks ----------------------------------------------------------------
// one mma.sync.MxNxK.f64 (N = 8): M = 8, K = 4 (Ampere's shape) or M = 16, K = 4 / 8 / 16 (sm_90)
template <int M, int K>
__device__ __forceinline__ void peak_mma(double (&c)[M / 4], const double (&a)[M * K / 32], const double (&b)[K / 4]) {
    if constexpr (M == 8)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                     : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
    else if constexpr (K == 4)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    else if constexpr (K == 8)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                     "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                       "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// register-resident operands, 16 independent accumulators per warp, `iters` rounds of 16 instructions
template <int M, int K>
__global__ void __launch_bounds__(256) dmma_peak_kernel(double* out, int iters) {
    double c[16][M / 4], a[M * K / 32], b[K / 4];
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int j = 0; j < M / 4; ++j) c[i][j] = 0.0;
#pragma unroll
    for (int j = 0; j < M * K / 32; ++j) a[j] = 1.0 + (threadIdx.x + j) * 1e-9;
#pragma unroll
    for (int j = 0; j < K / 4; ++j) b[j] = 1.0 - (threadIdx.x + j) * 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) peak_mma<M, K>(c[i], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int j = 0; j < M / 4; ++j) s += c[i][j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void __launch_bounds__(256) dfma_peak_kernel(double* out, int iters) {
    double c[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) c[i] = i * 1e-3;
    const double a = 1.0 + threadIdx.x * 1e-12, b = 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) c[i] = fma(c[i], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += c[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

extern "C" {

int b200gp_version(void) { return 100; }

int b200gp_create(int device, void* stream, b200gp_ctx** out) {
    if (!out) return 1;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0 || device < 0 || device >= count) {
        cudaGetLastError();
        return 3;  // no usable CUDA device: the host raises, there is no CPU fallback
    }
    b200gp_ctx* c = new b200gp_ctx();
    c->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete c; return 3; }
    if (stream) {
        c->stream = (cudaStream_t)stream;
    } else {
        if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; return 3; }
        c->own_stream = true;
    }
    cudaEventCreate(&c->ev0);
    cudaEventCreate(&c->ev1);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->num_sms = prop.multiProcessorCount;
    memset(&c->prof, 0, sizeof(c->prof));
    *out = c;
    return 0;
}

int b200gp_destroy(b200gp_ctx* ctx) {
    if (!ctx) return 0;
    cudaSetDevice(ctx->device);
    ctx->flush_timers();
    for (auto e : ctx->event_pool) cudaEventDestroy(e);
    ctx->trim();
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
    if (ctx->stream_solve) cudaStreamDestroy(ctx->stream_solve);
    if (ctx->stream_hi) cudaStreamDestroy(ctx->stream_hi);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return 0;
}

const char* b200gp_last_error(b200gp_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int64_t b200gp_launch_count(b200gp_ctx* ctx) { return ctx ? ctx->launches : 0; }

// plain integer options: key -> member (validated in b200gp_set_option); defaults = the member initialisers in common.cuh
static const struct OptEntry { const char* key; int64_t b200gp_ctx::*field; } kOptions[] = {
    {"nb", &b200gp_ctx::nb},
    {"peak_iters", &b200gp_ctx::peak_iters},
    {"qs_tree", &b200gp_ctx::qs_tree},
    {"qs_chunk", &b200gp_ctx::qs_chunk},
    {"qs_chunk_max", &b200gp_ctx::qs_chunk_max},
    {"qsm_chunk", &b200gp_ctx::qsm_chunk},
    {"qsm_sequential_redos", &b200gp_ctx::qsm_sequential_redos},
    {"build_fast", &b200gp_ctx::build_fast},
    {"qs_kernel", &b200gp_ctx::qs_kernel},
    {"qs_occupancy", &b200gp_ctx::qs_occupancy},
    {"nb_batched", &b200gp_ctx::nb_batched},
    {"ozaki_slices", &b200gp_ctx::oz_slices},
    {"ozaki_prefetch", &b200gp_ctx::oz_prefetch},
    {"ozaki_layout", &b200gp_ctx::oz_layout},
    {"ozaki_pairing", &b200gp_ctx::oz_pairing},
    {"build_ahead", &b200gp_ctx::build_ahead},
    {"ozaki_lookahead", &b200gp_ctx::oz_lookahead},
    {"ozaki_cluster", &b200gp_ctx::oz_cluster},
    {"ozaki_min_n", &b200gp_ctx::oz_min_n},
    {"ozaki_l2promo", &b200gp_ctx::oz_l2promo},
    {"ozaki_subpanel", &b200gp_ctx::oz_subpanel},
    {"ozaki_splitk", &b200gp_ctx::oz_splitk},
    {"solve_overlap", &b200gp_ctx::solve_overlap},
    {"mg_splitk", &b200gp_ctx::mg_splitk},
    {"ozaki_splitk_force", &b200gp_ctx::oz_splitk_force},
};

static void validate_option(const char* key, int64_t value) {
    if (!strcmp(key, "nb") || !strcmp(key, "nb_batched")) {
        if (value < TILE || value % TILE) throw GpError(std::string("option ") + key + " must be a positive multiple of 128");
    } else if (!strcmp(key, "peak_iters")) {
        if (value < 16) throw GpError("option peak_iters must be >= 16");
    } else if (!strcmp(key, "qs_tree") || !strcmp(key, "ozaki_layout")) {
        if (value != 0 && value != 1) throw GpError(std::string("option ") + key + " must be 0 or 1");
    } else if (!strcmp(key, "qs_chunk")) {
        if (value != 0 && (value < 4 || value > 4096)) throw GpError("option qs_chunk must be 0 (auto) or in [4, 4096]");
    } else if (!strcmp(key, "ozaki_slices")) {
        if (value < 0 || value > 8) throw GpError("option ozaki_slices must be in [0, 8]");
    }
}

int b200gp_set_option(b200gp_ctx* ctx, const char* key, int64_t value) {
    API_BEGIN(ctx)
    if (!strcmp(key, "profile")) {
        _ctx->flush_timers();
        _ctx->profile = (value != 0);
        return 0;
    }
    if (!strcmp(key, "trim")) {
        _ctx->trim();
        return 0;
    }
    if (!strcmp(key, "reset")) {   // every tuning option back to the library default
        const b200gp_ctx defaults;
        for (const OptEntry& o : kOptions) _ctx->*(o.field) = defaults.*(o.field);
        return 0;
    }
    for (const OptEntry& o : kOptions) {
        if (strcmp(key, o.key)) continue;
        validate_option(key, value);
        if (!strcmp(key, "ozaki_pairing")) value = (value == 2) ? 2 : (value ? 1 : 0);
        else if (!strcmp(key, "build_ahead")) value = value ? 1 : 0;
        _ctx->*(o.field) = value;
        return 0;
    }
    throw GpError(std::string("unknown option ") + key);
    API_END
}

int b200gp_get_option(b200gp_ctx* ctx, const char* key, int64_t* value) {
    API_BEGIN(ctx)
    if (!value) throw GpError("get_option: null output");
    if (!strcmp(key, "profile")) { *value = _ctx->profile ? 1 : 0; return 0; }
    for (const OptEntry& o : kOptions)
        if (!strcmp(key, o.key)) { *value = _ctx->*(o.field); return 0; }
    throw GpError(std::string("unknown option ") + key);
    API_END
}

int b200gp_get_profile(b200gp_ctx* ctx, b200gp_profile* out, int reset) {
    API_BEGIN(ctx)
    _ctx->flush_timers();
    *out = _ctx->prof;
    if (reset) memset(&_ctx->prof, 0, sizeof(_ctx->prof));
    API_END
}

// TFLOP/s of dmma_peak_kernel<M, K> on all SMs, timed after one warm-up launch.  peak_iters counts work in units of
// 16 m8n8k4 instructions per warp, so every shape runs the same flop count.
static double dmma_shape_tflops(b200gp_ctx* ctx, int m, int k, double* buf, int blocks, int threads) {
    const int iters = (int)std::max<int64_t>(1, ctx->peak_iters * 8 * 4 / (m * k));
    float ms = 0;
    for (int rep = 0; rep < 2; ++rep) {  // first pass warms up
        cudaEventRecord(ctx->ev0, ctx->stream);
        if (m == 8) dmma_peak_kernel<8, 4><<<blocks, threads, 0, ctx->stream>>>(buf, iters);
        else if (k == 4) dmma_peak_kernel<16, 4><<<blocks, threads, 0, ctx->stream>>>(buf, iters);
        else if (k == 8) dmma_peak_kernel<16, 8><<<blocks, threads, 0, ctx->stream>>>(buf, iters);
        else dmma_peak_kernel<16, 16><<<blocks, threads, 0, ctx->stream>>>(buf, iters);
        cudaEventRecord(ctx->ev1, ctx->stream);
        CUDA_CHECK(cudaEventSynchronize(ctx->ev1));
        cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
    }
    ctx->launches += 2;
    // per warp per instruction: m * 8 * k FMA = 2 m 8 k flop
    return (double)blocks * (threads / 32) * (double)iters * 16.0 * (2.0 * m * 8 * k) / (ms * 1e-3) / 1e12;
}

int b200gp_measure_dmma_shape(b200gp_ctx* ctx, int m, int n, int k, double* tflops) {
    API_BEGIN(ctx)
    if (!tflops) throw GpError("measure_dmma_shape: null output");
    if (n != 8 || !((m == 8 && k == 4) || (m == 16 && (k == 4 || k == 8 || k == 16))))
        throw GpError("measure_dmma_shape: the fp64 mma shapes are m8n8k4, m16n8k4, m16n8k8 and m16n8k16");
    const int blocks = _ctx->num_sms * 4, threads = 256;
    double* buf = (double*)_ctx->alloc((size_t)blocks * threads * 8);
    *tflops = dmma_shape_tflops(_ctx, m, k, buf, blocks, threads);
    _ctx->release(buf, (size_t)blocks * threads * 8);
    API_END
}

int b200gp_measure_fp64_peak(b200gp_ctx* ctx, double* dmma_tflops, double* dfma_tflops) {
    API_BEGIN(ctx)
    const int blocks = _ctx->num_sms * 4, threads = 256;
    const int iters = (int)_ctx->peak_iters;
    double* buf = (double*)_ctx->alloc((size_t)blocks * threads * 8);
    *dmma_tflops = dmma_shape_tflops(_ctx, 16, dmma::MK, buf, blocks, threads);   // the shape the GEMM mainloops issue
    float ms = 0;
    for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(_ctx->ev0, _ctx->stream);
        dfma_peak_kernel<<<blocks, threads, 0, _ctx->stream>>>(buf, iters);
        cudaEventRecord(_ctx->ev1, _ctx->stream);
        CUDA_CHECK(cudaEventSynchronize(_ctx->ev1));
        cudaEventElapsedTime(&ms, _ctx->ev0, _ctx->ev1);
    }
    *dfma_tflops = (double)blocks * threads * (double)iters * 16.0 * 2.0 / (ms * 1e-3) / 1e12;
    _ctx->launches += 2;
    _ctx->release(buf, (size_t)blocks * threads * 8);
    API_END
}

}  // extern "C"
