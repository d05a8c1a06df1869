// Fixed-point (Ozaki-style) Cholesky update on the Hopper tensor cores: wgmma s8 x s8 -> s32 with both operands in
// shared memory, fed by TMA (multicast inside a thread-block cluster) through an mbarrier ring; int32 accumulators live
// in registers.
//
// The N^3/3 flop of `linalg.cholesky` (src/tinygp/solvers/direct.py:53) can be moved from the fp64 tensor pipe (DMMA)
// onto the int8 tensor pipe:
//
//   * |L_ik| <= sqrt(K_ii) for a Cholesky factor, so every row of L has the a-priori scale
//     rs_i = 2^ceil(log2 sqrt(K_ii)) and  x_ik = L_ik / rs_i  lies in [-1, 1].
//   * x is cut into S signed 7-bit digits (first digit 6 bits):  x = sum_s q_s 2^-(6+7s) , q_s in int8,
//     with exact remainders (every step is exact in fp64).  Digits are stored as S int8 planes.
//   * sum_k L_ik L_jk = rs_i rs_j sum_{s,t} 2^-(12+7(s+t)) (q_s[i,:] . q_t[j,:])  where each integer dot
//     product is EXACT in int32; pairs with equal s+t = g share one accumulator, pairs with
//     s+t >= S are dropped (<= 2^-(6+7(S-1)) relative to the row scale: 2^-55 for S = 8).
//   * left-looking block columns: column block J is generated (K tiles), then
//     C -= L[rows, 0:c0] L[c0:c0+nb, 0:c0]^T runs with K = c0 (all previous panels at once), so each C tile
//     is converted int32 -> fp64 only S times in total; then the panel is factored in fp64 on the DMMA
//     path (dense.cu) and its digits are cut.
//
// Kernel (one CTA per 128 x 128 tile of C, or 256 x 128 for the wide variant; 288 threads):
//   warps 0-3, 4-7: two consumer warpgroups; warpgroup c owns the rows [c * 64 MW, (c + 1) * 64 MW) of the tile and issues
//                   wgmma.m64n128k32 from the ring stages, then converts its accumulators and updates C in fp64
//   warp 8        : TMA producer (cp.async.bulk.tensor, 128-byte swizzle, 192 KB ring)
// The two warpgroups work on the same stages independently, so the epilogue of one overlaps the MMAs of the other.
#include "common.cuh"
#include "kprog.cuh"
#include <cuda.h>
#include <limits.h>

namespace oz {

constexpr int TM = 128;          // rows of a launch tile (Args.tiles_m counts these)
constexpr int TN = 256;          // columns of a launch tile (Args.tiles_n counts these)
constexpr int CTN = 128;         // columns of one CTA tile (the wgmma N)
constexpr int KC = 128;          // int8 K elements per pipeline stage (= one 128-byte swizzle row)
constexpr int B_BYTES = CTN * KC;            // 16 KiB
constexpr int RING_BYTES = 192 * 1024;
constexpr int THREADS = 288;                 // 2 consumer warpgroups + 1 producer warp
constexpr int BOXR = 32;                     // rows per TMA box (a 4 x 1 cluster multicasts 32-row slices of B)
constexpr uint32_t SPIN_LIMIT = 1u << 26;    // bounded waits: a protocol bug must not hang the GPU

// MW = m64 blocks per consumer warpgroup: 1 (128-row CTA tile) or 2 (the wide 256-row tile)
template <int MW>
struct Geo {
    static constexpr int ROWS = 128 * MW;
    static constexpr int A_BYTES = ROWS * KC;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = RING_BYTES / STAGE_BYTES;              // 6 or 4
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

struct Args {
    double* C; int64_t ldc;            // fp64 tile base: C[(row0 + i) * ldc + col0 + j]
    const double* rs;                  // row scales (power of two), indexed by global row
    int64_t row0, col0;                // global row / col of tile (0,0)
    int tiles_m, tiles_n;              // TM x TN launch tiles
    int K;                             // int8 K extent (multiple of KC)
    int k_begin;                       // first K column (multiple of KC)
    int S;                             // number of digit planes used
    int64_t b_row0;                    // first global row of the B operand (= col0 for the Cholesky update)
    int64_t n_rows;                    // rows of the matrix (for masking the last column tile)
    int prefetch;                      // L2 prefetch distance in K-chunks (0 = off)
    int skip_upper;                    // skip tiles entirely above the diagonal
    int layout;                        // digit-plane layout: 0 plane-major [s][row][k], 1 chunk-major [k/128][row][s][128]
    int pg_single;                     // diagnostic: paired-group loop structure (kc outer) with ONE group per pass
    int* error_flag;
    unsigned long long* dbg;           // optional in-kernel cycle counters (see DBG_* below); nullptr = off
    // split-K of the tail cluster tiles (nseg <= 1 = off): cluster indices >= split_from (ntail of them) are cut into nseg K
    // segments of kseg columns that run as extra clusters of the SAME launch; segment 0 updates C, segment sg >= 1
    // accumulates into its own zero-filled fp64 scratch tile Cseg[(sg - 1) * ntail + tail index][rows][cols] of the cluster
    // tile that splitk_fixup_kernel adds to C afterwards in a fixed order.
    int nseg, kseg, split_from, ntail;
    double* Cseg;
    int no_split;                      // launcher hint: keep one K range per tile (sharded path: bit-identical for any rank count)
};

// in-kernel cycle counters (diagnostics, option-free: on when Args.dbg != nullptr).  Sums over CTAs of clock64() deltas;
// the MMA / EPI slots are taken by consumer warpgroup 0.
enum { DBG_PROD_WAIT = 0, DBG_PROD_TOTAL = 1, DBG_MMA_WAIT_FULL = 2, DBG_MMA_WAIT_TEMPTY = 3, DBG_MMA_TOTAL = 4,
       DBG_EPI_WAIT_TFULL = 5, DBG_EPI_TOTAL = 6, DBG_CTAS = 7, DBG_CTA_TOTAL = 8, DBG_N = 16 };

// ONE 3-D map (k, row, plane) -- or 4-D for the chunk-major layout -- serves every stage: cycling through per-plane
// descriptors would make every TMA issue miss the descriptor cache
struct Maps { CUtensorMap all; };

// ---- PTX wrappers -----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t local_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(r) : "r"(local_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];\n" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// returns false on timeout (the caller raises the abort flag)
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, volatile int* abort_flag) {
    for (uint32_t it = 0; it < SPIN_LIMIT; ++it) {
        if (mbar_try_wait(bar, parity)) return true;
        if ((it & 1023u) == 1023u && *abort_flag) return false;
    }
    *abort_flag = 1;
    return false;
}
// mbar_wait with an optional cycle counter around it
__device__ __forceinline__ bool mbar_wait_t(uint64_t* bar, uint32_t parity, volatile int* abort_flag, bool prof,
                                            unsigned long long& acc) {
    if (!prof) return mbar_wait(bar, parity, abort_flag);
    const long long t0 = clock64();
    const bool r = mbar_wait(bar, parity, abort_flag);
    acc += (unsigned long long)(clock64() - t0);
    return r;
}
__device__ __forceinline__ void dbg_add(unsigned long long* dbg, int slot, unsigned long long v) {
    if (dbg) atomicAdd(dbg + slot, v);
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* map, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];\n" ::"l"(map), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_load_3d_mc(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                               uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4, %5}], [%2], %6;\n" ::"r"(smem_u32(smem_dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];\n" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d_mc(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3,
                                               uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;\n" ::"r"(smem_u32(smem_dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

// K-major operand, 128-byte swizzle (the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): stride byte offset 1024 B
// between 8-row groups, leading byte offset unused; stage bases are 1024-byte aligned, so the base offset is 0 and a K step
// of 32 bytes inside the swizzle atom is a plain advance of the start address
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;                 // SWIZZLE_128B
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }
__device__ __forceinline__ void wg_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;\n" ::: "memory"); }

// d (64 x 128 int32, 64 registers per thread) (+)= A (64 x 32 int8) B (128 x 32 int8)^T
__device__ __forceinline__ void wgmma_i8(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p;\n\t}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(accumulate)
        : "memory");
}

// one stage (K = 128) of one m64 block: four k32 instructions
__device__ __forceinline__ void mma_stage(uint32_t (&d)[64], uint32_t a_addr, uint32_t b_addr, uint32_t& accumulate) {
#pragma unroll
    for (int kk = 0; kk < KC / 32; ++kk) {
        wgmma_i8(d, make_desc(a_addr + kk * 32), make_desc(b_addr + kk * 32), accumulate);
        accumulate = 1;
    }
}

// ---- epilogue of one digit group (or a pair of groups) for one m64 block ------------------------------------------
// Accumulator fragment of wgmma m64nN (32-bit): thread (warp w, lane l) holds rows 16 w + l / 4 (registers 4 i, 4 i + 1)
// and 16 w + l / 4 + 8 (4 i + 2, 4 i + 3) at columns 8 i + 2 (l % 4) + {0, 1}.
// C[row, col] += sc_row * rs_col * (acc0 + 2^-7 acc1).  The read-modify-write is issued in batches (loads first, then the
// arithmetic, then the stores), so that consecutive 16-byte accesses are not serialised on a possible alias.
template <bool TWO>
__device__ __forceinline__ void epi_rmw(const uint32_t (&d0)[64], const uint32_t (&d1)[64], double* crow0, double* crow1,
                                        const double* __restrict__ rs, int64_t gc_lane, int64_t n_cols, bool ok0, bool ok1,
                                        double sc0, double sc1) {
#pragma unroll
    for (int ib = 0; ib < CTN / 8; ib += 4) {
        double2 c0v[4], c1v[4], rj[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t gc = gc_lane + 8 * (ib + j);
            const bool in = gc < n_cols;
            rj[j] = in ? __ldg(reinterpret_cast<const double2*>(rs + gc)) : make_double2(0.0, 0.0);
            c0v[j] = (in && ok0) ? *reinterpret_cast<const double2*>(crow0 + gc) : make_double2(0.0, 0.0);
            c1v[j] = (in && ok1) ? *reinterpret_cast<const double2*>(crow1 + gc) : make_double2(0.0, 0.0);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int e = 4 * (ib + j);
            double t0x = (double)(int)d0[e], t0y = (double)(int)d0[e + 1];
            double t1x = (double)(int)d0[e + 2], t1y = (double)(int)d0[e + 3];
            if (TWO) {   // group g0 + 1 is 2^-7 of group g0: a0 + a1 2^-7 is exact (|a| < 2^31), one rounding per pair
                t0x = fma((double)(int)d1[e], 0.0078125, t0x);
                t0y = fma((double)(int)d1[e + 1], 0.0078125, t0y);
                t1x = fma((double)(int)d1[e + 2], 0.0078125, t1x);
                t1y = fma((double)(int)d1[e + 3], 0.0078125, t1y);
            }
            c0v[j].x = fma(sc0 * rj[j].x, t0x, c0v[j].x);
            c0v[j].y = fma(sc0 * rj[j].y, t0y, c0v[j].y);
            c1v[j].x = fma(sc1 * rj[j].x, t1x, c1v[j].x);
            c1v[j].y = fma(sc1 * rj[j].y, t1y, c1v[j].y);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t gc = gc_lane + 8 * (ib + j);
            if (gc < n_cols) {
                if (ok0) *reinterpret_cast<double2*>(crow0 + gc) = c0v[j];
                if (ok1) *reinterpret_cast<double2*>(crow1 + gc) = c1v[j];
            }
        }
    }
}

// PG ("paired groups"): two digit groups g0 = 2P, g1 = 2P + 1 are accumulated at once in two register accumulators.
// Per K chunk the ring then carries stages i = 0..g1 holding (A plane i, B plane g1 - i); stage i feeds
//   A_i x B_{g1-i} -> accumulator 1 (group g1)   and   A_{i-1} (previous stage) x B_{g1-i} -> accumulator 0 (group g0),
// so S = 8 needs 20 stage loads per K chunk instead of 36 for the same MMAs.
// Pass P of the paired loop covers digit group g0 and, if `two`, g0 + 1.  A paired pass streams g1 + 1 stages per K chunk
// and a single pass g0 + 1, so for an odd plane count the UNPAIRED group is the cheap group 0, not the expensive last one:
// S = 7 -> (0) (1,2) (3,4) (5,6) = 1 + 3 + 5 + 7 = 16 stage loads per K chunk for the 28 pair products (instead of
// 2 + 4 + 6 + 7 = 19 with the single group last, or 28 unpaired); S = 8 -> (0,1) (2,3) (4,5) (6,7) = 20 for 36.
__device__ __forceinline__ void pg_pass(int S, int pg_single, int P, int& g0, bool& two) {
    if (pg_single) { g0 = P; two = false; return; }
    const int odd = S & 1;
    if (odd && P == 0) { g0 = 0; two = false; return; }
    g0 = 2 * P - odd;
    two = (g0 + 1 < S);
}

// ---- the tile kernel ----------------------------------------------------------------------------
// Cluster of CM x CN CTAs (cluster rank r: cm = r % CM, cn = r / CM) working on CM x CN neighbouring CTA tiles.
// The A tile (rows of ti) is needed by the CN CTAs of a cluster row and the B tile (rows of tj) by the CM
// CTAs of a cluster column: every CTA fetches only its 1/CN slice of A and 1/CM slice of B and TMA-multicasts
// it to its mates, which divides the L2 -> SM operand traffic.
// A stage slot of CTA X is written by X's row and column mates, so X's consumers release it on the `empty` barrier of
// each of them (2 warpgroups x (CM + CN - 1) arrivals per phase).
template <int CM, int CN, bool PG, int MW>
__global__ void __launch_bounds__(THREADS, 1) i8_update_kernel(const __grid_constant__ Maps maps, const Args g) {
    using G = Geo<MW>;
    constexpr int ROWS = G::ROWS, A_BYTES = G::A_BYTES, STAGE_BYTES = G::STAGE_BYTES, STAGES = G::STAGES;
    static_assert((ROWS / CN) % BOXR == 0 && (CTN / CM) % BOXR == 0, "slice must be whole TMA boxes");
    static_assert(!(PG && MW > 1), "two accumulators of two m64 blocks do not fit the register file");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
    uint64_t* full = bars;                  // [STAGES]
    uint64_t* empty = bars + STAGES;        // [STAGES]
    volatile int* abort_flag = reinterpret_cast<volatile int*>(bars + 2 * STAGES);

    constexpr int CS = CM * CN;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int crank = 0;
    if (CS > 1) asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(crank));
    const int cm = crank % CM, cn = crank / CM;
    // cluster tiles: (CM * ROWS) x (CN * CTN); tj fastest, so co-resident CTAs share every A row panel in L2
    const int ctn = (2 * g.tiles_n + CN - 1) / CN;
    int cluster_id = (int)blockIdx.x / CS;
    int seg = 0, tail_idx = 0;
    const bool split = (g.nseg > 1 && cluster_id >= g.split_from);
    if (split) {                                             // tail clusters: segment slowest
        const int idx = cluster_id - g.split_from;
        seg = idx / g.ntail; tail_idx = idx - seg * g.ntail;
        cluster_id = g.split_from + tail_idx;
    }
    const int ci = cluster_id / ctn, cj = cluster_id % ctn;
    const int seg_k0 = g.k_begin + seg * g.kseg;             // first K column of this tile's segment
    const int seg_K = split ? ((g.K - seg * g.kseg < g.kseg) ? (g.K - seg * g.kseg) : g.kseg) : g.K;
    const int64_t crow_lo = g.row0 + (int64_t)ci * CM * ROWS, ccol_lo = g.col0 + (int64_t)cj * CN * CTN;
    const int64_t grow0 = crow_lo + (int64_t)cm * ROWS;      // global row of this CTA's tile row 0
    const int64_t gcol0 = ccol_lo + (int64_t)cn * CTN;       // global col of this CTA's tile col 0
    // cluster-uniform decision
    if (g.skip_upper && crow_lo + (int64_t)CM * ROWS - 1 < ccol_lo) return;   // every tile of the cluster lies above the diagonal
    // Pairs with s + t >= S are dropped everywhere.  Off the diagonal they are zero-mean; on the diagonal they
    // are sums of squares (a systematic bias), which cut_digits_kernel accumulates exactly per row and
    // diag_correct_kernel subtracts from C_ii -- so every tile does the same S(S+1)/2 products.
    const int S = g.S;

    uint16_t mask_a = 0, mask_b = 0;
#pragma unroll
    for (int c = 0; c < CN; ++c) mask_a |= (uint16_t)(1u << (cm + CM * c));
#pragma unroll
    for (int m = 0; m < CM; ++m) mask_b |= (uint16_t)(1u << (m + CM * cn));
    const uint16_t mask_all = mask_a | mask_b;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 2 * (CM + CN - 1)); }
        *abort_flag = 0;
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    if (CS > 1) cluster_sync_all();   // mates' barriers must be initialised before any multicast lands

    const int KT = seg_K / KC;
    const int64_t brow0 = g.b_row0 + (gcol0 - g.col0);      // global row of the B operand's first row

    const bool prof = (g.dbg != nullptr);
    const long long t_cta0 = prof ? clock64() : 0;
    if (warp == 8) {
        // ===== TMA producer =====
        if (lane == 0) {
            unsigned long long w_prod = 0;
            const long long t_role0 = prof ? clock64() : 0;
            const int kchunk0 = seg_k0 / KC;
            int stage = 0;
            uint32_t phase = 0;
            bool ok = true;
            // one BOXR-row x 128-byte box of digit plane `pl` at K chunk kc into this CTA's (and its mates') current stage
            auto load_box = [&](uint8_t* dst, int kc, int row, int pl, bool mc, uint16_t mask) {
                if (g.layout == 1) {
                    if (mc) tma_load_4d_mc(dst, &maps.all, full + stage, 0, pl, row, kchunk0 + kc, mask);
                    else tma_load_4d(dst, &maps.all, full + stage, 0, pl, row, kchunk0 + kc);
                } else {
                    if (mc) tma_load_3d_mc(dst, &maps.all, full + stage, seg_k0 + kc * KC, row, pl, mask);
                    else tma_load_3d(dst, &maps.all, full + stage, seg_k0 + kc * KC, row, pl);
                }
            };
            // one ring stage: (A plane s, B plane t) of K chunk kc
            auto issue_stage = [&](int s, int t, int kc) {
                if (!mbar_wait_t(empty + stage, phase ^ 1, abort_flag, prof, w_prod)) { ok = false; return; }
                uint8_t* a_dst = smem + stage * STAGE_BYTES;
                uint8_t* b_dst = a_dst + A_BYTES;
                mbar_expect_tx(full + stage, STAGE_BYTES);   // own + mates' slices land on this barrier
                constexpr int A_ROWS = ROWS / CN, B_ROWS = CTN / CM;
                if (g.prefetch > 0 && g.layout == 0 && kc + g.prefetch < KT) {   // own slices, `prefetch` K-chunks ahead, into L2
                    const int kp = seg_k0 + (kc + g.prefetch) * KC;
#pragma unroll
                    for (int bx = 0; bx < A_ROWS / BOXR; ++bx)
                        tma_prefetch_3d(&maps.all, kp, (int)grow0 + cn * A_ROWS + bx * BOXR, s);
#pragma unroll
                    for (int bx = 0; bx < B_ROWS / BOXR; ++bx)
                        tma_prefetch_3d(&maps.all, kp, (int)brow0 + cm * B_ROWS + bx * BOXR, t);
                }
#pragma unroll
                for (int bx = 0; bx < A_ROWS / BOXR; ++bx) {
                    const int r = cn * A_ROWS + bx * BOXR;
                    load_box(a_dst + r * KC, kc, (int)grow0 + r, s, CN > 1, mask_a);
                }
#pragma unroll
                for (int bx = 0; bx < B_ROWS / BOXR; ++bx) {
                    const int r = cm * B_ROWS + bx * BOXR;
                    load_box(b_dst + r * KC, kc, (int)brow0 + r, t, CM > 1, mask_b);
                }
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            };
            if constexpr (PG) {
                const int npass = g.pg_single ? S : (S + 1) / 2;
                for (int P = 0; P < npass && ok; ++P) {
                    int g0; bool two;
                    pg_pass(S, g.pg_single, P, g0, two);
                    const int top = two ? g0 + 1 : g0;
                    for (int kc = 0; kc < KT && ok; ++kc)
                        for (int i = 0; i <= top && ok; ++i) issue_stage(i, top - i, kc);
                }
            } else {
                for (int gi = 0; gi < S && ok; ++gi) {
                    const int s_lo = (gi - (S - 1) > 0) ? gi - (S - 1) : 0, s_hi = (gi < S - 1) ? gi : S - 1;
                    for (int s = s_lo; s <= s_hi && ok; ++s)
                        for (int kc = 0; kc < KT && ok; ++kc) issue_stage(s, gi - s, kc);
                }
            }
            if (prof) { dbg_add(g.dbg, DBG_PROD_WAIT, w_prod); dbg_add(g.dbg, DBG_PROD_TOTAL, (unsigned long long)(clock64() - t_role0)); }
        }
    } else {
        // ===== consumer warpgroup wg: wgmma on rows [wg * 64 MW, (wg + 1) * 64 MW) of the tile, then the fp64 epilogue =====
        const int wg = warp >> 2, wl = threadIdx.x & 127;
        const bool leader = (wl == 0);
        const bool prof_wg = prof && wg == 0 && leader;
        unsigned long long w_full = 0, t_epi = 0;
        const long long t_role0 = prof_wg ? clock64() : 0;
        // this thread's rows (two per m64 block) and the first of its columns
        const int rloc = wg * 64 * MW + 16 * (wl >> 5) + ((wl & 31) >> 2);
        const int64_t gc_lane = gcol0 + 2 * (lane & 3);
        double* crow[MW][2];
        bool rok[MW][2];
        double rsi[MW][2];
#pragma unroll
        for (int mw = 0; mw < MW; ++mw)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int lr = rloc + 64 * mw + 8 * h;
                const int64_t gr = grow0 + lr;
                rok[mw][h] = gr < g.n_rows;           // padding tiles of an incomplete cluster do no stores
                rsi[mw][h] = rok[mw][h] ? g.rs[gr] : 0.0;
                // segment >= 1: this cluster's scratch tile, addressed like C through a virtual base (columns are GLOBAL indices)
                crow[mw][h] = (seg == 0) ? g.C + (rok[mw][h] ? gr : 0) * g.ldc
                                         : g.Cseg + ((int64_t)(seg - 1) * g.ntail + tail_idx) * ((int64_t)CM * ROWS * CN * CTN)
                                               + (gr - crow_lo) * (CN * CTN) - ccol_lo;
            }
        // release a stage in every CTA whose producer writes into it (row- and column-mates, this CTA included)
        auto release = [&](int st) {
            if (!leader) return;
            if (CS == 1) { mbar_arrive(empty + st); return; }
            const uint32_t local = smem_u32(empty + st);
#pragma unroll
            for (int r = 0; r < CS; ++r)
                if ((mask_all >> r) & 1) mbar_arrive_cluster(mapa(local, (uint32_t)r));
        };
        uint32_t acc0[MW][64], acc1[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            acc1[i] = 0;
#pragma unroll
            for (int mw = 0; mw < MW; ++mw) acc0[mw][i] = 0;
        }
        int stage = 0;
        uint32_t phase = 0;
        bool ok = true;
        const uint32_t a_off = (uint32_t)(wg * 64 * MW * KC);
        if constexpr (PG) {
            const int npass = g.pg_single ? S : (S + 1) / 2;
            for (int P = 0; P < npass && ok; ++P) {
                int g0; bool two;
                pg_pass(S, g.pg_single, P, g0, two);
                const int top = two ? g0 + 1 : g0;
                uint32_t accum0 = 0, accum1 = 0;
                for (int kc = 0; kc < KT && ok; ++kc) {
                    uint32_t prev_a = 0;
                    int prev_stage = 0;
                    for (int i = 0; i <= top; ++i) {
                        if (!mbar_wait_t(full + stage, phase, abort_flag, prof_wg, w_full)) { ok = false; break; }
                        const uint32_t a_addr = smem_u32(smem + stage * STAGE_BYTES) + a_off;
                        const uint32_t b_addr = smem_u32(smem + stage * STAGE_BYTES + A_BYTES);
                        wg_fence();
                        if (two) {
                            mma_stage(acc1, a_addr, b_addr, accum1);                        // A_i x B_{top-i}: group top
                            if (i >= 1) mma_stage(acc0[0], prev_a, b_addr, accum0);         // A_{i-1} x B_{top-i}: group top - 1
                            wg_commit();
                            wg_wait0();
                            // stage i-1 is now dead: its A was just used for the last time, its B one step ago
                            if (i >= 1) release(prev_stage);
                            if (i == top) release(stage);
                        } else {
                            mma_stage(acc0[0], a_addr, b_addr, accum0);
                            wg_commit();
                            wg_wait0();
                            release(stage);
                        }
                        prev_a = a_addr;
                        prev_stage = stage;
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
                if (!ok) break;
                // group g0 weighs 2^-(12 + 7 g0); group g0 + 1 is 2^-7 of that.  a0 + a1 2^-7 is exact in fp64
                // (|a| < 2^31), so the pair costs ONE rounding and one read-modify-write of the fp64 tile.
                const long long te0 = prof_wg ? clock64() : 0;
                const double wgt = __longlong_as_double((long long)(1023 - (12 + 7 * g0)) << 52);
                const double sc0 = -(rsi[0][0] * wgt), sc1 = -(rsi[0][1] * wgt);
                if (two) epi_rmw<true>(acc0[0], acc1, crow[0][0], crow[0][1], g.rs, gc_lane, g.n_rows, rok[0][0], rok[0][1], sc0, sc1);
                else epi_rmw<false>(acc0[0], acc0[0], crow[0][0], crow[0][1], g.rs, gc_lane, g.n_rows, rok[0][0], rok[0][1], sc0, sc1);
                if (prof_wg) t_epi += (unsigned long long)(clock64() - te0);
            }
        } else {
            for (int gi = 0; gi < S && ok; ++gi) {
                uint32_t accumulate = 0;
                const int s_lo = (gi - (S - 1) > 0) ? gi - (S - 1) : 0, s_hi = (gi < S - 1) ? gi : S - 1;
                for (int s = s_lo; s <= s_hi && ok; ++s) {
                    for (int kc = 0; kc < KT; ++kc) {
                        if (!mbar_wait_t(full + stage, phase, abort_flag, prof_wg, w_full)) { ok = false; break; }
                        const uint32_t a_addr = smem_u32(smem + stage * STAGE_BYTES) + a_off;
                        const uint32_t b_addr = smem_u32(smem + stage * STAGE_BYTES + A_BYTES);
                        wg_fence();
#pragma unroll
                        for (int mw = 0; mw < MW; ++mw) {
                            uint32_t acc_flag = accumulate;
                            mma_stage(acc0[mw], a_addr + (uint32_t)(mw * 64 * KC), b_addr, acc_flag);
                        }
                        accumulate = 1;
                        wg_commit();
                        wg_wait0();
                        release(stage);
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
                if (!ok) break;
                const long long te0 = prof_wg ? clock64() : 0;
                // weight 2^-(12 + 7 gi), exact power of two
                const double wgt = __longlong_as_double((long long)(1023 - (12 + 7 * gi)) << 52);
#pragma unroll
                for (int mw = 0; mw < MW; ++mw)
                    epi_rmw<false>(acc0[mw], acc0[mw], crow[mw][0], crow[mw][1], g.rs, gc_lane, g.n_rows, rok[mw][0], rok[mw][1],
                                   -(rsi[mw][0] * wgt), -(rsi[mw][1] * wgt));
                if (prof_wg) t_epi += (unsigned long long)(clock64() - te0);
            }
        }
        if (prof_wg) {
            dbg_add(g.dbg, DBG_MMA_WAIT_FULL, w_full);
            dbg_add(g.dbg, DBG_EPI_TOTAL, t_epi);
            dbg_add(g.dbg, DBG_MMA_TOTAL, (unsigned long long)(clock64() - t_role0));
        }
    }

    __syncthreads();
    if (CS > 1) cluster_sync_all();   // no CTA may exit while mates still multicast into it / arrive on its barriers
    if (prof && threadIdx.x == 0) { dbg_add(g.dbg, DBG_CTAS, 1ull); dbg_add(g.dbg, DBG_CTA_TOTAL, (unsigned long long)(clock64() - t_cta0)); }
    if (threadIdx.x == 0 && *abort_flag) atomicExch(g.error_flag, 1);
}

// ---- digit cutting -------------------------------------------------------------------------------
// planes[s][row * ldq + col] for rows [r0, np), cols [c0, c0 + ncols); 16 columns per thread.
// Also accumulates, per row, the dropped diagonal pairs  sum_{s+t>=S} 2^-(12+7(s+t)) sum_k q_s q_t  (exact integer
// sums, fp64 weights) into corr[slot][row] with slot = 512-column group: two warps -> two commutative adds.
// ST > 0: the plane count is a compile-time constant, so the digit table q[ST][16] lives in registers and every loop over
// planes / digit pairs is unrolled; ST = 0 keeps the run-time count (q in local memory: 512 B of stack per thread).
template <int ST>
__global__ void __launch_bounds__(256, 2) cut_digits_kernel_t(const double* __restrict__ mat, int64_t ld, const double* __restrict__ rs,
                                                           int64_t r0, int64_t nrows, int64_t c0, int64_t ncols,
                                                           int8_t* planes, int64_t plane_stride, int64_t ldq, int S_rt,
                                                           double* corr /* [ncols/512 slots][np] for this panel */, int64_t np,
                                                           int layout) {
    const int S = (ST > 0) ? ST : S_rt;
    const int64_t groups_per_row = ncols / 16;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = idx < nrows * groups_per_row;
    const int64_t row = r0 + (active ? idx / groups_per_row : 0);
    const int64_t col = c0 + (active ? (idx % groups_per_row) * 16 : 0);
    double dropped = 0.0;
    if (active && ST > 0) {
        // two halves of 8 columns: the digit table of a half (ST x 8 ints) and the packed words of the first half are all
        // that stays live, the dropped-pair sums are carried across the halves as ST - 1 exact integer accumulators
        const double inv = 1.0 / rs[row];  // power of two: exact
        const double4* src = reinterpret_cast<const double4*>(mat + row * ld + col);
        constexpr int SS = (ST > 0) ? ST : 1;
        uint32_t pk[SS][4];
        int acc[SS];                       // acc[g - ST] for g = ST .. 2 ST - 2 (last entry unused)
#pragma unroll
        for (int g = 0; g < SS; ++g) acc[g] = 0;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            double x[8];
#pragma unroll
            for (int v = 0; v < 2; ++v) {
                const double4 d = src[2 * hf + v];
                x[4 * v + 0] = d.x * inv * 64.0; x[4 * v + 1] = d.y * inv * 64.0;
                x[4 * v + 2] = d.z * inv * 64.0; x[4 * v + 3] = d.w * inv * 64.0;
            }
            int q[SS][8];
#pragma unroll
            for (int sd = 0; sd < SS; ++sd) {
#pragma unroll
                for (int v = 0; v < 2; ++v) {
                    uint32_t wv = 0;
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        double& xx = x[4 * v + e];
                        double qd = rint(xx);
                        qd = fmin(fmax(qd, -127.0), 127.0);   // |x| <= 64 (+ rounding) by construction
                        xx = (xx - qd) * 128.0;               // exact
                        const int qi = (int)qd;
                        q[sd][4 * v + e] = qi;
                        wv |= ((uint32_t)(uint8_t)(int8_t)qi) << (8 * e);
                    }
                    pk[sd][2 * hf + v] = wv;
                }
            }
            // dropped pairs (s + t >= S), grouped by g = s + t so each group is one exact integer sum
#pragma unroll
            for (int gsum = SS; gsum <= 2 * (SS - 1); ++gsum) {
#pragma unroll
                for (int sdig = gsum - (SS - 1); sdig <= SS - 1; ++sdig) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) acc[gsum - SS] += q[sdig][e] * q[gsum - sdig][e];
                }
            }
        }
#pragma unroll
        for (int sd = 0; sd < SS; ++sd) {
            // plane-major [s][row][k], or chunk-major [k / 128][row][s][128] (np rows per chunk slab)
            const int64_t off = (layout == 1) ? (((col >> 7) * np + row) * S + sd) * 128 + (col & 127)
                                              : (int64_t)sd * plane_stride + row * ldq + col;
            *reinterpret_cast<uint4*>(planes + off) = make_uint4(pk[sd][0], pk[sd][1], pk[sd][2], pk[sd][3]);
        }
#pragma unroll
        for (int gsum = SS; gsum <= 2 * (SS - 1); ++gsum)
            dropped += (double)acc[gsum - SS] * __longlong_as_double((long long)(1023 - (12 + 7 * gsum)) << 52);
    } else if (active) {
        const double inv = 1.0 / rs[row];  // power of two: exact
        double x[16];
        const double4* src = reinterpret_cast<const double4*>(mat + row * ld + col);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const double4 d = src[v];
            x[4 * v + 0] = d.x * inv * 64.0; x[4 * v + 1] = d.y * inv * 64.0;
            x[4 * v + 2] = d.z * inv * 64.0; x[4 * v + 3] = d.w * inv * 64.0;
        }
        int q[8][16];
        for (int s = 0; s < S; ++s) {
            uint32_t packed[4];
#pragma unroll
            for (int v = 0; v < 4; ++v) {
                uint32_t wv = 0;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    double& xx = x[4 * v + e];
                    double qd = rint(xx);
                    qd = fmin(fmax(qd, -127.0), 127.0);   // |x| <= 64 (+ rounding) by construction
                    xx = (xx - qd) * 128.0;               // exact
                    const int qi = (int)qd;
                    q[s][4 * v + e] = qi;
                    wv |= ((uint32_t)(uint8_t)(int8_t)qi) << (8 * e);
                }
                packed[v] = wv;
            }
            const int64_t off = (layout == 1) ? (((col >> 7) * np + row) * S + s) * 128 + (col & 127)
                                              : (int64_t)s * plane_stride + row * ldq + col;
            *reinterpret_cast<uint4*>(planes + off) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
        }
        for (int gsum = S; gsum <= 2 * (S - 1); ++gsum) {
            int acc = 0;
            for (int sdig = gsum - (S - 1); sdig <= S - 1; ++sdig) {
                const int tdig = gsum - sdig;
#pragma unroll
                for (int e = 0; e < 16; ++e) acc += q[sdig][e] * q[tdig][e];
            }
            dropped += (double)acc * __longlong_as_double((long long)(1023 - (12 + 7 * gsum)) << 52);
        }
    }
    // 32 threads (one warp) cover 512 columns of one row when ncols >= 512; reduce and add once per warp
    const int lanes_per_row = (groups_per_row < 32) ? (int)groups_per_row : 32;
    for (int o = lanes_per_row >> 1; o > 0; o >>= 1) dropped += __shfl_xor_sync(0xffffffffu, dropped, o);
    if (active && ((threadIdx.x & 31) % lanes_per_row) == 0) {
        const int64_t slot = (col - c0) / 512;
        const double r2 = rs[row] * rs[row];
        corr[slot * np + row] = r2 * dropped;   // one writer per (slot, row)
    }
}

// test helper: plane-major [s][row][k] -> chunk-major [k / 128][row][s][128], 16 bytes per thread
static void launch_cut_digits(cudaStream_t st, int64_t nthreads, const double* mat, int64_t ld, const double* rs, int64_t r0,
                              int64_t nrows, int64_t c0, int64_t ncols, int8_t* planes, int64_t plane_stride, int64_t ldq, int S,
                              double* corr, int64_t np, int layout) {
    const unsigned grid = (unsigned)((nthreads + 255) / 256);
#define CUT(STv) cut_digits_kernel_t<STv><<<grid, 256, 0, st>>>(mat, ld, rs, r0, nrows, c0, ncols, planes, plane_stride, ldq, S, corr, np, layout)
    switch (S) {
        case 8: CUT(8); break;
        case 7: CUT(7); break;
        case 6: CUT(6); break;
        default: CUT(0); break;
    }
#undef CUT
}

__global__ void relayout_chunk_major_kernel(const int8_t* __restrict__ src, int8_t* __restrict__ dst, int64_t rows, int64_t K, int S) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t per_plane = rows * (K / 16);
    if (idx >= per_plane * S) return;
    const int s = (int)(idx / per_plane);
    const int64_t rem = idx % per_plane, row = rem / (K / 16), col = (rem % (K / 16)) * 16;
    const uint4 v = *reinterpret_cast<const uint4*>(src + (int64_t)s * rows * K + row * K + col);
    *reinterpret_cast<uint4*>(dst + (((col >> 7) * rows + row) * S + s) * 128 + (col & 127)) = v;
}

// C_ii -= sum over previous panels/slots of corr[.][i] for the rows of block column [c0, c0+kb)
__global__ void diag_correct_kernel(double* mat, int64_t ld, const double* corr, int64_t nslots, int64_t np, int64_t c0,
                                    int64_t kb) {
    const int64_t i = c0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c0 + kb) return;
    double s = 0.0;
    for (int64_t t = 0; t < nslots; ++t) s += corr[t * np + i];   // fixed order: deterministic
    mat[i * ld + i] -= s;
}

// rs[i] = 2^ceil(log2 sqrt(K_ii)), K_ii = kdiag + diag[i]; identity pad rows get 1
__global__ void row_scale_kernel(double kdiag, const double* __restrict__ diag, int64_t n, int64_t np, double* rs) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= np) return;
    double v = 1.0;
    if (i < n) {
        const double kii = kdiag + diag[i];
        if (kii > 0.0 && isfinite(kii)) {
            const int e = ilogb(kii);                        // 2^e <= kii < 2^(e+1)
            const int h = (e + 1 >= 0) ? (e + 2) / 2 : -((-(e + 1)) / 2);  // ceil((e+1)/2)
            v = scalbn(1.0, h);
        }
    }
    rs[i] = v;
}

// ---- host side -------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p)
            throw GpError("cuTensorMapEncodeTiled is not available from the driver");
        fn = (EncodeTiledFn)p;
    }
    return fn;
}

// planes: S int8 matrices [rows][ldq] (plane-major) or the chunk-major layout; box = 128 bytes (k) x BOXR rows, 128-byte swizzle
Maps make_maps(int8_t* planes, int64_t plane_stride, int64_t rows, int64_t ldq, int S, int layout = 0, int l2promo = 3) {
    Maps m{};
    EncodeTiledFn enc = get_encode();
    const CUtensorMapL2promotion promo = (l2promo == 0) ? CU_TENSOR_MAP_L2_PROMOTION_NONE
                                         : (l2promo == 1) ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B
                                         : (l2promo == 2) ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                                          : CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
    if (layout == 1) {   // chunk-major: [k / 128][row][plane][128]
        cuuint64_t dims[4] = {(cuuint64_t)KC, (cuuint64_t)S, (cuuint64_t)rows, (cuuint64_t)(ldq / KC)};
        cuuint64_t strides[3] = {(cuuint64_t)KC, (cuuint64_t)S * KC, (cuuint64_t)rows * S * KC};
        cuuint32_t box[4] = {(cuuint32_t)KC, 1u, (cuuint32_t)BOXR, 1u};
        cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
        CUresult r = enc(&m.all, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, planes, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) throw GpError("cuTensorMapEncodeTiled (4-D) failed");
        return m;
    }
    cuuint64_t dims[3] = {(cuuint64_t)ldq, (cuuint64_t)rows, (cuuint64_t)S};
    cuuint64_t strides[2] = {(cuuint64_t)ldq, (cuuint64_t)plane_stride};
    cuuint32_t box[3] = {(cuuint32_t)KC, (cuuint32_t)BOXR, 1u};
    cuuint32_t estr[3] = {1u, 1u, 1u};
    CUresult r = enc(&m.all, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, planes, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw GpError("cuTensorMapEncodeTiled (3-D) failed");
    return m;
}

// cluster-tile geometry of a launch: ctm x ctn cluster tiles of (CM * ROWS) x (CN * CTN)
struct ClusterGrid { int cs, ctm, ctn; int64_t rows, cols; };
static ClusterGrid cluster_grid(const Args& a, int CM, int CN, int MW) {
    ClusterGrid q;
    q.cs = CM * CN;
    q.rows = (int64_t)CM * 128 * MW;
    q.cols = (int64_t)CN * CTN;
    q.ctm = (int)(((int64_t)a.tiles_m * TM + q.rows - 1) / q.rows);
    q.ctn = (int)(((int64_t)a.tiles_n * TN + q.cols - 1) / q.cols);
    return q;
}
static bool cluster_above_diagonal(const Args& a, const ClusterGrid& q, int cid) {
    const int ci = cid / q.ctn, cj = cid % q.ctn;
    return a.skip_upper && a.row0 + (int64_t)ci * q.rows + q.rows - 1 < a.col0 + (int64_t)cj * q.cols;
}

template <int CM, int CN, bool PG, int MW>
static void launch_cfg(b200gp_ctx* ctx, const Maps& maps, const Args& a) {
    constexpr int SMEM = Geo<MW>::SMEM_BYTES;
    static bool attr = false;
    if (!attr) {
        CUDA_CHECK(cudaFuncSetAttribute(i8_update_kernel<CM, CN, PG, MW>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        attr = true;
    }
    const ClusterGrid q = cluster_grid(a, CM, CN, MW);
    const int64_t nclusters = (int64_t)q.ctm * q.ctn;
    if (nclusters <= 0 || a.K <= 0) return;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)((nclusters + (a.nseg > 1 ? (int64_t)(a.nseg - 1) * a.ntail : 0)) * q.cs));
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = SMEM;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = q.cs;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, i8_update_kernel<CM, CN, PG, MW>, maps, a));
    ctx->launches++;
    // int8 ops issued (mirrors the kernel's cluster-uniform decisions)
    int64_t active = 0;
    for (int c = 0; c < nclusters; ++c) active += cluster_above_diagonal(a, q, c) ? 0 : 1;
    ctx->prof.i8_ops += 2.0 * (double)active * 0.5 * a.S * (a.S + 1) * (double)q.rows * (double)q.cols * (double)a.K;
}

// cluster shape code: 1 = wide 256 x 128 tile per CTA (both m64 blocks of a warpgroup share every B stage; no pairing, no
// cluster); 2 = 2 x 1 cluster (B slices multicast to the CTA below, 256 x 128 per cluster) with tail split-K (default);
// 11 = 1x1 (no multicast), 21 = 2x1, 12 = 1x2, 22 = 2x2, 41 = 4x1, 42 = 4x2 (CTA tiles of 128 x 128, TMA multicast)
static void launch_update_one(b200gp_ctx* ctx, const Maps& maps, const Args& a) {
    if (ctx->oz_cluster == 1) { launch_cfg<1, 1, false, 2>(ctx, maps, a); return; }
    switch ((int)ctx->oz_cluster) {
#define OZ_CFG(CMv, CNv) \
    do { if (ctx->oz_pairing) launch_cfg<CMv, CNv, true, 1>(ctx, maps, a); else launch_cfg<CMv, CNv, false, 1>(ctx, maps, a); } while (0)
        case 11: OZ_CFG(1, 1); break;
        case 12: OZ_CFG(1, 2); break;
        case 22: OZ_CFG(2, 2); break;
        case 41: OZ_CFG(4, 1); break;
        case 42: OZ_CFG(4, 2); break;
        default: OZ_CFG(2, 1); break;   // 2 and 21
#undef OZ_CFG
    }
}

// Exactness of the int32 accumulators: every digit satisfies |q| <= 64 (cut_digits_kernel), a digit group g holds at
// most S pair products, so |accumulator| <= S * 4096 * K and the integer sums are exact while S * 4096 * K < 2^31:
// K <= 74880 for S = 7, 65408 for S = 8 (multiples of KC).  That covers every block column up to N = 65536 + nb in one
// launch; longer K ranges (N = 131072) are split into segments, each an independent exact update of the fp64 tile.
// (Typical sums are ~1e6 -- the bound is about the worst case, not the expected one.)
int max_exact_k(int S) {
    const int64_t k = (((int64_t)1 << 31) - 1) / (4096LL * (S > 0 ? S : 1));
    return (int)((k / KC) * KC);
}

// tail cluster tile `ti` (cluster index split_from + ti): C[tile] += sum_s scratch[s][ti] in the fixed order s = 0, 1, ...
// (deterministic)
__global__ void __launch_bounds__(256) splitk_fixup_kernel(double* __restrict__ C, int64_t ldc, int64_t row0, int64_t col0,
                                                           int ctn, int64_t trows, int64_t tcols, int split_from, int ntail,
                                                           int nextra, const double* __restrict__ scr, int64_t n_rows) {
    const int ti = blockIdx.y;
    const int cid = split_from + ti, ci = cid / ctn, cj = cid % ctn;
    const int64_t prow0 = row0 + (int64_t)ci * trows, gcol0 = col0 + (int64_t)cj * tcols;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // 2 columns per thread
    const int64_t r = idx / (tcols / 2), c = (idx % (tcols / 2)) * 2;
    if (r >= trows || prow0 + r >= n_rows || gcol0 + c >= n_rows) return;
    double2* cp = reinterpret_cast<double2*>(C + (prow0 + r) * ldc + gcol0 + c);
    double2 v = *cp;
    for (int sg = 0; sg < nextra; ++sg) {
        const double2 w = *reinterpret_cast<const double2*>(scr + ((int64_t)sg * ntail + ti) * (trows * tcols) + r * tcols + c);
        v.x += w.x; v.y += w.y;
    }
    *cp = v;
}

// Split-K of the default (code 2) launch's LAST, partially filled wave (option "ozaki_splitk" = E > 0: on, E = cost of a
// tile's fixed part -- epilogue passes, pipeline fill -- in K columns; 0 = off).  A block-column launch has T active cluster
// tiles of EQUAL duration for `slots` SM pairs: floor(T / slots) full waves and a last wave of r = T mod slots tiles that
// leaves slots - r SM pairs idle for a whole tile time; the last block columns have the longest tiles and the fewest of
// them.  The r tail tiles -- the last cluster indices of the launch, scheduled last -- are cut into s = floor(slots / r) K
// segments that run as s r <= slots short tiles of the SAME launch: segment 0 updates C, segment sg >= 1 accumulates into its
// own zero-filled fp64 scratch tile, added to C afterwards in a fixed order.  Every segment's integer sums are exact, so the
// only change is the order of s fp64 additions per element of a tail tile.
struct SplitPlan { int nseg = 1, kseg = 0, split_from = 0, ntail = 0; };
static SplitPlan choose_splitk(b200gp_ctx* ctx, const Args& a, const ClusterGrid& q) {
    SplitPlan p;
    p.kseg = a.K;
    const int64_t E = ctx->oz_splitk;
    if (ctx->oz_cluster != 2 || a.no_split || a.K < 2 * KC) return p;
    const int nclus = q.ctm * q.ctn;
    auto seg_len = [&](int s) { return (int)((((int64_t)a.K + s - 1) / s + KC - 1) / KC) * KC; };
    if (ctx->oz_splitk_force > 1) {   // tests: every tile, this many segments whatever the cost model says
        int s = (int)ctx->oz_splitk_force;
        if (s > a.K / KC) s = a.K / KC;
        p.kseg = seg_len(s);
        p.nseg = (a.K + p.kseg - 1) / p.kseg;
        p.split_from = 0; p.ntail = nclus;
        return p;
    }
    if (E <= 0) return p;
    const int slots = ctx->num_sms / q.cs > 0 ? ctx->num_sms / q.cs : 1;
    // active tiles in launch order; the tail starts at the (full waves * slots)-th one
    int64_t active = 0;
    for (int c = 0; c < nclus; ++c) active += cluster_above_diagonal(a, q, c) ? 0 : 1;
    const int64_t r = active % slots, full = active - r;
    if (r == 0) return p;
    int s = (int)(slots / r);
    while (s > 1 && seg_len(s) < 1024) --s;          // segments shorter than ~8 K chunks are all epilogue
    if (s > 16) s = 16;
    if (s < 2) return p;
    const int kseg = seg_len(s), nseg = (a.K + kseg - 1) / kseg;
    // worth it?  tail wave (K + E) against (kseg + E) + scratch traffic (zero-fill, fix-up) ~ 0.02 K-columns per tile-segment
    if ((double)kseg + (double)E > 0.9 * ((double)a.K + (double)E) || nseg < 2) return p;
    int64_t seen = 0;
    int split_from = nclus;
    for (int c = 0; c < nclus; ++c) {
        if (cluster_above_diagonal(a, q, c)) continue;
        if (seen == full) { split_from = c; break; }
        ++seen;
    }
    if (split_from >= nclus) return p;
    p.nseg = nseg; p.kseg = kseg; p.split_from = split_from; p.ntail = nclus - split_from;
    return p;
}

static void launch_update_splitk(b200gp_ctx* ctx, const Maps& maps, const Args& a) {
    const ClusterGrid q = cluster_grid(a, 2, 1, 1);   // the code-2 launch shape
    const SplitPlan p = choose_splitk(ctx, a, q);
    if (p.nseg <= 1) { launch_update_one(ctx, maps, a); return; }
    const size_t tile_doubles = (size_t)(q.rows * q.cols);
    const size_t need = (size_t)(p.nseg - 1) * p.ntail * tile_doubles * 8;
    size_t scr_bytes = (size_t)64 << 20;    // size classes (powers of two) so that the context's buffer cache hits
    while (scr_bytes < need) scr_bytes <<= 1;
    Scratch scr(ctx, scr_bytes);
    CUDA_CHECK(cudaMemsetAsync(scr.p, 0, need, ctx->stream));
    Args b = a;
    b.nseg = p.nseg; b.kseg = p.kseg; b.split_from = p.split_from; b.ntail = p.ntail;
    b.Cseg = scr.f64();
    launch_update_one(ctx, maps, b);
    dim3 grid((unsigned)((tile_doubles / 2 + 255) / 256), (unsigned)p.ntail);
    splitk_fixup_kernel<<<grid, 256, 0, ctx->stream>>>(a.C, a.ldc, a.row0, a.col0, q.ctn, q.rows, q.cols, p.split_from, p.ntail,
                                                      p.nseg - 1, scr.f64(), a.n_rows);
    CUDA_CHECK(cudaGetLastError());
    ctx->launches++;
}

void launch_update(b200gp_ctx* ctx, const Maps& maps, const Args& a) {
    const int kmax = max_exact_k(a.S);
    if (a.K <= kmax) {
        launch_update_splitk(ctx, maps, a);
        return;
    }
    for (int k0 = 0; k0 < a.K; k0 += kmax) {
        Args b = a;
        b.k_begin = a.k_begin + k0;
        b.K = (a.K - k0 < kmax) ? (a.K - k0) : kmax;
        launch_update_one(ctx, maps, b);
    }
}

// ---- int8 tensor peak: wgmma back to back from resident shared-memory operands (both warpgroups of every SM) ----------
constexpr int PEAK_SMEM = 2 * 64 * KC + B_BYTES + 1024;
__global__ void __launch_bounds__(256, 1) i8_peak_kernel(int iters, int* sink) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    for (int i = threadIdx.x; i < (2 * 64 * KC + B_BYTES) / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(smem)[i] = 0x01010101u;
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // generic-proxy smem writes -> async proxy (wgmma)
    __syncthreads();
    const int wg = threadIdx.x >> 7;
    const uint32_t a_addr = smem_u32(smem) + (uint32_t)(wg * 64 * KC), b_addr = smem_u32(smem) + 2 * 64 * KC;
    uint32_t d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0;
    wg_fence();
    for (int it = 0; it < iters; ++it) {
        uint32_t acc = 1;
        mma_stage(d, a_addr, b_addr, acc);
        wg_commit();
        wg_wait1();
    }
    wg_wait0();
    // every product is 1 x 1 summed over K = 128 per stage: the result is known, a wrong one marks the measurement invalid
    if (d[0] != (uint32_t)iters * (uint32_t)KC) atomicExch(sink, 1);
}

}  // namespace oz

// ================================================================================================
// left-looking factorisation driver
// ================================================================================================
void dense_panel_factor(b200gp_dense* s, int64_t k0, int64_t kb);                       // dense.cu
void dense_panel_factor_rows(b200gp_dense* s, int64_t k0, int64_t kb, int64_t r0, int64_t r1);   // dense.cu
struct BuildRegionArgs { int64_t r0, r1, c0, ncols; };
void dense_build_rows(b200gp_dense* s, const BuildRegionArgs& a);                        // dense.cu
void dense_build_region(b200gp_dense* s, int64_t r0, int64_t c0, int64_t ncols);          // dense.cu
double dense_kernel_diag_value(const KProg& P);                                           // dense.cu
void dense_trsv_fwd_blocks(b200gp_dense* s, double* y_dev, double* x_dev, int j_begin, int j_end);   // dense.cu

void dense_factor_ozaki(b200gp_dense* s, int S) {
    b200gp_ctx* ctx = s->ctx;
    const int64_t np = s->np, ld = np;
    int64_t NB = ctx->nb;
    {   // power of two >= 256 (the digit-cutting kernel reduces per 512-column group with warp shuffles)
        int64_t p2 = 256;
        while (p2 * 2 <= NB) p2 *= 2;
        NB = p2;
    }
    if (S < 2) S = 2;
    if (S > 8) S = 8;
    const bool lookahead = ctx->oz_lookahead != 0;

    const size_t plane_stride = (size_t)np * np;
    int8_t* planes = (int8_t*)ctx->alloc(plane_stride * S);
    double* rs = (double*)ctx->alloc((size_t)np * 8);
    int* err = (int*)ctx->alloc(sizeof(int));
    CUDA_CHECK(cudaMemsetAsync(err, 0, sizeof(int), ctx->stream));
    // Two-level blocking (option "ozaki_subpanel" = SB, 0 = off): the fp64 panel factorisation works on SB-wide
    // sub-panels; the update of sub-panel s by the sub-panels before it INSIDE the block column (K = s * SB <= NB - SB)
    // also runs on the int8 pipe.  The DMMA work of a block column drops from ~NB^2/2 to ~SB^2/2 per row.
    int64_t SB = lookahead ? 0 : ctx->oz_subpanel;
    if (SB < 256 || SB >= NB || (NB % SB) != 0 || (SB % 256) != 0) SB = 0;
    const int64_t slots_per_panel = SB ? (NB / SB) : ((NB + 511) / 512);
    const int64_t ncol_all = (np + NB - 1) / NB;
    const size_t corr_bytes = (size_t)ncol_all * slots_per_panel * np * 8;
    double* corr = (double*)ctx->alloc(corr_bytes);
    CUDA_CHECK(cudaMemsetAsync(corr, 0, corr_bytes, ctx->stream));
    int big = INT_MAX;
    CUDA_CHECK(cudaMemcpyAsync(s->info_dev, &big, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    oz::row_scale_kernel<<<(unsigned)((np + 255) / 256), 256, 0, ctx->stream>>>(dense_kernel_diag_value(s->prog), s->diag_dev,
                                                                               s->n, np, rs);
    ctx->launches++;
    const int layout = (int)ctx->oz_layout;
    oz::Maps maps = oz::make_maps(planes, (int64_t)plane_stride, np, np, S, layout, (int)ctx->oz_l2promo);

    // Two streams: `upd` (the context stream) runs build + int8 updates, `pan` (high priority) runs the fp64
    // panel factorisation and the digit cutting.  Update J is split into the part that only needs panels
    // < J-1 (runs UNDER the factorisation of panel J-1) and the short K = nb part that needs panel J-1.
    cudaStream_t upd = ctx->stream, pan = ctx->stream;
    if (lookahead) {
        if (!ctx->stream2) {
            int lo = 0, hi = 0;
            CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
            CUDA_CHECK(cudaStreamCreateWithPriority(&ctx->stream2, cudaStreamNonBlocking, hi));
        }
        pan = ctx->stream2;
    }
    const int ncol = (int)((np + NB - 1) / NB);
    // fused forward substitution (log_probability): y <- resid; after panel J is final its 128-blocks are substituted on a
    // side stream while the int8 update of column J + 1 runs (the substitution kernels fit beside the update's CTAs)
    cudaStream_t sol = nullptr;
    cudaEvent_t ev_panel = nullptr;
    double *fy = nullptr, *fx = nullptr;
    if (ctx->fuse_resid != nullptr && !lookahead) {
        if (!ctx->stream_solve) CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->stream_solve, cudaStreamNonBlocking));
        sol = ctx->stream_solve;
        fy = (double*)ctx->alloc((size_t)np * 8);
        fx = (double*)ctx->alloc((size_t)np * 8);
        CUDA_CHECK(cudaMemsetAsync(fy, 0, (size_t)np * 8, ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(fy, ctx->fuse_resid, (size_t)ctx->fuse_n * 8, cudaMemcpyDefault, ctx->stream));
        ev_panel = ctx->get_event();
        CUDA_CHECK(cudaEventRecord(ev_panel, ctx->stream));
        CUDA_CHECK(cudaStreamWaitEvent(sol, ev_panel, 0));
    }
    std::vector<cudaEvent_t> ev_upd(ncol), ev_cut(ncol);
    if (lookahead) {
        for (int j = 0; j < ncol; ++j) { ev_upd[j] = ctx->get_event(); ev_cut[j] = ctx->get_event(); }
        cudaEvent_t e0 = ctx->get_event();   // pan must see the row scales / info reset issued on upd
        CUDA_CHECK(cudaEventRecord(e0, upd));
        CUDA_CHECK(cudaStreamWaitEvent(pan, e0, 0));
        ctx->event_pool.push_back(e0);
    }

    auto update = [&](int64_t c0, int64_t kb, int64_t k_begin, int64_t k_len) {
        if (k_len <= 0) return;
        oz::Args a{};
        a.C = s->mat; a.ldc = ld; a.rs = rs;
        a.row0 = c0; a.col0 = c0; a.b_row0 = c0;
        a.tiles_m = (int)((np - c0) / oz::TM);
        a.tiles_n = (int)((kb + oz::TN - 1) / oz::TN);
        a.K = (int)k_len; a.k_begin = (int)k_begin; a.S = S; a.n_rows = np; a.skip_upper = 1; a.error_flag = err;
        a.prefetch = (int)ctx->oz_prefetch; a.pg_single = (ctx->oz_pairing == 2); a.layout = layout;
        ProfTimer t(ctx, &ctx->prof.syrk_ms);
        oz::launch_update(ctx, maps, a);
        ctx->prof.syrk_flop += 2.0 * (double)(np - c0) * (double)kb * (double)k_len;  // fp64-equivalent flop
        ctx->prof.syrk_launches++;
    };

    // Option "build_ahead": the kernel tiles of block column J+1 depend on nothing but X, so they are generated on a side
    // stream while the int8 update of column J runs (its CTAs leave most issue slots of an SM idle, and its last,
    // partially filled wave leaves whole SMs idle) instead of serially in front of update J+1.  Same values.
    const bool build_ahead = (ctx->build_ahead != 0) && !lookahead;
    cudaEvent_t ev_build = nullptr;
    if (build_ahead) {
        if (!ctx->stream2) CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->stream2, cudaStreamNonBlocking));
        ev_build = ctx->get_event();
        CUDA_CHECK(cudaEventRecord(ev_build, upd));                  // X / diag uploads and the resets above
        CUDA_CHECK(cudaStreamWaitEvent(ctx->stream2, ev_build, 0));
    }

    for (int J = 0; J < ncol; ++J) {
        const int64_t c0 = (int64_t)J * NB;
        const int64_t kb = (NB < np - c0) ? NB : (np - c0);
        // ---- stream upd: generate the block column, then C -= L[c0:, 0:c0] L[c0:c0+kb, 0:c0]^T on the int8 pipe
        ctx->stream = upd;
        if (build_ahead && J >= 1) CUDA_CHECK(cudaStreamWaitEvent(upd, ev_build, 0));   // generated during iteration J-1
        else dense_build_region(s, c0, c0, kb);
        if (lookahead) {
            if (J >= 2) update(c0, kb, 0, (int64_t)(J - 1) * NB);                 // panels 0 .. J-2
            if (J >= 1) {
                CUDA_CHECK(cudaStreamWaitEvent(upd, ev_cut[J - 1], 0));
                update(c0, kb, (int64_t)(J - 1) * NB, NB);                        // panel J-1
            }
        } else if (J >= 1) {
            update(c0, kb, 0, c0);
        }
        if (build_ahead && J + 1 < ncol) {   // column J+1 is not touched by anything else until its own update
            const int64_t c1 = c0 + NB, kb1 = (NB < np - c1) ? NB : (np - c1);
            ctx->stream = ctx->stream2;
            try {
                dense_build_region(s, c1, c1, kb1);
            } catch (...) {
                ctx->stream = upd;
                throw;
            }
            ctx->stream = upd;
            CUDA_CHECK(cudaEventRecord(ev_build, ctx->stream2));
        }
        if (J >= 1) {   // exact diagonal part of the dropped digit pairs (all previous panels)
            oz::diag_correct_kernel<<<(unsigned)((kb + 255) / 256), 256, 0, upd>>>(s->mat, ld, corr, (int64_t)J * slots_per_panel,
                                                                                  np, c0, kb);
            ctx->launches++;
        }
        if (lookahead) {
            CUDA_CHECK(cudaEventRecord(ev_upd[J], upd));
            CUDA_CHECK(cudaStreamWaitEvent(pan, ev_upd[J], 0));
        }
        // ---- stream pan: factor the panel in fp64 (DMMA path), then cut the digits of the rows below it
        ctx->stream = pan;
        if (SB) {
            for (int64_t sp = 0; sp * SB < kb; ++sp) {
                const int64_t cs = c0 + sp * SB;
                const int64_t sw = (SB < c0 + kb - cs) ? SB : (c0 + kb - cs);
                if (sp > 0) {   // C[cs:, cs:cs+sw] -= L[cs:, c0:cs] L[cs:cs+sw, c0:cs]^T with the digits cut a moment ago
                    oz::Args a{};
                    a.C = s->mat; a.ldc = ld; a.rs = rs;
                    a.row0 = cs; a.col0 = cs; a.b_row0 = cs;
                    a.tiles_m = (int)((np - cs) / oz::TM);
                    a.tiles_n = (int)((sw + oz::TN - 1) / oz::TN);
                    a.K = (int)(cs - c0); a.k_begin = (int)c0; a.S = S; a.n_rows = np; a.skip_upper = 1; a.error_flag = err;
                    a.prefetch = 0; a.pg_single = (ctx->oz_pairing == 2); a.layout = layout;
                    {
                        ProfTimer t(ctx, &ctx->prof.syrk_ms);
                        oz::launch_update(ctx, maps, a);
                        ctx->prof.syrk_flop += 2.0 * (double)(np - cs) * (double)sw * (double)(cs - c0);
                        ctx->prof.syrk_launches++;
                    }
                    oz::diag_correct_kernel<<<(unsigned)((sw + 255) / 256), 256, 0, pan>>>(
                        s->mat, ld, corr + (size_t)J * slots_per_panel * np, sp, np, cs, sw);
                    ctx->launches++;
                }
                {
                    ProfTimer t(ctx, &ctx->prof.panel_ms);
                    dense_panel_factor(s, cs, sw);
                }
                if (cs + sw < np) {
                    const int64_t nrows = np - (cs + sw);
                    const int64_t nthreads = nrows * (sw / 16);
                    ProfTimer t(ctx, &ctx->prof.build_ms);
                    oz::launch_cut_digits(pan, nthreads, s->mat, ld, rs, cs + sw, nrows, cs, sw, planes, (int64_t)plane_stride, np, S,
                        corr + ((size_t)J * slots_per_panel + sp) * np, np, layout);
                    ctx->launches++;
                }
            }
        } else {
        {
            ProfTimer t(ctx, &ctx->prof.panel_ms);
            dense_panel_factor(s, c0, kb);
        }
        if (c0 + kb < np) {
            const int64_t nrows = np - (c0 + kb);
            const int64_t nthreads = nrows * (kb / 16);
            ProfTimer t(ctx, &ctx->prof.build_ms);
            oz::launch_cut_digits(pan, nthreads, s->mat, ld, rs, c0 + kb, nrows, c0, kb, planes, (int64_t)plane_stride, np, S,
                corr + (size_t)J * slots_per_panel * np, np, layout);
            ctx->launches++;
        }
        }
        if (lookahead) CUDA_CHECK(cudaEventRecord(ev_cut[J], pan));
        if (sol) {   // columns [c0, c0 + kb) of L and their inverted diagonal blocks are final on `pan`
            CUDA_CHECK(cudaEventRecord(ev_panel, pan));
            CUDA_CHECK(cudaStreamWaitEvent(sol, ev_panel, 0));
            ctx->stream = sol;
            try {
                dense_trsv_fwd_blocks(s, fy, fx, (int)(c0 / TILE), (int)((c0 + kb) / TILE));
            } catch (...) {
                ctx->stream = upd;
                throw;
            }
            ctx->stream = pan;
        }
    }
    ctx->stream = upd;
    if (sol) {   // join
        CUDA_CHECK(cudaEventRecord(ev_panel, sol));
        CUDA_CHECK(cudaStreamWaitEvent(upd, ev_panel, 0));
        ctx->event_pool.push_back(ev_panel);
        ctx->fuse_y = fy; ctx->fuse_x = fx;
    }
    CUDA_CHECK(cudaGetLastError());
    if (ev_build) ctx->event_pool.push_back(ev_build);
    if (lookahead) {
        CUDA_CHECK(cudaStreamWaitEvent(upd, ev_cut[ncol - 1], 0));   // join
        for (int j = 0; j < ncol; ++j) { ctx->event_pool.push_back(ev_upd[j]); ctx->event_pool.push_back(ev_cut[j]); }
    }
    int herr = 0;
    CUDA_CHECK(cudaMemcpyAsync(&s->info, s->info_dev, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(&herr, err, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->release(planes, plane_stride * S);
    ctx->release(rs, (size_t)np * 8);
    ctx->release(err, sizeof(int));
    ctx->release(corr, corr_bytes);
    if (herr) throw GpError("int8 tensor update: pipeline wait timed out (internal protocol error)");
    if (s->info == INT_MAX) s->info = 0;
    if (s->info > s->n) s->info = 0;
}

// ---- diagnostics entry point: C -= sum_{s+t<S} 2^-(12+7(s+t)) rs_i rs_j Q_s[rows] Q_t[rows_b]^T ----------
extern "C" int b200gp_i8_update_test(b200gp_ctx* ctx, const int8_t* planes_host, int S, int64_t rows, int64_t K,
                                     const double* rs_host, double* C_host /* rows x rows, in/out */) {
    API_BEGIN(ctx)
    if (rows % 256 || K % 128 || S < 1 || S > 8) throw GpError("i8 test: rows % 256 == 0, K % 128 == 0, 1 <= S <= 8");
    const size_t pstride = (size_t)rows * K;
    int8_t* planes = (int8_t*)_ctx->alloc(pstride * S);
    double* rs = (double*)_ctx->alloc((size_t)rows * 8);
    double* C = (double*)_ctx->alloc((size_t)rows * rows * 8);
    int* err = (int*)_ctx->alloc(sizeof(int));
    CUDA_CHECK(cudaMemsetAsync(err, 0, sizeof(int), _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(planes, planes_host, pstride * S, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(rs, rs_host, (size_t)rows * 8, cudaMemcpyHostToDevice, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(C, C_host, (size_t)rows * rows * 8, cudaMemcpyHostToDevice, _ctx->stream));
    const int layout = (int)_ctx->oz_layout;
    int8_t* planes_cm = nullptr;
    if (layout == 1) {
        planes_cm = (int8_t*)_ctx->alloc(pstride * S);
        const int64_t nthr = (int64_t)S * rows * (K / 16);
        oz::relayout_chunk_major_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, _ctx->stream>>>(planes, planes_cm, rows, K, S);
        _ctx->launches++;
    }
    oz::Maps maps = oz::make_maps(layout == 1 ? planes_cm : planes, (int64_t)pstride, rows, K, S, layout);
    oz::Args a{};
    a.layout = layout;
    a.C = C; a.ldc = rows; a.rs = rs; a.row0 = 0; a.col0 = 0; a.b_row0 = 0;
    a.tiles_m = (int)(rows / oz::TM); a.tiles_n = (int)(rows / oz::TN);
    a.K = (int)K; a.k_begin = 0; a.S = S; a.n_rows = rows; a.skip_upper = 0; a.error_flag = err;
    a.prefetch = (int)_ctx->oz_prefetch; a.pg_single = (_ctx->oz_pairing == 2);
    oz::launch_update(_ctx, maps, a);
    int herr = 0;
    CUDA_CHECK(cudaMemcpyAsync(C_host, C, (size_t)rows * rows * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(&herr, err, sizeof(int), cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    _ctx->release(planes, pstride * S);
    if (planes_cm) _ctx->release(planes_cm, pstride * S);
    _ctx->release(rs, (size_t)rows * 8);
    _ctx->release(C, (size_t)rows * rows * 8);
    _ctx->release(err, sizeof(int));
    if (herr) throw GpError("i8 test: pipeline wait timed out");
    API_END
}

// ---- micro-benchmark of ONE update launch shape (diagnostics): rows x cols fp64 tile block, K int8 columns ----------
// planes are filled on the device with a hash pattern (|q| <= 64); `variant` = the ozaki_cluster code, the other switches
// come from the context options.  Returns the mean launch time and, if dbg_out != nullptr, the in-kernel cycle counters
// of the LAST launch (DBG_* slots).
__global__ void fill_planes_kernel(int8_t* p, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n / 16; i += stride) {
        uint32_t w[4];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            uint32_t h = (uint32_t)(i * 4 + v) * 2654435761u;
            h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
            uint32_t o = 0;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int q = (int)((h >> (8 * e)) & 0x7f) - 63;   // [-63, 64]
                o |= ((uint32_t)(uint8_t)(int8_t)q) << (8 * e);
            }
            w[v] = o;
        }
        reinterpret_cast<uint4*>(p)[i] = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

extern "C" int b200gp_i8_update_bench(b200gp_ctx* ctx, int64_t rows, int64_t cols, int64_t K, int S, int reps,
                                      int64_t ldq /* row stride of a digit plane, 0 = K */, int64_t ldc /* 0 = cols */,
                                      double* ms_out, unsigned long long* dbg_out /* 16 or null */) {
    API_BEGIN(ctx)
    if (ldq <= 0) ldq = K;
    if (ldc <= 0) ldc = cols;
    if (rows % 256 || cols % 256 || K % 128 || S < 1 || S > 8 || cols > rows || reps < 1 || ldq < K || ldq % 128 || ldc < cols)
        throw GpError("i8 bench: rows % 256 == 0, cols % 256 == 0, cols <= rows, K % 128 == 0, 1 <= S <= 8, ldq >= K, ldc >= cols");
    const size_t pstride = (size_t)rows * ldq;
    Scratch planes_b(_ctx, pstride * S), rs_b(_ctx, (size_t)rows * 8), C_b(_ctx, (size_t)rows * ldc * 8);
    Scratch err_b(_ctx, sizeof(int)), dbg_b(_ctx, oz::DBG_N * 8);
    int8_t* planes = (int8_t*)planes_b.p;
    double* rs = rs_b.f64();
    int* err = (int*)err_b.p;
    unsigned long long* dbg = (unsigned long long*)dbg_b.p;
    CUDA_CHECK(cudaMemsetAsync(err, 0, sizeof(int), _ctx->stream));
    CUDA_CHECK(cudaMemsetAsync(C_b.p, 0, (size_t)rows * ldc * 8, _ctx->stream));
    fill_planes_kernel<<<_ctx->num_sms * 8, 256, 0, _ctx->stream>>>(planes, pstride * S);
    {
        std::vector<double> ones((size_t)rows, 1.0);
        CUDA_CHECK(cudaMemcpyAsync(rs, ones.data(), (size_t)rows * 8, cudaMemcpyHostToDevice, _ctx->stream));
        CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    }
    const int layout = (int)_ctx->oz_layout;   // layout 1 reads the same bytes through the 4-D map (timing only)
    oz::Maps maps = oz::make_maps(planes, (int64_t)pstride, rows, ldq, S, layout, (int)_ctx->oz_l2promo);
    oz::Args a{};
    a.layout = layout;
    a.C = C_b.f64(); a.ldc = ldc; a.rs = rs; a.row0 = 0; a.col0 = 0; a.b_row0 = 0;
    a.tiles_m = (int)(rows / oz::TM); a.tiles_n = (int)(cols / oz::TN);
    a.K = (int)K; a.k_begin = 0; a.S = S; a.n_rows = rows; a.skip_upper = 0; a.error_flag = err;
    a.prefetch = (int)_ctx->oz_prefetch; a.pg_single = (_ctx->oz_pairing == 2);
    a.dbg = nullptr;
    oz::launch_update(_ctx, maps, a);   // warm-up
    cudaEventRecord(_ctx->ev0, _ctx->stream);
    for (int r = 0; r < reps; ++r) oz::launch_update(_ctx, maps, a);
    cudaEventRecord(_ctx->ev1, _ctx->stream);
    CUDA_CHECK(cudaEventSynchronize(_ctx->ev1));
    float ms = 0;
    cudaEventElapsedTime(&ms, _ctx->ev0, _ctx->ev1);
    *ms_out = (double)ms / reps;
    if (dbg_out) {
        CUDA_CHECK(cudaMemsetAsync(dbg, 0, oz::DBG_N * 8, _ctx->stream));
        a.dbg = dbg;
        oz::launch_update(_ctx, maps, a);
        CUDA_CHECK(cudaMemcpyAsync(dbg_out, dbg, oz::DBG_N * 8, cudaMemcpyDeviceToHost, _ctx->stream));
    }
    int herr = 0;
    CUDA_CHECK(cudaMemcpyAsync(&herr, err, sizeof(int), cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    if (herr) throw GpError("i8 bench: pipeline wait timed out");
    API_END
}

extern "C" int b200gp_measure_i8_peak(b200gp_ctx* ctx, double* tops) {
    API_BEGIN(ctx)
    CUDA_CHECK(cudaFuncSetAttribute(oz::i8_peak_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, oz::PEAK_SMEM));
    int* sink = (int*)_ctx->alloc(sizeof(int));
    CUDA_CHECK(cudaMemsetAsync(sink, 0, sizeof(int), _ctx->stream));
    const int iters = (int)((_ctx->peak_iters < 200000) ? _ctx->peak_iters * 4 : 800000);
    float ms = 0;
    for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(_ctx->ev0, _ctx->stream);
        oz::i8_peak_kernel<<<_ctx->num_sms, 256, oz::PEAK_SMEM, _ctx->stream>>>(iters, sink);
        cudaEventRecord(_ctx->ev1, _ctx->stream);
        CUDA_CHECK(cudaEventSynchronize(_ctx->ev1));
        cudaEventElapsedTime(&ms, _ctx->ev0, _ctx->ev1);
    }
    CUDA_CHECK(cudaGetLastError());
    _ctx->launches += 2;
    int bad = 0;
    CUDA_CHECK(cudaMemcpy(&bad, sink, sizeof(int), cudaMemcpyDeviceToHost));
    _ctx->release(sink, sizeof(int));
    if (bad) throw GpError("i8 peak: wrong accumulator value");
    // per SM and iteration: 2 warpgroups x 4 instructions x 64 x 128 x 32 MAC
    *tops = (double)_ctx->num_sms * (double)iters * 2.0 * 4.0 * 2.0 * 64.0 * oz::CTN * 32.0 / (ms * 1e-3) / 1e12;
    API_END
}

// ================================================================================================
// Multi-GPU (one process per GPU) step API for ONE dense factorisation sharded over ranks.
//
// Every rank holds the full matrix buffer and all digit planes.  For block column J the rows [c0, np) are
// split into equal chunks; rank r generates + int8-updates only ITS chunk of C_J, the chunks are all-gathered
// by the host (torch.distributed / NCCL over NVLink, one collective per block column:
// rows x nb x 8 bytes), and every rank then runs the (cheap, deterministic) fp64 panel factorisation and the
// digit cutting redundantly -- so there is no owner, no panel broadcast and no second collective.
// The N^3/3 part (the int8 update) is divided by the number of GPUs; communication totals 8 N^2/2 bytes.
// ================================================================================================
struct b200gp_mg {
    b200gp_ctx* ctx = nullptr;
    b200gp_dense* s = nullptr;
    int S = 8;
    int64_t NB = 1024;
    int ncol = 0;
    int8_t* planes = nullptr;
    size_t plane_stride = 0;
    double* rs = nullptr;
    double* corr = nullptr;
    size_t corr_bytes = 0;
    int64_t slots_per_panel = 0;
    int* err = nullptr;
    oz::Maps maps{};
    // streaming mode: no full fp64 matrix; a rolling np x NB column buffer, forward solve + log-det per panel
    bool streaming = false;
    double* colbuf = nullptr;
    bool colbuf_external = false;   // the rolling column buffer is the caller's (torch / NCCL-registered) memory
    double* y = nullptr;       // np, right-hand side being reduced
    double* x = nullptr;       // np, alpha
    double* logparts = nullptr;  // ncol partial sums of log L_ii
};

void dense_trsv_fwd_blocks(b200gp_dense* s, double* y_dev, double* x_dev, int j_begin, int j_end);   // dense.cu
void dense_logdiag_partial(b200gp_dense* s, int64_t c0, int64_t count, double* out_dev);             // dense.cu
b200gp_dense* dense_alloc_for_prog(b200gp_ctx* ctx, const KProg& prog, const double* X, int64_t n, int ndim,
                                   const double* diag);   // dense.cu

extern "C" {

int b200gp_mg_create(b200gp_ctx* ctx, const double* prog, int n_instr, const double* X, int64_t n, int ndim,
                     const double* diag, const double* resid, int slices, int streaming, b200gp_mg** out) {
    API_BEGIN(ctx)
    KProg P = parse_prog(prog, n_instr, ndim);
    b200gp_mg* m = new b200gp_mg();
    m->ctx = _ctx;
    m->streaming = (streaming != 0);
    int64_t p2 = 256;
    while (p2 * 2 <= _ctx->nb) p2 *= 2;
    m->NB = p2;
    if (!m->streaming) {
        m->s = dense_alloc_for_prog(_ctx, P, X, n, ndim, diag);
    } else {
        // hand-built dense object without the np x np matrix
        if (ndim < 1 || ndim > 16) throw GpError("dense: ndim must be in [1, 16]");
        b200gp_dense* s = new b200gp_dense();
        s->ctx = _ctx; s->n = n; s->np = ((n + TILE - 1) / TILE) * TILE; s->ld = m->NB;
        s->has_prog = true; s->prog = P; s->ndim = ndim; s->owns_inputs = true;
        s->linv = (double*)_ctx->alloc((size_t)(s->np / TILE) * TILE * TILE * sizeof(double));
        s->info_dev = (int*)_ctx->alloc(sizeof(int));
        s->X_dev = (double*)_ctx->alloc((size_t)n * ndim * sizeof(double));
        s->diag_dev = (double*)_ctx->alloc((size_t)n * sizeof(double));
        CUDA_CHECK(cudaMemcpyAsync(s->X_dev, X, (size_t)n * ndim * sizeof(double), cudaMemcpyDefault, _ctx->stream));
        CUDA_CHECK(cudaMemcpyAsync(s->diag_dev, diag, (size_t)n * sizeof(double), cudaMemcpyDefault, _ctx->stream));
        m->s = s;
        m->colbuf = (double*)_ctx->alloc((size_t)s->np * m->NB * 8);
    }
    const int64_t np = m->s->np;
    m->S = (slices < 2) ? 2 : (slices > 8 ? 8 : slices);
    m->y = (double*)_ctx->alloc((size_t)np * 8);
    m->x = (double*)_ctx->alloc((size_t)np * 8);
    CUDA_CHECK(cudaMemsetAsync(m->y, 0, (size_t)np * 8, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(m->y, resid, (size_t)n * 8, cudaMemcpyDefault, _ctx->stream));
    m->ncol = (int)((np + m->NB - 1) / m->NB);
    m->plane_stride = (size_t)np * np;
    m->planes = (int8_t*)_ctx->alloc(m->plane_stride * m->S);
    m->rs = (double*)_ctx->alloc((size_t)np * 8);
    m->err = (int*)_ctx->alloc(sizeof(int));
    m->slots_per_panel = (m->NB + 511) / 512;
    m->corr_bytes = (size_t)m->ncol * m->slots_per_panel * np * 8;
    m->corr = (double*)_ctx->alloc(m->corr_bytes);
    m->logparts = (double*)_ctx->alloc((size_t)m->ncol * 8);
    CUDA_CHECK(cudaMemsetAsync(m->logparts, 0, (size_t)m->ncol * 8, _ctx->stream));
    CUDA_CHECK(cudaMemsetAsync(m->err, 0, sizeof(int), _ctx->stream));
    CUDA_CHECK(cudaMemsetAsync(m->corr, 0, m->corr_bytes, _ctx->stream));
    int big = INT_MAX;
    CUDA_CHECK(cudaMemcpyAsync(m->s->info_dev, &big, sizeof(int), cudaMemcpyHostToDevice, _ctx->stream));
    oz::row_scale_kernel<<<(unsigned)((np + 255) / 256), 256, 0, _ctx->stream>>>(dense_kernel_diag_value(m->s->prog),
                                                                                m->s->diag_dev, m->s->n, np, m->rs);
    _ctx->launches++;
    m->maps = oz::make_maps(m->planes, (int64_t)m->plane_stride, np, np, m->S);
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    *out = m;
    API_END
}

int b200gp_mg_free(b200gp_mg* m) {
    if (!m) return 0;
    API_BEGIN(m->ctx)
    _ctx->release(m->planes, m->plane_stride * m->S);
    _ctx->release(m->rs, (size_t)m->s->np * 8);
    _ctx->release(m->err, sizeof(int));
    _ctx->release(m->corr, m->corr_bytes);
    _ctx->release(m->logparts, (size_t)m->ncol * 8);
    _ctx->release(m->y, (size_t)m->s->np * 8);
    _ctx->release(m->x, (size_t)m->s->np * 8);
    if (m->streaming) {
        if (!m->colbuf_external) _ctx->release(m->colbuf, (size_t)m->s->np * m->NB * 8);
        m->s->mat = nullptr;
    }
    dense_destroy(m->s);
    delete m;
    API_END
}

// streaming mode: use the caller's contiguous buffer of `rows` x nb doubles as the rolling block column (rows >= np), so
// that a rank's row chunk of the column is ONE contiguous range and the block column can be all-gathered IN PLACE
// (no pack / unpack copies around the collective)
int b200gp_mg_use_colbuf(b200gp_mg* m, double* buf_dev, int64_t rows) {
    API_BEGIN(m->ctx)
    if (!m->streaming) throw GpError("mg_use_colbuf: only the streaming mode has a rolling column buffer");
    if (!buf_dev || rows < m->s->np) throw GpError("mg_use_colbuf: the buffer must hold at least np rows");
    if (!m->colbuf_external) _ctx->release(m->colbuf, (size_t)m->s->np * m->NB * 8);
    m->colbuf = buf_dev;
    m->colbuf_external = true;
    API_END
}

int b200gp_mg_geometry(b200gp_mg* m, int64_t* np, int64_t* nb, int* ncol) {
    API_BEGIN(m->ctx)
    *np = m->s->np; *nb = m->NB; *ncol = m->ncol;
    API_END
}

// generate rows [r0, r1) of block column J and subtract L[r0:r1, 0:c0] L[c0:c0+kb, 0:c0]^T (int8 tensor update)
int b200gp_mg_update_rows(b200gp_mg* m, int J, int64_t r0, int64_t r1) {
    API_BEGIN(m->ctx)
    b200gp_dense* s = m->s;
    const int64_t np = s->np, c0 = (int64_t)J * m->NB;
    const int64_t kb = (m->NB < np - c0) ? m->NB : (np - c0);
    if (r1 > np) r1 = np;
    if (r0 < c0 || r0 % oz::TM || r1 % oz::TM) throw GpError("mg_update_rows: rows must be 128-aligned and >= c0");
    if (m->streaming) s->mat = m->colbuf - c0;   // virtual base: (r, c) of this block column -> colbuf[r * NB + (c - c0)]
    if (r1 <= r0) return 0;
    {   // build only my rows
        BuildRegionArgs br{r0, r1, c0, kb};
        dense_build_rows(s, br);
    }
    if (J >= 1) {
        oz::Args a{};
        a.C = s->mat; a.ldc = s->ld; a.rs = m->rs;
        a.row0 = r0; a.col0 = c0; a.b_row0 = c0;
        a.tiles_m = (int)((r1 - r0) / oz::TM);
        a.tiles_n = (int)((kb + oz::TN - 1) / oz::TN);
        a.K = (int)c0; a.k_begin = 0; a.S = m->S; a.n_rows = np; a.skip_upper = 1; a.error_flag = m->err;
        a.prefetch = (int)_ctx->oz_prefetch; a.pg_single = (_ctx->oz_pairing == 2);
        // the tail split depends on the tile count of THIS rank's rows, so with it the last bits of the result depend on the
        // rank count (option "mg_splitk" = 0 restores the rank-count-independent summation order: bit-identical for any G)
        a.no_split = (_ctx->mg_splitk == 0) ? 1 : 0;
        ProfTimer t(_ctx, &_ctx->prof.syrk_ms);
        oz::launch_update(_ctx, m->maps, a);
        _ctx->prof.syrk_flop += 2.0 * (double)(r1 - r0) * (double)kb * (double)c0;
        _ctx->prof.syrk_launches++;
    }
    API_END
}

// mat[r0:r1, c0:c0+kb] <-> contiguous device buffer [(r1-r0)][nb] (torch-owned, NCCL-visible)
int b200gp_mg_pack(b200gp_mg* m, int J, int64_t r0, int64_t r1, double* buf_dev) {
    API_BEGIN(m->ctx)
    const int64_t np = m->s->np, c0 = (int64_t)J * m->NB;
    const int64_t kb = (m->NB < np - c0) ? m->NB : (np - c0);
    if (r1 > np) r1 = np;
    if (r1 <= r0) return 0;
    CUDA_CHECK(cudaMemcpy2DAsync(buf_dev, (size_t)m->NB * 8, m->s->mat + r0 * m->s->ld + c0, (size_t)m->s->ld * 8,
                                 (size_t)kb * 8, (size_t)(r1 - r0), cudaMemcpyDeviceToDevice, _ctx->stream));
    API_END
}
int b200gp_mg_unpack(b200gp_mg* m, int J, int64_t r0, int64_t r1, const double* buf_dev) {
    API_BEGIN(m->ctx)
    const int64_t np = m->s->np, c0 = (int64_t)J * m->NB;
    const int64_t kb = (m->NB < np - c0) ? m->NB : (np - c0);
    if (r1 > np) r1 = np;
    if (r1 <= r0) return 0;
    CUDA_CHECK(cudaMemcpy2DAsync(m->s->mat + r0 * m->s->ld + c0, (size_t)m->s->ld * 8, buf_dev, (size_t)m->NB * 8,
                                 (size_t)kb * 8, (size_t)(r1 - r0), cudaMemcpyDeviceToDevice, _ctx->stream));
    API_END
}

// ---- the panel step, in two halves so that the fp64 triangular solve is sharded by rows as well --------------------
// mg_panel_factor: diagonal correction + factorisation of the diagonal block (every rank, redundantly: it needs the block's
// rows, which the host broadcasts from their owner) + triangular solve of THIS rank's rows [r0, r1) below the block.
// The host then all-gathers the finished column (in place) and calls mg_panel_finish: digit cutting of all rows and, in
// streaming mode, the forward-substitution / log-det step that consumes the column before it is overwritten.
int b200gp_mg_panel_factor(b200gp_mg* m, int J, int64_t r0, int64_t r1) {
    API_BEGIN(m->ctx)
    b200gp_dense* s = m->s;
    const int64_t np = s->np, c0 = (int64_t)J * m->NB;
    const int64_t kb = (m->NB < np - c0) ? m->NB : (np - c0);
    if (m->streaming) s->mat = m->colbuf - c0;
    if (J >= 1) {
        oz::diag_correct_kernel<<<(unsigned)((kb + 255) / 256), 256, 0, _ctx->stream>>>(
            s->mat, s->ld, m->corr, (int64_t)J * m->slots_per_panel, np, c0, kb);
        _ctx->launches++;
    }
    {
        ProfTimer t(_ctx, &_ctx->prof.panel_ms);
        dense_panel_factor_rows(s, c0, kb, r0, r1);
    }
    CUDA_CHECK(cudaGetLastError());
    API_END
}

static void mg_panel_tail(b200gp_mg* m, int J) {
    b200gp_ctx* _ctx = m->ctx;
    b200gp_dense* s = m->s;
    const int64_t np = s->np, c0 = (int64_t)J * m->NB;
    const int64_t kb = (m->NB < np - c0) ? m->NB : (np - c0);
    if (c0 + kb < np) {
        const int64_t nrows = np - (c0 + kb);
        const int64_t nthreads = nrows * (kb / 16);
        ProfTimer t(_ctx, &_ctx->prof.build_ms);
        oz::launch_cut_digits(_ctx->stream, nthreads, s->mat, s->ld, m->rs, c0 + kb, nrows, c0, kb, m->planes,
                              (int64_t)m->plane_stride, np, m->S, m->corr + (size_t)J * m->slots_per_panel * np, np, 0);
        _ctx->launches++;
    }
    if (m->streaming) {
        // this block column of L is about to be overwritten: consume it now (forward substitution + log-det)
        dense_trsv_fwd_blocks(s, m->y, m->x, (int)(c0 / TILE), (int)((c0 + kb) / TILE));
        const int64_t valid = (s->n > c0) ? ((s->n - c0 < kb) ? (s->n - c0) : kb) : 0;
        dense_logdiag_partial(s, c0, valid, m->logparts + J);
    }
    CUDA_CHECK(cudaGetLastError());
}

int b200gp_mg_panel_finish(b200gp_mg* m, int J) {
    API_BEGIN(m->ctx)
    if (m->streaming) m->s->mat = m->colbuf - (int64_t)J * m->NB;
    mg_panel_tail(m, J);
    API_END
}

// after the all-gather: diagonal correction, fp64 panel factorisation, digit cutting (identical on every rank)
int b200gp_mg_panel(b200gp_mg* m, int J) {
    API_BEGIN(m->ctx)
    b200gp_dense* s = m->s;
    const int64_t np = s->np, c0 = (int64_t)J * m->NB;
    const int64_t kb = (m->NB < np - c0) ? m->NB : (np - c0);
    if (J >= 1) {
        oz::diag_correct_kernel<<<(unsigned)((kb + 255) / 256), 256, 0, _ctx->stream>>>(
            s->mat, s->ld, m->corr, (int64_t)J * m->slots_per_panel, np, c0, kb);
        _ctx->launches++;
    }
    {
        ProfTimer t(_ctx, &_ctx->prof.panel_ms);
        dense_panel_factor(s, c0, kb);
    }
    mg_panel_tail(m, J);
    API_END
}

// forward solve + reductions on this rank's (complete) factor: gp.py:313-320
int b200gp_mg_finish(b200gp_mg* m, double* logp) {
    API_BEGIN(m->ctx)
    b200gp_dense* s = m->s;
    const int64_t np = s->np, n = s->n;
    int herr = 0;
    CUDA_CHECK(cudaMemcpyAsync(&s->info, s->info_dev, sizeof(int), cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(&herr, m->err, sizeof(int), cudaMemcpyDeviceToHost, _ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
    if (herr) throw GpError("int8 tensor update: pipeline wait timed out (internal protocol error)");
    if (s->info == INT_MAX) s->info = 0;
    (void)np;
    double ld;
    if (m->streaming) {
        std::vector<double> parts((size_t)m->ncol);
        CUDA_CHECK(cudaMemcpyAsync(parts.data(), m->logparts, (size_t)m->ncol * 8, cudaMemcpyDeviceToHost, _ctx->stream));
        CUDA_CHECK(cudaStreamSynchronize(_ctx->stream));
        ld = 0.0;
        for (double p : parts) ld += p;   // fixed order
    } else {
        dense_solve_vec_dev(s, m->y, m->x, false);
        ld = dense_logdet_half(s);
    }
    const double ss = dense_sumsq_dev(_ctx, m->x, n);
    double lp = -0.5 * ss - (ld + 0.5 * (double)n * log(2.0 * M_PI));
    if (s->info != 0 || !isfinite(lp)) lp = -INFINITY;
    *logp = lp;
    API_END
}

}  // extern "C"

// single-GPU fused log_probability through the same step functions (world size 1, streaming)
double ozaki_logp_streaming(b200gp_ctx* ctx, const KProg& P, const double* X, int64_t n, int ndim, const double* diag,
                            const double* resid, int S) {
    const std::vector<double> prog = kprog_encode(P);   // kprog.cuh: metric definitions + instructions
    const int n_rows = (int)(prog.size() / B200GP_PROG_STRIDE);
    b200gp_mg* m = nullptr;
    if (b200gp_mg_create(ctx, prog.data(), n_rows, X, n, ndim, diag, resid, S, 1, &m)) throw GpError(ctx->err);
    double lp = 0.0;
    int rc = 0;
    const int64_t np = m->s->np;
    for (int J = 0; J < m->ncol && !rc; ++J) {
        rc = b200gp_mg_update_rows(m, J, (int64_t)J * m->NB, np);
        if (!rc) rc = b200gp_mg_panel(m, J);
    }
    if (!rc) rc = b200gp_mg_finish(m, &lp);
    std::string err = ctx->err;
    b200gp_mg_free(m);
    if (rc) throw GpError(err);
    return lp;
}
