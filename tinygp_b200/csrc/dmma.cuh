// The fp64 tensor-core (DMMA) mainloop of every fp64 GEMM kernel: the warp tile and the 128 x 128 CTA tile with its
// cp.async operand ring (cta_tile_nt).  Its callers are dense.cu's gemm_nt_kernel (trailing and panel updates, the
// gradient's panel products) and grad.cu's tri_gemm_kernel (triangular inverse and the W contraction); each keeps only
// its tile schedule and its epilogue.
//
// Shape: mma.sync.m16n8k16.f64, Hopper's widest fp64 MMA (one DMMA.16x8x16 instruction).  On sm_90 the m16n8 shapes
// issue at a higher fp64 rate than Ampere's m8n8k4; MEASURED.md records the rates of all four shapes.
//
// Operands come from one shared-memory pipeline stage: SK = 32 doubles of K per row, rows K-contiguous (both operands
// of an NT product, C = A B^T), row stride LDS = 36 doubles.  The warp tile steps through a stage BK = 16 of K at a time.
// The padding 32 -> 36 makes the fragment loads of a half-warp (rows g = 0..3, k offsets t = 0..3) hit 16 distinct
// 8-byte bank pairs (row stride 72 words = 8 mod 32).
//
// A warp owns a WM x WN = 64 x 32 tile of C: 4 x 4 atoms of 16 x 8.  Its accumulators are kept as acc[8][4][2]:
// acc[m8][ni][q] is C(8 m8 + g, 8 ni + 2 t + q) of the warp tile (acc_row / acc_col), which is what the epilogues
// index.  Atom (mi, ni) accumulates into acc[2 mi][ni] (its rows g) and acc[2 mi + 1][ni] (its rows g + 8).
//
// Fragment layout of mma.m16n8k{4,8,16}.f64 (PTX ISA, "Matrix Fragments for mma.m16n8k*" with .f64), lane = 4 g + t:
//   A (16 x K, row): register i holds (row g + 8 (i mod 2), k t + 4 floor(i / 2))     K / 2 registers
//   B (K x 8, col):  register i holds (k t + 4 i, col g)                               K / 4 registers
//   C (16 x 8):      register i holds (row g + 8 floor(i / 2), col 2 t + (i mod 2))    4 registers
// The index functions below are __host__ __device__ so that tests/csrc/dmma_hostcheck.cu checks the loads and the
// accumulator map on the CPU with the same source.
#pragma once
#include <stdint.h>

namespace dmma {
constexpr int MK = 16;                  // K of one mma instruction
constexpr int BK = 16, LDS = 36;        // K step of the warp tile and padded row stride of a stage (doubles)
constexpr int WM = 64, WN = 32;         // warp tile
constexpr int AM = WM / 16, AN = WN / 8;
constexpr int AREG = MK / 2, BREG = MK / 4;
static_assert(BK % MK == 0, "a warp-tile K step holds whole mma K steps");

__host__ __device__ constexpr int a_row(int lane, int i) { return (lane >> 2) + 8 * (i & 1); }
__host__ __device__ constexpr int a_k(int lane, int i) { return (lane & 3) + 4 * (i >> 1); }
__host__ __device__ constexpr int b_k(int lane, int i) { return (lane & 3) + 4 * i; }
__host__ __device__ constexpr int b_col(int lane) { return lane >> 2; }
__host__ __device__ constexpr int c_row(int lane, int i) { return (lane >> 2) + 8 * (i >> 1); }
__host__ __device__ constexpr int c_col(int lane, int i) { return 2 * (lane & 3) + (i & 1); }
// element of the warp tile held by acc[m8][ni][q]
__host__ __device__ constexpr int acc_row(int lane, int m8) { return 8 * m8 + (lane >> 2); }
__host__ __device__ constexpr int acc_col(int lane, int ni, int q) { return 8 * ni + 2 * (lane & 3) + q; }

// fragments of A atom mi / B atom ni at K offset k0 of the stage; as / bs point at row 0, k 0 of the warp's rows
__host__ __device__ inline void load_a(double (&a)[AREG], const double* as, int lane, int mi, int k0) {
#pragma unroll
    for (int i = 0; i < AREG; ++i) a[i] = as[(16 * mi + a_row(lane, i)) * LDS + k0 + a_k(lane, i)];
}
__host__ __device__ inline void load_b(double (&b)[BREG], const double* bs, int lane, int ni, int k0) {
#pragma unroll
    for (int i = 0; i < BREG; ++i) b[i] = bs[(8 * ni + b_col(lane)) * LDS + k0 + b_k(lane, i)];
}

// {lo, hi} = the atom's accumulator rows g and g + 8
__device__ __forceinline__ void mma(double (&lo)[2], double (&hi)[2], const double (&a)[AREG], const double (&b)[BREG]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
        "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
        : "+d"(lo[0]), "+d"(lo[1]), "+d"(hi[0]), "+d"(hi[1])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
          "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// acc += (the warp's 64 rows of A) (its 32 rows of B)^T over BK of K
__device__ __forceinline__ void warp_tile_stage(double (&acc)[WM / 8][WN / 8][2], const double* as, const double* bs,
                                                int lane) {
#pragma unroll
    for (int k0 = 0; k0 < BK; k0 += MK) {
        double b[AN][BREG];
#pragma unroll
        for (int ni = 0; ni < AN; ++ni) load_b(b[ni], bs, lane, ni, k0);
#pragma unroll
        for (int mi = 0; mi < AM; ++mi) {
            double a[AREG];
            load_a(a, as, lane, mi, k0);
#pragma unroll
            for (int ni = 0; ni < AN; ++ni) mma(acc[2 * mi][ni], acc[2 * mi + 1][ni], a, b[ni]);
        }
    }
}

// ---- CTA tile: 128 x 128 of C, 8 warps (2 x 4) of warp tiles, 3-slot cp.async ring of SK-deep stages ----
// Each slot has a full and an empty mbarrier (after the ring, outside the memory a caller reuses).  A warp waits only for
// the stage it computes on and releases it when its MMAs are done, so there is no CTA barrier in the mainloop: the two
// warps of an SM sub-partition drift apart and the DMMAs of one overlap the fragment loads of the other.
constexpr int BM = 128, SK = 32, STAGES = 3, THREADS = 256;
constexpr int STAGE_DOUBLES = 2 * BM * LDS;                                 // A rows, then B rows
constexpr int RING_BYTES = STAGES * STAGE_DOUBLES * (int)sizeof(double);   // 221184
constexpr int SMEM_BYTES = RING_BYTES + 2 * STAGES * (int)sizeof(uint64_t);
static_assert(BM == 2 * WM && BM == 4 * WN && THREADS == 8 * 32, "8 warps of 2 x 4 warp tiles cover the CTA tile");
static_assert(SK % BK == 0 && SK <= LDS, "a stage holds whole warp-tile K steps");
static_assert(THREADS * 8 * 16 == BM * SK * (int)sizeof(double), "8 rows x 16 B per thread and operand fill a stage");

__device__ __forceinline__ void cp_async16(void* smem_ptr, const void* gptr) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_ptr);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gptr));
}
__device__ __forceinline__ unsigned bar_addr(uint64_t* bar) { return (unsigned)__cvta_generic_to_shared(bar); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar_addr(bar)), "r"(count) : "memory");
}
// one arrival once every cp.async this thread has issued so far has landed
__device__ __forceinline__ void mbar_arrive_cp_async(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(bar_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n"
        "WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@!p bra WAIT;\n\t}\n" ::"r"(bar_addr(bar)),
        "r"(parity)
        : "memory");
}

// K chunk kc of the CTA tile: its A rows start at a, lda doubles apart, its B rows at b, ldb apart; the chunk's SK
// columns start at column k of both
struct Operands {
    const double* a; int64_t lda;
    const double* b; int64_t ldb;
    int64_t k;
};

// acc = (the CTA tile's 128 rows of A) (its 128 rows of B)^T over kchunks chunks of SK, for warp (wm, wn) =
// (warp / 4, warp % 4) of the block's 8.  operands(kc) -> Operands gives chunk kc's rows; after_wait(kc) runs once
// stage kc has landed, before the warp's MMAs on it.
//
// Ring: chunk kc lives in slot kc % STAGES.  Every thread issues its copies of a chunk and arrives on the slot's full
// barrier when they land (THREADS arrivals); a warp waits on it before its fragment loads.  After its MMAs on chunk kc a
// warp arrives on the slot's empty barrier (8 arrivals) and then refills the slot of chunk kc - 1 with chunk
// kc + STAGES - 1, once every warp has released it.  The refill follows the MMAs, so its address arithmetic overlaps
// them (MEASURED.md), and a warp blocks there only on a warp a whole stage behind it.
//
// On return every copy has landed, but other warps may still read the last stages: a caller that reuses smem
// synchronises first.
template <class ChunkOperands, class AfterWait>
__device__ __forceinline__ void cta_tile_nt(double (&acc)[WM / 8][WN / 8][2], double* smem, int kchunks,
                                            ChunkOperands operands, AfterWait after_wait) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp >> 2, wn = warp & 3;
    uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(smem) + RING_BYTES);
    uint64_t* empty = full + STAGES;
    // each thread copies 8 rows x 16 B of A and of B per stage
    const int lrow = tid >> 4;         // 0..15  (+16 per i)
    const int lc16 = (tid & 15) * 2;   // double offset of the 16-byte chunk within the 256-byte row
    auto load_stage = [&](int slot, int kc) {
        const Operands o = operands(kc);
        const int64_t koff = o.k + lc16;
        double* as = smem + slot * STAGE_DOUBLES;
        double* bs = as + BM * LDS;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = lrow + i * 16;
            cp_async16(as + r * LDS + lc16, o.a + (int64_t)r * o.lda + koff);
            cp_async16(bs + r * LDS + lc16, o.b + (int64_t)r * o.ldb + koff);
        }
        mbar_arrive_cp_async(full + slot);
    };

#pragma unroll
    for (int mi = 0; mi < WM / 8; ++mi)
#pragma unroll
        for (int ni = 0; ni < WN / 8; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;

    if (tid == 0)
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full + s, THREADS);
            mbar_init(empty + s, THREADS / 32);
        }
    __syncthreads();   // the barriers are initialised before any thread arrives on them

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s)
        if (s < kchunks) load_stage(s, s);
    int slot = 0;
    unsigned phase = 0;   // parity of chunk kc's use of its slot: (kc / STAGES) & 1
    for (int kc = 0; kc < kchunks; ++kc) {
        mbar_wait(full + slot, phase);
        after_wait(kc);
        const double* as = smem + slot * STAGE_DOUBLES + wm * WM * LDS;
        const double* bs = smem + slot * STAGE_DOUBLES + BM * LDS + wn * WN * LDS;
#pragma unroll
        for (int k0 = 0; k0 < SK; k0 += BK) warp_tile_stage(acc, as + k0, bs + k0, lane);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + slot);
        const int nk = kc + STAGES - 1;
        if (nk < kchunks) {
            // chunk kc - 1's slot; its empty phase has chunk kc - 1's parity (none to wait for at kc = 0)
            const int prev = slot == 0 ? STAGES - 1 : slot - 1;
            if (kc > 0) mbar_wait(empty + prev, slot == 0 ? phase ^ 1 : phase);
            load_stage(prev, nk);
        }
        if (++slot == STAGES) {
            slot = 0;
            phase ^= 1;
        }
    }
}
}  // namespace dmma
