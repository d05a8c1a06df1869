// The fp64 tensor-core (DMMA) warp tile shared by every fp64 GEMM mainloop: dense.cu's gemm_nt_kernel (trailing and
// panel updates) and grad.cu's tri_gemm_kernel (triangular inverse and the W contraction).
//
// Shape: mma.sync.m16n8k16.f64, Hopper's widest fp64 MMA (one DMMA.16x8x16 instruction).  On sm_90 the m16n8 shapes
// issue at a higher fp64 rate than Ampere's m8n8k4; MEASURED.md records the rates of all four shapes.
//
// Operands come from one shared-memory pipeline stage: BK = 16 doubles of K per row, rows K-contiguous (both operands
// of an NT product, C = A B^T), row stride LDS = 20 doubles.  The padding 16 -> 20 makes the fragment loads of a
// half-warp (rows g = 0..3, k offsets t = 0..3) hit 16 distinct 8-byte bank pairs (row stride 40 words = 8 mod 32).
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

namespace dmma {
constexpr int MK = 16;                  // K of one mma instruction
constexpr int BK = 16, LDS = 20;        // stage depth and padded row stride (doubles)
constexpr int WM = 64, WN = 32;         // warp tile
constexpr int AM = WM / 16, AN = WN / 8;
constexpr int AREG = MK / 2, BREG = MK / 4;
static_assert(BK % MK == 0, "a stage holds whole mma K steps");

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

// acc += (the warp's 64 rows of A) (its 32 rows of B)^T over one stage of BK
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
}  // namespace dmma
