// TEST INFRASTRUCTURE: the DMMA warp tile of tinygp_b200/csrc/dmma.cuh (fragment loads, fragment coordinate maps and
// the accumulator map the epilogues use) run for one warp on the CPU.  Each mma atom is emulated from the 32 lanes'
// fragment registers through the coordinate maps, so an index slip in a load, a map or the epilogue shows up as a wrong
// product.  Whether the maps are the hardware's is checked on the GPU (tests/test_dmma_update_gpu.py).
// Built on demand by tests/test_dmma_fragments_on_host.py; never linked into libb200gp.so.
#include "../../tinygp_b200/csrc/dmma.cuh"
#include <cmath>
#include <vector>

using namespace dmma;

extern "C" {

// C (WM x WN, row-major) = A (WM x K) B (WN x K)^T, both row-major, K a multiple of BK, through the warp tile.
// Returns 0, or 1 if an atom element is not covered exactly once by the lanes' fragments, 2 if a fragment load read
// the row padding, 3 if the accumulator map does not write every C element exactly once.
int hostcheck_dmma_warp_tile(const double* A, const double* B, int K, double* C) {
    static double acc[32][WM / 8][WN / 8][2];
    for (int l = 0; l < 32; ++l)
        for (int m = 0; m < WM / 8; ++m)
            for (int n = 0; n < WN / 8; ++n) acc[l][m][n][0] = acc[l][m][n][1] = 0.0;
    std::vector<double> as(WM * LDS), bs(WN * LDS);
    for (int s = 0; s < K / BK; ++s) {
        // one shared-memory stage; the padding holds NaN so that reading it poisons the product
        for (int r = 0; r < WM; ++r)
            for (int c = 0; c < LDS; ++c) as[r * LDS + c] = c < BK ? A[r * K + s * BK + c] : NAN;
        for (int r = 0; r < WN; ++r)
            for (int c = 0; c < LDS; ++c) bs[r * LDS + c] = c < BK ? B[r * K + s * BK + c] : NAN;
        for (int k0 = 0; k0 < BK; k0 += MK) {
            double a[32][AM][AREG], b[32][AN][BREG];
            for (int l = 0; l < 32; ++l) {
                for (int mi = 0; mi < AM; ++mi) load_a(a[l][mi], as.data(), l, mi, k0);
                for (int ni = 0; ni < AN; ++ni) load_b(b[l][ni], bs.data(), l, ni, k0);
            }
            for (int mi = 0; mi < AM; ++mi)
                for (int ni = 0; ni < AN; ++ni) {
                    double At[16][MK], Bt[MK][8];
                    int na[16][MK] = {}, nb[MK][8] = {};
                    for (int l = 0; l < 32; ++l) {
                        for (int i = 0; i < AREG; ++i) {
                            At[a_row(l, i)][a_k(l, i)] = a[l][mi][i];
                            na[a_row(l, i)][a_k(l, i)]++;
                        }
                        for (int i = 0; i < BREG; ++i) {
                            Bt[b_k(l, i)][b_col(l)] = b[l][ni][i];
                            nb[b_k(l, i)][b_col(l)]++;
                        }
                    }
                    for (int r = 0; r < 16; ++r)
                        for (int k = 0; k < MK; ++k) {
                            if (na[r][k] != 1) return 1;
                            if (std::isnan(At[r][k])) return 2;
                        }
                    for (int k = 0; k < MK; ++k)
                        for (int c = 0; c < 8; ++c) {
                            if (nb[k][c] != 1) return 1;
                            if (std::isnan(Bt[k][c])) return 2;
                        }
                    // D += At Bt, scattered to the lanes' accumulators: c0, c1 -> acc[2 mi], c2, c3 -> acc[2 mi + 1]
                    for (int l = 0; l < 32; ++l)
                        for (int i = 0; i < 4; ++i) {
                            double d = 0.0;
                            for (int k = 0; k < MK; ++k) d += At[c_row(l, i)][k] * Bt[k][c_col(l, i)];
                            acc[l][2 * mi + (i >> 1)][ni][i & 1] += d;
                        }
                }
        }
    }
    std::vector<int> hits(WM * WN, 0);
    for (int l = 0; l < 32; ++l)
        for (int m = 0; m < WM / 8; ++m)
            for (int n = 0; n < WN / 8; ++n)
                for (int q = 0; q < 2; ++q) {
                    const int e = acc_row(l, m) * WN + acc_col(l, n, q);
                    C[e] = acc[l][m][n][q];
                    hits[e]++;
                }
    for (int e = 0; e < WM * WN; ++e)
        if (hits[e] != 1) return 3;
    return 0;
}

}  // extern "C"
