// TEST INFRASTRUCTURE: the second derivatives of a kernel program (tinygp_b200/csrc/kgrad.cuh: khess_eval, what the
// Hessian's second-derivative contraction in grad.cu runs for every element of a W tile) compiled for the CPU, so
// `-m "not gpu"` tests can check the SAME source against central differences of kgrad_eval and the oracle.
// Built on demand by tests/test_hessian_device_code_on_host.py; never linked into libb200gp.so.
#include "../../tinygp_b200/csrc/kgrad.cuh"

extern "C" {

// h[e * npair + q] = d^2 k / d slot pa[q] d slot pb[q] at the point pair (X1_e, X2_e), npair <= KHESS_PAIRS; *nslot =
// the program's slot count.  Returns 0, 3 (refused by kgrad_prepare), 4 (npair out of range) or 2 (parse error).
int hostcheck_khess(const double* prog, int n_rows, const double* X1, const double* X2, int64_t ne, int ndim,
                    const int* pa, const int* pb, int npair, double* h, int* nslot, char* err) {
    try {
        const KProg P = parse_prog_impl(prog, n_rows, ndim);
        KGrad G;
        if (!kgrad_prepare(P, G)) return 3;
        *nslot = G.nslot;
        if (npair < 1 || npair > KHESS_PAIRS) return 4;
        for (int64_t e = 0; e < ne; ++e) {
            const double* xa = X1 + e * ndim;
            const double* xb = X2 + e * ndim;
            khess_eval(P, G, ndim, [&](int d) { return xa[d] - xb[d]; }, pa, pb, npair, h + e * npair);
        }
        return 0;
    } catch (const std::exception& e) {
        snprintf(err, 256, "%s", e.what());
        return 2;
    }
}

// dk[e * KGRAD_MAX_SLOTS + s] = kgrad_eval at (X1_e, X2_e); mode 0: the normal form where the program has one, 1: the
// interpreter.  For the central differences.
int hostcheck_kgrad1(const double* prog, int n_rows, const double* X1, const double* X2, int64_t ne, int ndim, int mode,
                     double* dk) {
    try {
        const KProg P = parse_prog_impl(prog, n_rows, ndim);
        KGrad G;
        if (!kgrad_prepare(P, G)) return 3;
        for (int64_t e = 0; e < ne; ++e) {
            const double* xa = X1 + e * ndim;
            const double* xb = X2 + e * ndim;
            kgrad_eval(P, G, ndim, [&](int d) { return xa[d] - xb[d]; }, dk + e * KGRAD_MAX_SLOTS, mode == 0);
        }
        return 0;
    } catch (const std::exception&) { return 2; }
}

}  // extern "C"
