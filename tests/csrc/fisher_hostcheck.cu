// TEST INFRASTRUCTURE: the per-element code of the Fisher information's derivative build (tinygp_b200/csrc/kgrad.cuh:
// kgrad_element, what grad.cu's dk_build_kernel runs for every element of the np x np work buffer) compiled for the CPU,
// so `-m "not gpu"` tests can check the SAME source against the oracle's complex-step dK / d theta.
// Built on demand by tests/test_fisher_device_code_on_host.py; never linked into libb200gp.so.
#include "../../tinygp_b200/csrc/kgrad.cuh"

extern "C" {

// D (np x np, row-major) = kgrad_element(..., slot) for every element; *nslot = the program's slot count.  Returns 0,
// 3 (refused by kgrad_prepare) or 2 (parse error, message in err).
int hostcheck_dk_build(const double* prog, int n_rows, const double* X, int64_t n, int64_t np, int ndim, int slot,
                       double* D, int* nslot, char* err) {
    try {
        const KProg P = parse_prog_impl(prog, n_rows, ndim);
        KGrad G;
        if (!kgrad_prepare(P, G)) return 3;
        *nslot = G.nslot;
        for (int64_t i = 0; i < np; ++i)
            for (int64_t j = 0; j < np; ++j) D[i * np + j] = kgrad_element(P, G, ndim, X, n, i, j, slot);
        return 0;
    } catch (const std::exception& e) {
        snprintf(err, 256, "%s", e.what());
        return 2;
    }
}

}  // extern "C"
