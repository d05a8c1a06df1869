// TEST INFRASTRUCTURE: the coordinate derivatives of kgrad.cuh (kgrad_eval<true>, what the contraction epilogue of
// b200gp_dense_log_probability_grad_x inlines) compiled for the CPU, so `-m "not gpu"` tests can check the SAME source
// against central differences of kprog_eval.  Built on demand by tests/test_grad_x_device_code_on_host.py; never
// linked into libb200gp.so.
#include "../../tinygp_b200/csrc/kgrad.cuh"

extern "C" {

// for each pair (X1_i, X2_i): k[i], gx[i * KGRAD_MAX_DIM + d] = d k / d (x1 - x2)_d, and same_dk[i] = 1 if the slot
// derivatives of kgrad_eval<true> are bitwise equal to kgrad_eval<false>'s.  mode: 0 = the normal form when the program
// has one, 1 = always the interpreter; *is_fast reports whether the normal form ran.  Returns 0, 3 (refused by
// kgrad_prepare) or 2 (parse error, message in err).
int hostcheck_kgrad_x(const double* prog, int n_rows, const double* X1, const double* X2, int64_t npair, int ndim,
                      int mode, double* k, double* gx, int* same_dk, int* is_fast, char* err) {
    try {
        const KProg P = parse_prog_impl(prog, n_rows, ndim);
        KGrad G;
        if (!kgrad_prepare(P, G)) return 3;
        *is_fast = (G.fast && mode == 0) ? 1 : 0;
        for (int64_t i = 0; i < npair; ++i) {
            const double* xa = X1 + i * ndim;
            const double* xb = X2 + i * ndim;
            auto diff = [&](int d) { return xa[d] - xb[d]; };
            double dk0[KGRAD_MAX_SLOTS] = {}, dk1[KGRAD_MAX_SLOTS] = {};
            const double k0 = kgrad_eval(P, G, ndim, diff, dk0, mode == 0);
            k[i] = kgrad_eval<true>(P, G, ndim, diff, dk1, mode == 0, gx + i * KGRAD_MAX_DIM);
            same_dk[i] = (k0 == k[i]) ? 1 : 0;
            for (int s = 0; s < G.nslot; ++s)
                if (!(dk0[s] == dk1[s])) same_dk[i] = 0;
        }
        return 0;
    } catch (const std::exception& e) {
        snprintf(err, 256, "%s", e.what());
        return 2;
    }
}

// k(x1, x2) by the plain interpreter (kprog_eval), for finite differences
int hostcheck_keval_x(const double* prog, int n_rows, const double* X1, const double* X2, int64_t npair, int ndim,
                      double* k) {
    try {
        const KProg P = parse_prog_impl(prog, n_rows, ndim);
        for (int64_t i = 0; i < npair; ++i) {
            const double* xa = X1 + i * ndim;
            const double* xb = X2 + i * ndim;
            k[i] = kprog_eval(P, ndim, [&](int d) { return xa[d] - xb[d]; });
        }
        return 0;
    } catch (const std::exception&) { return 2; }
}

int hostcheck_kgrad_max_dim() { return KGRAD_MAX_DIM; }

}  // extern "C"
