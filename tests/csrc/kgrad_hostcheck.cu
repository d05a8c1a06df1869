// TEST INFRASTRUCTURE: the kernel-program derivatives of the dense gradient (tinygp_b200/csrc/kgrad.cuh: kgrad_prepare +
// kgrad_eval, what the contraction epilogue of grad.cu inlines) compiled for the CPU, so `-m "not gpu"` tests can check
// the SAME source against finite differences of kprog_eval and the oracle's closed forms.
// Built on demand by tests/test_grad_device_code_on_host.py; never linked into libb200gp.so.
#include "../../tinygp_b200/csrc/kgrad.cuh"

extern "C" {

// k(x1, x2) for each pair (X1_i, X2_i) and dk[i * nslot_max + s]; *nslot = the program's slot count.  mode: 0 = the
// normal form when the program has one, 1 = always the interpreter.  *is_fast reports whether the normal form ran.
// Returns 0, 3 (refused by kgrad_prepare) or 2 (parse error, message in err).
int hostcheck_kgrad(const double* prog, int n_rows, const double* X1, const double* X2, int64_t npair, int ndim, int mode,
                    double* k, double* dk, int* nslot, int* is_fast, char* err) {
    try {
        const KProg P = parse_prog_impl(prog, n_rows, ndim);
        KGrad G;
        if (!kgrad_prepare(P, G)) return 3;
        *nslot = G.nslot;
        *is_fast = (G.fast && mode == 0) ? 1 : 0;
        for (int64_t i = 0; i < npair; ++i) {
            const double* xa = X1 + i * ndim;
            const double* xb = X2 + i * ndim;
            k[i] = kgrad_eval(P, G, ndim, [&](int d) { return xa[d] - xb[d]; }, dk + i * KGRAD_MAX_SLOTS, mode == 0);
        }
        return 0;
    } catch (const std::exception& e) {
        snprintf(err, 256, "%s", e.what());
        return 2;
    }
}

// k(x1, x2) by the plain interpreter (kprog_eval), for finite differences
int hostcheck_keval(const double* prog, int n_rows, const double* X1, const double* X2, int64_t npair, int ndim, double* k) {
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

int hostcheck_kgrad_max_slots() { return KGRAD_MAX_SLOTS; }

}  // extern "C"
