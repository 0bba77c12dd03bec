// fiber_rhs_test.cpp -- C++ host test of the fiber RHS through skelly_b200/flow.hpp: the mirror returns bitwise what
// the C ABI returns, with and without the optional inputs, and its layout puts the boundary entries where
// apply_bc_rectangular does: a clamped minus end has x_0 / dt in rows 4n-14 .. 4n-12, a free plus end f_external of
// node n-1 in rows 4n-7 .. 4n-5 (fiber_finite_difference.cpp:377, 485).  The class matrices are random: this tests
// the mirror, not the numbers.
#include <skelly_b200/flow.hpp>

#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

using skelly_b200::Matrix;

int main() {
    const int n_fibers = 6, n = 16, nf = n_fibers * n, n4 = 4 * n, bc = n4 - 14;
    const double dt = 1e-2, eta = 1.0;
    std::mt19937_64 gen(11);
    std::uniform_real_distribution<double> U(-1.0, 1.0);
    Matrix r_fib(3, nf), D1(n, n), D2(n, n), D3(n, n), D4(n, n), P(bc, n4), v(3, nf), f(3, nf), empty;
    for (int fb = 0; fb < n_fibers; ++fb)
        for (int i = 0; i < n; ++i) {
            const double s = i / (n - 1.0);
            r_fib(0, fb * n + i) = 3.0 * fb + s;
            r_fib(1, fb * n + i) = 0.3 * std::sin(2.0 * s + fb);
            r_fib(2, fb * n + i) = 0.2 * std::cos(3.0 * s);
        }
    for (Matrix *m : {&D1, &D2, &D3, &D4, &v, &f})
        for (long i = 0; i < m->size(); ++i)
            m->data()[i] = U(gen);
    for (int r = 0; r < bc; ++r) { // block diagonal like P_downsample_bc (ffd.cpp:551-555)
        const int blk = std::min(r / (n - 4), 3);
        for (int c = blk * n; c < (blk + 1) * n; ++c)
            P(r, c) = U(gen) / n;
    }
    std::vector<skb_fiber_params> prm(n_fibers);
    std::vector<double> vg(n_fibers), fs(n_fibers), none;
    for (int fb = 0; fb < n_fibers; ++fb) {
        prm[fb] = skb_fiber_params{1.0 + 0.01 * fb, 2.5e-3, 0.0125, 500.0, 1.0, fb % 2, (fb / 2) % 2};
        vg[fb] = 0.1 * fb;
        fs[fb] = 0.5 - 0.2 * fb;
    }
    try {
        skelly_b200::FlowEngine eng(0);
        eng.set_fibers(r_fib, std::vector<int>(n_fibers, n), std::vector<double>(n_fibers, 1.0));
        eng.set_periphery(empty, empty);
        eng.set_bodies(empty, empty, empty);
        eng.set_fiber_class(n, D1, P);
        eng.set_fiber_class_derivatives(n, D2, D3, D4);
        bool same = true, layout = true;
        for (int full = 0; full < 2; ++full) {
            Matrix rhs = full ? eng.build_fiber_rhs(prm, vg, fs, v, f, dt, eta)
                              : eng.build_fiber_rhs(prm, none, none, empty, empty, dt, eta);
            Matrix ref(4 * nf, 1);
            if (skb_flow_build_fiber_rhs(eng.handle(), prm.data(), full ? vg.data() : nullptr,
                                         full ? fs.data() : nullptr, full ? v.data() : nullptr,
                                         full ? f.data() : nullptr, dt, eta, ref.data()) != SKB_OK)
                throw std::runtime_error(skb_last_error_string());
            for (long i = 0; i < rhs.size(); ++i)
                same = same && rhs.data()[i] == ref.data()[i];
            for (int fb = 0; fb < n_fibers; ++fb) {
                const double *r = rhs.data() + (size_t)fb * n4;
                for (int k = 0; k < 3; ++k) {
                    if (prm[fb].minus_clamped)
                        layout = layout && r[bc + k] == r_fib(k, fb * n) / dt;
                    if (!prm[fb].plus_hinged)
                        layout = layout && r[bc + 7 + k] == (full ? f(k, fb * n + n - 1) : 0.0);
                }
            }
        }
        printf("fiber_rhs_test: mirror vs C ABI %s, boundary entries %s\n", same ? "bitwise identical" : "DIFFER",
               layout ? "in place" : "MISPLACED");
        return same && layout ? 0 : 1;
    } catch (const std::exception &e) {
        fprintf(stderr, "%s\n", e.what());
        return 3;
    }
}
