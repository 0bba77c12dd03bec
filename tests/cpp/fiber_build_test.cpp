// fiber_build_test.cpp -- C++ host test of the device build of the per-fiber operators through skelly_b200/flow.hpp:
// build, read back, upload the read-back operators again (set_fiber_operators + set_fiber_preconditioner), and check
// that the matvec and the preconditioner give bitwise the same results on both, and that xs_ is x_ D_1_0 scaled by
// 2 / length_prev (ffd.cpp:62-68).  The class matrices are random: this tests the mirror, not the numbers.
#include <skelly_b200/flow.hpp>

#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

using skelly_b200::Matrix;

int main() {
    const int n_fibers = 6, n = 16, nf = n_fibers * n, n4 = 4 * n, bc = n4 - 14;
    std::mt19937_64 gen(7);
    std::uniform_real_distribution<double> U(-1.0, 1.0);
    Matrix r_fib(3, nf), D1(n, n), D2(n, n), D3(n, n), D4(n, n), P(bc, n4), x(4 * nf, 1), link(7, n_fibers), empty;
    for (int f = 0; f < n_fibers; ++f)
        for (int i = 0; i < n; ++i) {
            const double s = i / (n - 1.0);
            r_fib(0, f * n + i) = 3.0 * f + s;
            r_fib(1, f * n + i) = 0.3 * std::sin(2.0 * s + f);
            r_fib(2, f * n + i) = 0.2 * std::cos(3.0 * s);
        }
    for (Matrix *m : {&D1, &D2, &D3, &D4})
        for (long i = 0; i < m->size(); ++i)
            m->data()[i] = U(gen);
    for (int r = 0; r < bc; ++r) { // block diagonal like P_downsample_bc (ffd.cpp:551-555)
        const int blk = std::min(r / (n - 4), 3);
        for (int c = blk * n; c < (blk + 1) * n; ++c)
            P(r, c) = U(gen) / n;
    }
    for (long i = 0; i < x.size(); ++i) x.data()[i] = U(gen);
    for (long i = 0; i < link.size(); ++i) link.data()[i] = U(gen);
    std::vector<skb_fiber_params> prm(n_fibers);
    for (int f = 0; f < n_fibers; ++f)
        prm[f] = skb_fiber_params{1.0 + 0.01 * f, 2.5e-3, 0.0125, 500.0, 1.0, f % 2, (f / 2) % 2};
    try {
        skelly_b200::FlowEngine eng(0);
        eng.set_fibers(r_fib, std::vector<int>(n_fibers, n), std::vector<double>(n_fibers, 1.0));
        eng.set_periphery(empty, empty);
        eng.set_bodies(empty, empty, empty);
        eng.set_fiber_class(n, D1, P);
        eng.set_fiber_class_derivatives(n, D2, D3, D4);
        eng.build_fiber_operators(prm, 1e-2, 1.0);
        std::vector<double> A, F, Ai;
        Matrix xs, v_s, v_b;
        eng.get_fiber_operators(A, F, xs, Ai);
        Matrix res = eng.apply_matvec(x, empty, empty, empty, link, 1.0, v_s, v_b);
        Matrix y = eng.apply_fiber_preconditioner(x);

        double e_xs = 0, m_xs = 0;
        for (int f = 0; f < n_fibers; ++f)
            for (int i = 0; i < n; ++i)
                for (int k = 0; k < 3; ++k) {
                    double s = 0;
                    for (int j = 0; j < n; ++j)
                        s += r_fib(k, f * n + j) * D1(j, i);
                    s *= 2.0 / prm[f].length_prev;
                    e_xs = std::fmax(e_xs, std::fabs(s - xs(k, f * n + i)));
                    m_xs = std::fmax(m_xs, std::fabs(s));
                }

        std::vector<const double *> Ap, Fp, Aip;
        std::vector<double> lprev;
        std::vector<int> plus;
        for (int f = 0; f < n_fibers; ++f) {
            Ap.push_back(A.data() + (size_t)16 * n * n * f);
            Fp.push_back(F.data() + (size_t)12 * n * n * f);
            Aip.push_back(Ai.data() + (size_t)16 * n * n * f);
            lprev.push_back(prm[f].length_prev);
            plus.push_back(prm[f].plus_hinged);
        }
        eng.set_fiber_operators(Ap, Fp, xs, lprev, plus);
        eng.set_fiber_preconditioner(Aip);
        Matrix res2 = eng.apply_matvec(x, empty, empty, empty, link, 1.0, v_s, v_b);
        Matrix y2 = eng.apply_fiber_preconditioner(x);
        bool same = true;
        for (long i = 0; i < res.size(); ++i)
            same = same && res.data()[i] == res2.data()[i] && y.data()[i] == y2.data()[i];
        printf("fiber_build_test: xs rel err %.3e (gate 1e-13), matvec / preconditioner after the round trip %s\n",
               e_xs / m_xs, same ? "bitwise identical" : "DIFFER");
        return (e_xs / m_xs > 1e-13 || !same) ? 1 : 0;
    } catch (const std::exception &e) {
        fprintf(stderr, "%s\n", e.what());
        return 3;
    }
}
