// Executes the solve kernels of csrc/dks_wide.cuh on host threads (emu_shim.h) and compares them with a plain float64
// reference: y = ln(sum p1 / sum p0) - link(fnull) (or the identity link), beta = y P^T (bit for bit: the kernel's
// summation order is an ascending fma chain over the coalitions), phi = beta - delta d with the remainder in the last
// group, both classes.  Shapes chosen to hit every boundary of the tiling: an instance list that is a shuffled subset
// (count < n), a partial last tile of 128 instances, M - 1 not a multiple of 64, S not a multiple of 32, more instances
// than finish CTAs.  Prints the largest deviations; exit code 0 iff all are within tolerance.
#define DKS_HOST_EMULATION 1
#include "dks_wide.cuh"

#include <algorithm>
#include <cstdio>
#include <random>

using namespace dks;
using namespace dks::wide;

static int run_case(int n, int cnt, int G, int S, int N, int link, int sm_count, unsigned seed) {
    std::mt19937_64 rng(seed);
    std::uniform_real_distribution<double> U(0.0, 1.0);
    std::normal_distribution<double> Nrm(0.0, 1.0);
    const int C = 2, nA = G - 1, KP = kpad(G), S_pad = (S + 31) / 32 * 32;
    std::vector<float2> sums((size_t)n * S_pad);
    for (auto& v : sums) {                       // poison everything, then fill the valid cells
        v.x = std::nanf(""); v.y = std::nanf("");
    }
    for (int i = 0; i < n; ++i)
        for (int s = 0; s < S; ++s) {
            const double p1 = std::exp(-8.0 * U(rng)) * N;        // sum of N sigmoids, possibly tiny
            sums[(size_t)i * S_pad + s] = make_float2((float)p1, (float)(N - p1));
        }
    std::vector<double> PT((size_t)S_pad * KP, 0.0), dvec(KP, 0.0), dlink((size_t)n * C), y((size_t)n * S_pad, std::nan("")),
        beta((size_t)n * KP, std::nan("")), phi((size_t)C * n * G, std::nan(""));
    for (int s = 0; s < S; ++s)
        for (int k = 0; k < nA; ++k) PT[(size_t)s * KP + k] = Nrm(rng) * 1e-2;
    for (int k = 0; k < nA; ++k) dvec[k] = Nrm(rng) * 0.1;
    for (auto& v : dlink) v = Nrm(rng) * 3.0;
    const double fnull[2] = {0.37, 0.63};
    const double linkfnull[2] = {link == DKS_LINK_LOGIT ? std::log(0.37 / 0.63) : 0.37,
                                 link == DKS_LINK_LOGIT ? std::log(0.63 / 0.37) : 0.63};
    std::vector<int> list(n);
    for (int i = 0; i < n; ++i) list[i] = i;
    std::shuffle(list.begin(), list.end(), rng);

    WideParams p{};
    p.n = n; p.N = N; p.G = G; p.C = C; p.S = S; p.S_pad = S_pad; p.KP = KP; p.link = link;
    p.sums = sums.data(); p.PT = PT.data(); p.dvec = dvec.data(); p.dlink = dlink.data(); p.linkfnull = linkfnull;
    p.fnull = fnull; p.list = list.data(); p.count = &cnt; p.y = y.data(); p.beta = beta.data(); p.phi = phi.data();

    emu::launch(link_grid(S_pad, n, sm_count), dim3(256), wide_link_kernel, p);
    emu::launch(beta2_grid(KP, n), dim3(THREADS), wide_beta2_kernel, p);
    emu::launch(dim3(finish_grid(n, sm_count)), dim3(256), wide_finish_kernel, p);

    double ey = 0, ep = 0, esum = 0;
    int bad = 0, beta_mismatch = 0;
    std::vector<char> listed(n, 0);
    for (int m = 0; m < cnt; ++m) listed[list[m]] = 1;
    for (int i = 0; i < n; ++i) {
        if (!listed[i]) {                        // rows off the list must be untouched
            for (int k = 0; k < G; ++k)
                if (!std::isnan(phi[(size_t)i * G + k]) || !std::isnan(phi[(size_t)n * G + (size_t)i * G + k])) ++bad;
            for (int k = 0; k < KP; ++k)
                if (!std::isnan(beta[(size_t)i * KP + k])) ++bad;
            continue;
        }
        std::vector<double> yr(S_pad, 0.0);
        for (int s = 0; s < S; ++s) {
            const float2 a = sums[(size_t)i * S_pad + s];
            yr[s] = link == DKS_LINK_LOGIT ? std::log((double)a.x) - std::log((double)a.y) - linkfnull[1]
                                           : (double)a.x / N - fnull[1];
        }
        for (int s = 0; s < S_pad; ++s) ey = std::max(ey, std::fabs(yr[s] - y[(size_t)i * S_pad + s]));
        const double delta = dlink[(size_t)i * C + 1];
        double sum = 0.0;
        std::vector<double> want(G);
        for (int k = 0; k < KP; ++k) {           // padding coefficients included: zero columns of PT give zeros
            double b = 0.0;
            for (int s = 0; s < S_pad; ++s) b = std::fma(y[(size_t)i * S_pad + s], PT[(size_t)s * KP + k], b);   // kernel's y: isolates the product
            if (std::memcmp(&b, &beta[(size_t)i * KP + k], sizeof(double)) != 0) ++beta_mismatch;
            if (k >= nA) continue;
            want[k] = beta[(size_t)i * KP + k] - delta * dvec[k];
            sum += want[k];
        }
        want[nA] = delta - sum;
        double got_sum = 0.0;
        for (int k = 0; k < G; ++k) {
            double w = std::fabs(want[k]) < 1e-10 ? 0.0 : want[k];
            const double g1 = phi[(size_t)n * G + (size_t)i * G + k], g0 = phi[(size_t)i * G + k];
            ep = std::max(ep, std::fabs(g1 - w));
            if (g0 != -g1 && !(g0 == 0.0 && g1 == 0.0)) ++bad;
            got_sum += g1;
        }
        esum = std::max(esum, std::fabs(got_sum - delta));
    }
    std::printf("n=%d cnt=%d G=%d S=%d N=%d link=%d: |y-ref| %.2e  beta bits differ %d  |phi-ref| %.2e  |sum phi - delta| %.2e  "
                "bad %d\n", n, cnt, G, S, N, link, ey, beta_mismatch, ep, esum, bad);
    // y: the table log is good to ~2e-9 absolute; the finish step is float64 (association order may differ slightly)
    return (ey < 1e-8 && beta_mismatch == 0 && ep < 1e-11 && esum < 1e-9 && bad == 0) ? 0 : 1;
}

int main() {
    int rc = 0;
    rc |= run_case(150, 131, 200, 150, 40, DKS_LINK_LOGIT, 2, 1);       // 2 tiles of instances (last partial), KP = 256, S_pad = 160
    rc |= run_case(70, 70, 130, 97, 256, DKS_LINK_IDENTITY, 1, 2);      // KP = 192; more instances than finish CTAs (8)
    rc |= run_case(5, 3, 1024, 64, 16, DKS_LINK_LOGIT, 148, 3);         // the configs[3] width: KP = 1024
    rc |= run_case(64, 64, 129, 33, 100, DKS_LINK_LOGIT, 1, 4);         // one half-filled tile; smallest wide M
    rc |= run_case(300, 257, 193, 70, 30, DKS_LINK_LOGIT, 3, 5);        // three 128-instance tiles (last with one row), M - 1 = 192
    std::printf(rc ? "FAILED\n" : "OK\n");
    return rc;
}
