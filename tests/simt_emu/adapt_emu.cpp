// adapt_emu.cpp -- the adaptor-statistics kernels K5 / K5b (advancedhmc.jl_b200/csrc/ahmc_adapt.cu, unmodified) under the
// CPU SIMT emulator (block barriers, static shared variables, the last-block reduction).  TEST INFRASTRUCTURE ONLY.
#define AHMC_SIMT_EMULATION 1
#define __shared__ static  // this file's kernels use static shared variables only; blocks run one at a time
#include <cstdlib>
#include <cstdio>
#include <vector>

#include "ahmc_adapt.cu"
#include "emu_harness.h"

using namespace ahmc;

struct SumArgs {
    int D;
    long long N;
    const double* theta;
    long long ld;
    const double* alpha;
    double* partial;
    unsigned* counter;
    double* out;
};
template <int PASS>
static void sum_thunk(const void* p) {
    const SumArgs& a = *static_cast<const SumArgs*>(p);
    adapt_kernel<PASS>(a.D, a.N, a.theta, a.ld, a.alpha, a.partial, a.counter, a.out);
}
struct CovArgs {
    int D;
    long long N;
    const double* theta;
    long long ld;
    const double* mean;
    double* out;
};
static void cov_thunk(const void* p) {
    const CovArgs& a = *static_cast<const CovArgs*>(p);
    adapt_cov_kernel(a.D, a.N, a.theta, a.ld, a.mean, a.out);
}

extern "C" int emu_adapt(int D, long long N, const double* theta, const double* alpha, double* rec /* 2+2D */, double* cov /* D*D */) {
    const int blocks = (int)(N < 5 ? N : 5);
    std::vector<double> partial((size_t)blocks * (D + 1), 0.0);
    unsigned counter = 0;
    SumArgs s{D, N, theta, D, alpha, partial.data(), &counter, rec};
    emu_launch(sum_thunk<0>, &s, blocks, kAdaptThreads);
    emu_launch(sum_thunk<1>, &s, blocks, kAdaptThreads);
    const int T = (D + kCovTile - 1) / kCovTile;
    CovArgs c{D, N, theta, D, rec + 2, cov};
    emu_launch(cov_thunk, &c, T * (T + 1) / 2, 256);
    return 0;
}

#ifdef RACE_ADAPT
int main() {
    const int D = 37;
    const long long N = 300;
    std::vector<double> theta((size_t)N * D), alpha(N), rec(2 + 2 * D), cov((size_t)D * D);
    srand(2);
    for (auto& x : theta) x = rand() / (double)RAND_MAX - 0.5;
    for (auto& x : alpha) x = rand() / (double)RAND_MAX;
    const int rc = emu_adapt(D, N, theta.data(), alpha.data(), rec.data(), cov.data());
    std::printf("adapt D %d N %lld: rc %d n %.0f\n", D, N, rc, rec[0]);
    return rc != 0 || rec[0] != (double)N;
}
#endif
