// dense_adapt_emu.cpp -- runs the WelfordCov form of the per-chain adaptor (ahmc_chain_adapt.cuh) under the CPU SIMT
// emulator: the adaptive NUTS kernel (ahmc_nuts_kernel.cuh) and the adaptive static-HMC kernel (ahmc_leapfrog.cu) on a
// diagonal Gaussian with a per-chain Dense metric and the Philox streams, and the window-end estimate + Cholesky
// factorisation on its own, on a workspace the caller fills.  The sources are included unmodified (their host launch code is
// skipped with AHMC_SIMT_EMULATION).  Built with -DDENSE_ADAPT_RACE it is a ThreadSanitizer program of its own (see
// race_main.cpp for the method).  TEST INFRASTRUCTURE ONLY (tests/test_dense_adapt_cpu.py).
#define AHMC_SIMT_EMULATION 1
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "ahmc_nuts_kernel.cuh"
#include "ahmc_leapfrog.cu"

namespace ahmc {
double smem[1 << 16];  // the block's dynamic shared memory
}
void emu_launch(void (*kernel)(const void*), const void* args, int blocks, int threads);

using namespace ahmc;

struct EmuDenseAdapt {
    int32_t hmc;  // 0: adaptive NUTS (max_depth), 1: adaptive static HMC (n_steps)
    int32_t D;
    int64_t N;
    const double *mu, *w;          // target mean, 1/s^2
    const double *Minv0, *cholU0;  // starting per-chain Dense metric: N x (D x D) column-major each (stride D*D)
    double eps0;
    int32_t max_depth, n_steps;
    uint64_t seed;
    int32_t T, n_adapts, init_buffer, term_buffer, window_size, adapt_metric, n_min;
    const double *th_in, *g_in, *lp_in;  // N x D, N x D (-grad lp), N
    double *th_out, *r_out, *g_out, *lp_out, *lk_out;
    double *draws, *acc, *eps_trace;  // T x N x D, T x N, T x N
    int32_t* n_steps_out;             // T x N
    double *eps_rw, *minv_rw, *cholu_rw;  // N, N x D x D, N x D x D
    double* workspace;                // out: N x (D + D*D), the estimator state (mean, M) after the launch
};

template <int G, int E>
static void nuts_thunk(const void* p) {
    const NutsArgs& a = *static_cast<const NutsArgs*>(p);
    if (G == 32 && E >= 2 && E <= 8 && a.D == G * E)
        nuts_kernel<AHMC_MODEL_DIAG_GAUSS, kMetricDenseChain, G, E, false, AHMC_ADAPT_WELFORD_COV, true>(a);
    else nuts_kernel<AHMC_MODEL_DIAG_GAUSS, kMetricDenseChain, G, E, false, AHMC_ADAPT_WELFORD_COV, false>(a);
}
template <int G, int E>
static void hmc_thunk(const void* p) {
    hmc_kernel<AHMC_MODEL_DIAG_GAUSS, kMetricDenseChain, G, E, AHMC_ADAPT_WELFORD_COV>(*static_cast<const HmcArgs*>(p));
}
typedef void (*KernelFn)(const void*);

extern "C" int emu_dense_adapt(const EmuDenseAdapt* q) {
    int G, E;
    const int D = q->D;
    if (!pick_layout(D, &G, &E) || (G == 32 && E > 2)) return -1;
    KernelFn fn = nullptr;
#define AHMC_EMU_PICK(g, e) \
    if (G == g && E == e) fn = q->hmc ? hmc_thunk<g, e> : nuts_thunk<g, e>;
    AHMC_EMU_PICK(4, 1) AHMC_EMU_PICK(8, 1) AHMC_EMU_PICK(16, 1) AHMC_EMU_PICK(32, 1) AHMC_EMU_PICK(32, 2)
#undef AHMC_EMU_PICK
    if (!fn) return -2;
    AdaptDev ad{};
    ad.enabled = 1;
    ad.n_adapts = q->n_adapts;
    ad.delta = 0.8; ad.gamma = 0.05; ad.t0 = 10.0; ad.kappa = 0.75;
    ad.adapt_metric = q->adapt_metric;
    ad.n_min = q->n_min;
    if (!stan_window_schedule(ad, q->init_buffer, q->term_buffer, q->window_size, q->n_adapts)) return -3;
    ad.eps = q->eps_rw;
    ad.minv = q->minv_rw;
    ad.cholU = q->cholu_rw;
    ad.eps_trace = q->eps_trace;
    for (long long c = 0; c < q->N; ++c) q->eps_rw[c] = q->eps0;
    const ModelDev model{AHMC_MODEL_DIAG_GAUSS, D, q->mu, q->w, 0.0};
    const MetricDev metric{AHMC_METRIC_DENSE, q->Minv0, (long long)D * D, q->cholU0};
    const RngDev rng{q->seed, 0, nullptr, nullptr, 0, nullptr, 0, 0.0, 0.0};
    StatsDev st{};
    st.n_steps = q->n_steps_out;
    st.acceptance_rate = q->acc;
    const int blocks = (int)((q->N + kBlockThreads / G - 1) / (kBlockThreads / G));
    const long long adapt_doubles = chain_adapt_doubles(q->adapt_metric, D);
    std::vector<double> scratch;
    std::vector<double> r_in((size_t)q->N * D, 0.0);
    long long off = 0, stride = 0;
    if (q->hmc) {
        HmcArgs h{};
        LeapfrogArgs& a = h.lf;
        a.model = model; a.metric = metric; a.D = D; a.N = q->N; a.eps = 0.0; a.eps_chain = q->eps_rw;
        a.n_steps = q->n_steps; a.fwd = 1;
        a.th_in = q->th_in; a.r_in = r_in.data(); a.g_in = q->g_in; a.lp_in = q->lp_in; a.ld_in = D;
        a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out; a.ld_out = D;
        h.rng = rng; h.st = st; h.refresh = 1; h.n_transitions = q->T; h.draws = q->draws;
        h.ad = ad;
        scratch.assign((size_t)adapt_doubles * q->N, 0.0);
        h.scratch = scratch.data();
        h.scratch_stride = stride = adapt_doubles;
        emu_launch(fn, &h, blocks, kBlockThreads);
    } else {
        NutsArgs a{};
        a.model = model; a.metric = metric; a.D = D; a.N = q->N; a.eps = 0.0; a.eps_chain = q->eps_rw;
        a.max_depth = q->max_depth; a.delta_max = 1000.0; a.ad = ad; a.rng = rng; a.refresh = 1;
        a.th_in = q->th_in; a.r_in = r_in.data(); a.g_in = q->g_in; a.lp_in = q->lp_in; a.ld_in = D;
        a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out; a.ld_out = D;
        a.st = st; a.n_transitions = q->T; a.draws = q->draws;
        a.scratch_stride = stride = nuts_level_doubles(D, q->max_depth) + adapt_doubles;
        off = nuts_level_doubles(D, q->max_depth);
        scratch.assign((size_t)a.scratch_stride * q->N, 0.0);
        a.scratch = scratch.data();
        emu_launch(fn, &a, blocks, kBlockThreads);
    }
    if (q->workspace)
        for (long long c = 0; c < q->N; ++c)
            for (long long k = 0; k < adapt_doubles; ++k) q->workspace[c * adapt_doubles + k] = scratch[(size_t)(c * stride + off + k)];
    return 0;
}

// the window-end estimate of n draws on its own: workspace N x (D + D*D) (mean, M) in, the chains' Minv / cholU rows
// (N x D x D) in and out, ok[N] = whether the chain's metric was replaced
struct EmuEstimate {
    int32_t D;
    int64_t N;
    double n;
    double* W;
    double *minv, *cholu;
    int32_t* ok;
};
template <int G, int E>
static void estimate_thunk(const void* p) {
    const EmuEstimate& q = *static_cast<const EmuEstimate*>(p);
    const int l = threadIdx.x % G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + threadIdx.x / G;
    const bool act = chain0 < q.N;
    const long long chain = act ? chain0 : q.N - 1;
    AdaptDev ad{};
    ad.minv = q.minv;
    ad.cholU = q.cholu;
    const bool ok = ChainAdapt<G, E, AHMC_ADAPT_WELFORD_COV>::estimate_cov(ad, q.W + ((long long)q.D + (long long)q.D * q.D) * chain,
                                                                           act, q.n, chain, l, q.D);
    if (act && l == 0) q.ok[chain] = ok ? 1 : 0;
}
extern "C" int emu_dense_estimate(const EmuEstimate* q) {
    int G, E;
    if (!pick_layout(q->D, &G, &E) || (G == 32 && E > 2)) return -1;
    KernelFn fn = nullptr;
#define AHMC_EMU_PICK(g, e) \
    if (G == g && E == e) fn = estimate_thunk<g, e>;
    AHMC_EMU_PICK(4, 1) AHMC_EMU_PICK(8, 1) AHMC_EMU_PICK(16, 1) AHMC_EMU_PICK(32, 1) AHMC_EMU_PICK(32, 2)
#undef AHMC_EMU_PICK
    if (!fn) return -2;
    emu_launch(fn, q, (int)((q->N + kBlockThreads / G - 1) / (kBlockThreads / G)), kBlockThreads);
    return 0;
}

#ifdef DENSE_ADAPT_RACE
static int run(int hmc, int D, int N, int T) {
    std::vector<double> mu(D), w(D), Minv((size_t)N * D * D, 0.0), U((size_t)N * D * D, 0.0), th((size_t)N * D), g((size_t)N * D),
        lp(N, 0.0);
    srand(29 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u();
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {  // a diagonal starting metric per chain (its factor: the square roots)
            const double v = 0.7 + 0.6 * u();
            Minv[(size_t)c * D * D + d + (size_t)D * d] = v;
            U[(size_t)c * D * D + d + (size_t)D * d] = std::sqrt(v);
            const size_t i = (size_t)c * D + d;
            th[i] = u() - 0.5;
            g[i] = (th[i] - mu[d]) * w[d];
            lp[c] -= 0.5 * g[i] * (th[i] - mu[d]);
        }
    std::vector<double> o((size_t)3 * N * D), lpo(N), lko(N), draws((size_t)T * N * D), acc((size_t)T * N), tr((size_t)T * N);
    std::vector<double> eps(N), minv((size_t)N * D * D), cholu((size_t)N * D * D);
    std::vector<int32_t> ns((size_t)T * N);
    EmuDenseAdapt q{};
    q.hmc = hmc; q.D = D; q.N = N; q.mu = mu.data(); q.w = w.data(); q.Minv0 = Minv.data(); q.cholU0 = U.data(); q.eps0 = 0.2;
    q.max_depth = 4; q.n_steps = 5; q.seed = 17; q.T = T; q.n_adapts = T - 2; q.init_buffer = 2; q.term_buffer = 2;
    q.window_size = 3; q.adapt_metric = AHMC_ADAPT_WELFORD_COV; q.n_min = 3;
    q.th_in = th.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.draws = draws.data(); q.acc = acc.data(); q.eps_trace = tr.data();
    q.n_steps_out = ns.data(); q.eps_rw = eps.data(); q.minv_rw = minv.data(); q.cholu_rw = cholu.data();
    const int rc = emu_dense_adapt(&q);
    long steps = 0;
    for (auto s : ns) steps += s;
    std::printf("adaptive dense %s D %d N %d T %d: rc %d, %ld leapfrog steps\n", hmc ? "hmc" : "nuts", D, N, T, rc, steps);
    return rc != 0 || steps < (long)T * N;
}

int main() {
    // N fills its blocks (idle groups of a ragged block alias chain N - 1 and re-read its in-flight state: benign reads,
    // excluded here as in race_main.cpp)
    int bad = 0;
    bad |= run(0, 6, 16, 12);  // NUTS, four chains per warp
    bad |= run(1, 7, 16, 12);  // static HMC
    bad |= run(0, 40, 4, 8);   // one chain per warp
    bad |= run(1, 40, 4, 8);
    return bad;
}
#endif
