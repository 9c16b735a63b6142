// adapt_chain_emu.cpp -- runs the two adaptive persistent kernels (K3 adaptive NUTS, ahmc_nuts_kernel.cuh; K2 adaptive
// static HMC, ahmc_leapfrog.cu; both with the per-chain adaptor of ahmc_chain_adapt.cuh) under the CPU SIMT emulator, on
// a diagonal Gaussian with the Diag metric and the Philox streams.  The sources are included unmodified (their host launch
// code is skipped with AHMC_SIMT_EMULATION).  Built with -DRACE_ADAPT_CHAIN it is a ThreadSanitizer program of its own
// (emu_harness.h describes the method).  TEST INFRASTRUCTURE ONLY (tests/test_adapt_in_launch_cpu.py).
#define AHMC_SIMT_EMULATION 1
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "ahmc_nuts_kernel.cuh"
#include "ahmc_leapfrog.cu"
#include "emu_harness.h"

namespace ahmc {
double smem[1 << 16];  // the block's dynamic shared memory
}

using namespace ahmc;

struct EmuAdaptChain {
    int32_t hmc;  // 0: adaptive NUTS (max_depth), 1: adaptive static HMC (n_steps)
    int32_t D;
    int64_t N;
    const double *mu, *w, *Minv;  // target mean, 1/s^2; starting M^-1 (D, shared by the chains)
    double eps0;
    int32_t max_depth, n_steps;
    uint64_t seed;
    int32_t T, n_adapts, init_buffer, term_buffer, window_size, adapt_metric, n_min;
    const double *th_in, *g_in, *lp_in;  // N x D, N x D (-grad lp), N
    double *th_out, *r_out, *g_out, *lp_out, *lk_out;
    double *draws, *acc, *eps_trace;  // T x N x D, T x N, T x N
    int32_t* n_steps_out;             // T x N
    double *eps_rw, *minv_rw;         // N, N x D
};
EMU_EXPORT_SIZEOF(EmuAdaptChain);

// FORM: the adaptor's compiled estimator form (adapt_form), as the library's launchers pick it
template <int G, int E, int FORM>
static void nuts_thunk(const void* p) {
    const NutsArgs& a = *static_cast<const NutsArgs*>(p);
    if (G == 32 && E >= 2 && E <= 8 && a.D == G * E) nuts_kernel<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, G, E, false, FORM, true>(a);
    else nuts_kernel<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, G, E, false, FORM, false>(a);
}
template <int G, int E, int FORM>
static void hmc_thunk(const void* p) {
    hmc_kernel<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, G, E, FORM>(*static_cast<const HmcArgs*>(p));
}
typedef void (*KernelFn)(const void*);

extern "C" int emu_adapt_chain(const EmuAdaptChain* q) {
    int G, E;
    const int D = q->D;
    if (!pick_layout(D, &G, &E) || (G == 32 && E > 2)) return -1;
    KernelFn fn = nullptr;
    const bool nut = q->adapt_metric == AHMC_ADAPT_NUTPIE;
#define AHMC_EMU_PICK(g, e)                                                                                      \
    if (G == g && E == e)                                                                                       \
        fn = q->hmc ? (nut ? hmc_thunk<g, e, AHMC_ADAPT_NUTPIE> : hmc_thunk<g, e, AHMC_ADAPT_WELFORD>)           \
                    : (nut ? nuts_thunk<g, e, AHMC_ADAPT_NUTPIE> : nuts_thunk<g, e, AHMC_ADAPT_WELFORD>);
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
    ad.eps_trace = q->eps_trace;
    for (long long c = 0; c < q->N; ++c) q->eps_rw[c] = q->eps0;
    const ModelDev model{AHMC_MODEL_DIAG_GAUSS, D, q->mu, q->w, 0.0};
    const MetricDev metric{AHMC_METRIC_DIAG, q->Minv, 0, nullptr};
    const RngDev rng{q->seed, 0, nullptr, nullptr, 0, nullptr, 0, 0.0, 0.0};
    StatsDev st{};
    st.n_steps = q->n_steps_out;
    st.acceptance_rate = q->acc;
    const int blocks = (int)((q->N + kBlockThreads / G - 1) / (kBlockThreads / G));
    const long long adapt_doubles = (long long)chain_adapt_vectors(q->adapt_metric) * D;
    std::vector<double> scratch;
    std::vector<double> r_in((size_t)q->N * D, 0.0);
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
        h.scratch_stride = adapt_doubles;
        emu_launch(fn, &h, blocks, kBlockThreads);
    } else {
        NutsArgs a{};
        a.model = model; a.metric = metric; a.D = D; a.N = q->N; a.eps = 0.0; a.eps_chain = q->eps_rw;
        a.max_depth = q->max_depth; a.delta_max = 1000.0; a.ad = ad; a.rng = rng; a.refresh = 1;
        a.th_in = q->th_in; a.r_in = r_in.data(); a.g_in = q->g_in; a.lp_in = q->lp_in; a.ld_in = D;
        a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out; a.ld_out = D;
        a.st = st; a.n_transitions = q->T; a.draws = q->draws;
        a.scratch_stride = nuts_level_doubles(D, q->max_depth) + adapt_doubles;
        scratch.assign((size_t)a.scratch_stride * q->N, 0.0);
        a.scratch = scratch.data();
        emu_launch(fn, &a, blocks, kBlockThreads);
    }
    return 0;
}

#ifdef RACE_ADAPT_CHAIN
static int run(int hmc, int D, int N, int T, int adapt_metric) {
    std::vector<double> mu(D), w(D), Minv(D), th((size_t)N * D), g((size_t)N * D), lp(N, 0.0);
    srand(13 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u(), Minv[d] = 0.7 + 0.6 * u();
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {
            const size_t i = (size_t)c * D + d;
            th[i] = u() - 0.5;
            g[i] = (th[i] - mu[d]) * w[d];
            lp[c] -= 0.5 * g[i] * (th[i] - mu[d]);
        }
    std::vector<double> o((size_t)3 * N * D), lpo(N), lko(N), draws((size_t)T * N * D), acc((size_t)T * N), tr((size_t)T * N);
    std::vector<double> eps(N), minv((size_t)N * D);
    std::vector<int32_t> ns((size_t)T * N);
    EmuAdaptChain q{};
    q.hmc = hmc; q.D = D; q.N = N; q.mu = mu.data(); q.w = w.data(); q.Minv = Minv.data(); q.eps0 = 0.2; q.max_depth = 4;
    q.n_steps = 5; q.seed = 17; q.T = T; q.n_adapts = T - 2; q.init_buffer = 2; q.term_buffer = 2; q.window_size = 3;
    q.adapt_metric = adapt_metric; q.n_min = 3;
    q.th_in = th.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.draws = draws.data(); q.acc = acc.data(); q.eps_trace = tr.data();
    q.n_steps_out = ns.data(); q.eps_rw = eps.data(); q.minv_rw = minv.data();
    const int rc = emu_adapt_chain(&q);
    long steps = 0;
    for (auto s : ns) steps += s;
    std::printf("adaptive %s D %d N %d T %d adapt_metric %d: rc %d, %ld leapfrog steps\n", hmc ? "hmc" : "nuts", D, N, T,
                adapt_metric, rc, steps);
    return rc != 0 || steps < (long)T * N;
}

int main() {
    // N fills its blocks.  In a ragged block the idle groups alias chain N - 1 (`chain = N - 1`): like every persistent
    // kernel of the library they re-read that chain's in-flight state (its phase point, here also its step size) while
    // its owner group writes it, and discard what they computed -- benign reads, excluded here as in nuts_emu.cpp's main.
    int bad = 0;
    bad |= run(0, 6, 16, 12, 2);  // NUTS + NutpieVar, four chains per warp
    bad |= run(1, 6, 16, 12, 2);  // static HMC + NutpieVar
    bad |= run(1, 7, 16, 12, 1);  // static HMC + WelfordVar
    bad |= run(1, 5, 16, 10, 0);  // static HMC, step size only: no estimator workspace at all
    bad |= run(0, 40, 4, 8, 2);   // one chain per warp
    bad |= run(1, 40, 4, 8, 2);
    return bad;
}
#endif
