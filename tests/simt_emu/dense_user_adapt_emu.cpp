// dense_user_adapt_emu.cpp -- runs the WelfordCov form of the per-chain adaptor (ahmc_chain_adapt.cuh) for a run-time
// compiled target under the CPU SIMT emulator: the adaptive NUTS kernel (ahmc_nuts_kernel.cuh) and the adaptive static-HMC
// kernel (ahmc_leapfrog.cu) instantiated as NVRTC instantiates them for a Dense warm-up (AHMC_MODEL_USER,
// kMetricDenseChain, AHMC_ADAPT_WELFORD_COV), with the Philox streams.  The target is a correlated Gaussian written as a
// user would hand it over, params = [mu (D) | P (D x D, column-major)]: log pi = -(th - mu)' P (th - mu) / 2.
// Built with -DDENSE_USER_GROUP it is the group form (AHMC_USER_GROUPWISE: every lane of the group evaluates its rows of
// P (th - mu), the group sums the shares with ahmc_group_sum), without it the one-lane form.  A shuffle or __syncwarp here
// is a barrier of all 32 lanes of the warp, so a model call or an estimator exchange that some lane of the warp does not
// reach would never return.  The sources are included unmodified (their host launch code is skipped with
// AHMC_SIMT_EMULATION).  Built with -DDENSE_USER_ADAPT_RACE it is a ThreadSanitizer program of its own (race_main.cpp
// describes the method).  TEST INFRASTRUCTURE ONLY (tests/test_dense_user_adapt_cpu.py).
#define AHMC_SIMT_EMULATION 1
#define AHMC_NVRTC_USER_MODEL 1
#ifdef DENSE_USER_GROUP
#define AHMC_USER_GROUPWISE 1
#endif
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

// ---- the user's source
#ifdef DENSE_USER_GROUP
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    const double* mu = p;
    const double* P = p + D;
    double s = 0.0;
    for (int i = grp.lane; i < D; i += grp.size) {
        double acc = 0.0;
        for (int j = 0; j < D; ++j) acc = fma(P[i + (long long)D * j], th[j] - mu[j], acc);
        g[i] = -acc;
        s = fma(th[i] - mu[i], acc, s);
    }
    ahmc_group_sync(grp);
    const double S = ahmc_group_sum(grp, s);
    return grp.lane == 0 ? -0.5 * S : 0.0;
}
#else
__device__ double ahmc_user_logp_grad(const double* th, double* g, int D, const double* p) {
    const double* mu = p;
    const double* P = p + D;
    double s = 0.0;
    for (int i = 0; i < D; ++i) {
        double acc = 0.0;
        for (int j = 0; j < D; ++j) acc = fma(P[i + (long long)D * j], th[j] - mu[j], acc);
        g[i] = -acc;
        s = fma(th[i] - mu[i], acc, s);
    }
    return -0.5 * s;
}
#endif

struct EmuDenseUserAdapt {
    int32_t hmc;  // 0: adaptive NUTS (max_depth), 1: adaptive static HMC (n_steps)
    int32_t D;
    int64_t N;
    const double* params;          // [mu | P]
    const double *Minv0, *cholU0;  // starting metric: N x (D x D) column-major each (stride D*D), or one shared (stride 0)
    int64_t metric_stride;
    double eps0;
    int32_t max_depth, n_steps;
    uint64_t seed;
    int32_t T, n_adapts, init_buffer, term_buffer, window_size, adapt_metric, n_min;
    const double *th_in, *g_in, *lp_in;  // N x D, N x D (-grad lp), N
    double *th_out, *r_out, *g_out, *lp_out, *lk_out;
    double *draws, *acc, *eps_trace;  // T x N x D, T x N, T x N
    int32_t *n_steps_out, *tree_depth;  // T x N
    uint8_t *is_accept, *numerical;     // T x N
    double *eps_rw, *minv_rw, *cholu_rw;  // N, N x D x D, N x D x D
};

template <int G, int E>
static void nuts_thunk(const void* p) {
    const NutsArgs& a = *static_cast<const NutsArgs*>(p);
    if (G == 32 && E >= 2 && E <= 8 && a.D == G * E)
        nuts_kernel<AHMC_MODEL_USER, kMetricDenseChain, G, E, false, AHMC_ADAPT_WELFORD_COV, true>(a);
    else nuts_kernel<AHMC_MODEL_USER, kMetricDenseChain, G, E, false, AHMC_ADAPT_WELFORD_COV, false>(a);
}
template <int G, int E>
static void hmc_thunk(const void* p) {
    hmc_kernel<AHMC_MODEL_USER, kMetricDenseChain, G, E, AHMC_ADAPT_WELFORD_COV>(*static_cast<const HmcArgs*>(p));
}
typedef void (*KernelFn)(const void*);

extern "C" int emu_dense_user_adapt(const EmuDenseUserAdapt* q) {
    int G, E;
    const int D = q->D;
    if (!pick_layout(D, &G, &E)) return -1;
    KernelFn fn = nullptr;
#define AHMC_EMU_PICK(g, e) \
    if (G == g && E == e) fn = q->hmc ? hmc_thunk<g, e> : nuts_thunk<g, e>;
    AHMC_EMU_PICK(8, 1) AHMC_EMU_PICK(32, 2)
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
    ModelDev model{};
    model.kind = AHMC_MODEL_USER; model.D = D; model.p0 = q->params; model.c0 = 0.0;
    const MetricDev metric{AHMC_METRIC_DENSE, q->Minv0, (long long)q->metric_stride, q->cholU0};
    const RngDev rng{q->seed, 0, nullptr, nullptr, 0, nullptr, 0, 0.0, 0.0};
    StatsDev st{};
    st.n_steps = q->n_steps_out;
    st.acceptance_rate = q->acc;
    st.tree_depth = q->tree_depth;
    st.is_accept = q->is_accept;
    st.numerical_error = q->numerical;
    const int blocks = (int)((q->N + kBlockThreads / G - 1) / (kBlockThreads / G));
    const long long adapt_doubles = chain_adapt_doubles(q->adapt_metric, D);
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

#ifdef DENSE_USER_ADAPT_RACE
static int run(int hmc, int D, int N, int T) {
    std::vector<double> params((size_t)D + (size_t)D * D, 0.0), Minv((size_t)N * D * D, 0.0), U((size_t)N * D * D, 0.0),
        th((size_t)N * D), g((size_t)N * D), lp(N, 0.0);
    srand(31 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) {  // mean, and the precision of AR(1) correlations 0.5^|i-j| (tridiagonal)
        params[d] = u() - 0.5;
        const double dg = (d == 0 || d == D - 1) ? 1.0 : 1.25;
        params[D + d + (size_t)D * d] = dg / 0.75;
        if (d + 1 < D) params[D + d + (size_t)D * (d + 1)] = params[D + d + 1 + (size_t)D * d] = -0.5 / 0.75;
    }
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {  // a diagonal starting metric per chain (its factor: the square roots)
            const double v = 0.7 + 0.6 * u();
            Minv[(size_t)c * D * D + d + (size_t)D * d] = v;
            U[(size_t)c * D * D + d + (size_t)D * d] = std::sqrt(v);
            th[(size_t)c * D + d] = params[d] + u() - 0.5;
        }
    for (int c = 0; c < N; ++c)
        for (int i = 0; i < D; ++i) {
            double acc = 0.0;
            for (int j = 0; j < D; ++j) acc += params[D + i + (size_t)D * j] * (th[(size_t)c * D + j] - params[j]);
            g[(size_t)c * D + i] = acc;
            lp[c] -= 0.5 * acc * (th[(size_t)c * D + i] - params[i]);
        }
    std::vector<double> o((size_t)3 * N * D), lpo(N), lko(N), draws((size_t)T * N * D), acc((size_t)T * N), tr((size_t)T * N);
    std::vector<double> eps(N), minv((size_t)N * D * D), cholu((size_t)N * D * D);
    std::vector<int32_t> ns((size_t)T * N), td((size_t)T * N);
    std::vector<uint8_t> ia((size_t)T * N), ne((size_t)T * N);
    EmuDenseUserAdapt q{};
    q.hmc = hmc; q.D = D; q.N = N; q.params = params.data(); q.Minv0 = Minv.data(); q.cholU0 = U.data();
    q.metric_stride = (int64_t)D * D; q.eps0 = 0.2;
    q.max_depth = 4; q.n_steps = 5; q.seed = 19; q.T = T; q.n_adapts = T - 2; q.init_buffer = 2; q.term_buffer = 2;
    q.window_size = 3; q.adapt_metric = AHMC_ADAPT_WELFORD_COV; q.n_min = 3;
    q.th_in = th.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.draws = draws.data(); q.acc = acc.data(); q.eps_trace = tr.data();
    q.n_steps_out = ns.data(); q.tree_depth = td.data(); q.is_accept = ia.data(); q.numerical = ne.data();
    q.eps_rw = eps.data(); q.minv_rw = minv.data(); q.cholu_rw = cholu.data();
    const int rc = emu_dense_user_adapt(&q);
    long steps = 0;
    for (auto s : ns) steps += s;
    std::printf("adaptive dense user %s D %d N %d T %d: rc %d, %ld leapfrog steps\n", hmc ? "hmc" : "nuts", D, N, T, rc, steps);
    return rc != 0 || steps < (long)T * N;
}

int main() {
    // N fills its blocks (idle groups of a ragged block alias chain N - 1 and re-read its in-flight state: benign reads,
    // excluded here as in race_main.cpp)
    int bad = 0;
    bad |= run(0, 6, 16, 12);  // NUTS, four chains per warp
    bad |= run(1, 6, 16, 12);  // static HMC
    bad |= run(0, 40, 4, 8);   // one chain per warp
    bad |= run(1, 40, 4, 8);
    return bad;
}
#endif
