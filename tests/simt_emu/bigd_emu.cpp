// bigd_emu.cpp -- runs the D > 512 sampling kernels (advancedhmc.jl_b200/csrc/ahmc_bigd_hmc.cu: the static transition,
// its adaptive form and find_good_stepsize, all on the shared streamed step of ahmc_bigd.cuh) under the CPU SIMT emulator.
// The source is included unmodified (its host launch code is skipped with AHMC_SIMT_EMULATION).  Built with -DBIGD_RACE it
// is a ThreadSanitizer program of its own (see race_main.cpp for the method).  TEST INFRASTRUCTURE ONLY
// (tests/test_bigd_transitions_cpu.py).
#define AHMC_SIMT_EMULATION 1
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "ahmc_bigd_hmc.cu"

void emu_launch(void (*kernel)(const void*), const void* args, int blocks, int threads);

using namespace ahmc;

struct EmuBigd {
    int32_t model, metric;  // AHMC_MODEL_*, AHMC_METRIC_* (Unit / Diag)
    int32_t D;
    int64_t N;
    const double *p0, *p1;  // target mean, 1/s^2 (DIAG_GAUSS)
    double c0;
    const double* Minv;     // Diag: D, or D x N (per chain, minv_stride = D)
    int64_t minv_stride;
    const double* eps;      // N
    int32_t n_steps, T, refresh;
    uint64_t seed, offset;  // Philox key and the first transition's counter
    double partial_alpha;
    const double *normal_tape, *exp_tape;       // N x D, N (T == 1) or NULL (Philox)
    const double *th_in, *r_in, *g_in, *lp_in;  // N x D (ld = D), N
    double *th_out, *r_out, *g_out, *lp_out, *lk_out;
    double *draws, *acc, *H, *dH;               // T x N x D, T x N
    uint8_t *is_accept, *numerical_error;       // T x N
    // adaptive form (adapt_metric >= 0): eps_rw (N) in/out, minv_rw (N x D) out, eps_trace (T x N)
    int32_t adapt_metric, n_adapts, init_buffer, term_buffer, window_size, n_min;
    double *eps_rw, *minv_rw, *eps_trace;
};

template <int MODEL, int METRIC, int ADAPT>
static void hmc_thunk(const void* p) {
    hmc_big_kernel<MODEL, METRIC, ADAPT>(*static_cast<const HmcArgs*>(p));
}
template <int MODEL, int METRIC>
static void fe_thunk(const void* p) {
    find_eps_big_kernel<MODEL, METRIC>(*static_cast<const FindEpsArgs*>(p));
}
typedef void (*KernelFn)(const void*);

template <template <int, int> class P>
static KernelFn pick(int model, int metric) {
    const bool d = metric == AHMC_METRIC_DIAG;
    if (model == AHMC_MODEL_STD_NORMAL) return d ? P<AHMC_MODEL_STD_NORMAL, AHMC_METRIC_DIAG>::fn : P<AHMC_MODEL_STD_NORMAL, AHMC_METRIC_UNIT>::fn;
    if (model == AHMC_MODEL_DIAG_GAUSS) return d ? P<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG>::fn : P<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_UNIT>::fn;
    return d ? P<AHMC_MODEL_FUNNEL, AHMC_METRIC_DIAG>::fn : P<AHMC_MODEL_FUNNEL, AHMC_METRIC_UNIT>::fn;
}
template <int MODEL, int METRIC>
struct PlainHmc { static constexpr KernelFn fn = hmc_thunk<MODEL, METRIC, 0>; };
template <int MODEL, int METRIC>
struct WelfordHmc { static constexpr KernelFn fn = hmc_thunk<MODEL, AHMC_METRIC_DIAG, AHMC_ADAPT_WELFORD>; };
template <int MODEL, int METRIC>
struct NutpieHmc { static constexpr KernelFn fn = hmc_thunk<MODEL, AHMC_METRIC_DIAG, AHMC_ADAPT_NUTPIE>; };
template <int MODEL, int METRIC>
struct FindEps { static constexpr KernelFn fn = fe_thunk<MODEL, METRIC>; };

static int blocks_of(long long N) { return (int)((N + kBlockThreads / 32 - 1) / (kBlockThreads / 32)); }

extern "C" int emu_bigd_hmc(const EmuBigd* q) {
    const int D = q->D;
    const bool adapt = q->adapt_metric >= 0;
    KernelFn fn = adapt ? (q->adapt_metric == AHMC_ADAPT_NUTPIE ? pick<NutpieHmc>(q->model, q->metric) : pick<WelfordHmc>(q->model, q->metric))
                        : pick<PlainHmc>(q->model, q->metric);
    HmcArgs h{};
    LeapfrogArgs& a = h.lf;
    a.model = ModelDev{q->model, D, q->p0, q->p1, q->c0};
    a.metric = MetricDev{q->metric, q->Minv, q->minv_stride, nullptr};
    a.D = D; a.N = q->N; a.eps = 0.0; a.eps_chain = q->eps; a.n_steps = q->n_steps; a.fwd = 1;
    a.th_in = q->th_in; a.r_in = q->r_in; a.g_in = q->g_in; a.lp_in = q->lp_in; a.ld_in = D;
    a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out; a.ld_out = D;
    h.rng = RngDev{q->seed, q->offset, q->normal_tape, q->exp_tape, 1, nullptr, 0, q->partial_alpha, 0.0};
    h.st.is_accept = q->is_accept; h.st.acceptance_rate = q->acc; h.st.hamiltonian_energy = q->H;
    h.st.hamiltonian_energy_error = q->dH; h.st.numerical_error = q->numerical_error;
    h.refresh = q->refresh; h.n_transitions = q->T; h.draws = q->draws;
    if (adapt) {
        AdaptDev& ad = h.ad;
        ad.enabled = 1; ad.n_adapts = q->n_adapts;
        ad.delta = 0.8; ad.gamma = 0.05; ad.t0 = 10.0; ad.kappa = 0.75;
        ad.adapt_metric = q->adapt_metric; ad.n_min = q->n_min;
        if (!stan_window_schedule(ad, q->init_buffer, q->term_buffer, q->window_size, q->n_adapts)) return -3;
        ad.eps = q->eps_rw; ad.minv = q->minv_rw; ad.eps_trace = q->eps_trace;
        a.eps_chain = q->eps_rw;
    }
    h.scratch_stride = (long long)(kBigHmcVectors + (adapt ? chain_adapt_vectors(q->adapt_metric) : 0)) * D;
    std::vector<double> scratch((size_t)h.scratch_stride * q->N, 0.0);
    h.scratch = scratch.data();
    emu_launch(fn, &h, blocks_of(q->N), kBlockThreads);
    return 0;
}

extern "C" int emu_bigd_find_eps(int32_t model, int32_t metric, int32_t D, int64_t N, const double* p0, const double* p1, double c0,
                                 const double* Minv, int64_t minv_stride, const double* th, const double* g, const double* lp,
                                 const double* normal_tape, double eps0, int32_t max_iters, double* eps_out, double* r_out) {
    FindEpsArgs a{};
    a.model = ModelDev{model, D, p0, p1, c0};
    a.metric = MetricDev{metric, Minv, minv_stride, nullptr};
    a.D = D; a.N = N; a.th = th; a.g = g; a.lp = lp; a.ld = D; a.seed = 0; a.offset = 0; a.normal_tape = normal_tape;
    a.eps0 = eps0; a.max_iters = max_iters; a.eps_out = eps_out; a.r_out = r_out;
    std::vector<double> scratch((size_t)kBigFindEpsVectors * D * N, 0.0);
    a.scratch = scratch.data();
    emu_launch(pick<FindEps>(model, metric), &a, blocks_of(N), kBlockThreads);
    return 0;
}

#ifdef BIGD_RACE
// a persistent Philox run of each kernel form on a ragged block (N = 6: two warps of the second block idle)
static int run(int model, int metric, int adapt_metric, int D, int N, int T) {
    std::vector<double> mu(D), w(D), Minv(D), th((size_t)N * D), r((size_t)N * D, 0.0), g((size_t)N * D), lp(N, 0.0), eps(N, 0.05);
    srand(5 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u(), Minv[d] = 0.7 + 0.6 * u();
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {
            const size_t i = (size_t)c * D + d;
            th[i] = 0.3 * (u() - 0.5);
            g[i] = (th[i] - mu[d]) * w[d];
            lp[c] -= 0.5 * g[i] * (th[i] - mu[d]);
        }
    std::vector<double> o((size_t)3 * N * D), lpo(N), lko(N), draws((size_t)T * N * D), acc((size_t)T * N), H((size_t)T * N),
        dH((size_t)T * N), tr((size_t)T * N), epsrw(N, 0.05), minv((size_t)N * D);
    std::vector<uint8_t> ia((size_t)T * N), ne((size_t)T * N);
    EmuBigd q{};
    q.model = model; q.metric = metric; q.D = D; q.N = N; q.p0 = mu.data(); q.p1 = w.data(); q.Minv = Minv.data();
    q.eps = eps.data(); q.n_steps = 3; q.T = T; q.refresh = 1; q.seed = 9; q.partial_alpha = 0.3;
    q.th_in = th.data(); q.r_in = r.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D; q.lp_out = lpo.data(); q.lk_out = lko.data();
    q.draws = draws.data(); q.acc = acc.data(); q.H = H.data(); q.dH = dH.data(); q.is_accept = ia.data(); q.numerical_error = ne.data();
    q.adapt_metric = adapt_metric; q.n_adapts = T - 1; q.init_buffer = 1; q.term_buffer = 1; q.window_size = 2; q.n_min = 2;
    q.eps_rw = epsrw.data(); q.minv_rw = minv.data(); q.eps_trace = tr.data();
    const int rc = emu_bigd_hmc(&q);
    std::vector<double> eo(N);
    const int rc2 = emu_bigd_find_eps(model, metric, D, N, mu.data(), w.data(), 0.0, Minv.data(), 0, th.data(), g.data(), lp.data(), nullptr,
                                      0.1, 20, eo.data(), nullptr);
    int accepted = 0;
    for (auto x : ia) accepted += x;
    std::printf("bigd model %d metric %d adapt %d D %d N %d T %d: rc %d %d, %d accepted\n", model, metric, adapt_metric, D, N, T, rc, rc2,
                accepted);
    return rc != 0 || rc2 != 0;
}

int main() {
    int bad = 0;
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, -1, 600, 6, 3);
    bad |= run(AHMC_MODEL_FUNNEL, AHMC_METRIC_UNIT, -1, 530, 6, 2);
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, AHMC_ADAPT_WELFORD, 520, 6, 5);
    bad |= run(AHMC_MODEL_STD_NORMAL, AHMC_METRIC_DIAG, AHMC_ADAPT_NUTPIE, 520, 6, 5);
    return bad;
}
#endif
