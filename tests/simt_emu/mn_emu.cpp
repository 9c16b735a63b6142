// mn_emu.cpp -- the MultinomialTS static-transition kernel (advancedhmc.jl_b200/csrc/ahmc_multinomial.cu, unmodified)
// under the CPU SIMT emulator.  TEST INFRASTRUCTURE ONLY (tests/test_simt_emulation.py).
#define AHMC_SIMT_EMULATION 1
#include <cstdlib>
#include <cstdio>
#include <vector>

#include "ahmc_multinomial.cu"
#include "emu_harness.h"

namespace ahmc {
double smem[1 << 16];
}
using namespace ahmc;

struct EmuMn {
    int32_t model_kind, metric_kind, D;
    int64_t N;
    const double *p0, *p1;
    const double* Minv;
    const double* cholU;
    double eps;
    int32_t n_steps, n_fwd;
    const double *normal_tape, *unif_tape;
    const double *th_in, *g_in, *lp_in;
    double *th_out, *r_out, *g_out, *lp_out, *lk_out;
    double* acc;
    int32_t* index;
    double temper_alpha;
};
EMU_EXPORT_SIZEOF(EmuMn);

template <int MODEL, int METRIC, int G, int E>
static void mn_thunk(const void* p) { multinomial_kernel<MODEL, METRIC, G, E>(*static_cast<const MultinomialArgs*>(p)); }
typedef void (*KernelFn)(const void*);
template <int MODEL, int METRIC>
static KernelFn pick(int G, int E) {
    if (G == 4 && E == 1) return mn_thunk<MODEL, METRIC, 4, 1>;
    if (G == 8 && E == 1) return mn_thunk<MODEL, METRIC, 8, 1>;
    if (G == 32 && E == 2) return mn_thunk<MODEL, METRIC, 32, 2>;
    return nullptr;
}

extern "C" int emu_multinomial(const EmuMn* q) {
    int G, E;
    const int D = q->D;
    if (D <= 4) G = 4, E = 1;
    else if (D <= 8) G = 8, E = 1;
    else if (D > 32 && D <= 64) G = 32, E = 2;
    else return -1;
    std::vector<double> r_in((size_t)D * q->N, 0.0), energies((size_t)(q->n_steps + 1) * q->N, 0.0);
    MultinomialArgs a{};
    a.model = ModelDev{q->model_kind, D, q->p0, q->p1, 0.0};
    a.metric = MetricDev{q->metric_kind, q->Minv, 0, q->cholU};
    a.D = D;
    a.N = q->N;
    a.eps = q->eps;
    a.n_steps = q->n_steps;
    a.n_fwd = q->n_fwd;
    a.refresh = 1;
    a.rng = RngDev{1, 0, q->normal_tape, q->unif_tape, 1, nullptr, 0, 0.0, q->temper_alpha};
    a.th_in = q->th_in; a.r_in = r_in.data(); a.g_in = q->g_in; a.lp_in = q->lp_in;
    a.ld_in = D;
    a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out;
    a.ld_out = D;
    a.st = StatsDev{};
    a.st.acceptance_rate = q->acc;
    a.st.tree_depth = q->index;
    a.energies = energies.data();
    KernelFn fn = nullptr;
    const int m = q->model_kind, me = q->metric_kind;
    if (m == AHMC_MODEL_DIAG_GAUSS && me == AHMC_METRIC_DIAG) fn = pick<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG>(G, E);
    else if (m == AHMC_MODEL_FUNNEL && me == AHMC_METRIC_DENSE) fn = pick<AHMC_MODEL_FUNNEL, AHMC_METRIC_DENSE>(G, E);
    else if (m == AHMC_MODEL_DENSE_GAUSS && me == AHMC_METRIC_UNIT) fn = pick<AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_UNIT>(G, E);
    if (!fn) return -2;
    const int chains_per_block = kBlockThreads / G;
    emu_launch(fn, &a, (int)((q->N + chains_per_block - 1) / chains_per_block), kBlockThreads);
    return 0;
}

#ifdef RACE_MN
static int run(int model, int metric, int D, int N, int n, int n_fwd) {
    std::vector<double> mu(D), w(D), P, Minv, cholU, th((size_t)N * D), g((size_t)N * D), lp(N, 0.0);
    std::vector<double> normals((size_t)N * D), unif(N);
    srand(9 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u();
    if (model == AHMC_MODEL_DENSE_GAUSS) {
        P.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            P[(size_t)d * D + d] = 1.0 + 0.1 * u();
            if (d) P[(size_t)d * D + d - 1] = P[(size_t)(d - 1) * D + d] = 0.2;
        }
    }
    if (metric == AHMC_METRIC_DIAG) {
        Minv.resize(D);
        for (auto& x : Minv) x = 0.7 + 0.6 * u();
    }
    for (int c = 0; c < N; ++c) {
        unif[c] = u();
        for (int d = 0; d < D; ++d) th[(size_t)c * D + d] = u() - 0.5, normals[(size_t)c * D + d] = 2.0 * u() - 1.0;
    }
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {
            double gd = 0.0;
            if (model == AHMC_MODEL_DENSE_GAUSS)
                for (int k = 0; k < D; ++k) gd += P[(size_t)k * D + d] * (th[(size_t)c * D + k] - mu[k]);
            else gd = (th[(size_t)c * D + d] - mu[d]) * w[d];
            g[(size_t)c * D + d] = gd;
            lp[c] -= 0.5 * gd * (th[(size_t)c * D + d] - mu[d]);
        }
    std::vector<double> o((size_t)3 * N * D), lpo(N), lko(N), acc(N);
    std::vector<int32_t> idx(N);
    EmuMn q{};
    q.model_kind = model; q.metric_kind = metric; q.D = D; q.N = N; q.p0 = mu.data();
    q.p1 = model == AHMC_MODEL_DENSE_GAUSS ? P.data() : w.data();
    q.Minv = Minv.empty() ? nullptr : Minv.data(); q.eps = 0.2; q.n_steps = n; q.n_fwd = n_fwd;
    q.normal_tape = normals.data(); q.unif_tape = unif.data(); q.th_in = th.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.acc = acc.data(); q.index = idx.data();
    const int rc = emu_multinomial(&q);
    std::printf("mn model %d metric %d D %d N %d: rc %d acc0 %.6f\n", model, metric, D, N, rc, acc[0]);
    return rc != 0;
}

int main() {
    int bad = 0;
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 7, 21, 7, 3);    // four chains per warp, ragged block, both directions
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_UNIT, 6, 9, 5, 5);    // shared-memory precision slab
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 40, 5, 6, 0);    // one chain per warp, all backward
    return bad;
}
#endif
