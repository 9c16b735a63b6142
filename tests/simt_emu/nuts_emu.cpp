// nuts_emu.cpp -- runs the product's NUTS kernel source (ahmc_nuts_kernel.cuh) under the CPU SIMT emulator.
// TEST INFRASTRUCTURE ONLY: built by tests/test_simt_emulation.py with g++; the kernel header is included unmodified
// (its host launch code is skipped with AHMC_SIMT_EMULATION).
#define AHMC_SIMT_EMULATION 1
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "ahmc_nuts_kernel.cuh"
#include "emu_smem.h"
#include "emu_harness.h"

EMU_DEFINE_SMEM_ARENA();  // the block's dynamic shared memory (`extern __shared__ double smem[]` in the kernel)

using namespace ahmc;

struct EmuNuts {
    int32_t model_kind, metric_kind, D;
    int64_t N;
    const double *p0, *p1;
    double c0;
    const double* Minv;
    int64_t minv_stride;
    const double* cholU;
    double eps;
    const double* eps_chain;
    int32_t max_depth;
    double delta_max;
    int32_t sampler, criterion;
    uint64_t seed, offset;
    const double *normal_tape, *exp_tape;
    int64_t exp_stride;
    const uint8_t* dir_tape;
    int64_t dir_stride;
    double partial_alpha;
    int32_t refresh;
    const double *th_in, *r_in, *g_in, *lp_in;
    double *th_out, *r_out, *g_out, *lp_out, *lk_out;
    int32_t *n_steps, *tree_depth;
    uint8_t* numerical;
    double *acc, *dH, *dHmax;
    int32_t n_transitions;
    double* draws;
    int32_t adapt, n_adapts, init_buffer, term_buffer, window_size;
    double delta, gamma, t0, kappa;
    int32_t adapt_metric, n_min;
    double *eps_rw, *minv_rw, *eps_trace;
    double temper_alpha;
    int32_t coop_padded;  // 1: also hand the kernel column-padded copies of the dense matrices (one bulk copy per chunk)
    int64_t ld_in, ld_out;  // leading dimensions of the D x N inputs / outputs (0: D)
};
EMU_EXPORT_SIZEOF(EmuNuts);

template <int MODEL, int METRIC, int G, int E, bool VAR, bool ADAPT>
static constexpr bool coop_form() {  // like launch_nuts_v: dense operators, one chain per warp, default family
    return (MODEL == AHMC_MODEL_DENSE_GAUSS || METRIC == AHMC_METRIC_DENSE) && G == 32 && !VAR;
}
template <int MODEL, int METRIC, int G, int E, bool VAR, bool ADAPT>
static void thunk(const void* p) {
    const NutsArgs& a = *static_cast<const NutsArgs*>(p);
    if constexpr (coop_form<MODEL, METRIC, G, E, VAR, ADAPT>()) {
        if (E >= 2 && E <= 8 && a.D == G * E) nuts_kernel<MODEL, METRIC, G, E, VAR, ADAPT, true, true>(a);
        else nuts_kernel<MODEL, METRIC, G, E, VAR, ADAPT, false, true>(a);
        return;
    }
    if (G == 32 && E >= 2 && E <= 8 && a.D == G * E) {  // the full-tile instantiation (D a compile-time constant), like launch_nuts_v
        nuts_kernel<MODEL, METRIC, G, E, VAR, ADAPT, true>(a);
        return;
    }
    nuts_kernel<MODEL, METRIC, G, E, VAR, ADAPT, false>(a);
}

typedef void (*KernelFn)(const void*);

template <int MODEL, int METRIC, bool VAR, bool ADAPT>
static KernelFn by_layout(int G, int E) {
    if (G == 4 && E == 1) return thunk<MODEL, METRIC, 4, 1, VAR, ADAPT>;
    if (G == 8 && E == 1) return thunk<MODEL, METRIC, 8, 1, VAR, ADAPT>;
    if (G == 32 && E == 2) return thunk<MODEL, METRIC, 32, 2, VAR, ADAPT>;
    if (G == 16 && E == 1) return thunk<MODEL, METRIC, 16, 1, VAR, ADAPT>;
    if (G == 32 && E == 1) return thunk<MODEL, METRIC, 32, 1, VAR, ADAPT>;  // D in (16, 32]
    if (G == 32 && E == 4) return thunk<MODEL, METRIC, 32, 4, VAR, ADAPT>;
    if (G == 32 && E == 8) return thunk<MODEL, METRIC, 32, 8, VAR, ADAPT>;
    if constexpr (!VAR && !ADAPT) {
        if (G == 32 && E == 16) return thunk<MODEL, METRIC, 32, 16, VAR, ADAPT>;  // D in (256, 512]: 16-column chunks, 2 stages
    }
    return nullptr;
}

template <bool VAR, bool ADAPT>
static KernelFn by_model(int model, int metric, int G, int E) {
    if (model == AHMC_MODEL_STD_NORMAL && metric == AHMC_METRIC_UNIT) return by_layout<AHMC_MODEL_STD_NORMAL, AHMC_METRIC_UNIT, VAR, ADAPT>(G, E);
    if (model == AHMC_MODEL_DIAG_GAUSS && metric == AHMC_METRIC_DIAG) return by_layout<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, VAR, ADAPT>(G, E);
    if (model == AHMC_MODEL_FUNNEL && metric == AHMC_METRIC_DIAG) return by_layout<AHMC_MODEL_FUNNEL, AHMC_METRIC_DIAG, VAR, ADAPT>(G, E);
    if (ADAPT && !VAR && model == AHMC_MODEL_DENSE_GAUSS && metric == AHMC_METRIC_DIAG)  // adaptive family, cooperative form
        return by_layout<AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DIAG, false, true>(G, E);
    if (!ADAPT) {
        if (model == AHMC_MODEL_DENSE_GAUSS && metric == AHMC_METRIC_DENSE) return by_layout<AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, VAR, false>(G, E);
        if (model == AHMC_MODEL_DIAG_GAUSS && metric == AHMC_METRIC_UNIT) return by_layout<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_UNIT, VAR, false>(G, E);
        if (!VAR) {  // the other two dense-operator combinations of the COOP form
            if (model == AHMC_MODEL_DENSE_GAUSS && metric == AHMC_METRIC_DIAG) return by_layout<AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DIAG, false, false>(G, E);
            if (model == AHMC_MODEL_DIAG_GAUSS && metric == AHMC_METRIC_DENSE) return by_layout<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DENSE, false, false>(G, E);
            if (model == AHMC_MODEL_DENSE_GAUSS && metric == AHMC_METRIC_UNIT) return by_layout<AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_UNIT, false, false>(G, E);
            if (model == AHMC_MODEL_FUNNEL && metric == AHMC_METRIC_DENSE) return by_layout<AHMC_MODEL_FUNNEL, AHMC_METRIC_DENSE, false, false>(G, E);
        }
    }
    return nullptr;
}

// the product's host-side window schedule (ahmc_kernels.cuh), for the comparison with the oracle's
extern "C" int emu_window_schedule(int init_buffer, int term_buffer, int window_size, int n_adapts, int* ws, int* we, int* splits) {
    AdaptDev ad{};
    if (!stan_window_schedule(ad, init_buffer, term_buffer, window_size, n_adapts)) return -1;
    *ws = ad.window_start;
    *we = ad.window_end;
    for (int i = 0; i < ad.n_splits; ++i) splits[i] = ad.splits[i];
    return ad.n_splits;
}

extern "C" int emu_nuts(const EmuNuts* q) {
    int G, E;
    const int D = q->D;
    if (D <= 4) G = 4, E = 1;
    else if (D <= 8) G = 8, E = 1;
    else if (D <= 16) G = 16, E = 1;
    else if (D <= 32) G = 32, E = 1;  // (pick_layout, ahmc_leapfrog.cu)
    else if (D <= 64) G = 32, E = 2;
    else if (D > 64 && D <= 128) G = 32, E = 4;  // the headline layout
    else if (D > 128 && D <= 256) G = 32, E = 8;  // C5's layout
    else if (D > 256 && D <= 512) G = 32, E = 16;
    else return -1;
    NutsArgs a{};
    a.model = ModelDev{q->model_kind, D, q->p0, q->p1, q->c0};
    a.metric = MetricDev{q->metric_kind, q->Minv, q->minv_stride, q->cholU};
    std::vector<double> pad_p, pad_m, pad_u;
    if (q->coop_padded) {  // what ahmc_model_create / nuts_impl prepare on the device (launch_pad_columns)
        const int lds = coop_lds(D);
        auto pad = [&](const double* A, std::vector<double>& out) {
            out.assign((size_t)D * lds, 0.0);
            for (int k = 0; k < D; ++k)
                for (int r = 0; r < D; ++r) out[(size_t)k * lds + r] = A[(size_t)k * D + r];
            return out.data();
        };
        if (q->model_kind == AHMC_MODEL_DENSE_GAUSS) a.model.p1_coop = pad(q->p1, pad_p);
        if (q->metric_kind == AHMC_METRIC_DENSE) {
            a.metric.Minv_coop = pad(q->Minv, pad_m);
            if (q->cholU) a.metric.cholU_coop = pad(q->cholU, pad_u);
        }
    }
    a.D = D;
    a.N = q->N;
    a.eps = q->eps;
    a.eps_chain = q->eps_chain;
    a.max_depth = q->max_depth;
    a.delta_max = q->delta_max;
    a.sampler = q->sampler;
    a.criterion = q->criterion;
    a.rng = RngDev{q->seed, q->offset, q->normal_tape, q->exp_tape, q->exp_stride, q->dir_tape, q->dir_stride, q->partial_alpha, q->temper_alpha};
    a.refresh = q->refresh;
    a.th_in = q->th_in; a.r_in = q->r_in; a.g_in = q->g_in; a.lp_in = q->lp_in;
    a.ld_in = q->ld_in ? q->ld_in : D;
    a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out;
    a.ld_out = q->ld_out ? q->ld_out : D;
    a.st = StatsDev{};
    a.st.n_steps = q->n_steps;
    a.st.tree_depth = q->tree_depth;
    a.st.numerical_error = q->numerical;
    a.st.acceptance_rate = q->acc;
    a.st.hamiltonian_energy_error = q->dH;
    a.st.max_hamiltonian_energy_error = q->dHmax;
    a.n_transitions = q->n_transitions;
    a.draws = q->draws;
    if (q->adapt) {
        AdaptDev& ad = a.ad;
        ad.enabled = 1;
        ad.n_adapts = q->n_adapts;
        ad.delta = q->delta; ad.gamma = q->gamma; ad.t0 = q->t0; ad.kappa = q->kappa;
        ad.adapt_metric = q->adapt_metric;
        ad.n_min = q->n_min;
        if (!stan_window_schedule(ad, q->init_buffer, q->term_buffer, q->window_size, q->n_adapts)) return -3;  // as nuts_impl
        ad.eps = q->eps_rw;
        a.eps_chain = q->eps_rw;
        ad.minv = q->minv_rw;
        ad.eps_trace = q->eps_trace;
    }
    const long long stride = nuts_level_doubles(D, q->max_depth) + (q->adapt ? 2LL * D : 0);
    std::vector<double> scratch((size_t)stride * (size_t)q->N, 0.0);
    a.scratch = scratch.data();
    a.scratch_stride = stride;
    const bool var = q->sampler != 0 || q->criterion != 0;
    KernelFn fn = q->adapt ? by_model<false, true>(q->model_kind, q->metric_kind, G, E)
                           : (var ? by_model<true, false>(q->model_kind, q->metric_kind, G, E)
                                  : by_model<false, false>(q->model_kind, q->metric_kind, G, E));
    if (!fn) return -2;
    const bool dense_ops = q->model_kind == AHMC_MODEL_DENSE_GAUSS || q->metric_kind == AHMC_METRIC_DENSE;
    const bool coop = dense_ops && G == 32 && !var;  // blocks of kCoopWarps chains sharing the D x D products
    const int threads = coop ? kCoopThreads : kBlockThreads;
    const int chains_per_block = threads / G;
    const int blocks = (int)((q->N + chains_per_block - 1) / chains_per_block);
    size_t sm = 0;  // what launch_nuts_v asks for
    switch (E) {
        case 1: sm = nuts_smem_bytes<1>(coop, q->model_kind, q->metric_kind, D, G, q->max_depth); break;
        case 2: sm = nuts_smem_bytes<2>(coop, q->model_kind, q->metric_kind, D, G, q->max_depth); break;
        case 4: sm = nuts_smem_bytes<4>(coop, q->model_kind, q->metric_kind, D, G, q->max_depth); break;
        case 8: sm = nuts_smem_bytes<8>(coop, q->model_kind, q->metric_kind, D, G, q->max_depth); break;
        default: sm = nuts_smem_bytes<16>(coop, q->model_kind, q->metric_kind, D, G, q->max_depth); break;
    }
    emu_smem_begin(emu_smem_base(), sm, 0, coop ? "nuts_kernel (COOP)" : "nuts_kernel");
    emu_launch(fn, &a, blocks, threads);
    emu_smem_end();
    return 0;
}

#ifdef RACE_NUTS
static int run(int model, int metric, int D, int N, int T, int sampler, int criterion, bool adapt) {
    std::vector<double> mu(D), w(D), Minv, cholU, th((size_t)N * D), r((size_t)N * D, 0.0), g((size_t)N * D), lp(N, 0.0);
    std::vector<double> P;
    srand(7 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u();
    if (model == AHMC_MODEL_DENSE_GAUSS) {  // tridiagonal precision
        P.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            P[(size_t)d * D + d] = 1.0 + 0.1 * u();
            if (d) P[(size_t)d * D + d - 1] = P[(size_t)(d - 1) * D + d] = 0.2;
        }
    }
    if (metric == AHMC_METRIC_DIAG) {
        Minv.resize(D);
        for (auto& x : Minv) x = 0.7 + 0.6 * u();
    } else if (metric == AHMC_METRIC_DENSE) {  // diagonal matrices in dense storage: Minv and its Cholesky factor
        Minv.assign((size_t)D * D, 0.0);
        cholU.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            const double s = 0.8 + 0.4 * u();
            Minv[(size_t)d * D + d] = s * s;
            cholU[(size_t)d * D + d] = s;
        }
    }
    for (int c = 0; c < N; ++c) {
        for (int d = 0; d < D; ++d) th[(size_t)c * D + d] = u() - 0.5;
        for (int d = 0; d < D; ++d) {  // -grad log pi and log pi at theta
            double gd = 0.0;
            if (model == AHMC_MODEL_DENSE_GAUSS)
                for (int k = 0; k < D; ++k) gd += P[(size_t)k * D + d] * (th[(size_t)c * D + k] - mu[k]);
            else if (model == AHMC_MODEL_DIAG_GAUSS) gd = (th[(size_t)c * D + d] - mu[d]) * w[d];
            else gd = th[(size_t)c * D + d];
            g[(size_t)c * D + d] = gd;
            lp[c] -= 0.5 * gd * (th[(size_t)c * D + d] - (model == AHMC_MODEL_STD_NORMAL ? 0.0 : mu[d]));
        }
    }
    std::vector<double> o((size_t)3 * N * D), lpo(N), lko(N), acc((size_t)T * N), dH((size_t)T * N), dHm((size_t)T * N);
    std::vector<double> draws((size_t)T * N * D), eps_rw(N, 0.3), minv_rw((size_t)N * D, 0.0), trace((size_t)T * N);
    std::vector<int32_t> ns((size_t)T * N), td((size_t)T * N);
    std::vector<uint8_t> ne((size_t)T * N);
    EmuNuts q{};
    q.model_kind = model; q.metric_kind = metric; q.D = D; q.N = N;
    q.p0 = model == AHMC_MODEL_STD_NORMAL ? nullptr : mu.data();
    q.p1 = model == AHMC_MODEL_DENSE_GAUSS ? P.data() : (model == AHMC_MODEL_DIAG_GAUSS ? w.data() : nullptr);
    q.Minv = Minv.empty() ? nullptr : Minv.data();
    q.cholU = cholU.empty() ? nullptr : cholU.data();
    q.eps = 0.3; q.max_depth = 5; q.delta_max = 1000.0; q.sampler = sampler; q.criterion = criterion;
    q.seed = 11; q.refresh = 1;
    q.th_in = th.data(); q.r_in = r.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.n_steps = ns.data(); q.tree_depth = td.data(); q.numerical = ne.data();
    q.acc = acc.data(); q.dH = dH.data(); q.dHmax = dHm.data(); q.n_transitions = T; q.draws = draws.data();
    if (adapt) {
        q.adapt = 1; q.n_adapts = T - 2; q.init_buffer = 2; q.term_buffer = 2; q.window_size = 3;
        q.delta = 0.8; q.gamma = 0.05; q.t0 = 10.0; q.kappa = 0.75; q.adapt_metric = 1; q.n_min = 3;
        q.eps_rw = eps_rw.data(); q.minv_rw = minv_rw.data(); q.eps_trace = trace.data();
    }
    const int rc = emu_nuts(&q);
    long steps = 0;
    for (auto s : ns) steps += s;
    std::printf("nuts model %d metric %d D %d N %d sampler %d criterion %d adapt %d: rc %d, %ld leapfrog steps\n", model, metric, D, N,
                sampler, criterion, (int)adapt, rc, steps);
    return rc != 0 || steps < (long)T * N;
}

int main() {
    int bad = 0;
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 6, 9, 4, 0, 0, false);    // four chains per warp, ragged last block
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 40, 5, 3, 0, 0, false);   // one chain per warp (or the alt layouts)
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 100, 3, 2, 0, 0, false);  // the headline layout
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, 6, 5, 3, 0, 0, false);  // shared-memory operator slabs
    bad |= run(AHMC_MODEL_FUNNEL, AHMC_METRIC_DIAG, 5, 6, 3, 1, 2, false);        // SliceTS + strict criterion family
    bad |= run(AHMC_MODEL_STD_NORMAL, AHMC_METRIC_UNIT, 3, 7, 3, 0, 1, false);    // classic criterion
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, 40, 11, 2, 0, 0, false);  // COOP form: 8 chains per block share the D x D products
    // in-launch adaptation (chain workspace).  N fills its block: the idle groups of a ragged block alias the LAST chain
    // read-only (`chain = N - 1`, ahmc_nuts_kernel.cuh) and their unused load of its step size would be reported against the
    // owner's write-back of the adapted value -- a benign read, excluded here rather than suppressed.
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 6, 16, 12, 0, 0, true);
    return bad;
}
#endif
