// lf_emu.cpp -- runs the product's trajectory kernels (K1 leapfrog_kernel, K2 hmc_kernel, phasepoint, momentum; source:
// advancedhmc.jl_b200/csrc/ahmc_leapfrog.cu + ahmc_traj.cuh, unmodified) under the CPU SIMT emulator.
// TEST INFRASTRUCTURE ONLY (tests/test_simt_emulation.py).
#define AHMC_SIMT_EMULATION 1
#include <cstdlib>
#include <cstdio>
#include <vector>

#include "ahmc_leapfrog.cu"
#include "emu_smem.h"
#include "emu_harness.h"

EMU_DEFINE_SMEM_ARENA();  // the block's dynamic shared memory (`extern __shared__ double smem[]` in the kernels)
using namespace ahmc;

struct EmuLf {
    int32_t model_kind, metric_kind, D;
    int64_t N;
    const double *p0, *p1;
    double c0;
    const double* Minv;
    int64_t minv_stride;
    const double* cholU;
    double eps;
    const double* eps_chain;
    int32_t n_steps, fwd;
    double temper_alpha;
    const double *th_in, *r_in, *g_in, *lp_in;
    double *th_out, *r_out, *g_out, *lp_out, *lk_out, *dr_out;
    uint32_t* status;
    int32_t* steps_done;
    uint32_t flags;
    // K2 only
    int32_t hmc, refresh, n_transitions;
    uint64_t seed, offset;
    const double *normal_tape, *exp_tape;
    uint8_t* is_accept;
    double *acc, *dH;
    double* draws;
};
EMU_EXPORT_SIZEOF(EmuLf);

template <int MODEL, int METRIC, int G, int E>
static void lf_thunk(const void* p) { leapfrog_kernel<MODEL, METRIC, G, E>(*static_cast<const LeapfrogArgs*>(p)); }
template <int MODEL, int METRIC, int G, int E>
static void lfc_thunk(const void* p) { leapfrog_kernel<MODEL, METRIC, G, E, true>(*static_cast<const LeapfrogArgs*>(p)); }
template <int MODEL, int METRIC, int G, int E>
static void hmc_thunk(const void* p) { hmc_kernel<MODEL, METRIC, G, E>(*static_cast<const HmcArgs*>(p)); }
typedef void (*KernelFn)(const void*);

template <int MODEL, int METRIC>
static KernelFn pick(int G, int E, bool hmc, bool contig) {
    // full tile D == 64: the lane-contiguous instantiation the product's launcher picks (launch_lf_t)
    if constexpr (FastCapable<MODEL, METRIC>::value)
        if (contig && !hmc && G == 32 && E == 2) return lfc_thunk<MODEL, METRIC, 32, 2>;
    if (G == 4 && E == 1) return hmc ? hmc_thunk<MODEL, METRIC, 4, 1> : lf_thunk<MODEL, METRIC, 4, 1>;
    if (G == 8 && E == 1) return hmc ? hmc_thunk<MODEL, METRIC, 8, 1> : lf_thunk<MODEL, METRIC, 8, 1>;
    if (G == 32 && E == 2) return hmc ? hmc_thunk<MODEL, METRIC, 32, 2> : lf_thunk<MODEL, METRIC, 32, 2>;
    return nullptr;
}

extern "C" int emu_leapfrog(const EmuLf* q) {
    int G, E;
    const int D = q->D;
    if (D <= 4) G = 4, E = 1;
    else if (D <= 8) G = 8, E = 1;
    else if (D > 32 && D <= 64) G = 32, E = 2;
    else return -1;
    LeapfrogArgs a{};
    a.model = ModelDev{q->model_kind, D, q->p0, q->p1, q->c0};
    a.metric = MetricDev{q->metric_kind, q->Minv, q->minv_stride, q->cholU};
    a.D = D;
    a.N = q->N;
    a.eps = q->eps;
    a.eps_chain = q->eps_chain;
    a.n_steps = q->n_steps;
    a.fwd = q->fwd;
    a.temper_alpha = q->temper_alpha;
    a.th_in = q->th_in; a.r_in = q->r_in; a.g_in = q->g_in; a.lp_in = q->lp_in;
    a.ld_in = D;
    a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out; a.dr_out = q->dr_out;
    a.ld_out = D;
    a.status = q->status;
    a.steps_done = q->steps_done;
    a.flags = q->flags;
    HmcArgs h{};
    h.lf = a;
    h.rng = RngDev{q->seed, q->offset, q->normal_tape, q->exp_tape, 1, nullptr, 0, 0.0, q->temper_alpha > 0.0 ? q->temper_alpha : 0.0};
    h.st.is_accept = q->is_accept;
    h.st.acceptance_rate = q->acc;
    h.st.hamiltonian_energy_error = q->dH;
    h.refresh = q->refresh;
    h.n_transitions = q->n_transitions;
    h.draws = q->draws;
    KernelFn fn = nullptr;
    const int m = q->model_kind, me = q->metric_kind;
    const bool hm = q->hmc != 0;
    const bool contig = D == 64 && !(q->flags & AHMC_FLAG_EXACT_CHECKS) && !(q->temper_alpha > 0.0);
    if (m == AHMC_MODEL_STD_NORMAL && me == AHMC_METRIC_UNIT) fn = pick<AHMC_MODEL_STD_NORMAL, AHMC_METRIC_UNIT>(G, E, hm, contig);
    else if (m == AHMC_MODEL_DIAG_GAUSS && me == AHMC_METRIC_DIAG) fn = pick<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG>(G, E, hm, contig);
    else if (m == AHMC_MODEL_FUNNEL && me == AHMC_METRIC_DIAG) fn = pick<AHMC_MODEL_FUNNEL, AHMC_METRIC_DIAG>(G, E, hm, contig);
    else if (m == AHMC_MODEL_DENSE_GAUSS && me == AHMC_METRIC_DENSE) fn = pick<AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE>(G, E, hm, contig);
    if (!fn) return -2;
    const int chains_per_block = kBlockThreads / G;
    const int blocks = (int)((q->N + chains_per_block - 1) / chains_per_block);
    // K1's exact path and K2 use one operator slab per group (the pair kernel: per warp, as G = 32 does); the launcher's
    // occupancy padding for host-memory lanes only adds bytes the kernel never touches
    emu_smem_begin(emu_smem_base(), smem_bytes(m, me, D, G), 0, hm ? "hmc_kernel" : "leapfrog_kernel");
    emu_launch(fn, hm ? (const void*)&h : (const void*)&a, blocks, kBlockThreads);
    emu_smem_end();
    return 0;
}

#ifdef RACE_LF
static int run(int model, int metric, int D, int N, int n, int hmc) {
    std::vector<double> mu(D), w(D), P, Minv, cholU, th((size_t)N * D), r((size_t)N * D), g((size_t)N * D), lp(N, 0.0);
    srand(5 + D);
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
    } else if (metric == AHMC_METRIC_DENSE) {
        Minv.assign((size_t)D * D, 0.0);
        cholU.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            const double s = 0.8 + 0.4 * u();
            Minv[(size_t)d * D + d] = s * s;
            cholU[(size_t)d * D + d] = s;
        }
    }
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {
            th[(size_t)c * D + d] = u() - 0.5;
            r[(size_t)c * D + d] = u() - 0.5;
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
    std::vector<double> o((size_t)4 * N * D), lpo(N), lko(N), acc(N), dH(N);
    std::vector<uint32_t> st(N);
    std::vector<int32_t> done(N);
    std::vector<uint8_t> isacc(N);
    EmuLf q{};
    q.model_kind = model; q.metric_kind = metric; q.D = D; q.N = N; q.p0 = mu.data();
    q.p1 = model == AHMC_MODEL_DENSE_GAUSS ? P.data() : w.data();
    q.Minv = Minv.data(); q.cholU = cholU.empty() ? nullptr : cholU.data(); q.eps = 0.1; q.n_steps = n; q.fwd = 1;
    q.th_in = th.data(); q.r_in = r.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D; q.dr_out = o.data() + (size_t)3 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.status = st.data(); q.steps_done = done.data();
    q.hmc = hmc; q.refresh = 1; q.n_transitions = 1; q.seed = 3; q.is_accept = isacc.data(); q.acc = acc.data(); q.dH = dH.data();
    const int rc = emu_leapfrog(&q);
    std::printf("lf model %d metric %d D %d N %d hmc %d: rc %d lp0 %.6f\n", model, metric, D, N, hmc, rc, lpo[0]);
    return rc != 0;
}

int main() {
    int bad = 0;
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 7, 21, 12, 0);   // K1 fused fast path, four chains per warp, ragged block
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, 6, 9, 6, 0);   // K1 exact path with the shared-memory operator slabs
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 40, 5, 8, 0);    // one chain per warp
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 7, 21, 5, 1);    // K2: refresh + trajectory + Metropolis step
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, 6, 9, 4, 1);
    return bad;
}
#endif
