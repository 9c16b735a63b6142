// lf_emu.cpp -- runs the product's trajectory kernels (K1 leapfrog_kernel, K2 hmc_kernel, phasepoint, momentum; source:
// advancedhmc.jl_b200/csrc/ahmc_leapfrog.cu + ahmc_traj.cuh, unmodified) under the CPU SIMT emulator.
// TEST INFRASTRUCTURE ONLY (tests/test_simt_emulation.py).
#define AHMC_SIMT_EMULATION 1
#include <vector>

#include "ahmc_leapfrog.cu"
#include "emu_smem.h"

EMU_DEFINE_SMEM_ARENA();  // the block's dynamic shared memory (`extern __shared__ double smem[]` in the kernels)
void emu_launch(void (*kernel)(const void*), const void* args, int blocks, int threads);
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
