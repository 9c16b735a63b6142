// user_group_emu.cpp -- runs the product's kernels (phasepoint, the K1 trajectory, NUTS; sources ahmc_leapfrog.cu,
// ahmc_traj.cuh, ahmc_nuts_kernel.cuh, unmodified) for a run-time compiled target in the GROUP form (AHMC_USER_GROUPWISE:
// every lane of the chain's group runs ahmc_user_logp_grad_group) under the CPU SIMT emulator.  The target is Neal's funnel,
// written as a user would hand it to NVRTC.  A shuffle or __syncwarp here is a barrier of all 32 lanes of the warp, so a
// call site of the model that some lane of the warp does not reach would never return.
// TEST INFRASTRUCTURE ONLY (tests/test_user_group_cpu.py).
#define AHMC_SIMT_EMULATION 1
#define AHMC_NVRTC_USER_MODEL 1
#define AHMC_USER_GROUPWISE 1
#include <vector>

#include "ahmc_leapfrog.cu"
#include "ahmc_nuts_kernel.cuh"

namespace ahmc {
double smem[1 << 16];
}
void emu_launch(void (*kernel)(const void*), const void* args, int blocks, int threads);
using namespace ahmc;

// the user's source (the funnel tests/test_user_group_cpu.py compiles with NVRTC): lane 0 broadcasts e^-v, lane l of the
// group owns the coordinates d = l + G k, the sum of th_d^2 e^-v over them is reduced across the group, lane 0 adds the
// v terms
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    (void)p;
    const double v = th[0];
    const double ev = ahmc_group_bcast(grp, grp.lane == 0 ? exp(-v) : 0.0, 0);
    double s = 0.0;
    for (int d = grp.lane; d < D; d += grp.size) {
        if (d == 0) continue;
        const double gd = th[d] * ev;
        g[d] = -gd;
        s = fma(th[d], gd, s);
    }
    ahmc_group_sync(grp);
    const double S = ahmc_group_sum(grp, s);
    if (grp.lane != 0) return 0.0;
    g[0] = -v / 9.0 + (S - (D - 1)) * 0.5;
    return -v * v / 18.0 - (S + (D - 1) * v) * 0.5;
}

struct EmuUser {
    int32_t op;  // 0 phasepoint, 1 fused trajectory (K1), 2 one NUTS transition (MultinomialTS + GeneralisedNoUTurn)
    int32_t metric_kind, D;
    int64_t N;
    double c0;
    const double *Minv, *cholU;
    double eps;
    int32_t n_steps, max_depth;
    const double* exp_tape;
    int64_t exp_stride;
    const uint8_t* dir_tape;
    int64_t dir_stride;
    const double *th_in, *r_in, *g_in, *lp_in;  // g_in nullable for op 1: the gradient is then evaluated at the start
    double *th_out, *r_out, *g_out, *lp_out, *lk_out;
    int32_t *steps, *tree_depth;
    uint8_t* numerical;
    double* acc;
};

template <int M, int G, int E>
static void pp_thunk(const void* p) { phasepoint_kernel<AHMC_MODEL_USER, M, G, E>(*static_cast<const PhasepointArgs*>(p)); }
template <int M, int G, int E>
static void lf_thunk(const void* p) { leapfrog_kernel<AHMC_MODEL_USER, M, G, E>(*static_cast<const LeapfrogArgs*>(p)); }
template <int M, int G, int E>
static void nuts_thunk(const void* p) { nuts_kernel<AHMC_MODEL_USER, M, G, E, false, 0, false>(*static_cast<const NutsArgs*>(p)); }
typedef void (*KernelFn)(const void*);

template <int M, int G, int E>
static KernelFn pick_op(int op) { return op == 0 ? pp_thunk<M, G, E> : op == 1 ? lf_thunk<M, G, E> : nuts_thunk<M, G, E>; }
template <int M>
static KernelFn pick(int op, int G, int E) {
    if (G == 4 && E == 1) return pick_op<M, 4, 1>(op);
    if (G == 32 && E == 1) return pick_op<M, 32, 1>(op);
    if (G == 32 && E == 2) return pick_op<M, 32, 2>(op);
    return nullptr;
}

extern "C" int emu_user_group(const EmuUser* q) {
    int G, E;
    const int D = q->D;
    if (!pick_layout(D, &G, &E)) return -1;
    KernelFn fn = q->metric_kind == AHMC_METRIC_UNIT   ? pick<AHMC_METRIC_UNIT>(q->op, G, E)
                  : q->metric_kind == AHMC_METRIC_DIAG ? pick<AHMC_METRIC_DIAG>(q->op, G, E)
                                                       : pick<AHMC_METRIC_DENSE>(q->op, G, E);
    if (!fn) return -2;
    const ModelDev model{AHMC_MODEL_USER, D, nullptr, nullptr, q->c0};
    const MetricDev metric{q->metric_kind, q->Minv, 0, q->cholU};
    const int blocks = (int)((q->N + kBlockThreads / G - 1) / (kBlockThreads / G));
    PhasepointArgs pa{};
    LeapfrogArgs la{};
    NutsArgs na{};
    std::vector<double> scratch;
    const void* args = nullptr;
    if (q->op == 0) {
        pa.model = model; pa.metric = metric; pa.D = D; pa.N = q->N;
        pa.th = q->th_in; pa.r = q->r_in; pa.lp = q->lp_out; pa.g = q->g_out; pa.lk = q->lk_out; pa.dr = nullptr;
        pa.ld = D;
        args = &pa;
    } else if (q->op == 1) {
        la.model = model; la.metric = metric; la.D = D; la.N = q->N;
        la.eps = q->eps; la.n_steps = q->n_steps; la.fwd = 1;
        la.th_in = q->th_in; la.r_in = q->r_in; la.g_in = q->g_in; la.lp_in = q->lp_in;
        la.ld_in = D;
        la.th_out = q->th_out; la.r_out = q->r_out; la.g_out = q->g_out; la.lp_out = q->lp_out; la.lk_out = q->lk_out;
        la.ld_out = D;
        la.steps_done = q->steps;
        la.flags = AHMC_FLAG_EXACT_CHECKS;
        args = &la;
    } else {
        na.model = model; na.metric = metric; na.D = D; na.N = q->N;
        na.eps = q->eps; na.max_depth = q->max_depth; na.delta_max = 1000.0;
        na.rng = RngDev{1, 0, nullptr, q->exp_tape, q->exp_stride, q->dir_tape, q->dir_stride, 0.0, 0.0};
        na.refresh = 0;
        na.th_in = q->th_in; na.r_in = q->r_in; na.g_in = q->g_in; na.lp_in = q->lp_in;
        na.ld_in = D;
        na.th_out = q->th_out; na.r_out = q->r_out; na.g_out = q->g_out; na.lp_out = q->lp_out; na.lk_out = q->lk_out;
        na.ld_out = D;
        na.st.n_steps = q->steps;
        na.st.tree_depth = q->tree_depth;
        na.st.numerical_error = q->numerical;
        na.st.acceptance_rate = q->acc;
        na.n_transitions = 1;
        const long long stride = nuts_level_doubles(D, q->max_depth);
        scratch.assign((size_t)stride * (size_t)q->N, 0.0);
        na.scratch = scratch.data();
        na.scratch_stride = stride;
        args = &na;
    }
    emu_launch(fn, args, blocks, kBlockThreads);
    return 0;
}
