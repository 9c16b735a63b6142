// ahmc_bigd.cu -- `step` and `phasepoint` for D > 512 (the reference has no bound on D, src/metric.jl:52-72): the
// register-resident layouts of K1 stop at 512 coordinates per chain, so here a warp STREAMS its chain through registers in
// tiles of 512 coordinates, the state living in the output arrays (L1 / L2 resident between the two passes of a step).
// The step itself is big_step (ahmc_bigd.cuh), shared with the transition and step-size kernels of ahmc_bigd_hmc.cu.
// Targets: std-normal, diagonal Gaussian, Neal's funnel; metrics: Unit, Diag (shared or per chain).  Dense operators at
// D > 512 need the tiled GEMM form inside a CTA-per-tile kernel and are reported as unsupported.
#include "ahmc_bigd.cuh"
#include "ahmc_dispatch.cuh"

namespace ahmc {

template <int MODEL, int METRIC>
__global__ void __launch_bounds__(kBlockThreads) leapfrog_big_kernel(const LeapfrogArgs a) {
    const int l = threadIdx.x % 32;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / 32) + threadIdx.x / 32;
    if (chain0 >= a.N) return;  // whole warps: no cross-warp collectives here
    const long long chain = chain0;
    if (a.only_mask && a.only_mask[chain] == 0) return;
    const int D = a.D;
    double eps = a.eps_chain ? __ldg(a.eps_chain + chain) : a.eps;
    eps = a.fwd ? eps : -eps;  // integrator.jl:226
    BigModel<MODEL> mo{a.model.p0, a.model.p1, a.model.c0, D};
    const double* Mi = METRIC == AHMC_METRIC_DIAG ? a.metric.Minv + a.metric.chain_stride * chain : nullptr;
    double* th = a.th_out + a.ld_out * chain;
    double* r = a.r_out + a.ld_out * chain;
    double* g = a.g_out + a.ld_out * chain;
    // state -> output arrays (in place when z_out aliases z_in)
    for (int d0 = 0; d0 < D; d0 += kBigTile) {
        double t[kBigE];
        if (th != a.th_in + a.ld_in * chain) { tile_load(t, a.th_in + a.ld_in * chain, d0, l, D); tile_store(th, t, d0, l, D); }
        if (r != a.r_in + a.ld_in * chain) { tile_load(t, a.r_in + a.ld_in * chain, d0, l, D); tile_store(r, t, d0, l, D); }
        if (a.g_in && g != a.g_in + a.ld_in * chain) { tile_load(t, a.g_in + a.ld_in * chain, d0, l, D); tile_store(g, t, d0, l, D); }
    }
    __syncwarp();
    bool fin = true;
    if (!a.g_in) big_eval<MODEL>(mo, th, g, l, D, fin);  // no cached gradient: dH/dtheta at the start point
    __syncwarp();
    double lp = 0.0, lk = 0.0;
    int steps = 0;
    fin = true;
    double* dr = a.dr_out ? a.dr_out + a.ld_out * chain : nullptr;
    for (int i = 1; i <= a.n_steps; ++i) {
        const bool f = big_step<MODEL, METRIC>(mo, Mi, eps, th, r, g, dr, l, D, lp, lk);
        steps = i;
        if (!f) {  // the non-finite phase point is what is returned (integrator.jl:252-258)
            fin = false;
            break;
        }
    }
    if (l == 0) {
        a.lp_out[chain] = lp;
        a.lk_out[chain] = lk;
        if (a.status) a.status[chain] = fin ? 0u : AHMC_STATUS_NONFINITE;
        if (a.steps_done) a.steps_done[chain] = steps;
        if (!fin && a.min_break) atomicMin(a.min_break, steps);
    }
}

template <int MODEL, int METRIC>
__global__ void __launch_bounds__(kBlockThreads) phasepoint_big_kernel(const PhasepointArgs a) {
    const int l = threadIdx.x % 32;
    const long long chain = (long long)blockIdx.x * (kBlockThreads / 32) + threadIdx.x / 32;
    if (chain >= a.N) return;
    const int D = a.D;
    BigModel<MODEL> mo{a.model.p0, a.model.p1, a.model.c0, D};
    const double* Mi = METRIC == AHMC_METRIC_DIAG ? a.metric.Minv + a.metric.chain_stride * chain : nullptr;
    bool fin = true;
    const double lp = big_eval<MODEL>(mo, a.th + a.ld * chain, a.g + a.ld * chain, l, D, fin);
    double lk_part = 0.0;
    for (int d0 = 0; d0 < D; d0 += kBigTile) {
        double rr[kBigE], dr[kBigE];
        tile_load(rr, a.r + a.ld * chain, d0, l, D);
#pragma unroll
        for (int e = 0; e < kBigE; ++e) {
            const int d = d0 + l + 32 * e;
            const double mi = METRIC == AHMC_METRIC_DIAG ? (d < D ? __ldg(Mi + d) : 0.0) : 1.0;
            dr[e] = mi * rr[e];
            lk_part = METRIC == AHMC_METRIC_DIAG ? fma(rr[e] * rr[e], mi, lk_part) : fma(rr[e], rr[e], lk_part);
        }
        if (a.dr) tile_store(a.dr + a.ld * chain, dr, d0, l, D);
    }
    const double lk = -0.5 * Grp<32>::sum(lk_part);
    if (l == 0) {
        a.lp[chain] = map_nonfinite(lp);
        a.lk[chain] = map_nonfinite(lk);
    }
}

bool bigd_supported(int model_kind, int metric_kind) {
    return (model_kind == AHMC_MODEL_STD_NORMAL || model_kind == AHMC_MODEL_DIAG_GAUSS || model_kind == AHMC_MODEL_FUNNEL) &&
           (metric_kind == AHMC_METRIC_UNIT || metric_kind == AHMC_METRIC_DIAG);
}

cudaError_t launch_leapfrog_big(const LeapfrogArgs& a, cudaStream_t st) {
    if (!bigd_supported(a.model.kind, a.metric.kind) || a.temper_alpha > 0.0) return cudaErrorNotSupported;
    return with_model_metric(BigModels{}, BigMetrics{}, a.model.kind, a.metric.kind,
                             [&](auto M, auto K) { return launch_warps(leapfrog_big_kernel<M, K>, a.N, 32, 0, st, a); }, cudaErrorNotSupported);
}
cudaError_t launch_phasepoint_big(const PhasepointArgs& a, cudaStream_t st) {
    if (!bigd_supported(a.model.kind, a.metric.kind)) return cudaErrorNotSupported;
    return with_model_metric(BigModels{}, BigMetrics{}, a.model.kind, a.metric.kind,
                             [&](auto M, auto K) { return launch_warps(phasepoint_big_kernel<M, K>, a.N, 32, 0, st, a); }, cudaErrorNotSupported);
}

}  // namespace ahmc
