// ahmc_chain_adapt.cuh -- the per-chain `StanHMCAdaptor` of the adaptive persistent launches (K2 adaptive static HMC,
// K3 adaptive NUTS): the reference's vectorised adaptors, one state per chain, updated by the chain's own group right
// after each of its transitions, so no chain waits for another:
//   * NesterovDualAveraging (stepsize.jl:178-210): DAState in registers (every lane of the group holds the same values);
//   * the windowed metric estimator (massmatrix.jl:141-157 WelfordVar, :172-250 NutpieVar) in the chain's workspace, its
//     vectors owned lane-wise like every other group vector (element e of lane l = coordinate l + G*e);
//   * the window schedule, the reset at window ends (stan_adaptor.jl:13-50, 137-159) and finalize! (stepsize.jl:54-62).
#pragma once
#include "ahmc_kernels.cuh"

namespace ahmc {

// D-vectors of estimator state per chain: none for step size only, (mean, M2) of theta for WelfordVar, and for NutpieVar
// also (mean, M2) of the gradient
__host__ __device__ inline int chain_adapt_vectors(int adapt_metric) {
    return adapt_metric == AHMC_ADAPT_NUTPIE ? 4 : (adapt_metric == AHMC_ADAPT_WELFORD ? 2 : 0);
}

// EST: the compiled estimator form -- AHMC_ADAPT_WELFORD (serves step size only and WelfordVar, selected at run time by
// ad.adapt_metric) or AHMC_ADAPT_NUTPIE.  A compile-time choice, so that the WelfordVar form carries no NutpieVar code.
template <int G, int E, int EST>
struct ChainAdapt {
    double mu, xbar, Hbar, m;  // DAState (stepsize.jl:27-36)
    double n;                  // draws in the estimator's current window
    // (W, the chain's chain_adapt_vectors(adapt_metric) workspace vectors, is passed in by the caller: a kernel recomputes
    //  the address more cheaply than it keeps it in registers)

    static __device__ __forceinline__ void clear(const AdaptDev& ad, double* W, int l, int D) {
        if (!ad.adapt_metric) return;  // step size only: no estimator, no workspace
        double zero[E];
#pragma unroll
        for (int e = 0; e < E; ++e) zero[e] = 0.0;
        vstore<G, E>(W, zero, l, D);
        vstore<G, E>(W + D, zero, l, D);
        if constexpr (EST == AHMC_ADAPT_NUTPIE) {
            vstore<G, E>(W + 2LL * D, zero, l, D);
            vstore<G, E>(W + 3LL * D, zero, l, D);
        }
    }

    // push! of x into the Welford state (WMU, WMU + D) (massmatrix.jl:141-149), n = draws including this one; with `est`,
    // get_estimation (:152-157) of each coordinate goes through out(e, estimate)
    template <class Out>
    static __device__ __forceinline__ void push(double* WMU, const double* x, double n, bool est, int l, int D, Out out) {
        double xs[E], wmu[E], wm2[E];
        vload_nc<G, E>(xs, x, l, D);
        vload_nc<G, E>(wmu, WMU, l, D);
        vload_nc<G, E>(wm2, WMU + D, l, D);
        const double f = (n - 1.0) / n;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const double dl = xs[e] - wmu[e];
            wmu[e] = wmu[e] + dl / n;
            wm2[e] = wm2[e] + dl * dl * f;
        }
        if (est) {
            const double c1 = n / ((n + 5.0) * (n - 1.0)), c2 = 1e-3 * (5.0 / (n + 5.0));
#pragma unroll
            for (int e = 0; e < E; ++e) out(e, c1 * wm2[e] + c2);
        }
        vstore<G, E>(WMU, wmu, l, D);
        vstore<G, E>(WMU + D, wm2, l, D);
    }

    // adapt_stepsize! (stepsize.jl:178-210), one chain, with acceptance statistic alpha
    __device__ __forceinline__ void adapt_stepsize(const AdaptDev& ad, double alpha, double& eps) {
        const double amin = (alpha != alpha) ? alpha : (alpha < 1.0 ? alpha : 1.0);  // min(1, alpha)
        const double m1 = m + 1.0;
        const double eta_H = 1.0 / (m1 + ad.t0);
        const double Hn = (1.0 - eta_H) * Hbar + eta_H * (ad.delta - amin);
        const double x = mu - Hn * (sqrt(m1) / ad.gamma);
        const double eta_x = pow(m1, -ad.kappa);
        const double xn = (1.0 - eta_x) * xbar + eta_x * x;
        const double en = exp(x);
        if (finite_d(en)) {  // else the previous state stays (stepsize.jl:199-203, per chain)
            m = m1;
            Hbar = Hn;
            xbar = xn;
            eps = en;
        }
    }
    // is_window_end (stan_adaptor.jl:135)
    static __device__ __forceinline__ bool window_end(const AdaptDev& ad, int it) {
        bool split = false;
        for (int q = 0; q < ad.n_splits; ++q) split = split || (ad.splits[q] == it);
        return split;
    }
    // the scalar part of the reset at a window end: reset!(ssa) and the estimator's draw count
    __device__ __forceinline__ void reset(double eps) {
        m = 0.0;
        mu = log(10.0 * eps);
        xbar = Hbar = 0.0;
        n = 0.0;
    }

    // DAState(eps) and empty estimators (massmatrix.jl:109-118); reports the starting eps and M^-1
    __device__ __forceinline__ void begin(const AdaptDev& ad, double* W, double eps, const double (&minv)[E], long long chain, int l,
                                          int D) {
        mu = log(10.0 * eps);
        xbar = Hbar = m = n = 0.0;
        clear(ad, W, l, D);
        if (ad.minv) vstore<G, E>(ad.minv + (long long)D * chain, minv, l, D);
        if (l == 0) ad.eps[chain] = eps;
    }

    // iteration `it` (1-based, sampler.jl:182) produced the draw (th, g = -grad lp; the sign is irrelevant to a variance)
    // with acceptance statistic alpha; si = (it - 1) * N + chain.  Updates eps and minv (the chain's M^-1, in registers).
    __device__ __forceinline__ void update(const AdaptDev& ad, double* W, int it, long long si, double alpha, const double* th,
                                           const double* g, double& eps, double (&minv)[E], long long chain, int l, int D) {
        if (ad.eps_trace && l == 0) ad.eps_trace[si] = eps;
        if (it > ad.n_adapts) return;
        adapt_stepsize(ad, alpha, eps);
        const bool split = window_end(ad, it);
        if (ad.adapt_metric && it >= ad.window_start && it <= ad.window_end) {
            if constexpr (EST == AHMC_ADAPT_NUTPIE) {
                // NutpieVar (massmatrix.jl:235-248): positions and gradients, M^-1 = sqrt(est(theta) ./ est(gradient));
                // est(gradient) is parked in minv, which is overwritten only at an estimate
                n += 1.0;
                const bool est = split && n >= (double)ad.n_min;  // update! (massmatrix.jl:60-62)
                push(W + 2LL * D, g, n, est, l, D, [&](int e, double v) { minv[e] = v; });
                push(W, th, n, est, l, D, [&](int e, double v) { minv[e] = sqrt(v / minv[e]); });
                if (est) {
#pragma unroll
                    for (int e = 0; e < E; ++e) minv[e] = (l + G * e < D) ? minv[e] : 0.0;
                    vstore<G, E>(ad.minv + (long long)D * chain, minv, l, D);
                }
            } else {
                // push!(::WelfordVar, theta) (massmatrix.jl:141-149) with the new draw
                double th_new[E], wmu[E], wm2[E];
                vload_nc<G, E>(th_new, th, l, D);
                vload_nc<G, E>(wmu, W, l, D);
                vload_nc<G, E>(wm2, W + D, l, D);
                n += 1.0;
                const double f = (n - 1.0) / n;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const double dl = th_new[e] - wmu[e];
                    wmu[e] = wmu[e] + dl / n;
                    wm2[e] = wm2[e] + dl * dl * f;
                }
                if (split && n >= (double)ad.n_min) {  // update! + get_estimation (massmatrix.jl:60-62, 152-157)
                    const double c1 = n / ((n + 5.0) * (n - 1.0)), c2 = 1e-3 * (5.0 / (n + 5.0));
#pragma unroll
                    for (int e = 0; e < E; ++e) minv[e] = (l + G * e < D) ? c1 * wm2[e] + c2 : 0.0;
                    vstore<G, E>(ad.minv + (long long)D * chain, minv, l, D);
                }
                vstore<G, E>(W, wmu, l, D);
                vstore<G, E>(W + D, wm2, l, D);
            }
        }
        if (split) {  // reset!(ssa); reset!(pc) (stan_adaptor.jl:155-158; stepsize.jl:38-52)
            reset(eps);
            clear(ad, W, l, D);
        }
        if (it == ad.n_adapts) eps = exp(xbar);  // finalize! (stepsize.jl:54-62)
        if (l == 0) ad.eps[chain] = eps;
    }
};

}  // namespace ahmc
