// ahmc_chain_adapt.cuh -- the per-chain `StanHMCAdaptor` of the adaptive persistent launches (K2 adaptive static HMC,
// K3 adaptive NUTS): the reference's vectorised adaptors, one state per chain, updated by the chain's own group right
// after each of its transitions, so no chain waits for another:
//   * NesterovDualAveraging (stepsize.jl:178-210): DAState in registers (every lane of the group holds the same values);
//   * the windowed metric estimator (massmatrix.jl:141-157 WelfordVar, :172-250 NutpieVar, :284-340 WelfordCov) in the
//     chain's workspace, its vectors owned lane-wise like every other group vector (element e of lane l = coordinate
//     l + G*e; WelfordCov's D x D matrix: rows l + G*e of every column);
//   * the window schedule, the reset at window ends (stan_adaptor.jl:13-50, 137-159) and finalize! (stepsize.jl:54-62).
#pragma once
#include "ahmc_kernels.cuh"

namespace ahmc {

// D-vectors of estimator state per chain: none for step size only, (mean, M2) of theta for WelfordVar, and for NutpieVar
// also (mean, M2) of the gradient
__host__ __device__ inline int chain_adapt_vectors(int adapt_metric) {
    return adapt_metric == AHMC_ADAPT_NUTPIE ? 4 : (adapt_metric == AHMC_ADAPT_WELFORD ? 2 : 0);
}
// doubles of estimator state per chain, every estimator: WelfordCov keeps the mean and the full D x D matrix M (D + D^2)
__host__ __device__ inline long long chain_adapt_doubles(int adapt_metric, int D) {
    return adapt_metric == AHMC_ADAPT_WELFORD_COV ? (long long)D + (long long)D * D : (long long)chain_adapt_vectors(adapt_metric) * D;
}

// The metric the trajectories of an adaptive launch read.  The WelfordCov form (Dense metric) reads the chain's own
// Minv_chain / cholU_chain rows when the call provides them -- the launch writes them at every window end -- and the
// call's metric otherwise (step size only); the other forms read the call's metric.
template <int ADAPT>
__device__ __forceinline__ const MetricDev& adapt_launch_metric(const MetricDev& m, const AdaptDev& ad, int D, MetricDev& rows) {
    if constexpr (ADAPT == AHMC_ADAPT_WELFORD_COV) {
        if (!ad.minv || !ad.cholU) return m;
        rows = MetricDev{AHMC_METRIC_DENSE, ad.minv, (long long)D * D, ad.cholU, nullptr, nullptr};
        return rows;
    } else {
        return m;
    }
}

// EST: the compiled estimator form -- AHMC_ADAPT_WELFORD (serves step size only and WelfordVar, selected at run time by
// ad.adapt_metric), AHMC_ADAPT_NUTPIE, or AHMC_ADAPT_WELFORD_COV (Dense metric: step size only or WelfordCov).  A
// compile-time choice, so that the WelfordVar form carries no NutpieVar or WelfordCov code.
//
// The WelfordCov form exchanges data between the lanes of a group (the rank-one update reads every coordinate of the draw,
// the Cholesky factorisation broadcasts pivots through memory), so its entry points (begin_dense, update_cov) are called
// by every lane of the warp at a warp-uniform point, each group with its own `act` predicate.
template <int G, int E, int EST>
struct ChainAdapt {
    double mu, xbar, Hbar, m;  // DAState (stepsize.jl:27-36)
    double n;                  // draws in the estimator's current window
    // (W, the chain's chain_adapt_vectors(adapt_metric) workspace vectors, is passed in by the caller: a kernel recomputes
    //  the address more cheaply than it keeps it in registers)

    static __device__ __forceinline__ void clear(const AdaptDev& ad, double* W, int l, int D) {
        if (!ad.adapt_metric) return;  // step size only: no estimator, no workspace
        if constexpr (EST != AHMC_ADAPT_WELFORD_COV) {  // (WelfordCov: clear_cov, warp-uniform)
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
        if constexpr (EST != AHMC_ADAPT_WELFORD_COV) {
            if (ad.minv) vstore<G, E>(ad.minv + (long long)D * chain, minv, l, D);
        }
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

    // ---- WelfordCov (massmatrix.jl:284-340), Dense metric.  Workspace W: mu[D], then M (D x D, column-major).
    // D x D copy, lanes over the rows of every column
    static __device__ __forceinline__ void mat_copy(double* dst, const double* src, bool act, int l, int D) {
        if (!act) return;
        for (int j = 0; j < D; ++j) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int i = l + G * e;
                if (i < D) dst[i + (long long)D * j] = src[i + (long long)D * j];
            }
        }
    }
    // the empty estimator (reset!, massmatrix.jl:317-322)
    static __device__ __forceinline__ void clear_cov(const AdaptDev& ad, double* W, bool act, int l, int D) {
        if (!act || !ad.adapt_metric) return;
        for (int j = -1; j < D; ++j) {  // j = -1: the mean
            double* col = W + D + (long long)D * j;
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int i = l + G * e;
                if (i < D) col[i] = 0.0;
            }
        }
    }
    // begin: the starting metric of chain `chain` (the call's shared or per-chain M^-1 and factor) into the chain's
    // Minv_chain / cholU_chain rows, so that the launch always reads the chain's own rows; empty estimator
    static __device__ __forceinline__ void begin_dense(const AdaptDev& ad, const MetricDev& m, double* W, bool act, long long chain,
                                                       int l, int D) {
        if (ad.minv && ad.cholU) {  // (the entry points require the metric's factor with an adaptive Dense launch)
            const long long DD = (long long)D * D;
            mat_copy(ad.minv + DD * chain, m.Minv + m.chain_stride * chain, act, l, D);
            if (m.cholU) mat_copy(ad.cholU + DD * chain, m.cholU + m.chain_stride * chain, act, l, D);
        }
        clear_cov(ad, W, act, l, D);
        __syncwarp();
    }
    // push!(::WelfordCov, s) (massmatrix.jl:324-333), literally: delta = s - mu, mu += delta / n, M += (s - mu) * delta'
    // (the full matrix, no symmetrisation); n = draws including this one
    static __device__ __forceinline__ void push_cov(double* W, const double* s, bool act, double n, int l, int D) {
        double mu[E], a[E];
        if (act) {
            double xs[E];
            vload_nc<G, E>(xs, s, l, D);
            vload_nc<G, E>(mu, W, l, D);
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const double dl = xs[e] - mu[e];
                mu[e] = mu[e] + dl / n;
                a[e] = xs[e] - mu[e];
            }
            double* M = W + D;
            for (int j = 0; j < D; ++j) {
                const double dj = s[j] - W[j];  // delta_j: W still holds the previous mean
                double* col = M + (long long)D * j;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int i = l + G * e;
                    if (i < D) col[i] = col[i] + a[e] * dj;
                }
            }
        }
        __syncwarp();  // every lane of the group has read the previous mean
        if (act) vstore<G, E>(W, mu, l, D);
    }
    // get_estimation (massmatrix.jl:335-340) of n >= n_min draws at a window end, then renew(::DenseEuclideanMetric)
    // (metric.jl:105-120): the upper Cholesky factor of Symmetric(M^-1) (its upper triangle).  Row k of the factor is
    //   U[k][j] = (A[k][j] - sum_{m<k} U[m][k] U[m][j]) / U[k][k]  (j > k),   U[k][k] = sqrt(A[k][k] - sum_{m<k} U[m][k]^2)
    // with A = M^-1, lanes over j.  While it is computed the factor lives where neither the metric in use nor the estimate
    // is: U[m][j] (m < j) in the strictly lower triangle of the chain's cholU_chain row (at (j, m); only the upper triangle
    // of a factor is ever read), the diagonal in the estimator's mean (cleared at this window end anyway).  Only when every
    // pivot is positive and finite are the chain's Minv_chain and cholU_chain rows replaced; otherwise -- rounding or
    // non-finite draws, where the reference throws PosDefException -- the chain keeps its previous M^-1 and factor.
    // Returns whether the metric was replaced.
    static __device__ __forceinline__ bool estimate_cov(const AdaptDev& ad, double* W, bool act, double n, long long chain, int l,
                                                        int D) {
        const double c1 = n / ((n + 5.0) * (n - 1.0)), c2 = 1e-3 * (5.0 / (n + 5.0));
        const long long DD = (long long)D * D;
        const double* M = W + D;
        double* dg = W;
        double* Ur = ad.cholU + DD * chain;
        double* Mr = ad.minv + DD * chain;
        __syncwarp();  // M, updated row-wise by every lane, is read along its rows below
        for (int k = 0; k < D; ++k) {
            double v[E];
            if (act) {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int j = l + G * e;
                    v[e] = 0.0;
                    if (j >= k && j < D) {
                        double acc = c1 * M[k + (long long)D * j] + (j == k ? c2 : 0.0);
                        for (int m = 0; m < k; ++m) acc -= Ur[k + (long long)D * m] * Ur[j + (long long)D * m];
                        v[e] = acc;
                        if (j == k) dg[k] = sqrt(acc);
                    }
                }
            }
            __syncwarp();  // the pivot is in memory
            if (act) {
                const double piv = dg[k];
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int j = l + G * e;
                    if (j > k && j < D) Ur[j + (long long)D * k] = v[e] / piv;
                }
            }
            __syncwarp();  // row k is in memory before row k + 1 reads it
        }
        bool ok = true;
        if (act) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int j = l + G * e;
                if (j < D) ok = ok && finite_d(dg[j]) && dg[j] > 0.0;
            }
        }
        ok = Grp<G>::all(ok) && act;
        if (ok) {
            for (int j = 0; j < D; ++j) {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int i = l + G * e;
                    if (i < D) {
                        Mr[i + (long long)D * j] = c1 * M[i + (long long)D * j] + (i == j ? c2 : 0.0);
                        if (i < j) Ur[i + (long long)D * j] = Ur[j + (long long)D * i];
                        else if (i == j) Ur[i + (long long)D * j] = dg[j];
                    }
                }
            }
        }
        __syncwarp();
        if (act) {  // the scratch triangle back to zeros: the factor is upper triangular
            for (int j = 0; j < D; ++j) {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int i = l + G * e;
                    if (i > j && i < D) Ur[i + (long long)D * j] = 0.0;
                }
            }
        }
        __syncwarp();
        return ok;
    }
    // `update` of the WelfordCov form: iteration `it` of a group with `act` produced the draw th (its th_out row) with
    // acceptance statistic alpha; every lane of the warp calls
    __device__ __forceinline__ void update_cov(const AdaptDev& ad, double* W, bool act, int it, long long si, double alpha,
                                               const double* th, double& eps, long long chain, int l, int D) {
        if (act && ad.eps_trace && l == 0) ad.eps_trace[si] = eps;
        const bool in = act && it <= ad.n_adapts;
        if (in) adapt_stepsize(ad, alpha, eps);
        const bool split = in && window_end(ad, it);
        const bool push = in && ad.adapt_metric && it >= ad.window_start && it <= ad.window_end;
        if (push) n += 1.0;
        __syncwarp();  // the draw's coordinates, stored by every lane of the group, are visible to all of them
        if (__any_sync(FULL, push)) push_cov(W, th, push, n, l, D);
        const bool est = push && split && n >= (double)ad.n_min;  // update! (massmatrix.jl:60-62)
        if (__any_sync(FULL, est)) estimate_cov(ad, W, est, n, chain, l, D);
        if (split) reset(eps);  // reset!(ssa); reset!(pc)
        if (__any_sync(FULL, split)) {
            clear_cov(ad, W, split, l, D);
            __syncwarp();
        }
        if (in && it == ad.n_adapts) eps = exp(xbar);  // finalize!
        if (in && l == 0) ad.eps[chain] = eps;
    }
};

}  // namespace ahmc
