// ahmc_traj.cuh -- the fused n-step leapfrog trajectory of ONE chain group, shared by K1 (`step`,
// src/integrator.jl:216-265) and K2 (static `transition`, src/trajectory.jl:271-300).
//
// Two code paths (see DESIGN.md "K1"):
//
//  * EXACT (every model x metric): per step the reference's op sequence with FMAs and the reference's
//    `isfinite(z)` test (hamiltonian.jl:141-142); the energies themselves are reduced by warp shuffles only at
//    the step the chain stops on (leapfrog_step_lean: the per-step test is decided from lane partials).  A non-finite
//    chain stops on its own and its phase point AT the break step is what is handed to `done`
//    (integrator.jl:252-258 returns the non-finite z).
//
//  * FAST (separable Gaussian targets STD_NORMAL / DIAG_GAUSS with Unit / Diag metric, no tempering):
//    state in shifted coordinates x = theta - m, the two half kicks of consecutive steps merged,
//    per-coordinate constants a = eps*Minv, b = eps/s^2 precomputed: a step is 2 dependent DFMAs per
//    coordinate and no reduction.  The reference's per-step `isfinite` control flow stays exact by a
//    magnitude argument: with K = (1+max|a|)(1+max|b|) the sup-norm of (x, r) grows by at most K per
//    step, so checking the exponent fields of (x, r) against 2^200 every floor(100/log2 K) steps
//    PROVES that every intermediate phase point, energies included, was finite (|x|,|r| < 2^300,
//    parameters < 2^100, so squares summed over D < 2^31 coordinates stay below 2^731).  A chain that
//    fails a check, or whose parameters are outside the proof's range, is re-run by the exact path in
//    the same launch.  When n*log2(K) <= 240 the periodic test collapses to ONE test of the loaded state
//    against 2^(300 - n*log2 K) (the headline shape: K = 121, n = 32 -> 2^76).
//
// The caller supplies a functor F with
//    void init(double (&th)[E], double (&r)[E], double (&g)[E])   -- (re)materialise the start state
//    void done(th, r, g, dr, lp, lk, fin, steps)                  -- consume the end state (stores)
//    bool has_g()                                                 -- false: init() leaves g unset, recompute it from theta
//    static constexpr bool kContig                                -- true: the fast path uses init_c / done_c, the same
//                                                                    calls on lane-contiguous vectors (ahmc_device.cuh)
//    static constexpr bool kChainMinv                             -- true: a Diag metric's M^-1 is the functor's register
//                                                                    vector minv[E] (a chain adapting its own metric inside
//                                                                    the launch), not `metric.Minv`
// `done` is called exactly once per valid chain, by all lanes of the chain's group.
#pragma once
#include "ahmc_device.cuh"

namespace ahmc {

template <int MODEL, int METRIC>
struct FastCapable {
    static constexpr bool value = (MODEL == AHMC_MODEL_STD_NORMAL || MODEL == AHMC_MODEL_DIAG_GAUSS) &&
                                  (METRIC == AHMC_METRIC_UNIT || METRIC == AHMC_METRIC_DIAG);
};

// The fast path's constants: per coordinate a = eps*Minv, b = eps*w, the mean m and w itself, and the magnitude proof's
// segment length and entry threshold.  One set serves every chain with the same eps and M^-1 (both chains of a K1 pair
// when eps is a scalar and M^-1 is shared).  C: the lane layout of the state vectors (the coefficients follow it).
template <int MODEL, int METRIC, int G, int E, bool C>
struct FastCoef {
    double ca[E], cb[E], mu[E], wi[E];
    double he, inv_eps;
    int cseg, tb;
    bool bad;  // eps or the coefficients outside the proof's range: every chain using them goes to the exact path

    __device__ __forceinline__ void load_model(const ModelDev& model, int l, int D) {
        if constexpr (MODEL == AHMC_MODEL_DIAG_GAUSS) {
            lload<C, G, E>(wi, model.p1, l, D);
            lload<C, G, E>(mu, model.p0, l, D);
        } else {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                wi[e] = lin<C, G, E>(l, e, D) ? 1.0 : 0.0;
                mu[e] = 0.0;
            }
        }
    }
    // mi: the chain's M^-1 (read for a Diag metric only); needs load_model first
    __device__ __forceinline__ void make(const double (&mi)[E], double eps, int n, int l, int D) {
        constexpr int T200 = expo_bits(200), T100 = expo_bits(100), T50 = expo_bits(50);
        // |eps| must be in [2^-100, 2^50] for the proof below and for the 1/eps rescaling of the last step
        inv_eps = 1.0 / eps;
        bad = big_d(eps, T50) | big_d(inv_eps, T100);
        he = 0.5 * eps;
        unsigned amax = 0u, bmax = 0u;  // top 32 bits of max|a|, max|b| (monotone in the magnitude)
#pragma unroll
        for (int e = 0; e < E; ++e) {
            ca[e] = eps * ((METRIC == AHMC_METRIC_DIAG) ? mi[e] : (lin<C, G, E>(l, e, D) ? 1.0 : 0.0));
            cb[e] = eps * wi[e];
            const unsigned ha = (unsigned)__double2hiint(ca[e]) & 0x7fffffffu;
            const unsigned hb = (unsigned)__double2hiint(cb[e]) & 0x7fffffffu;
            amax = ha > amax ? ha : amax;
            bmax = hb > bmax ? hb : bmax;
        }
        amax = grp_umax<G>(amax);
        bmax = grp_umax<G>(bmax);
        bad |= (amax >= 0x7ff00000u) | (bmax >= 0x7ff00000u);  // Inf / NaN coefficients
        // upper bounds of max|a|, max|b| rebuilt from their high words (+1 in the last place of the high word)
        const double Amax = __hiloint2double((int)(amax + 1u), 0);
        const double Bmax = __hiloint2double((int)(bmax + 1u), 0);
        // K = (1+A)(1+B) bounds the per-step growth of max(|x|,|r|); log2(K) <= exponent(K) + 1 = ek
        const double K = (1.0 + Amax) * (1.0 + Bmax);
        int ek = ((__double2hiint(K) >> 20) & 0x7ff) - 1023 + 1;  // K >= 1: ek >= 1
        if (ek > 100 || !(K >= 1.0)) bad = true;                  // also catches NaN / Inf
        ek = ek < 1 ? 1 : (ek > 100 ? 100 : ek);
        // Segments of `cseg` steps, each entered only if max(|x|,|r|) < 2^tb with tb + cseg*ek <= 300: every
        // intermediate phase point of the segment is then below 2^300 and finite, energies included.  When the whole
        // trajectory fits one segment (n*ek <= 240: the entry threshold is still >= 2^60) the test on the loaded state
        // is the only one; otherwise test against 2^200 every floor(100/ek) steps.
        if (n * ek <= 240) {
            cseg = n;
            tb = (1023 + 300 - n * ek) << 20;
        } else {
            cseg = 100 / ek;
            tb = T200;
        }
    }
    // shifted coordinate x = theta - m and the first half kick, which uses the CACHED gradient (integrator.jl:237);
    // without one it is recomputed exactly as ModelOps::eval does: (theta - m) * w
    __device__ __forceinline__ void enter(double (&x)[E], double (&r)[E], const double (&g0)[E], bool have_g) const {
#pragma unroll
        for (int e = 0; e < E; ++e) {
            x[e] = x[e] - mu[e];
            const double ge = have_g ? g0[e] : ((MODEL == AHMC_MODEL_DIAG_GAUSS) ? x[e] * wi[e] : x[e]);
            r[e] = fma(-he, ge, r[e]);
        }
    }
    // the first segment's entry test
    __device__ __forceinline__ bool test(const double (&x)[E], const double (&r)[E]) const {
        bool s = false;
#pragma unroll
        for (int e = 0; e < E; ++e) s |= big_d(x[e], tb) | big_d(r[e], tb);
        return s;
    }
    // the first n - 1 steps (2 dependent DFMAs per coordinate), testing the entry of every later segment
    __device__ __forceinline__ bool steps(double (&x)[E], double (&r)[E], int n) const {
        bool s = false;
        int left = n;  // steps still to take; the last one is the split (drift, gradient, half kick, energies) step
        for (;;) {
            const bool last = left <= cseg;
            const int m = last ? left - 1 : cseg;
            for (int j = 0; j < m; ++j) {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    x[e] = fma(ca[e], r[e], x[e]);
                    r[e] = fma(-cb[e], x[e], r[e]);
                }
            }
            if (last) break;
            left -= m;
#pragma unroll
            for (int e = 0; e < E; ++e) s |= big_d(x[e], tb) | big_d(r[e], tb);
        }
        return s;
    }
    // last step: drift, gradient, half kick, energies (x back to theta).  g = x*w and dH/dr = Minv*r are recovered from the
    // per-coordinate constants as (x*b)/eps and (r*a)/eps (one extra rounding, ~1e-16 relative)
    __device__ __forceinline__ void last(double (&x)[E], double (&r)[E], double (&g)[E], double (&dr)[E], double& lp,
                                         double& lk, double c0, int l, int D) const {
        double lp_part = 0.0, lk_part = 0.0;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            x[e] = fma(ca[e], r[e], x[e]);
            g[e] = (MODEL == AHMC_MODEL_DIAG_GAUSS) ? (x[e] * cb[e]) * inv_eps : (lin<C, G, E>(l, e, D) ? x[e] : 0.0);
            r[e] = fma(-he, g[e], r[e]);
            lp_part = fma(x[e], g[e], lp_part);
            dr[e] = (METRIC == AHMC_METRIC_DIAG) ? (r[e] * ca[e]) * inv_eps : r[e];
            lk_part = fma(r[e], dr[e], lk_part);
            x[e] = x[e] + mu[e];
        }
        lp = fma(-0.5, Grp<G>::sum(lp_part), c0);
        lk = -0.5 * Grp<G>::sum(lk_part);
    }
};

// The exact path of a chain group: every model x metric, run only when some group of the warp needs it (need_exact: a
// valid chain that is not already done).  Called by all lanes of the warp.
template <int MODEL, int METRIC, int G, int E, class F>
__device__ __forceinline__ void exact_trajectory(const ModelDev& model, const MetricDev& metric, int D, long long chain,
                                                 bool need_exact, int l, double* xs, double eps, int n,
                                                 double temper_alpha, F& f) {
    if (!__any_sync(FULL, need_exact)) return;

    ModelOps<MODEL, G, E> mo;
    MetricOps<METRIC, G, E> me;
    mo.load(model, l, D);
    me.load(metric, chain, l, D);
    if constexpr (F::kChainMinv) {
#pragma unroll
        for (int e = 0; e < E; ++e) me.Minv[e] = f.minv[e];
    }
    ChainState<E> s;
    f.init(s.th, s.r, s.g);
    if (!f.has_g()) mo.eval(s.th, s.g, xs, l);  // no cached gradient handed over: dH/dtheta at the start point
    s.lp = 0.0;
    s.lk = 0.0;
    double dr[E];
    const double sa = temper_alpha > 0.0 ? sqrt(temper_alpha) : 1.0;
    bool active = need_exact;
    for (int i = 1; i <= n; ++i) {
        double t1 = 1.0, t2 = 1.0;
        if (temper_alpha > 0.0) {  // integrator.jl:198-209
            t1 = (2 * (i - 1) + 1 <= n) ? sa : 1.0 / sa;
            t2 = (2 * (i - 1) + 2 <= n) ? sa : 1.0 / sa;
        }
        const bool fin = leapfrog_step_lean<MODEL, METRIC, G, E>(s, mo, me, eps, dr, xs, l, t1, t2, i == n);
        if (active && (!fin || i == n)) {
            f.done(s.th, s.r, s.g, dr, s.lp, s.lk, fin, i);
            active = false;
        }
        if (!__any_sync(FULL, active)) break;
    }
}

template <int MODEL, int METRIC, int G, int E, class F>
__device__ __forceinline__ void run_trajectory(const ModelDev& model, const MetricDev& metric, int D,
                                               long long chain, bool valid, int l, double* xs, double eps, int n,
                                               double temper_alpha, uint32_t flags, F& f) {
    bool need_exact = valid;

    if constexpr (FastCapable<MODEL, METRIC>::value) {
        const bool fast_on = !(flags & AHMC_FLAG_EXACT_CHECKS) && !(temper_alpha > 0.0);
        if (fast_on) {
            constexpr bool C = F::kContig;
            FastCoef<MODEL, METRIC, G, E, C> k;
            double x[E], r[E];
            {
                double g0[E], mi[E];
                if constexpr (C) f.init_c(x, r, g0);
                else f.init(x, r, g0);
                if constexpr (METRIC == AHMC_METRIC_DIAG) {
                    if constexpr (F::kChainMinv) {
#pragma unroll
                        for (int e = 0; e < E; ++e) mi[e] = f.minv[e];
                    } else {
                        lload<C, G, E>(mi, metric.Minv + metric.chain_stride * chain, l, D);
                    }
                }
                k.load_model(model, l, D);
                k.make(mi, eps, n, l, D);
                k.enter(x, r, g0, f.has_g());
            }
            bool suspicious = k.bad | k.test(x, r);
            suspicious |= k.steps(x, r, n);
            double g[E], dr[E], lp, lk;
            k.last(x, r, g, dr, lp, lk, model.c0, l, D);
            suspicious = Grp<G>::any(suspicious);
            need_exact = valid && suspicious;
            if (valid && !suspicious) {  // finite by the magnitude proof
                if constexpr (C) f.done_c(x, r, g, dr, lp, lk, true, n);
                else f.done(x, r, g, dr, lp, lk, true, n);
            }
        }
    }
    exact_trajectory<MODEL, METRIC, G, E>(model, metric, D, chain, need_exact, l, xs, eps, n, temper_alpha, f);
}

}  // namespace ahmc
