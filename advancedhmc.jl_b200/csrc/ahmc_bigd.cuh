// ahmc_bigd.cuh -- the device code every D > 512 kernel shares (ahmc_bigd.cu: `step`, `phasepoint`; ahmc_bigd_hmc.cu:
// `rand_momentum`, static transitions with and without in-launch adaptation, `find_good_stepsize`).  A warp STREAMS its
// chain through registers in tiles of 512 coordinates (the same 32 lanes x 16 coordinates vector ops as the widest
// register-resident layout); coordinate d of a tile is owned by lane d mod 32, so a lane only ever re-reads what it wrote
// itself, and the only cross-lane traffic is the warp reductions and the funnel's theta_1.
#pragma once
#include "ahmc_kernels.cuh"

namespace ahmc {

constexpr int kBigE = 16, kBigTile = 32 * kBigE;  // coordinates per tile

template <int MODEL>
struct BigModel {
    const double *m, *w;
    double c0;
    int D;
    // per-tile contribution to the quantity the gradient needs from the whole vector (funnel: sum_{d>=1} th_d^2)
    __device__ __forceinline__ double pre(const double (&th)[kBigE], int d0, int l) const {
        double p = 0.0;
        if (MODEL == AHMC_MODEL_FUNNEL) {
#pragma unroll
            for (int e = 0; e < kBigE; ++e) {
                const int d = d0 + l + 32 * e;
                if (d >= 1 && d < D) p = fma(th[e], th[e], p);
            }
        }
        return p;
    }
    // g tile (MINUS gradient) and the tile's lp partial; v, ev, S: funnel globals (S = e^{-v} sum_{d>=1} th_d^2)
    __device__ __forceinline__ double grad(const double (&th)[kBigE], double (&g)[kBigE], int d0, int l, double v, double ev, double S) const {
        double part = 0.0;
#pragma unroll
        for (int e = 0; e < kBigE; ++e) {
            const int d = d0 + l + 32 * e;
            const bool in = d < D;
            if (MODEL == AHMC_MODEL_STD_NORMAL) {
                g[e] = in ? th[e] : 0.0;
                part = fma(g[e], g[e], part);
            } else if (MODEL == AHMC_MODEL_DIAG_GAUSS) {
                const double diff = in ? th[e] - __ldg(m + d) : 0.0;
                g[e] = in ? diff * __ldg(w + d) : 0.0;
                part = fma(diff, g[e], part);
            } else {  // funnel
                if (d == 0) g[e] = v / 9.0 - (S - (double)(D - 1)) * 0.5;
                else g[e] = in ? th[e] * ev : 0.0;
            }
        }
        return part;
    }
    __device__ __forceinline__ double lp(double part_sum, double v, double S) const {
        if (MODEL == AHMC_MODEL_FUNNEL) return c0 - v * v / 18.0 - (S + (double)(D - 1) * v) * 0.5;
        return fma(-0.5, part_sum, c0);
    }
};

__device__ __forceinline__ void tile_load(double (&x)[kBigE], const double* base, int d0, int l, int D) {
#pragma unroll
    for (int e = 0; e < kBigE; ++e) {
        const int d = d0 + l + 32 * e;
        x[e] = d < D ? base[d] : 0.0;
    }
}
__device__ __forceinline__ void tile_store(double* base, const double (&x)[kBigE], int d0, int l, int D) {
#pragma unroll
    for (int e = 0; e < kBigE; ++e) {
        const int d = d0 + l + 32 * e;
        if (d < D) base[d] = x[e];
    }
}
// gradient / lp of the chain's current theta (in `th` array, global), written to g; returns lp (all lanes) and finiteness of g
template <int MODEL>
__device__ __forceinline__ double big_eval(const BigModel<MODEL>& mo, const double* th, double* g, int l, int D, bool& fin) {
    double S = 0.0, v = 0.0, ev = 0.0;
    if (MODEL == AHMC_MODEL_FUNNEL) {
        for (int d0 = 0; d0 < D; d0 += kBigTile) {
            double t[kBigE];
            tile_load(t, th, d0, l, D);
            S += mo.pre(t, d0, l);
        }
        v = th[0];
        ev = exp(-v);
        S = Grp<32>::sum(S) * ev;
    }
    double part = 0.0;
    for (int d0 = 0; d0 < D; d0 += kBigTile) {
        double t[kBigE], gg[kBigE];
        tile_load(t, th, d0, l, D);
        part += mo.grad(t, gg, d0, l, v, ev, S);
#pragma unroll
        for (int e = 0; e < kBigE; ++e) fin = fin && finite_d(gg[e]);
        tile_store(g, gg, d0, l, D);
    }
    return mo.lp(Grp<32>::sum(part), v, S);
}

// ONE leapfrog step (src/integrator.jl:235-247) of a chain whose state (th, r, g = -grad lp) lives in global memory and
// is updated in place; every D > 512 kernel integrates with this, so a step is the same arithmetic everywhere.
//   pass 1 over the tiles:  r -= eps/2 g;  theta += eps dH/dr(r);  accumulate what the gradient needs from ALL of theta
//                           (the funnel's sum over i >= 2 of theta_i^2 e^{-v});
//   pass 2 over the tiles:  g = -grad lp(theta);  r -= eps/2 g;  accumulate lp, the kinetic energy and the isfinite test.
// Mi: the chain's Diag M^-1 (METRIC == AHMC_METRIC_DIAG); dr_out: nullable, receives dH/dr.  Returns isfinite(z)
// (hamiltonian.jl:141-142); lp and lk come back with a non-finite value mapped to -Inf.  MINV_RO = false: M^-1 is written
// by the same launch (a chain adapting its own metric), so it is not read through the read-only data cache.
template <bool MINV_RO>
__device__ __forceinline__ double big_minv(const double* Mi, int d) { return MINV_RO ? __ldg(Mi + d) : Mi[d]; }
template <int MODEL, int METRIC, bool MINV_RO = true>
__device__ __forceinline__ bool big_step(const BigModel<MODEL>& mo, const double* Mi, double eps, double* th, double* r, double* g,
                                         double* dr_out, int l, int D, double& lp, double& lk) {
    const double he = 0.5 * eps;
    // pass 1: half kick with the cached gradient, drift
    double S = 0.0;
    for (int d0 = 0; d0 < D; d0 += kBigTile) {
        double t[kBigE], rr[kBigE], gg[kBigE];
        tile_load(t, th, d0, l, D);
        tile_load(rr, r, d0, l, D);
        tile_load(gg, g, d0, l, D);
#pragma unroll
        for (int e = 0; e < kBigE; ++e) {
            const int d = d0 + l + 32 * e;
            rr[e] = fma(-he, gg[e], rr[e]);
            const double dr = METRIC == AHMC_METRIC_DIAG ? (d < D ? big_minv<MINV_RO>(Mi, d) : 0.0) * rr[e] : rr[e];
            t[e] = fma(eps, dr, t[e]);
        }
        S += mo.pre(t, d0, l);
        tile_store(th, t, d0, l, D);
        tile_store(r, rr, d0, l, D);
    }
    __syncwarp();
    double v = 0.0, ev = 0.0;
    if (MODEL == AHMC_MODEL_FUNNEL) {
        v = th[0];
        ev = exp(-v);
        S = Grp<32>::sum(S) * ev;
    }
    // pass 2: gradient at the new position, second half kick, energies, isfinite(z) (hamiltonian.jl:141-142)
    double lp_part = 0.0, lk_part = 0.0;
    bool f = true;
    for (int d0 = 0; d0 < D; d0 += kBigTile) {
        double t[kBigE], rr[kBigE], gg[kBigE], dr[kBigE];
        tile_load(t, th, d0, l, D);
        tile_load(rr, r, d0, l, D);
        lp_part += mo.grad(t, gg, d0, l, v, ev, S);
#pragma unroll
        for (int e = 0; e < kBigE; ++e) {
            const int d = d0 + l + 32 * e;
            rr[e] = fma(-he, gg[e], rr[e]);
            const double mi = METRIC == AHMC_METRIC_DIAG ? (d < D ? big_minv<MINV_RO>(Mi, d) : 0.0) : 1.0;
            dr[e] = mi * rr[e];
            lk_part = METRIC == AHMC_METRIC_DIAG ? fma(rr[e] * rr[e], mi, lk_part) : fma(rr[e], rr[e], lk_part);
            f = f && finite_d(gg[e]) && finite_d(dr[e]);
        }
        tile_store(r, rr, d0, l, D);
        tile_store(g, gg, d0, l, D);
        if (dr_out) tile_store(dr_out, dr, d0, l, D);
    }
    __syncwarp();
    lp = mo.lp(Grp<32>::sum(lp_part), v, S);
    lk = -0.5 * Grp<32>::sum(lk_part);
    f = Grp<32>::all(f) && finite_d(lp) && finite_d(lk);
    lp = map_nonfinite(lp);
    lk = map_nonfinite(lk);
    return f;
}

}  // namespace ahmc
