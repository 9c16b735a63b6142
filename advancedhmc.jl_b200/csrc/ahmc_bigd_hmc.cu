// ahmc_bigd_hmc.cu -- sampling for D > 512 in the streaming form of ahmc_bigd.cuh (one warp per chain, tiles of 512
// coordinates, the chain's vectors in global memory): `rand_momentum` (metric.jl:290-320), the static EndPointTS
// transition as the persistent loop of hmc_kernel (sampler.jl:182, trajectory.jl:271-300, 863-880), its in-launch
// adaptive form (the per-chain StanHMCAdaptor of ahmc_chain_adapt.cuh) and the one-launch `find_good_stepsize`
// (trajectory.jl:768-837).  Every leapfrog step is big_step, the step of `step` at D > 512.
//
// Per-chain workspace (HmcArgs::scratch, FindEpsArgs::scratch), D-vectors:
//   transition:  theta0, g0, r0 -- the start point and its refreshed momentum, so that a reverted transition restores
//                theta, -grad lp and lp bit for bit even when z_out aliases z_in (the trajectory runs in z_out);
//                then the adaptor's estimator (2 WelfordVar, 4 NutpieVar) in tile blocks, see BigChainAdapt;
//   find_eps:    r0, then the probe's theta, r, g (the start theta and g stay in the read-only input).
#include "ahmc_bigd.cuh"
#include "ahmc_chain_adapt.cuh"
#ifndef AHMC_SIMT_EMULATION
#include "ahmc_dispatch.cuh"
#endif

namespace ahmc {

// standard normals of tile d0 under the G = 32 counter rule of philox_normals extended past E = 16: coordinate d uses
// Philox block (d mod 32) + 32 floor(floor(d/32) / 2), the cosine for even floor(d/32), the sine for odd.  The draw is a
// pure function of (seed, offset, chain, d); its first 512 coordinates are the D = 512 draw.  (The block index stays below
// 2^24, the bits `offset << 24` leaves free, for D < 2^25.)
__device__ __forceinline__ void big_normals(const double* tape, uint64_t seed, uint64_t offset, long long chain, int d0, int l, int D,
                                            double (&z)[kBigE]) {
    if (tape) {
        tile_load(z, tape + (long long)D * chain, d0, l, D);
        return;
    }
#pragma unroll
    for (int q = 0; q < kBigE / 2; ++q) {
        uint32_t o[4];
        Philox::gen(seed, (uint64_t)chain, (offset << 24) ^ (STREAM_NORMAL << 60) ^ (uint64_t)(d0 / 2 + l + 32 * q), o);
        const double u1 = Philox::u01(o[0], o[1]), u2 = Philox::u01(o[2], o[3]);
        const double rad = sqrt(-2.0 * log(u1));
        double sn, cs;
        sincospi(2.0 * u2, &sn, &cs);
        z[2 * q] = (d0 + l + 32 * (2 * q) < D) ? rad * cs : 0.0;
        z[2 * q + 1] = (d0 + l + 32 * (2 * q + 1) < D) ? rad * sn : 0.0;
    }
}
// r = z / sqrt(M^-1) for a Diag metric (metric.jl:290-320), zero past D
template <int METRIC>
__device__ __forceinline__ void big_scale_momentum(double (&r)[kBigE], const double* Mi, int d0, int l, int D) {
    if (METRIC == AHMC_METRIC_DIAG) {
#pragma unroll
        for (int e = 0; e < kBigE; ++e) {
            const int d = d0 + l + 32 * e;
            r[e] = d < D ? r[e] / sqrt(Mi[d]) : 0.0;
        }
    }
}
// lane partial of the kinetic energy of tile d0, the same expression as big_step's
template <int METRIC>
__device__ __forceinline__ double big_kinetic_part(const double (&r)[kBigE], const double* Mi, int d0, int l, int D, double part) {
#pragma unroll
    for (int e = 0; e < kBigE; ++e) {
        const int d = d0 + l + 32 * e;
        const double mi = METRIC == AHMC_METRIC_DIAG ? (d < D ? Mi[d] : 0.0) : 1.0;
        part = METRIC == AHMC_METRIC_DIAG ? fma(r[e] * r[e], mi, part) : fma(r[e], r[e], part);
    }
    return part;
}

template <int METRIC>
__global__ void __launch_bounds__(kBlockThreads) momentum_big_kernel(const MomentumArgs a) {
    const int l = threadIdx.x % 32;
    const long long chain = (long long)blockIdx.x * (kBlockThreads / 32) + threadIdx.x / 32;
    if (chain >= a.N) return;
    const int D = a.D;
    const double* Mi = METRIC == AHMC_METRIC_DIAG ? a.metric.Minv + a.metric.chain_stride * chain : nullptr;
    for (int d0 = 0; d0 < D; d0 += kBigTile) {
        double r[kBigE];
        big_normals(a.normal_tape, a.seed, a.offset, chain, d0, l, D, r);
        big_scale_momentum<METRIC>(r, Mi, d0, l, D);
        tile_store(a.r + a.ld * chain, r, d0, l, D);
    }
}

// The per-chain StanHMCAdaptor of ChainAdapt with the chain's vectors in global memory: dual averaging in registers
// (ChainAdapt's own code), the estimator pushed and read tile by tile with ChainAdapt::push, M^-1 in the adaptor's
// Minv_chain output row, which is also the metric the chain's trajectories use.  Estimator workspace AW: 2D doubles per
// estimated quantity (theta; NutpieVar also the gradient at AW + 2D); tile d0's (mean, M2) block starts at 2 d0 and holds
// Dt = min(512, D - d0) means followed by Dt M2 -- the layout push(base, x, n, est, l, Dt) reads.
template <int EST>
struct BigChainAdapt {
    using CA = ChainAdapt<32, kBigE, EST>;
    using Block = ChainAdapt<32, kBigE, AHMC_ADAPT_WELFORD>;  // clears one (mean, M2) block
    CA ca;

    static __device__ __forceinline__ int tile_len(int d0, int D) { return D - d0 < kBigTile ? D - d0 : kBigTile; }
    static __device__ __forceinline__ void clear(const AdaptDev& ad, double* AW, int l, int D) {
        for (int d0 = 0; d0 < D; d0 += kBigTile) {
            Block::clear(ad, AW + 2LL * d0, l, tile_len(d0, D));
            if constexpr (EST == AHMC_ADAPT_NUTPIE) Block::clear(ad, AW + 2LL * D + 2LL * d0, l, tile_len(d0, D));
        }
    }
    // DAState(eps), empty estimators, the starting M^-1 (Mi0) into the chain's Minv_chain row (massmatrix.jl:109-118)
    __device__ __forceinline__ void begin(const AdaptDev& ad, double* AW, double eps, const double* Mi0, long long chain, int l, int D) {
        ca.mu = log(10.0 * eps);
        ca.xbar = ca.Hbar = ca.m = ca.n = 0.0;
        clear(ad, AW, l, D);
        if (ad.minv) {
            for (int d0 = 0; d0 < D; d0 += kBigTile) {
                double x[kBigE];
                tile_load(x, Mi0, d0, l, D);
                tile_store(ad.minv + (long long)D * chain, x, d0, l, D);
            }
        }
        if (l == 0) ad.eps[chain] = eps;
    }
    // ChainAdapt::update with the estimator streamed: iteration `it` produced the draw (th, g = -grad lp) with acceptance
    // statistic alpha; si = (it - 1) * N + chain
    __device__ __forceinline__ void update(const AdaptDev& ad, double* AW, int it, long long si, double alpha, const double* th,
                                           const double* g, double& eps, long long chain, int l, int D) {
        if (ad.eps_trace && l == 0) ad.eps_trace[si] = eps;
        if (it > ad.n_adapts) return;
        ca.adapt_stepsize(ad, alpha, eps);
        const bool split = CA::window_end(ad, it);
        if (ad.adapt_metric && it >= ad.window_start && it <= ad.window_end) {
            ca.n += 1.0;
            const bool est = split && ca.n >= (double)ad.n_min;  // update! (massmatrix.jl:60-62)
            double* minv = ad.minv + (long long)D * chain;
            for (int d0 = 0; d0 < D; d0 += kBigTile) {
                const int Dt = tile_len(d0, D);
                double mv[kBigE];
                if constexpr (EST == AHMC_ADAPT_NUTPIE) {  // M^-1 = sqrt(est(theta) ./ est(gradient)) (massmatrix.jl:235-248)
                    CA::push(AW + 2LL * D + 2LL * d0, g + d0, ca.n, est, l, Dt, [&](int e, double v) { mv[e] = v; });
                    CA::push(AW + 2LL * d0, th + d0, ca.n, est, l, Dt, [&](int e, double v) { mv[e] = sqrt(v / mv[e]); });
                } else {  // WelfordVar (massmatrix.jl:141-157)
                    CA::push(AW + 2LL * d0, th + d0, ca.n, est, l, Dt, [&](int e, double v) { mv[e] = v; });
                }
                if (est) tile_store(minv, mv, d0, l, D);
            }
        }
        if (split) {  // reset!(ssa); reset!(pc) (stan_adaptor.jl:155-158; stepsize.jl:38-52)
            ca.reset(eps);
            clear(ad, AW, l, D);
        }
        if (it == ad.n_adapts) eps = exp(ca.xbar);  // finalize! (stepsize.jl:54-62)
        if (l == 0) ad.eps[chain] = eps;
    }
};

// n_transitions static-HMC transitions per chain in one launch: refresh, kinetic energy, L streamed steps (stopping at the
// first non-finite one), the Metropolis test with the same exponential draw as hmc_kernel, accept (momentum flipped) or
// revert to the start point (its momentum flipped), stats and draws.  ADAPT != 0: the adaptor's estimator form, iterations
// 1..n_adapts also adapt the chain's step size and (Diag) M^-1.
template <int MODEL, int METRIC, int ADAPT = 0>
__global__ void __launch_bounds__(kBlockThreads) hmc_big_kernel(const HmcArgs h) {
    const LeapfrogArgs& a = h.lf;
    const int l = threadIdx.x % 32;
    const long long chain = (long long)blockIdx.x * (kBlockThreads / 32) + threadIdx.x / 32;
    if (chain >= a.N) return;  // whole warps
    const int D = a.D;
    double eps = a.eps_chain ? a.eps_chain[chain] : a.eps;
    const BigModel<MODEL> mo{a.model.p0, a.model.p1, a.model.c0, D};
    const double* Mi = METRIC == AHMC_METRIC_DIAG ? a.metric.Minv + a.metric.chain_stride * chain : nullptr;
    double* W = h.scratch + h.scratch_stride * chain;
    double *th0 = W, *g0 = W + D, *r0 = W + 2LL * D;
    double* th = a.th_out + a.ld_out * chain;
    double* r = a.r_out + a.ld_out * chain;
    double* g = a.g_out + a.ld_out * chain;
    BigChainAdapt<ADAPT == AHMC_ADAPT_NUTPIE ? AHMC_ADAPT_NUTPIE : AHMC_ADAPT_WELFORD> cad{};
    double* AW = W + (long long)kBigHmcVectors * D;
    if constexpr (ADAPT != 0) {
        __syncwarp();  // every lane has read its starting eps (ad.eps) before lane 0 writes it back
        cad.begin(h.ad, AW, eps, Mi, chain, l, D);
        if (h.ad.adapt_metric) Mi = h.ad.minv + (long long)D * chain;
        __syncwarp();
    }
    for (int t = 0; t < h.n_transitions; ++t) {
        const bool first = (t == 0);
        const double* sth = first ? a.th_in + a.ld_in * chain : th;
        const double* sg = first ? a.g_in + a.ld_in * chain : g;
        const double* sr = first ? a.r_in + a.ld_in * chain : r;
        const long long si = (long long)t * a.N + chain;
        const uint64_t off = h.rng.offset + (uint64_t)t;
        const double lp0 = map_nonfinite(first ? a.lp_in[chain] : a.lp_out[chain]);
        // refresh (hamiltonian.jl:213-220, 243-254): the start point into the workspace and z_out, the new momentum into both
        double lk_part = 0.0;
        for (int d0 = 0; d0 < D; d0 += kBigTile) {
            double tt[kBigE], gg[kBigE], rr[kBigE];
            tile_load(tt, sth, d0, l, D);
            tile_load(gg, sg, d0, l, D);
            if (h.refresh) {
                big_normals(h.rng.normal_tape, h.rng.seed, off, chain, d0, l, D, rr);
                big_scale_momentum<METRIC>(rr, Mi, d0, l, D);
                if (h.rng.partial_alpha != 0.0) {  // PartialMomentumRefreshment
                    double rp[kBigE];
                    tile_load(rp, sr, d0, l, D);
                    const double al = h.rng.partial_alpha, be = sqrt(1.0 - al * al);
#pragma unroll
                    for (int e = 0; e < kBigE; ++e) rr[e] = al * rp[e] + be * rr[e];
                }
            } else {
                tile_load(rr, sr, d0, l, D);
            }
            lk_part = big_kinetic_part<METRIC>(rr, Mi, d0, l, D, lk_part);
            tile_store(th0, tt, d0, l, D);
            tile_store(g0, gg, d0, l, D);
            tile_store(r0, rr, d0, l, D);
            if (sth != th) tile_store(th, tt, d0, l, D);
            if (sg != g) tile_store(g, gg, d0, l, D);
            tile_store(r, rr, d0, l, D);
        }
        const double lk0 = map_nonfinite(-0.5 * Grp<32>::sum(lk_part));
        const double H0 = -(lp0 + lk0);
        const double ex = h.rng.exp_tape ? h.rng.exp_tape[chain] : philox_exp(h.rng.seed, off, chain, 0);
        __syncwarp();
        double lp = 0.0, lk = 0.0;
        bool fin = true;
        int steps = 0;
        for (int i = 1; i <= a.n_steps; ++i) {
            fin = big_step<MODEL, METRIC, ADAPT == 0>(mo, Mi, eps, th, r, g, nullptr, l, D, lp, lk);
            steps = i;
            if (!fin) break;
        }
        // mh_accept_ratio + accept_phasepoint! + momentum flip (trajectory.jl:283, 312-332, 869-877)
        const double H1 = -(lp + lk);
        const bool accept = H1 < H0 + ex;
        const double alpha = mh_accept_ratio(H0, H1);
        double* dro = h.draws ? h.draws + si * D : nullptr;
        for (int d0 = 0; d0 < D; d0 += kBigTile) {
            double tt[kBigE], rr[kBigE];
            if (accept) {
                tile_load(rr, r, d0, l, D);
                if (dro) {
                    tile_load(tt, th, d0, l, D);
                    tile_store(dro, tt, d0, l, D);
                }
            } else {
                double gg[kBigE];
                tile_load(tt, th0, d0, l, D);
                tile_load(gg, g0, d0, l, D);
                tile_load(rr, r0, d0, l, D);
                tile_store(th, tt, d0, l, D);
                tile_store(g, gg, d0, l, D);
                if (dro) tile_store(dro, tt, d0, l, D);
            }
#pragma unroll
            for (int e = 0; e < kBigE; ++e) rr[e] = -rr[e];
            tile_store(r, rr, d0, l, D);
        }
        const double lpn = accept ? lp : lp0, lkn = accept ? lk : lk0;
        if (l == 0) {
            const double H = -(lpn + lkn);
            a.lp_out[chain] = lpn;
            a.lk_out[chain] = lkn;
            if (a.status) a.status[chain] = fin ? 0u : AHMC_STATUS_NONFINITE;
            if (a.steps_done) a.steps_done[chain] = steps;
            record_stats(h.st, si, a.n_steps, accept, alpha, lpn, H, H0, !finite_d(H1));  // nsteps(tau), nominal (trajectory.jl:288)
        }
        if constexpr (ADAPT != 0) {  // iteration t + 1 of `sample` (sampler.jl:182)
            __syncwarp();
            cad.update(h.ad, AW, t + 1, si, alpha, th, g, eps, chain, l, D);
        }
        __syncwarp();  // lane 0's lp_out is the next transition's lp0 on every lane
    }
}

// find_good_stepsize (trajectory.jl:768-837) for one chain per warp, the whole search in one launch, in the control flow of
// find_eps_kernel; every probe A(h, z, eps) (:753-757) copies the start point into the probe vectors and takes one big_step,
// so chain c's result is the host-side search's (which probes through the D > 512 `step`) bit for bit.
template <int MODEL, int METRIC>
__global__ void __launch_bounds__(kBlockThreads) find_eps_big_kernel(const FindEpsArgs a) {
    const int l = threadIdx.x % 32;
    const long long chain = (long long)blockIdx.x * (kBlockThreads / 32) + threadIdx.x / 32;
    if (chain >= a.N) return;
    const int D = a.D;
    const BigModel<MODEL> mo{a.model.p0, a.model.p1, a.model.c0, D};
    const double* Mi = METRIC == AHMC_METRIC_DIAG ? a.metric.Minv + a.metric.chain_stride * chain : nullptr;
    double* W = a.scratch + (long long)kBigFindEpsVectors * D * chain;
    double *r0 = W, *pth = W + D, *pr = W + 2LL * D, *pg = W + 3LL * D;
    const double* th0 = a.th + a.ld * chain;
    const double* g0 = a.g + a.ld * chain;
    double lk_part = 0.0;
    for (int d0 = 0; d0 < D; d0 += kBigTile) {
        double rr[kBigE];
        big_normals(a.normal_tape, a.seed, a.offset, chain, d0, l, D, rr);
        big_scale_momentum<METRIC>(rr, Mi, d0, l, D);
        lk_part = big_kinetic_part<METRIC>(rr, Mi, d0, l, D, lk_part);
        tile_store(r0, rr, d0, l, D);
        if (a.r_out) tile_store(a.r_out + a.ld * chain, rr, d0, l, D);
    }
    const double lk0 = map_nonfinite(-0.5 * Grp<32>::sum(lk_part));
    const double H = -(map_nonfinite(a.lp[chain]) + lk0);  // energy(z) (hamiltonian.jl:149,194)
    auto probe = [&](double eps) -> double {                // H' of A(h, z, eps) (trajectory.jl:753-757)
        for (int d0 = 0; d0 < D; d0 += kBigTile) {
            double x[kBigE];
            tile_load(x, th0, d0, l, D);
            tile_store(pth, x, d0, l, D);
            tile_load(x, r0, d0, l, D);
            tile_store(pr, x, d0, l, D);
            tile_load(x, g0, d0, l, D);
            tile_store(pg, x, d0, l, D);
        }
        __syncwarp();
        double lp, lk;
        big_step<MODEL, METRIC>(mo, Mi, eps, pth, pr, pg, nullptr, l, D, lp, lk);
        return -(lp + lk);
    };
    const double log_a_min = 2.0 * -0.6931471805599453, log_a_cross = -0.6931471805599453, log_a_max = log(0.75);
    double eps = a.eps0, eps_p = a.eps0;
    double dH = H - probe(eps);
    const bool too_high = dH > log_a_cross;
    for (int it = 0; it < a.max_iters; ++it) {  // crossing step (:796-810)
        eps_p = too_high ? 2.0 * eps : 0.5 * eps;
        dH = H - probe(eps);
        if (too_high != (dH > log_a_cross)) break;
        eps = eps_p;
    }
    double lo = fmin(eps, eps_p), hi = fmax(eps, eps_p);  // minmax (:818)
    for (int it = 0; it < a.max_iters; ++it) {             // bisection (:822-834)
        const double mid = 0.5 * (lo + hi);
        dH = H - probe(mid);
        if (dH > log_a_max) {
            lo = mid;
        } else if (dH < log_a_min) {
            hi = mid;
        } else {
            lo = mid;
            break;
        }
    }
    if (l == 0) a.eps_out[chain] = lo;
}

#ifndef AHMC_SIMT_EMULATION  // host launch code (skipped by the CPU SIMT emulation harness, tests/simt_emu/)
cudaError_t launch_rand_momentum_big(const MomentumArgs& a, cudaStream_t st) {
    return with_kind(BigMetrics{}, a.metric.kind, [&](auto K) { return launch_warps(momentum_big_kernel<K>, a.N, 32, 0, st, a); },
                     cudaErrorNotSupported);
}

cudaError_t launch_hmc_big(const HmcArgs& a, cudaStream_t st) {
    const LeapfrogArgs& lf = a.lf;
    if (!bigd_supported(lf.model.kind, lf.metric.kind) || a.rng.temper_alpha > 0.0) return cudaErrorNotSupported;
    auto run = [&](auto form, auto metrics) {
        return with_model_metric(BigModels{}, metrics, lf.model.kind, lf.metric.kind,
                                 [&](auto M, auto K) { return launch_warps(hmc_big_kernel<M, K, form>, lf.N, 32, 0, st, a); });
    };
    if (!a.ad.enabled) return run(IC<0>{}, BigMetrics{});
    // the adaptive form: Diag metric only (the chain adapts its diagonal M^-1)
    if (adapt_kernel(a.ad, a.lf.metric).form == AHMC_ADAPT_NUTPIE) return run(IC<AHMC_ADAPT_NUTPIE>{}, Kinds<AHMC_METRIC_DIAG>{});
    return run(IC<AHMC_ADAPT_WELFORD>{}, Kinds<AHMC_METRIC_DIAG>{});
}

cudaError_t launch_find_eps_big(const FindEpsArgs& a, cudaStream_t st) {
    if (!bigd_supported(a.model.kind, a.metric.kind)) return cudaErrorNotSupported;
    return with_model_metric(BigModels{}, BigMetrics{}, a.model.kind, a.metric.kind,
                             [&](auto M, auto K) { return launch_warps(find_eps_big_kernel<M, K>, a.N, 32, 0, st, a); }, cudaErrorNotSupported);
}
#endif  // AHMC_SIMT_EMULATION

}  // namespace ahmc
