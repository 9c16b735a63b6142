// ahmc_leapfrog.cu -- K1: the fused leapfrog trajectory kernel (`step(lf, h, z, n_steps)`,
// src/integrator.jl:216-265) + `phasepoint` (src/hamiltonian.jl:115-119) + `rand_momentum`
// (src/metric.jl:290-320).
//
// One launch integrates every chain for all n_steps: a chain's theta, r and -grad(lp) are read once
// from HBM (coalesced runs of G doubles per group), stay in registers for the whole trajectory and
// are written once.  Two code paths share the kernel:
//
//  * EXACT path (every model x metric): per step the reference's op sequence with FMAs, the kinetic
//    and potential energies reduced by warp shuffles, and the reference's `isfinite(z)` test
//    (hamiltonian.jl:141-142) -- a non-finite chain stops on its own (default) and its phase point at
//    the break step is what is returned, as integrator.jl:252-258 does.
//
//  * FAST path (separable Gaussian targets STD_NORMAL / DIAG_GAUSS with Unit / Diag metric, no
//    tempering): state is kept in shifted coordinates x = theta - m, the two half kicks of
//    consecutive steps are merged and the per-coordinate constants a = eps*Minv, b = eps/s^2 are
//    precomputed, so a step costs 2 dependent DFMAs per coordinate and no reduction.  Exactness of the
//    reference's per-step `isfinite` control flow is kept by a magnitude argument: with
//    K = (1+max|a|)(1+max|b|) the sup-norm of (x, r) grows by at most K per step, so checking the
//    exponent fields of (x, r) against 2^200 every floor(100/log2 K) steps PROVES every intermediate
//    phase point (incl. its energies) was finite; a chain that fails a check (or whose parameters are
//    outside the proof's range) is simply re-run by the exact path inside the same launch.
#ifndef __CUDACC_RTC__
#include <cstdlib>
#endif
#include "ahmc_chain_adapt.cuh"
#include "ahmc_kernels.cuh"
#include "ahmc_traj.cuh"
#if !defined(AHMC_SIMT_EMULATION) && !defined(__CUDACC_RTC__)
#include "ahmc_dispatch.cuh"
#endif

namespace ahmc {

// the register-resident layout of D; with_layout (ahmc_dispatch.cuh) instantiates the kernels for exactly these 8 pairs
bool pick_layout(int D, int* G, int* E) {
    if (D < 1) return false;
    if (D <= 4) { *G = 4; *E = 1; return true; }
    if (D <= 8) { *G = 8; *E = 1; return true; }
    if (D <= 16) { *G = 16; *E = 1; return true; }
    if (D <= 32) { *G = 32; *E = 1; return true; }
    if (D <= 64) { *G = 32; *E = 2; return true; }
    if (D <= 128) { *G = 32; *E = 4; return true; }
    if (D <= 256) { *G = 32; *E = 8; return true; }
    if (D <= 512) { *G = 32; *E = 16; return true; }
    return false;
}

// K1 functor: start state = z_in, end state -> z_out (+ status / steps_done / min_break).  CONTIG: the fast path moves
// the state with lane-contiguous 128/256-bit accesses (init_c / done_c); the exact path always uses the interleaved form.
template <int G, int E, bool CONTIG = false>
struct StepIO {
    static constexpr bool kContig = CONTIG;
    static constexpr bool kChainMinv = false;
    const LeapfrogArgs& a;
    long long chain;
    int l;
    __device__ __forceinline__ bool has_g() const { return a.g_in != nullptr; }
    __device__ __forceinline__ void init(double (&th)[E], double (&r)[E], double (&g)[E]) const {
        vload_nc<G, E>(th, a.th_in + a.ld_in * chain, l, a.D);
        vload_nc<G, E>(r, a.r_in + a.ld_in * chain, l, a.D);
        if (a.g_in) vload_nc<G, E>(g, a.g_in + a.ld_in * chain, l, a.D);
    }
    __device__ __forceinline__ void init_c(double (&th)[E], double (&r)[E], double (&g)[E]) const {
        cload<E>(th, a.th_in + a.ld_in * chain, l, a.D);
        cload<E>(r, a.r_in + a.ld_in * chain, l, a.D);
        // issued unconditionally so that all three loads are in flight together (without a cached gradient theta is
        // read a second time and the value ignored)
        cload<E>(g, (a.g_in ? a.g_in : a.th_in) + a.ld_in * chain, l, a.D);
    }
    __device__ __forceinline__ void scalars(double lp, double lk, bool fin, int steps) const {
        if (l == 0) {
            a.lp_out[chain] = lp;
            a.lk_out[chain] = lk;
            if (a.status) a.status[chain] = fin ? 0u : AHMC_STATUS_NONFINITE;
            if (a.steps_done) a.steps_done[chain] = steps;
            if (!fin && a.min_break) atomicMin(a.min_break, steps);
        }
    }
    __device__ __forceinline__ void done(const double (&th)[E], const double (&r)[E], const double (&g)[E],
                                         const double (&dr)[E], double lp, double lk, bool fin, int steps) const {
        vstore<G, E>(a.th_out + a.ld_out * chain, th, l, a.D);
        vstore<G, E>(a.r_out + a.ld_out * chain, r, l, a.D);
        vstore<G, E>(a.g_out + a.ld_out * chain, g, l, a.D);
        if (a.dr_out) vstore<G, E>(a.dr_out + a.ld_out * chain, dr, l, a.D);
        scalars(lp, lk, fin, steps);
    }
    __device__ __forceinline__ void done_c(const double (&th)[E], const double (&r)[E], const double (&g)[E],
                                           const double (&dr)[E], double lp, double lk, bool fin, int steps) const {
        cstore<E>(a.th_out + a.ld_out * chain, th, l, a.D);
        cstore<E>(a.r_out + a.ld_out * chain, r, l, a.D);
        cstore<E>(a.g_out + a.ld_out * chain, g, l, a.D);
        if (a.dr_out) cstore<E>(a.dr_out + a.ld_out * chain, dr, l, a.D);
        scalars(lp, lk, fin, steps);
    }
};

// Occupancy of the one-chain-per-group kernel: 7 blocks of 4 warps per SM, i.e. <= 72 registers per thread.  With one
// chain per warp the headline batch (4096 chains x D=128) would be one full wave of 3696 warps plus a 10 % tail on an
// H100; capping at 8 blocks (64 registers) made it one wave but measured no faster (H100 SXM, 400 W power limit, L2
// flushed: 14.5 against 14.4 us per launch), since the load, compute and store phases of one wave do not overlap.  The
// headline shape now runs leapfrog_pair_kernel (below: two chains per warp, 4 blocks per SM, one wave).  The cap makes
// the (rarely taken) exact fallback of the separable kernels spill a little, which is the right trade.  Wider layouts
// (E >= 8) and non-separable models keep the default budget.
template <int MODEL, int METRIC, int E>
constexpr int min_blocks_per_sm() {
    return (FastCapable<MODEL, METRIC>::value && E <= 4) ? 7 : 1;
}
// The funnel trajectory kernel (exact path only) sits at 95 registers uncapped = 5 blocks per SM = two waves for 4096
// chains; capped it spills ~50 bytes outside the step loop and runs in one.  Its transition kernel would spill inside
// the loop, so that one keeps the default.
// The transition kernel of a general target: 128 registers (4 blocks per SM) are enough for E <= 4 without spills; left
// alone it takes ~140 and loses a block per SM.
template <int MODEL, int METRIC, int E>
constexpr int min_blocks_hmc() {
    return (FastCapable<MODEL, METRIC>::value && E <= 4) ? 7 : ((!is_dense_metric(METRIC) && MODEL != AHMC_MODEL_DENSE_GAUSS && E <= 4) ? 4 : 1);
}
template <int MODEL, int METRIC, int E>
constexpr int min_blocks_lf() {
    return (MODEL == AHMC_MODEL_FUNNEL && !is_dense_metric(METRIC) && E <= 4) ? 7 : min_blocks_per_sm<MODEL, METRIC, E>();
}

template <int MODEL, int METRIC, int G, int E, bool CONTIG = false>
__global__ void __launch_bounds__(kBlockThreads, min_blocks_lf<MODEL, METRIC, E>()) leapfrog_kernel(const LeapfrogArgs a) {
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + grp_in_block;
    const long long chain = chain0 < a.N ? chain0 : a.N - 1;  // tail groups shadow the last chain, never store
    const bool valid = chain0 < a.N && (!a.only_mask || a.only_mask[chain] != 0);
    double* xs = smem + (size_t)grp_in_block * slab_vectors<MODEL>() * a.D;
    double eps = a.eps_chain ? __ldg(a.eps_chain + chain) : a.eps;
    eps = a.fwd ? eps : -eps;  // integrator.jl:226
    StepIO<G, E, CONTIG> io{a, chain, l};
    run_trajectory<MODEL, METRIC, G, E>(a.model, a.metric, a.D, chain, valid, l, xs, eps, a.n_steps, a.temper_alpha,
                                        a.flags, io);
}

// K1's fast path on lane-contiguous full tiles (D = 64, 128; launched only without tempering or exact checks): warp w
// integrates TWO chains, A = 2w and B = 2w + 1, one after the other, and B's loads are issued only once A's state has
// arrived and passed its magnitude test, so they are in flight while A integrates and stores.  With one chain per warp
// every warp of the wave issues its loads at once, DRAM serves them interleaved, and the whole wave then computes with
// HBM idle and stores at once.  Each chain goes through run_trajectory's fast-path arithmetic (FastCoef) op for op, so
// the results are bit-identical to the one-chain kernel.  SHARED: scalar eps and a shared M^-1, so A's coefficient
// registers serve B too (what keeps the pair within 128 registers at E = 4); otherwise B builds its own after A is done.
// 4 blocks of 4 warps per SM (<= 128 registers): the headline 4096 chains are 2048 warps, one wave on 132 SMs.
template <int MODEL, int METRIC, int E, bool SHARED>
__global__ void __launch_bounds__(kBlockThreads, 4) leapfrog_pair_kernel(const LeapfrogArgs a) {
    constexpr int G = 32;
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int w = threadIdx.x / G;
    const long long cA0 = 2 * ((long long)blockIdx.x * (kBlockThreads / G) + w), cB0 = cA0 + 1;
    const long long cA = cA0 < a.N ? cA0 : a.N - 1, cB = cB0 < a.N ? cB0 : a.N - 1;  // past N: shadow the last chain
    const bool vA = cA0 < a.N && (!a.only_mask || a.only_mask[cA] != 0);
    const bool vB = cB0 < a.N && (!a.only_mask || a.only_mask[cB] != 0);
    const int D = a.D, n = a.n_steps;
    double epsA = a.eps_chain ? __ldg(a.eps_chain + cA) : a.eps, epsB = a.eps_chain ? __ldg(a.eps_chain + cB) : a.eps;
    epsA = a.fwd ? epsA : -epsA;  // integrator.jl:226
    epsB = a.fwd ? epsB : -epsB;
    StepIO<G, E, true> ioA{a, cA, l}, ioB{a, cB, l};
    FastCoef<MODEL, METRIC, G, E, true> k;
    const bool have_g = ioA.has_g();

    double xA[E], rA[E];
    {
        double g0[E], mi[E];
        ioA.init_c(xA, rA, g0);
        if constexpr (METRIC == AHMC_METRIC_DIAG) cload<E>(mi, a.metric.Minv + a.metric.chain_stride * cA, l, D);
        k.load_model(a.model, l, D);
        k.make(mi, epsA, n, l, D);
        k.enter(xA, rA, g0, have_g);
    }
    bool sA = k.bad | k.test(xA, rA);

    // B's loads.  Left alone the compiler issues them together with A's at the top of the kernel.  Their address is made
    // to depend on a vote over A's test, which reads every element of A's state, through a term that is zero at run time
    // but not to the compiler (%laneid equals l, which it cannot prove): the loads leave once A's state has arrived.
#ifdef AHMC_SIMT_EMULATION
    const unsigned lane = threadIdx.x % 32;
#else
    unsigned lane;
    asm("mov.u32 %0, %%laneid;" : "=r"(lane));
#endif
    const long long offB = a.ld_in * cB + (long long)(__any_sync(FULL, sA) & (lane ^ (unsigned)l));
    double xB[E], rB[E], gB[E], miB[E];
    cload<E>(xB, a.th_in + offB, l, D);
    cload<E>(rB, a.r_in + offB, l, D);
    cload<E>(gB, (a.g_in ? a.g_in : a.th_in) + offB, l, D);
    if constexpr (METRIC == AHMC_METRIC_DIAG && !SHARED) cload<E>(miB, a.metric.Minv + a.metric.chain_stride * cB, l, D);

    bool needA, needB;
    {
        sA |= k.steps(xA, rA, n);
        double g[E], dr[E], lp, lk;
        k.last(xA, rA, g, dr, lp, lk, a.model.c0, l, D);
        sA = Grp<G>::any(sA);
        needA = vA && sA;
        if (vA && !sA) ioA.done_c(xA, rA, g, dr, lp, lk, true, n);
    }
    {
        if constexpr (!SHARED) k.make(miB, epsB, n, l, D);
        k.enter(xB, rB, gB, have_g);
        bool sB = k.bad | k.test(xB, rB);
        sB |= k.steps(xB, rB, n);
        double g[E], dr[E], lp, lk;
        k.last(xB, rB, g, dr, lp, lk, a.model.c0, l, D);
        sB = Grp<G>::any(sB);
        needB = vB && sB;
        if (vB && !sB) ioB.done_c(xB, rB, g, dr, lp, lk, true, n);
    }

    // a chain that failed its proof is re-run alone by the exact path, A then B, each with the whole warp
    if (!__any_sync(FULL, needA || needB)) return;
    double* xs = smem + (size_t)w * slab_vectors<MODEL>() * D;
    exact_trajectory<MODEL, METRIC, G, E>(a.model, a.metric, D, cA, needA, l, xs, epsA, n, a.temper_alpha, ioA);
    exact_trajectory<MODEL, METRIC, G, E>(a.model, a.metric, D, cB, needB, l, xs, epsB, n, a.temper_alpha, ioB);
}

// ---------------------------------------------------------------------------------------------
// K2: one static-HMC transition (sampler.jl:48-58 + trajectory.jl:271-300, 312-340, 863-880)
// ---------------------------------------------------------------------------------------------
// ADAPT: the chain adapts its own step size and diagonal M^-1 inside the launch (minv: its current M^-1, alpha: the
// acceptance statistic of the transition just made, for dual averaging)
template <int METRIC, int G, int E, bool ADAPT = false>
struct HmcIO {
    const HmcArgs& h;
    long long chain;
    int l;
    const double* src_th;  // start point of THIS transition (z_in for the first, z_out afterwards)
    const double* src_g;
    long long stat_idx;    // t*N + chain
    double H0, lp0, lk0, ex;
    double r0[E];
    double minv[ADAPT ? E : 1];
    mutable double alpha;

    static constexpr bool kContig = false;
    static constexpr bool kChainMinv = ADAPT;
    __device__ __forceinline__ bool has_g() const { return true; }
    __device__ __forceinline__ void init(double (&th)[E], double (&r)[E], double (&g)[E]) const {
        vload_nc<G, E>(th, src_th, l, h.lf.D);
        vload_nc<G, E>(g, src_g, l, h.lf.D);
#pragma unroll
        for (int e = 0; e < E; ++e) r[e] = r0[e];
    }
    // mh_accept_ratio + accept_phasepoint! + momentum flip + stats
    __device__ __forceinline__ void done(const double (&th)[E], const double (&r)[E], const double (&g)[E],
                                         const double (&dr)[E], double lp, double lk, bool fin, int steps) const {
        const LeapfrogArgs& a = h.lf;
        const double H1 = -(lp + lk);                   // energy(z') (hamiltonian.jl:149,194)
        const bool accept = H1 < H0 + ex;               // trajectory.jl:869-877
        const double alpha = mh_accept_ratio(H0, H1);
        double* tho = a.th_out + a.ld_out * chain;
        double* ro = a.r_out + a.ld_out * chain;
        double* go = a.g_out + a.ld_out * chain;
        double* dro = h.draws ? h.draws + stat_idx * a.D : nullptr;
        double lpn, lkn;
        if (accept) {
            double nr[E];
#pragma unroll
            for (int e = 0; e < E; ++e) nr[e] = -r[e];  // flip (trajectory.jl:283)
            vstore<G, E>(tho, th, l, a.D);
            vstore<G, E>(ro, nr, l, a.D);
            vstore<G, E>(go, g, l, a.D);
            if (dro) vstore<G, E>(dro, th, l, a.D);
            lpn = lp;
            lkn = lk;
        } else {  // revert (trajectory.jl:312-332)
            double t0[E], g0[E], nr[E];
            vload_nc<G, E>(t0, src_th, l, a.D);
            vload_nc<G, E>(g0, src_g, l, a.D);
#pragma unroll
            for (int e = 0; e < E; ++e) nr[e] = -r0[e];
            vstore<G, E>(tho, t0, l, a.D);
            vstore<G, E>(ro, nr, l, a.D);
            vstore<G, E>(go, g0, l, a.D);
            if (dro) vstore<G, E>(dro, t0, l, a.D);
            lpn = lp0;
            lkn = lk0;
        }
        if (l == 0) {
            const double H = -(lpn + lkn);
            a.lp_out[chain] = lpn;
            a.lk_out[chain] = lkn;
            if (a.status) a.status[chain] = fin ? 0u : AHMC_STATUS_NONFINITE;
            if (a.steps_done) a.steps_done[chain] = steps;
            record_stats(h.st, stat_idx, a.n_steps, accept, alpha, lpn, H, H0, !finite_d(H1));  // nsteps(tau), nominal (trajectory.jl:288)
        }
        this->alpha = alpha;
        (void)dr;
    }
};

// One launch = n_transitions static-HMC transitions per chain (the reference's `for i in 1:n_samples` loop,
// sampler.jl:182): state is re-read from the output phase point, which stays L2-resident.  ADAPT != 0 (the adaptor's estimator form, ahmc_chain_adapt.cuh): iterations
// 1..n_adapts also run the chain's own StanHMCAdaptor (ahmc_chain_adapt.cuh) on its acceptance rate and draw.
template <int MODEL, int METRIC, int G, int E, int ADAPT = 0>
__global__ void __launch_bounds__(kBlockThreads, min_blocks_hmc<MODEL, METRIC, E>()) hmc_kernel(const HmcArgs h) {
    extern __shared__ double smem[];
    const LeapfrogArgs& a = h.lf;
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + grp_in_block;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = a.D;
    double* xs = smem + (size_t)grp_in_block * slab_vectors<MODEL>() * D;
    double eps = a.eps_chain ? __ldg(a.eps_chain + chain) : a.eps;
    constexpr bool kCov = ADAPT == AHMC_ADAPT_WELFORD_COV;  // (METRIC = kMetricDenseChain: the chain's own rows)

    MetricOps<METRIC, G, E> me;
    MetricDev rows;
    const MetricDev& md = adapt_launch_metric<ADAPT>(a.metric, h.ad, D, rows);
    if constexpr (!kCov) me.load(md, chain, l, D);
    HmcIO<METRIC, G, E, (ADAPT != 0 && !kCov)> io{h, chain, l};
    ChainAdapt<G, E, ADAPT == AHMC_ADAPT_NUTPIE ? AHMC_ADAPT_NUTPIE : (kCov ? AHMC_ADAPT_WELFORD_COV : AHMC_ADAPT_WELFORD)> cad{};
    if constexpr (ADAPT) {
        __syncwarp();  // every lane has read its starting eps (ad.eps) before lane 0 writes it back
        if constexpr (kCov) cad.begin_dense(h.ad, a.metric, h.scratch + h.scratch_stride * chain, valid, chain, l, D);
        if (valid) cad.begin(h.ad, h.scratch + h.scratch_stride * chain, eps, me.Minv, chain, l, D);
    }
    if constexpr (kCov) me.load(md, chain, l, D);  // the rows begin_dense filled
    for (int t = 0; t < h.n_transitions; ++t) {
        const bool first = (t == 0);
        io.src_th = first ? a.th_in + a.ld_in * chain : a.th_out + a.ld_out * chain;
        io.src_g = first ? a.g_in + a.ld_in * chain : a.g_out + a.ld_out * chain;
        io.stat_idx = (long long)t * a.N + chain;
        const uint64_t off = h.rng.offset + (uint64_t)t;
        // refresh (hamiltonian.jl:213-220): new momentum, kinetic energy; lp is the cached value (quirk Q2:
        // the reference recomputes it from theta -- same number)
        if (h.refresh) {
            draw_momentum(me, h.rng.normal_tape, h.rng.seed, off, chain, l, D, io.r0);
            if (h.rng.partial_alpha != 0.0) {  // PartialMomentumRefreshment (hamiltonian.jl:243-254)
                double rp[E];
                vload_nc<G, E>(rp, first ? a.r_in + a.ld_in * chain : a.r_out + a.ld_out * chain, l, D);
                const double al = h.rng.partial_alpha, be = sqrt(1.0 - al * al);
#pragma unroll
                for (int e = 0; e < E; ++e) io.r0[e] = al * rp[e] + be * io.r0[e];
            }
        } else {
            vload_nc<G, E>(io.r0, first ? a.r_in + a.ld_in * chain : a.r_out + a.ld_out * chain, l, D);
        }
        {
            double dr0[E];
            io.lk0 = map_nonfinite(kinetic<METRIC, G, E>(me, io.r0, dr0, xs, l));
        }
        io.lp0 = map_nonfinite(first ? a.lp_in[chain] : a.lp_out[chain]);
        io.H0 = -(io.lp0 + io.lk0);
        io.ex = h.rng.exp_tape ? h.rng.exp_tape[chain] : philox_exp(h.rng.seed, off, chain, 0);
        if constexpr (ADAPT && !kCov) {
#pragma unroll
            for (int e = 0; e < E; ++e) io.minv[e] = me.Minv[e];
        }
        run_trajectory<MODEL, METRIC, G, E>(a.model, md, D, chain, valid, l, xs, eps, a.n_steps, h.rng.temper_alpha, a.flags, io);
        if constexpr (kCov) {  // every lane of the warp calls (the estimator exchanges data across the group)
            cad.update_cov(h.ad, h.scratch + h.scratch_stride * chain, valid, t + 1, io.stat_idx, io.alpha, a.th_out + a.ld_out * chain,
                           eps, chain, l, D);
        } else if constexpr (ADAPT) {  // iteration t + 1 of `sample` (sampler.jl:182)
            if (valid)
                cad.update(h.ad, h.scratch + h.scratch_stride * chain, t + 1, io.stat_idx, io.alpha, a.th_out + a.ld_out * chain, a.g_out + a.ld_out * chain, eps, me.Minv,
                           chain, l, D);
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// find_good_stepsize (trajectory.jl:768-837), one independent search per chain, the WHOLE search in one launch:
// momentum draw, H, the direction probe, the crossing loop (doubling / halving until the one-step acceptance ratio
// crosses 1/2) and the bisection (until it lies in (1/4, 3/4]).  Every probe A(h, z, eps) (:753-757) is one exact
// leapfrog step from the chain's start point held in registers.  Loops are warp-uniform (groups that finished keep
// stepping with their final eps and ignore the result), so shuffles stay convergent when several chains share a warp.
// Mirrors the reference's control flow literally, including its quirk of probing with eps (not eps') in the crossing loop.
// ---------------------------------------------------------------------------------------------
template <int MODEL, int METRIC, int G, int E>
__global__ void __launch_bounds__(kBlockThreads) find_eps_kernel(const FindEpsArgs a) {
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + grp_in_block;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = a.D;
    double* xs = smem + (size_t)grp_in_block * slab_vectors<MODEL>() * D;
    ModelOps<MODEL, G, E> mo;
    MetricOps<METRIC, G, E> me;
    mo.load(a.model, l, D);
    me.load(a.metric, chain, l, D);
    ChainState<E> z0;
    vload_nc<G, E>(z0.th, a.th + a.ld * chain, l, D);
    vload_nc<G, E>(z0.g, a.g + a.ld * chain, l, D);
    draw_momentum(me, a.normal_tape, a.seed, a.offset, chain, l, D, z0.r);
    if (a.r_out && valid) vstore<G, E>(a.r_out + a.ld * chain, z0.r, l, D);
    double dr[E];
    const double lk0 = map_nonfinite(kinetic<METRIC, G, E>(me, z0.r, dr, xs, l));
    const double H = -(map_nonfinite(a.lp[chain]) + lk0);  // energy(z) (hamiltonian.jl:149,194)
    auto probe = [&](double eps) -> double {                // H' of A(h, z, eps) (trajectory.jl:753-757)
        ChainState<E> s = z0;
        leapfrog_step<MODEL, METRIC, G, E>(s, mo, me, eps, dr, xs, l);
        return -(s.lp + s.lk);
    };
    const double log_a_min = 2.0 * -0.6931471805599453, log_a_cross = -0.6931471805599453, log_a_max = log(0.75);
    double eps = a.eps0, eps_p = a.eps0;
    double dH = H - probe(eps);
    const bool too_high = dH > log_a_cross;
    bool active = true;
    for (int it = 0; it < a.max_iters; ++it) {  // crossing step (:796-810)
        if (!__any_sync(FULL, active)) break;
        if (active) eps_p = too_high ? 2.0 * eps : 0.5 * eps;
        dH = H - probe(eps);
        if (active) {
            if (too_high != (dH > log_a_cross)) active = false;
            else eps = eps_p;
        }
    }
    double lo = fmin(eps, eps_p), hi = fmax(eps, eps_p);  // minmax (:818)
    active = true;
    for (int it = 0; it < a.max_iters; ++it) {  // bisection (:822-834)
        if (!__any_sync(FULL, active)) break;
        const double mid = 0.5 * (lo + hi);
        dH = H - probe(active ? mid : lo);
        if (active) {
            if (dH > log_a_max) lo = mid;
            else if (dH < log_a_min) hi = mid;
            else {
                lo = mid;
                active = false;
            }
        }
    }
    if (valid && l == 0) a.eps_out[chain] = lo;
}

// ---------------------------------------------------------------------------------------------
// phasepoint(h, theta, r)  (hamiltonian.jl:115-119)
// ---------------------------------------------------------------------------------------------
template <int MODEL, int METRIC, int G, int E>
__global__ void __launch_bounds__(kBlockThreads) phasepoint_kernel(const PhasepointArgs a) {
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + grp_in_block;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = a.D;
    double* xs = smem + (size_t)grp_in_block * slab_vectors<MODEL>() * D;
    ModelOps<MODEL, G, E> mo;
    MetricOps<METRIC, G, E> me;
    mo.load(a.model, l, D);
    me.load(a.metric, chain, l, D);
    double th[E], r[E], g[E], dr[E];
    vload_nc<G, E>(th, a.th + a.ld * chain, l, D);
    vload_nc<G, E>(r, a.r + a.ld * chain, l, D);
    double lp = map_nonfinite(mo.eval(th, g, xs, l));
    double lk = map_nonfinite(kinetic<METRIC, G, E>(me, r, dr, xs, l));
    if (valid) {
        vstore<G, E>(a.g + a.ld * chain, g, l, D);
        if (a.dr) vstore<G, E>(a.dr + a.ld * chain, dr, l, D);
        if (l == 0) {
            a.lp[chain] = lp;
            a.lk[chain] = lk;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// rand_momentum  (metric.jl:290-320)
// ---------------------------------------------------------------------------------------------
template <int METRIC, int G, int E>
__global__ void __launch_bounds__(kBlockThreads) momentum_kernel(const MomentumArgs a) {
    const int l = threadIdx.x % G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + threadIdx.x / G;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = a.D;
    MetricOps<METRIC, G, E> me;
    me.load(a.metric, chain, l, D);
    double r[E];
    draw_momentum(me, a.normal_tape, a.seed, a.offset, chain, l, D, r);
    if (valid) vstore<G, E>(a.r + a.ld * chain, r, l, D);
}

// ---------------------------------------------------------------------------------------------
// split-step kernels: the generic path for a user-supplied gradient (hamiltonian.jl:45-48 closure)
// ---------------------------------------------------------------------------------------------
// first half of integrator.jl:235-240: temper, r -= eps/2 g, theta += eps dH/dr(r)
template <int METRIC, int G, int E>
__global__ void __launch_bounds__(kBlockThreads) kick_drift_kernel(const SplitArgs a) {
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + grp_in_block;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = a.D;
    double* xs = smem + (size_t)grp_in_block * D;
    const bool active = valid && a.status[chain] == 0u;
    double eps = a.eps_chain ? __ldg(a.eps_chain + chain) : a.eps;
    eps = a.fwd ? eps : -eps;
    MetricOps<METRIC, G, E> me;
    me.load(a.metric, chain, l, D);
    double th[E], r[E], g[E], dr[E];
    vload_nc<G, E>(th, a.th + a.ld * chain, l, D);
    vload_nc<G, E>(r, a.r + a.ld * chain, l, D);
    vload_nc<G, E>(g, a.g + a.ld * chain, l, D);
    const double he = 0.5 * eps;
#pragma unroll
    for (int e = 0; e < E; ++e) r[e] = fma(-he, g[e], r[e] * a.mul);
    me.dHdr(r, dr, xs, l);
#pragma unroll
    for (int e = 0; e < E; ++e) th[e] = fma(eps, dr[e], th[e]);
    if (active) {
        vstore<G, E>(a.th + a.ld * chain, th, l, D);
        vstore<G, E>(a.r + a.ld * chain, r, l, D);
    }
}

// second half of integrator.jl:242-258: g = -grad, r -= eps/2 g, temper, energies, isfinite(z).
// no_kick = 1 turns it into the tail of `phasepoint` (hamiltonian.jl:115-119): r untouched, status ignored,
// cb_grad / cb_lp may be NULL (then only lk / dH/dr are produced).
template <int METRIC, int G, int E>
__global__ void __launch_bounds__(kBlockThreads) kick_energy_kernel(const SplitArgs a) {
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + grp_in_block;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = a.D;
    double* xs = smem + (size_t)grp_in_block * D;
    const bool active = valid && (a.no_kick || a.status[chain] == 0u);
    double eps = a.eps_chain ? __ldg(a.eps_chain + chain) : a.eps;
    eps = a.fwd ? eps : -eps;
    MetricOps<METRIC, G, E> me;
    me.load(a.metric, chain, l, D);
    double r[E], g[E], dr[E];
    vload_nc<G, E>(r, a.r + a.ld * chain, l, D);
    if (a.cb_grad) {
        vload_nc<G, E>(g, a.cb_grad + a.ld * chain, l, D);
#pragma unroll
        for (int e = 0; e < E; ++e) g[e] = -g[e];  // dH/dtheta = DualValue(lp, -grad) (hamiltonian.jl:47)
    } else {
#pragma unroll
        for (int e = 0; e < E; ++e) g[e] = 0.0;
    }
    if (!a.no_kick) {
        const double he = 0.5 * eps;
#pragma unroll
        for (int e = 0; e < E; ++e) r[e] = fma(-he, g[e], r[e]) * a.mul;
    }
    const double lk = kinetic<METRIC, G, E>(me, r, dr, xs, l);
    const double lp = a.cb_lp ? a.cb_lp[chain] : 0.0;
    bool fin = true;
#pragma unroll
    for (int e = 0; e < E; ++e) fin = fin && finite_d(g[e]) && finite_d(dr[e]);
    fin = Grp<G>::all(fin) && finite_d(lp) && finite_d(lk);
    if (active) {
        if (!a.no_kick) vstore<G, E>(a.r + a.ld * chain, r, l, D);
        if (a.cb_grad) vstore<G, E>(a.g + a.ld * chain, g, l, D);
        if (a.dr) vstore<G, E>(a.dr + a.ld * chain, dr, l, D);
        if (l == 0) {
            if (a.cb_lp) a.lp[chain] = map_nonfinite(lp);
            a.lk[chain] = map_nonfinite(lk);
            if (!a.no_kick) {
                if (a.steps_done) a.steps_done[chain] = a.step_index;
                if (!fin) {
                    a.status[chain] = AHMC_STATUS_NONFINITE;
                    if (a.any_nonfinite) *a.any_nonfinite = 1;
                }
            }
        }
    }
}

// mh_accept_ratio + accept_phasepoint! + flip + stats, element-parallel over the group (trajectory.jl:271-300)
template <int G, int E>
__global__ void __launch_bounds__(kBlockThreads) mh_select_kernel(const MhArgs a) {
    const int l = threadIdx.x % G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + threadIdx.x / G;
    if (chain0 >= a.N) return;
    const long long chain = chain0;
    const int D = a.D;
    const double lp0 = map_nonfinite(a.lp0[chain]), lk0 = a.lk0[chain];
    const double lp1 = a.lp[chain], lk1 = a.lk[chain];
    const double H0 = -(lp0 + lk0), H1 = -(lp1 + lk1);
    const double ex = a.rng.exp_tape ? a.rng.exp_tape[chain] : philox_exp(a.rng.seed, a.rng.offset, chain, 0);
    const bool accept = H1 < H0 + ex;
    const double alpha = mh_accept_ratio(H0, H1);
    double t[E];
    if (accept) {
        vload_nc<G, E>(t, a.r + a.ld * chain, l, D);
#pragma unroll
        for (int e = 0; e < E; ++e) t[e] = -t[e];
        vstore<G, E>(a.r + a.ld * chain, t, l, D);
    } else {
        vload_nc<G, E>(t, a.th0 + a.ld0 * chain, l, D);
        vstore<G, E>(a.th + a.ld * chain, t, l, D);
        vload_nc<G, E>(t, a.g0 + a.ld0 * chain, l, D);
        vstore<G, E>(a.g + a.ld * chain, t, l, D);
        vload_nc<G, E>(t, a.r0 + (long long)D * chain, l, D);
#pragma unroll
        for (int e = 0; e < E; ++e) t[e] = -t[e];
        vstore<G, E>(a.r + a.ld * chain, t, l, D);
    }
    if (l == 0) {
        const double lpn = accept ? lp1 : lp0, lkn = accept ? lk1 : lk0;
        const double H = -(lpn + lkn);
        a.lp[chain] = lpn;
        a.lk[chain] = lkn;
        record_stats(a.st, chain, a.n_steps, accept, alpha, lpn, H, H0, !finite_d(H1));
    }
}

#ifndef AHMC_SIMT_EMULATION  // host launch code (skipped by the CPU SIMT emulation harness, tests/simt_emu/)
// ---------------------------------------------------------------------------------------------
// dispatch
// ---------------------------------------------------------------------------------------------
#ifndef __CUDACC_RTC__  // host launch code (the kernels above are also compiled at run time for user targets, ahmc_user.cu)
// can the fast path of this launch use the lane-contiguous vector layout?  (full tile D == 32*E, rows and coefficient
// vectors aligned to the vector width)
template <int E>
static bool contig_ok(const LeapfrogArgs& a) {
    constexpr int V = E >= 4 ? 4 : E;
    const uintptr_t m = (uintptr_t)(8 * V - 1);
    auto al = [&](const void* p) { return ((uintptr_t)p & m) == 0; };
    if (a.D != 32 * E || a.ld_in % V || a.ld_out % V) return false;  // full tiles only: no bounds predicate in the kernel
    if (!al(a.th_in) || !al(a.r_in) || !al(a.g_in) || !al(a.th_out) || !al(a.r_out) || !al(a.g_out) || !al(a.dr_out)) return false;
    if (a.metric.kind == AHMC_METRIC_DIAG && (!al(a.metric.Minv) || a.metric.chain_stride % V)) return false;
    if (a.model.kind == AHMC_MODEL_DIAG_GAUSS && (!al(a.model.p0) || !al(a.model.p1))) return false;
    return true;
}

// dynamic shared memory of a K1 launch (the pair kernel's exact path uses one group's slab per warp, as G = 32 does)
static size_t lf_smem(int model, int metric, int G, const LeapfrogArgs& a) {
    size_t sm = smem_bytes(model, metric, a.D, G);
    const int occ = a.resident_blocks_per_sm;
    if (occ > 0) {
        // occupancy throttle (host-memory lanes): pad the dynamic shared memory so that only this many CTAs fit on
        // an SM; the grid then runs in staggered waves, some CTAs storing while others are still loading
        const size_t pad = (size_t)(227 * 1024) / (size_t)occ - 1024;
        if (pad > sm) sm = pad;
    }
    return sm;
}
template <int MODEL, int METRIC, int G, int E, bool CONTIG>
static cudaError_t launch_lf_c(const LeapfrogArgs& a, cudaStream_t st) {
    return launch_warps(leapfrog_kernel<MODEL, METRIC, G, E, CONTIG>, a.N, G, lf_smem(MODEL, METRIC, G, a), st, a);
}
template <int MODEL, int METRIC, int G, int E>
static cudaError_t launch_lf_t(const LeapfrogArgs& a, cudaStream_t st) {
    if constexpr (FastCapable<MODEL, METRIC>::value && G == 32 && E >= 2) {
        if (!(a.flags & AHMC_FLAG_EXACT_CHECKS) && !(a.temper_alpha > 0.0) && contig_ok<E>(a)) {
            if constexpr (E <= 4) {
                // the pair kernel: 2 chains per warp, 8 per block
                const size_t sm = lf_smem(MODEL, METRIC, G, a);
                const bool shared = !a.eps_chain && (METRIC != AHMC_METRIC_DIAG || a.metric.chain_stride == 0);
                const long long blocks = (a.N + 2 * (kBlockThreads / G) - 1) / (2 * (kBlockThreads / G));
                return shared ? launch_kernel(leapfrog_pair_kernel<MODEL, METRIC, E, true>, blocks, kBlockThreads, sm, st, a)
                              : launch_kernel(leapfrog_pair_kernel<MODEL, METRIC, E, false>, blocks, kBlockThreads, sm, st, a);
            } else {
                // D = 256, 512: two chains' state and in-flight loads do not fit 128 registers; one chain per warp
                return launch_lf_c<MODEL, METRIC, G, E, true>(a, st);
            }
        }
    }
    return launch_lf_c<MODEL, METRIC, G, E, false>(a, st);
}

// the entry points with a D > 512 streaming form and a run-time compiled form: past D = 512 `big`, for a user target its
// compiled kernel `uk` on the template metric kind `metric_kind` (estimator form `form`), else `builtin(G, E)` at the
// register-resident layout of D
template <class Args, class Builtin>
static cudaError_t front_door(const Args& a, int D, long long N, const ModelDev& model, int metric_kind,
                              cudaError_t (*big)(const Args&, cudaStream_t), int uk, int form, cudaStream_t st,
                              int* n_launches, Builtin&& builtin) {
    int G, E;
    if (D > 512) {  // beyond the register-resident layouts: the streaming form (ahmc_bigd.cu, ahmc_bigd_hmc.cu)
        if (n_launches) *n_launches += 1;
        return big(a, st);
    }
    if (!pick_layout(D, &G, &E)) return cudaErrorInvalidValue;
    if (n_launches) *n_launches += 1;
    if (model.kind == AHMC_MODEL_USER) {  // run-time compiled kernels of a user target (ahmc_user.cu)
        const int cpb = kBlockThreads / G;
        return user_launch((UserModule*)model.user, uk, metric_kind, G, E, &a, (unsigned)((N + cpb - 1) / cpb),
                           smem_bytes(AHMC_MODEL_USER, metric_kind, D, G), st, form);
    }
    return builtin(G, E);
}

cudaError_t launch_leapfrog(const LeapfrogArgs& a, cudaStream_t st, int* n_launches) {
    return front_door(a, a.D, a.N, a.model, metric_form(a.metric), launch_leapfrog_big, UK_LEAPFROG, 0, st, n_launches, [&](int G, int E) {
        return with_model_metric_layout(AllModels{}, AllMetrics{}, a.model.kind, metric_form(a.metric), G, E,
                                        [&](auto M, auto K, auto g, auto e) { return launch_lf_t<M, K, g, e>(a, st); });
    });
}

cudaError_t launch_find_eps(const FindEpsArgs& a, cudaStream_t st, int* n_launches) {
    return front_door(a, a.D, a.N, a.model, metric_form(a.metric), launch_find_eps_big, UK_FIND_EPS, 0, st, n_launches, [&](int G, int E) {
        return with_model_metric_layout(AllModels{}, AllMetrics{}, a.model.kind, metric_form(a.metric), G, E, [&](auto M, auto K, auto g, auto e) {
            return launch_warps(find_eps_kernel<M, K, g, e>, a.N, g, smem_bytes(M, K, a.D, g), st, a);
        });
    });
}

cudaError_t launch_phasepoint(const PhasepointArgs& a, cudaStream_t st, int* n_launches) {
    return front_door(a, a.D, a.N, a.model, metric_form(a.metric), launch_phasepoint_big, UK_PHASEPOINT, 0, st, n_launches, [&](int G, int E) {
        return with_model_metric_layout(AllModels{}, AllMetrics{}, a.model.kind, metric_form(a.metric), G, E, [&](auto M, auto K, auto g, auto e) {
            return launch_warps(phasepoint_kernel<M, K, g, e>, a.N, g, smem_bytes(M, K, a.D, g), st, a);
        });
    });
}

cudaError_t launch_hmc(const HmcArgs& a, cudaStream_t st, int* n_launches) {
    const LeapfrogArgs& lf = a.lf;
    const AdaptKernel ak = a.ad.enabled ? adapt_kernel(a.ad, lf.metric) : AdaptKernel{metric_form(lf.metric), 0};
    return front_door(a, lf.D, lf.N, lf.model, ak.metric_kind, launch_hmc_big, a.ad.enabled ? UK_HMC_ADAPT : UK_HMC, ak.form, st,
                      n_launches, [&](int G, int E) -> cudaError_t {
        auto run = [&](auto form, auto metrics) {
            return with_model_metric_layout(AllModels{}, metrics, lf.model.kind, ak.metric_kind, G, E, [&](auto M, auto K, auto g, auto e) {
                return launch_warps(hmc_kernel<M, K, g, e, form>, lf.N, g, smem_bytes(M, K, lf.D, g), st, a);
            });
        };
        // the adaptive forms run on the metric their estimator adapts: Diag, or for WelfordCov the chain's own Dense rows
        switch (ak.form) {
            case 0: return run(IC<0>{}, AllMetrics{});
            case AHMC_ADAPT_WELFORD_COV: return run(IC<AHMC_ADAPT_WELFORD_COV>{}, Kinds<kMetricDenseChain>{});
            case AHMC_ADAPT_NUTPIE: return run(IC<AHMC_ADAPT_NUTPIE>{}, Kinds<AHMC_METRIC_DIAG>{});
            default: return run(IC<AHMC_ADAPT_WELFORD>{}, Kinds<AHMC_METRIC_DIAG>{});
        }
    });
}

// the kernels without a model (split step, momentum draw): f(METRIC, G, E) for the metric form, at the layout of D
template <class F>
static cudaError_t metric_layout(int D, const MetricDev& metric, int* n_launches, F&& f) {
    int G, E;
    if (!pick_layout(D, &G, &E)) return cudaErrorInvalidValue;
    if (n_launches) *n_launches += 1;
    return with_kind(AllMetrics{}, metric_form(metric), [&](auto K) {
        return with_layout(G, E, [&](auto g, auto e) { return f(K, g, e); });
    });
}

cudaError_t launch_kick_drift(const SplitArgs& a, cudaStream_t st, int* n_launches) {
    return metric_layout(a.D, a.metric, n_launches, [&](auto K, auto g, auto e) {
        return launch_warps(kick_drift_kernel<K, g, e>, a.N, g, smem_bytes(AHMC_MODEL_STD_NORMAL, K, a.D, g), st, a);
    });
}
cudaError_t launch_kick_energy(const SplitArgs& a, cudaStream_t st, int* n_launches) {
    return metric_layout(a.D, a.metric, n_launches, [&](auto K, auto g, auto e) {
        return launch_warps(kick_energy_kernel<K, g, e>, a.N, g, smem_bytes(AHMC_MODEL_STD_NORMAL, K, a.D, g), st, a);
    });
}
cudaError_t launch_mh_select(const MhArgs& a, cudaStream_t st, int* n_launches) {
    int G, E;
    if (!pick_layout(a.D, &G, &E)) return cudaErrorInvalidValue;
    if (n_launches) *n_launches += 1;
    return with_layout(G, E, [&](auto g, auto e) { return launch_warps(mh_select_kernel<g, e>, a.N, g, 0, st, a); });
}

cudaError_t launch_rand_momentum(const MomentumArgs& a, cudaStream_t st, int* n_launches) {
    if (a.D > 512) {
        if (n_launches) *n_launches += 1;
        return launch_rand_momentum_big(a, st);
    }
    return metric_layout(a.D, a.metric, n_launches, [&](auto K, auto g, auto e) {
        return launch_warps(momentum_kernel<K, g, e>, a.N, g, 0, st, a);
    });
}

#endif  // AHMC_SIMT_EMULATION

#endif  // __CUDACC_RTC__

}  // namespace ahmc
