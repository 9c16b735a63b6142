// ahmc_nuts_kernel.cuh -- K3: one NUTS transition per chain (MultinomialTS + GeneralisedNoUTurn), the
// reference's recursive doubling tree (src/trajectory.jl:626-742) run ITERATIVELY by one warp-group
// per chain, so divergent U-turn termination stays inside the group.
//
// Recursion -> iteration.  `build_tree(depth j)` is a post-order walk over 2^j leaves; the only state
// the recursion keeps alive is, per level k, the FIRST half-subtree waiting for its sibling.  We keep
// exactly that ("pending[k]") in a per-chain workspace and drive the merges like a binary counter:
// after leaf i, level k merges iff bit k of i is set.  Per pending level:
//   rho      = sum of momenta over its leaves            (TurnStatistic, :462-467)
//   rfirst   = momentum of its first-built leaf          (zleft or zright of the half tree)
//   cand     = (theta, r, -grad lp, lp, lk) of its multinomial candidate  (:131-136)
//   scalars  = lw (log weight), sum_alpha, n_alpha, dH_max               (:512-542)
// Semantics preserved (SURVEY 8a N1-N8): leaf weights H0 - H' (:174-176); one randexp per internal
// combine in post-order (:191-195, :667) and one for the top-level mh_accept only if the new subtree
// did not terminate (:708-713); a terminated first half is returned without building/combining its
// sibling (:652) -- the terminated node "floats" up through levels whose bit is 0 and is combined at
// levels whose bit is 1, exactly as the unwinding recursion does; divergence iff
// !(-H0 < delta_max - H') (:503-507); direction = sign of the step size (:640, integrator.jl:221-226).
//
// Control flow is warp-uniform (`__any_sync` guarded blocks, per-group predicates) so that groups of
// G < 32 lanes sharing a warp can sit at different tree positions while shuffles stay convergent.
//
// The kernel is compiled in families, one translation unit each (build time): the default sampler/criterion
// (ahmc_nuts.cu), the SliceTS / Classic / Strict variants (ahmc_nuts_var.cu), and the forms that adapt step size and
// metric per chain inside the launch: diagonal WelfordVar (ahmc_nuts_adapt.cu), NutpieVar (ahmc_nuts_nutpie.cu) and, for
// the Dense metric, WelfordCov (ahmc_nuts_cov.cu).
#pragma once
#include "ahmc_chain_adapt.cuh"
#if !defined(AHMC_SIMT_EMULATION) && !defined(__CUDACC_RTC__)
#include "ahmc_dispatch.cuh"
#endif

namespace ahmc {

// workspace layout per chain (doubles): LEFT edge (theta,r,g) | RIGHT edge | rho_tree | M^-1 r of the LEFT edge | of the
// RIGHT edge (Dense metric: the whole-tree criterion then needs no D x D product -- a leaf's dH/dr is parked when the leaf
// becomes an edge) | per level k (7 vectors): 0 rho, 1 rfirst, 2 cand theta, 3 cand r, 4 cand g, 5 rlast (Strict),
// 6 theta_first (Classic)
constexpr int kLevelVecs = 7;
// (+ chain_adapt_vectors(adapt_metric) vectors at the end for the estimator state of the adaptive form, ahmc_chain_adapt.cuh)
__host__ __device__ inline long long nuts_level_doubles(int D, int max_depth) {
    return (long long)(9 + kLevelVecs * (max_depth > 0 ? max_depth : 1)) * D;
}

__device__ __forceinline__ double logaddexp(double a, double b) {  // LogExpFunctions.logaddexp
    double delta = (a == b) ? 0.0 : fabs(a - b);
    double mx = (a != a || b != b) ? CUDART_NAN : (a > b ? a : b);
    return mx + log1p(exp(-delta));
}
__device__ __forceinline__ double maxabs(double a, double b) { return fabs(a) > fabs(b) ? a : b; }  // :526

constexpr int kLevelScalars = 7;  // lw (m), sum_alpha, n_alpha, dH_max, cand lp, cand lk, ww (w)

// Instruction-count cuts of the tree walk (random draws, logaddexp and the leaf's exp dominated it), tape-identical to the
// recursive oracle:
//   * variates are prefetched lane-parallel: lane l of the chain's group generates uniform #(base + l) of the Philox
//     stream (one block per LANE instead of one per DRAW), a draw is then a group broadcast of one register; direction
//     bits come from a cached block (128 doublings each);
//   * multinomial weights are carried as (m, w) pairs -- log-weight = m + log(w), m = the largest leaf log-weight under
//     the node, w in [1, #leaves] -- and the combine decides in the probability domain, u < w_p / (w_p + w_c): one exp per
//     combine, NO log / log1p anywhere in the tree walk (same events; oracle/nuts_iterative.py max_weights);
//   * the acceptance statistic sum_alpha = sum over leaves of exp(min(0, -dH)) is order-free: a leaf parks dH in one
//     lane's register and the exponentials are taken G at a time, one per lane;
//   * FULLTILE = true: the instantiation for D == G * E (64, 128, 256) in which D is a compile-time constant -- the `d < D`
//     guard of every vector load / store and most of the workspace address arithmetic fold away.

// Occupancy: the tree walk is a long chain of dependent, mostly fixed-latency instructions, so throughput scales with
// resident warps per scheduler; cap registers so that this many 4-warp blocks fit per SM (4 was measured slower: spills).
template <int E>
constexpr int nuts_min_blocks() { return E <= 4 ? 3 : (E <= 8 ? 2 : 1); }

// VAR = false: MultinomialTS + GeneralisedNoUTurn only (what `NUTS(delta)` builds); VAR = true additionally compiles
// SliceTS (trajectory.jl:102-109,144-145,164-166,178-189,202,500-502) and the Classic / StrictGeneralised criteria
// (trajectory.jl:551-557, 579-613), selected at run time by a.sampler / a.criterion.
//
// ADAPT = 0: no adaptation; else the estimator form of the chain's in-launch adaptor (ahmc_chain_adapt.cuh):
// AHMC_ADAPT_WELFORD (step size only or WelfordVar, by a.ad.adapt_metric), AHMC_ADAPT_NUTPIE, or AHMC_ADAPT_WELFORD_COV
// (METRIC = kMetricDenseChain: the chain's trajectories read its own M^-1 / factor rows, which its adaptor rewrites at
// window ends).
//
// COOP = true (dense operators, one chain per warp, default family): the block has kCoopWarps warps and every D x D product
// (dH/dr with a Dense metric, grad lp of a dense Gaussian) is a CTA-wide rendezvous -- the matrix is streamed from L2 into
// shared memory once per BLOCK and each element feeds kCoopWarps FMAs (matvec_coop, ahmc_device.cuh) instead of every warp
// re-reading the whole matrix from L2 for its own chain (1.5 MB per leaf per chain at D = 256: the r01 kernel was L2-bound).
// All warps of a block must then reach the product sites together: the votes that steer the loop around them are block-wide,
// and a warp whose chain is idle or finished keeps taking part (its results are ignored, like idle groups of a warp).
// A per-chain Dense metric (METRIC = kMetricDenseChain) never runs in this form: each warp reads its own matrices.
// (the tile flag must not be called FULL: that is the namespace's all-lanes mask used by every *_sync below)
template <int MODEL, int METRIC, int G, int E, bool VAR, int ADAPT, bool FULLTILE, bool COOP = false>
__global__ void __launch_bounds__(COOP ? kCoopThreads : kBlockThreads, COOP ? 1 : nuts_min_blocks<E>()) nuts_kernel(const NutsArgs a) {
    static_assert(!COOP || (G == 32 && !VAR && METRIC != kMetricDenseChain), "COOP: one chain per warp, default family, one matrix");
    constexpr bool kCov = ADAPT == AHMC_ADAPT_WELFORD_COV;
    constexpr int kThreads = COOP ? kCoopThreads : kBlockThreads;
    // warp-uniform predicate -> uniform over everything that must stay in step (the warp, or the block when COOP)
    auto any_peer = [](bool p) -> bool {
        if constexpr (COOP) return __syncthreads_or(p ? 1 : 0) != 0;
        else return __any_sync(FULL, p);
    };
    // Dense metric: a merge needs dH/dr = M^-1 r of the pending half's first leaf -- a D x D product.  The default family
    // caches the vector (slot 1 of the level holds M^-1 r_first instead of r_first) so merges do no dense product at all.
    constexpr bool STORE_DR = !VAR && is_dense_metric(METRIC);
    const int samp = VAR ? a.sampler : 0;    // 0 MultinomialTS, 1 SliceTS
    const int crit = VAR ? a.criterion : 0;  // 0 Generalised, 1 Classic, 2 StrictGeneralised
    double lu = 0.0;                         // SliceTS slice variable (log space)
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    constexpr int kGroups = kThreads / G;
    const long long chain0 = (long long)blockIdx.x * kGroups + grp_in_block;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = FULLTILE ? G * E : a.D;
    const bool dense = (MODEL == AHMC_MODEL_DENSE_GAUSS) || is_dense_metric(METRIC) || (MODEL == AHMC_MODEL_USER);
    constexpr int kSlab = slab_vectors<MODEL>();
    double* xs = COOP ? smem : smem + (size_t)grp_in_block * kSlab * D;  // dense / user-target slab (unused otherwise)
    const int maxd = a.max_depth > 0 ? a.max_depth : 1;
    double* lv = smem + (COOP ? (size_t)coop_smem_doubles(D, coop_kc<E>()) : dense ? (size_t)kGroups * kSlab * D : 0) +
                 (size_t)grp_in_block * maxd * kLevelScalars;
    double* LW = lv;
    double* SA = lv + maxd;
    double* NA = lv + 2 * maxd;
    double* DH = lv + 3 * maxd;
    double* CLP = lv + 4 * maxd;
    double* CLK = lv + 5 * maxd;
    double* WW = lv + 6 * maxd;  // (m, w) weights: LW holds m, WW holds w
    double ww_tree = 1.0, ww_c = 1.0;

    double* base = a.scratch + a.scratch_stride * chain;
    double* LEFT = base;
    double* RIGHT = base + 3 * (long long)D;
    double* RHO = base + 6 * (long long)D;
    double* LEFT_DR = base + 7 * (long long)D;   // Dense metric only
    double* RIGHT_DR = base + 8 * (long long)D;
    auto level = [&](int k) { return base + (9 + kLevelVecs * (long long)k) * D; };

    double eps_c = a.eps_chain ? __ldg(a.eps_chain + chain) : a.eps;
    // adaptive family: the chain's adaptor (ahmc_chain_adapt.cuh), its estimator state behind the tree workspace
    ChainAdapt<G, E, ADAPT == AHMC_ADAPT_NUTPIE ? AHMC_ADAPT_NUTPIE : (kCov ? AHMC_ADAPT_WELFORD_COV : AHMC_ADAPT_WELFORD)> cad{};
    auto cad_ws = [&]() { return base + nuts_level_doubles(D, a.max_depth); };

    ModelOps<MODEL, G, E> mo;
    MetricOps<METRIC, G, E> me;
    mo.load(a.model, l, D);
    if constexpr (kCov) {  // the chain's own rows, filled before the first momentum draw
        MetricDev rows;
        cad.begin_dense(a.ad, a.metric, cad_ws(), valid, chain, l, D);
        me.load(adapt_launch_metric<ADAPT>(a.metric, a.ad, D, rows), chain, l, D);
    } else {
        me.load(a.metric, chain, l, D);
    }
    if constexpr (COOP) {
        mo.coop = smem;
        me.coop = smem;
        coop_begin<E>(smem, D);  // the pipeline's mbarriers (block barrier inside)
    }

    int nexp = 0, ndir = 0;
    uint64_t off = a.rng.offset;  // Philox transition counter of the transition this group is working on
    // Lane-parallel variate prefetch: lane l of the chain's group holds uniform #(vbase + l) of the (chain, transition)
    // stream -- one Philox block per LANE instead of one per DRAW -- and a draw is a group broadcast of one register.
    // peek_u() must be called by every lane of the warp at a warp-uniform point (it shuffles); the take_*() below then
    // consume the peeked value inside the per-chain (divergent) bookkeeping.  Same stream, same values as philox_exp().
    double vbuf = 0.0;
    int vbase = -(1 << 30);
    auto peek_u = [&]() -> double {
        const bool tape = a.rng.exp_tape && nexp < a.rng.exp_stride;
        const bool need = !tape && (nexp < vbase || nexp >= vbase + G);
        if (__any_sync(FULL, need)) {
            if (need) {
                vbase = (nexp / G) * G;
                const int kk = vbase + l;
                uint32_t o[4];
                Philox::gen(a.rng.seed, (uint64_t)chain, (off << 24) ^ (STREAM_EXP << 60) ^ (uint64_t)(kk >> 1), o);
                vbuf = (kk & 1) ? Philox::u01(o[2], o[3]) : Philox::u01(o[0], o[1]);
            }
        }
        return Grp<G>::bcast(vbuf, (nexp - vbase) & (G - 1));
    };
    auto take_exp = [&](double u_pk) -> double {  // randexp
        int k = nexp++;
        if (a.rng.exp_tape && k < a.rng.exp_stride) return a.rng.exp_tape[chain * a.rng.exp_stride + k];
        return -log(u_pk);
    };
    auto take_unif = [&](double u_pk) -> double {  // SliceTS: rand(rng)
        int k = nexp++;
        if (a.rng.exp_tape && k < a.rng.exp_stride) return a.rng.exp_tape[chain * a.rng.exp_stride + k];
        return u_pk;
    };
    auto take_u_of_exp = [&](double u_pk) -> double {  // u = exp(-randexp): the uniform behind the exponential
        int k = nexp++;
        if (a.rng.exp_tape && k < a.rng.exp_stride) return exp(-a.rng.exp_tape[chain * a.rng.exp_stride + k]);
        return u_pk;
    };
    uint32_t cdir[4] = {0u, 0u, 0u, 0u};
    int cdir_blk = -1;  // cached Philox block of direction bits (128 doublings per block)
    auto next_dir = [&]() -> bool {
        int k = ndir++;
        if (a.rng.dir_tape && k < a.rng.dir_stride) return a.rng.dir_tape[chain * a.rng.dir_stride + k] != 0;
        if ((k >> 7) != cdir_blk) {
            cdir_blk = k >> 7;
            Philox::gen(a.rng.seed, (uint64_t)chain, (off << 24) ^ (STREAM_DIR << 60) ^ (uint64_t)cdir_blk, cdir);
        }
        return (cdir[(k >> 5) & 3] >> (k & 31)) & 1u;
    };
    // Deferred acceptance statistic: sum_alpha = sum over the leaves built of exp(min(0, -dH)) is order-free, so the leaf
    // only parks its dH in one lane's register and the exponentials are taken G at a time, one per lane.
    double abuf = 0.0, sa_acc = 0.0;
    int acnt = 0;
    auto alpha_flush = [&](bool mine) {  // warp-uniform call; `mine`: this group flushes now
        double v = (mine && l < acnt) ? exp(jl_min0(-abuf)) : 0.0;
        v = Grp<G>::sum(v);
        if (mine) {
            sa_acc += v;
            acnt = 0;
        }
    };

    // ---- per-transition state (a launch runs n_transitions transitions per chain: the reference's
    //      `for i in 1:n_samples` loop, sampler.jl:182, each chain advancing at its own pace)
    ChainState<E> s;
    double dr[E];
    double H0 = 0.0, zc_lp = 0.0, zc_lk = 0.0;
    double lw_tree = 0.0, sa_tree = 0.0, dh_tree = 0.0;
    int na_tree = 0, j = 0;
    bool term_dyn = false, term_num = false;
    bool done = true, in_sub = false;
    int i = 0, jsub = 0, v = 1;
    int t = 0;
    bool finished = !valid;
    bool need_init = valid;

    while (true) {
        // ---------------------------------------------------------------- (I) begin a transition:
        // z0 = refresh (sampler.jl:55; hamiltonian.jl:213-220) with the cached lp / gradient;
        // tree = BinaryTree(z0, z0, rho = z0.r, 0, 0, 0); sampler = MultinomialTS(z0, lw = 0) (:682-688, :155)
        if (any_peer(need_init)) {
            const bool first = (t == 0);
            double rn[E], drn[E];
            if (need_init) {
                off = a.rng.offset + (uint64_t)t;
                nexp = 0;
                ndir = 0;
                vbase = -(1 << 30);
                cdir_blk = -1;
                sa_acc = 0.0;
                acnt = 0;
                vload_nc<G, E>(s.th, first ? a.th_in + a.ld_in * chain : a.th_out + a.ld_out * chain, l, D);
                vload_nc<G, E>(s.g, first ? a.g_in + a.ld_in * chain : a.g_out + a.ld_out * chain, l, D);
            }
            if (a.refresh) {  // (written out, not draw_momentum: sharing it changes the variant family's generated code)
                if (a.rng.normal_tape) {
                    vload_nc<G, E>(rn, a.rng.normal_tape + (long long)D * chain, l, D);
                } else {
                    philox_normals<G, E>(a.rng.seed, off, chain, l, D, rn);
                }
                me.rand_momentum(rn, l);
                if (a.rng.partial_alpha != 0.0) {  // PartialMomentumRefreshment (hamiltonian.jl:243-254)
                    double rp[E];
                    vload_nc<G, E>(rp, first ? a.r_in + a.ld_in * chain : a.r_out + a.ld_out * chain, l, D);
                    const double al = a.rng.partial_alpha, be = sqrt(1.0 - al * al);
#pragma unroll
                    for (int e = 0; e < E; ++e) rn[e] = al * rp[e] + be * rn[e];
                }
            } else {
                vload_nc<G, E>(rn, first ? a.r_in + a.ld_in * chain : a.r_out + a.ld_out * chain, l, D);
            }
            const double lk0 = map_nonfinite(kinetic<METRIC, G, E>(me, rn, drn, xs, l));
            double u_init = 0.0;
            if (VAR && samp == 1) u_init = peek_u();  // the slice variable's randexp (variate #0 of the transition)
            if (need_init) {
#pragma unroll
                for (int e = 0; e < E; ++e) s.r[e] = rn[e];
                s.lp = first ? map_nonfinite(a.lp_in[chain]) : zc_lp;
                s.lk = lk0;
                H0 = -(s.lp + s.lk);  // energy(z0) (:682)
                zc_lp = s.lp;
                zc_lk = s.lk;
                vstore<G, E>(LEFT, s.th, l, D);
                vstore<G, E>(LEFT + D, s.r, l, D);
                vstore<G, E>(LEFT + 2 * (long long)D, s.g, l, D);
                vstore<G, E>(RIGHT, s.th, l, D);
                vstore<G, E>(RIGHT + D, s.r, l, D);
                vstore<G, E>(RIGHT + 2 * (long long)D, s.g, l, D);
                if constexpr (is_dense_metric(METRIC)) {  // M^-1 r0 (from the kinetic energy above) for both edges
                    vstore<G, E>(LEFT_DR, drn, l, D);
                    vstore<G, E>(RIGHT_DR, drn, l, D);
                }
                vstore<G, E>(RHO, s.r, l, D);
                vstore<G, E>(a.th_out + a.ld_out * chain, s.th, l, D);
                vstore<G, E>(a.r_out + a.ld_out * chain, s.r, l, D);
                vstore<G, E>(a.g_out + a.ld_out * chain, s.g, l, D);
                if (ADAPT && first) cad.begin(a.ad, cad_ws(), eps_c, me.Minv, chain, l, D);  // (WelfordCov: the scalars only)
                lw_tree = 0.0;
                ww_tree = 1.0;
                if (VAR && samp == 1) {  // SliceTS(rng, z0) = SliceTS(z0, neg_energy(z0) - randexp(rng), 1) (:144-145)
                    lu = (s.lp + s.lk) - take_exp(u_init);
                    lw_tree = 1.0;  // n = 1
                }
                sa_tree = 0.0;
                dh_tree = 0.0;
                na_tree = 0;
                j = 0;
                term_dyn = false;
                term_num = false;
                done = !(j < a.max_depth);
                in_sub = false;
                need_init = false;
            }
        }
        // ---------------------------------------------------------------- (F) finish a transition: stats (:725-739), draw
        {
            const bool fl = !finished && done && !in_sub && acnt > 0;
            if (__any_sync(FULL, fl)) alpha_flush(fl);
        }
        {
            const bool fin_now = !finished && done && !in_sub;
            if (fin_now) sa_tree = sa_acc;
            if (fin_now) {
                const long long si = (long long)t * a.N + chain;
                if (a.draws) {
                    double tt[E];
                    vload_nc<G, E>(tt, a.th_out + a.ld_out * chain, l, D);
                    vstore<G, E>(a.draws + si * D, tt, l, D);
                }
                if (l == 0) {
                    const double H = -(zc_lp + zc_lk);
                    a.lp_out[chain] = zc_lp;
                    a.lk_out[chain] = zc_lk;
                    const StatsDev& st = a.st;
                    if (st.n_steps) st.n_steps[si] = na_tree;
                    if (st.is_accept) st.is_accept[si] = 1;
                    if (st.acceptance_rate) st.acceptance_rate[si] = sa_tree / (double)na_tree;
                    if (st.log_density) st.log_density[si] = zc_lp;
                    if (st.hamiltonian_energy) st.hamiltonian_energy[si] = H;
                    if (st.hamiltonian_energy_error) st.hamiltonian_energy_error[si] = H - H0;
                    if (st.max_hamiltonian_energy_error) st.max_hamiltonian_energy_error[si] = dh_tree;
                    if (st.tree_depth) st.tree_depth[si] = j;
                    if (st.numerical_error) st.numerical_error[si] = term_num ? 1 : 0;
                }
                if constexpr (ADAPT && !kCov)  // iteration t + 1 of `sample` (sampler.jl:182): alpha = this transition's acceptance rate
                    cad.update(a.ad, cad_ws(), t + 1, si, sa_tree / (double)na_tree, a.th_out + a.ld_out * chain, a.g_out + a.ld_out * chain,
                               eps_c, me.Minv, chain, l, D);
                ++t;
                if (t < a.n_transitions) need_init = true;
                else finished = true;
            }
            if constexpr (kCov) {  // the WelfordCov form exchanges data across the group: every lane of the warp calls
                // (a group that just finished a transition has advanced t: it was iteration t, entry (t - 1) * N + chain)
                if (__any_sync(FULL, fin_now))
                    cad.update_cov(a.ad, cad_ws(), fin_now, t, (long long)(t - 1) * a.N + chain, sa_tree / (double)na_tree,
                                   a.th_out + a.ld_out * chain, eps_c, chain, l, D);
            }
        }
        if (any_peer(need_init)) continue;

        // ---------------------------------------------------------------- (A) start a doubling (:691-706)
        const bool start = !finished && !done && !in_sub;
        if (__any_sync(FULL, start)) {
            if (start) {
                const bool vleft = next_dir();  // rand(rng, Bool) (:693)
                v = vleft ? -1 : 1;
                const double* edge = vleft ? LEFT : RIGHT;
                vload_nc<G, E>(s.th, edge, l, D);
                vload_nc<G, E>(s.r, edge + D, l, D);
                vload_nc<G, E>(s.g, edge + 2 * (long long)D, l, D);
                jsub = j;
                i = 0;
                in_sub = true;
            }
        }
        if (!any_peer(in_sub)) break;

        // ---------------------------------------------------------------- (B) one leaf (:638-647)
        {
            double t1, t2;  // a leaf is `step(lf, h, z, v)` with |v| = 1: sqrt(alpha) before, 1/sqrt(alpha) after
            temper_muls(a.rng.temper_alpha, 1, 1, t1, t2);
            leapfrog_step<MODEL, METRIC, G, E>(s, mo, me, v > 0 ? eps_c : -eps_c, dr, xs, l, t1, t2);
        }
        const double nE = s.lp + s.lk;  // neg_energy(z')
        const double H1 = -nE;
        const double dH = H1 - H0;
        double lw_c = H0 + nE;                               // MultinomialTS(s, H0, z') (:174-176)
        double sa_c = 0.0;  // (deferred: see alpha_flush)
        if (in_sub) {
            if (l == acnt) abuf = dH;
            ++acnt;
        }
        {
            const bool fl = in_sub && acnt == G;
            if (__any_sync(FULL, fl)) alpha_flush(fl);
        }
        double na_c = 1.0, dh_c = dH;
        bool tnum_c = !(-H0 < a.delta_max + -H1);            // Termination(...) (:503-507)
        if (VAR && samp == 1) {
            lw_c = (lu <= nE) ? 1.0 : 0.0;                   // SliceTS(s, H0, z'): n = Int(lu <= neg_energy) (:164-166)
            tnum_c = !(lu < a.delta_max + -H1);              // Termination(::SliceTS) (:500-502)
        }
        bool tdyn_c = false;
        ww_c = 1.0;  // a leaf: (m, w) = (H0 - H', 1)
        double rho_cur[E];
#pragma unroll
        for (int e = 0; e < E; ++e) rho_cur[e] = s.r[e];  // TurnStatistic(z.r)
        int cand_cur = -1;  // -1: the leaf in registers; k >= 0: candidate stored in level slot k

        // ---------------------------------------------------------------- (C) post-order merges (:649-673)
        bool merging = in_sub;
        bool complete = false;
        int k = 0;
        while (__any_sync(FULL, merging)) {
            if (merging && k == jsub) {
                complete = true;
                merging = false;
            }
            const bool bit = merging && ((i >> k) & 1);
            const bool term_c = tnum_c || tdyn_c;
            const bool do_comb = merging && bit;
            const bool do_store = merging && !bit && !term_c;
            const bool do_float = merging && !bit && term_c;  // terminated first half: returned as is (:652)
            if (__any_sync(FULL, do_comb)) {
                double rho_p[E], rf_p[E], t1[E];
#pragma unroll
                for (int e = 0; e < E; ++e) rho_p[e] = rf_p[e] = 0.0;
                const double* L = level(k);
                if (do_comb) {
                    if (k == 0) {
                        vload_nc<G, E>(rho_p, L + 3 * (long long)D, l, D);  // level 0: rho = rfirst = rlast = cand r
#pragma unroll
                        for (int e = 0; e < E; ++e) rf_p[e] = rho_p[e];
                    } else {
                        vload_nc<G, E>(rho_p, L, l, D);
                        vload_nc<G, E>(rf_p, L + D, l, D);
                    }
                }
                bool uturn_extra = false;
                if (VAR && crit == 2) {
                    // StrictGeneralisedNoUTurn (:579-613).  F = first-built half (pending), S = second-built half (current).
                    //   check A: rho = F.rho + S.rfirst, against dH/dr(F.rfirst), dH/dr(S.rfirst)
                    //   check B: rho = S.rho + F.rlast,  against dH/dr(r_leaf),  dH/dr(F.rlast)
                    // (v = +1: A = check_left_subtree, B = check_right_subtree; v = -1: the other way round)
                    double rsf[E], rl_p[E], tA[E], tB[E];
#pragma unroll
                    for (int e = 0; e < E; ++e) rsf[e] = rl_p[e] = 0.0;
                    if (do_comb && !term_c) {  // (a node that already terminated floats up unchanged: its level slots
                                               //  below k were never written, and the verdict cannot change any more)
                        if (k == 0) {
#pragma unroll
                            for (int e = 0; e < E; ++e) {
                                rsf[e] = s.r[e];      // S is the leaf itself
                                rl_p[e] = rho_p[e];   // F is a single leaf
                            }
                        } else {
                            const double* P = level(k - 1);
                            vload_nc<G, E>(rsf, (k == 1) ? P + 3 * (long long)D : P + D, l, D);
                            vload_nc<G, E>(rl_p, L + 5 * (long long)D, l, D);
                        }
                    }
                    me.dHdr(rf_p, t1, xs, l);
                    me.dHdr(rsf, tA, xs, l);
                    me.dHdr(rl_p, tB, xs, l);
                    double a1 = 0.0, a2 = 0.0, b1 = 0.0, b2 = 0.0;
#pragma unroll
                    for (int e = 0; e < E; ++e) {
                        const double ra = rho_p[e] + rsf[e];
                        const double rb = rho_cur[e] + rl_p[e];
                        a1 = fma(ra, t1[e], a1);
                        a2 = fma(ra, tA[e], a2);
                        b1 = fma(rb, dr[e], b1);
                        b2 = fma(rb, tB[e], b2);
                    }
                    a1 = Grp<G>::sum(a1);
                    a2 = Grp<G>::sum(a2);
                    b1 = Grp<G>::sum(b1);
                    b2 = Grp<G>::sum(b2);
                    uturn_extra = (a1 <= 0.0) || (a2 <= 0.0) || (b1 <= 0.0) || (b2 <= 0.0);
                }
                if (do_comb) {
#pragma unroll
                    for (int e = 0; e < E; ++e) rho_cur[e] += rho_p[e];  // combine(ts) (:467)
                }
                double d1 = 0.0, d2 = 0.0;
                bool uturn;
                if (STORE_DR) {  // dH/dr of the pending half's first leaf was cached when that leaf was stored
#pragma unroll
                    for (int e = 0; e < E; ++e) t1[e] = 0.0;
                    if (do_comb) vload_nc<G, E>(t1, L + D, l, D);
                } else {
                    me.dHdr(rf_p, t1, xs, l);
                }
                if (VAR && crit == 1) {
                    // ClassicNoUTurn (:551-557): s = dot(dtheta, dH/dr(-r_left)) >= 0 || dot(-dtheta, dH/dr(r_right)) >= 0
                    // with dtheta = theta_right - theta_left; q = -dtheta
                    double thf[E];
#pragma unroll
                    for (int e = 0; e < E; ++e) thf[e] = 0.0;
                    if (do_comb) vload_nc<G, E>(thf, (k == 0) ? L + 2 * (long long)D : L + 6 * (long long)D, l, D);
#pragma unroll
                    for (int e = 0; e < E; ++e) {
                        const double q = (v > 0) ? (thf[e] - s.th[e]) : (s.th[e] - thf[e]);
                        d1 = fma(q, t1[e], d1);
                        d2 = fma(q, dr[e], d2);
                    }
                    d1 = Grp<G>::sum(d1);
                    d2 = Grp<G>::sum(d2);
                    uturn = (d1 >= 0.0) || (d2 >= 0.0);
                } else {
                    // isterminated(GeneralisedNoUTurn) on the merged node (:566-570, :615-617)
#pragma unroll
                    for (int e = 0; e < E; ++e) {
                        d1 = fma(rho_cur[e], t1[e], d1);
                        d2 = fma(rho_cur[e], dr[e], d2);
                    }
                    d1 = Grp<G>::sum(d1);
                    d2 = Grp<G>::sum(d2);
                    uturn = (d1 <= 0.0) || (d2 <= 0.0) || uturn_extra;
                }
                const double u_comb = peek_u();
                if (do_comb) {
                    const double lw_p = LW[k], sa_p = 0.0, na_p = NA[k], dh_p = DH[k];  // sum(alpha): see alpha_flush
                    if (VAR && samp == 1) {  // combine(rng, s1::SliceTS, s2) (:178-183)
                        const double n = lw_p + lw_c;
                        if (n * take_unif(u_comb) < lw_p) cand_cur = k;
                        lw_c = n;
                    } else {  // combine(rng, s1, s2) (:191-195) on (m, w) weights, decided in the probability domain
                        const double u = take_u_of_exp(u_comb);
                        const double ww_p = WW[k];
                        const double dlw = lw_p - lw_c;          // m_p - m_c
                        const double tt = (lw_p == lw_c) ? 1.0 : exp(-fabs(dlw));  // like logaddexp: equal (even -Inf) -> 1; NaN in -> NaN
                        double w_new, p_first;
                        if (dlw >= 0.0) {
                            w_new = fma(ww_c, tt, ww_p);
                            p_first = ww_p / w_new;
                            lw_c = lw_p;
                        } else {  // m_c is the larger one, or dlw is NaN (both -Inf: m stays -Inf; a NaN weight: m becomes NaN)
                            w_new = fma(ww_p, tt, ww_c);
                            p_first = ww_p * tt / w_new;
                            lw_c = (lw_p != lw_p) ? lw_p : lw_c;
                        }
                        if ((dlw == dlw) && (u < p_first)) cand_cur = k;  // lw < lw_p + randexp  <=>  u < w_p / (w_p + w_c)
                        ww_c = w_new;
                    }
                    sa_c = (v > 0) ? sa_p + sa_c : sa_c + sa_p;  // treeleft + treeright (:538)
                    na_c += na_p;
                    dh_c = (v > 0) ? maxabs(dh_p, dh_c) : maxabs(dh_c, dh_p);
                    tdyn_c = tdyn_c || uturn;
                }
            }
            if (__any_sync(FULL, do_store)) {
                if (do_store) {
                    double* L = level(k);
                    if (k > 0) {
                        // first-built leaf of this node = first-built leaf of the half merged last (level k-1),
                        // whose slot is still intact (level 0 keeps it as its candidate momentum)
                        double t[E];
                        const double* P = level(k - 1);
                        vload_nc<G, E>(t, (k == 1 && !STORE_DR) ? P + 3 * (long long)D : P + D, l, D);
                        vstore<G, E>(L + D, t, l, D);
                        vstore<G, E>(L, rho_cur, l, D);
                        if (VAR && crit == 2) vstore<G, E>(L + 5 * (long long)D, s.r, l, D);  // rlast = the current leaf
                        if (VAR && crit == 1) {                                                // theta of the first-built leaf
                            vload_nc<G, E>(t, (k == 1) ? P + 2 * (long long)D : P + 6 * (long long)D, l, D);
                            vstore<G, E>(L + 6 * (long long)D, t, l, D);
                        }
                    }
                    if (STORE_DR && k == 0) vstore<G, E>(L + D, dr, l, D);  // M^-1 r of this leaf, for the merge above
                    double clp, clk;
                    if (cand_cur < 0) {
                        vstore<G, E>(L + 2 * (long long)D, s.th, l, D);
                        vstore<G, E>(L + 3 * (long long)D, s.r, l, D);
                        vstore<G, E>(L + 4 * (long long)D, s.g, l, D);
                        clp = s.lp;
                        clk = s.lk;
                    } else {
                        const double* S = level(cand_cur);
                        double t[E];
                        vload_nc<G, E>(t, S + 2 * (long long)D, l, D);
                        vstore<G, E>(L + 2 * (long long)D, t, l, D);
                        vload_nc<G, E>(t, S + 3 * (long long)D, l, D);
                        vstore<G, E>(L + 3 * (long long)D, t, l, D);
                        vload_nc<G, E>(t, S + 4 * (long long)D, l, D);
                        vstore<G, E>(L + 4 * (long long)D, t, l, D);
                        clp = CLP[cand_cur];
                        clk = CLK[cand_cur];
                    }
                    if (l == 0) {
                        WW[k] = ww_c;
                        LW[k] = lw_c;
                        NA[k] = na_c;
                        DH[k] = dh_c;
                        CLP[k] = clp;
                        CLK[k] = clk;
                    }
                    merging = false;
                }
                __syncwarp();
            }
            if (do_comb || do_float) ++k;
        }

        // ---------------------------------------------------------------- (D) subtree complete (:707-722)
        if (any_peer(complete)) {
            const bool sub_term = tnum_c || tdyn_c;
            bool accept = false;
            const double u_top = peek_u();
            if (complete && !sub_term) {
                j = j + 1;
                if (VAR && samp == 1) accept = lw_tree * take_unif(u_top) < lw_c;  // mh_accept(::SliceTS) (:202)
                else accept = take_u_of_exp(u_top) < (ww_c / ww_tree) * exp(lw_c - lw_tree);  // lw_T < lw_c + randexp (:204-206)
            }
            if (accept) {  // zcand = sampler'.zcand
                if (cand_cur < 0) {
                    vstore<G, E>(a.th_out + a.ld_out * chain, s.th, l, D);
                    vstore<G, E>(a.r_out + a.ld_out * chain, s.r, l, D);
                    vstore<G, E>(a.g_out + a.ld_out * chain, s.g, l, D);
                    zc_lp = s.lp;
                    zc_lk = s.lk;
                } else {
                    const double* S = level(cand_cur);
                    double t[E];
                    vload_nc<G, E>(t, S + 2 * (long long)D, l, D);
                    vstore<G, E>(a.th_out + a.ld_out * chain, t, l, D);
                    vload_nc<G, E>(t, S + 3 * (long long)D, l, D);
                    vstore<G, E>(a.r_out + a.ld_out * chain, t, l, D);
                    vload_nc<G, E>(t, S + 4 * (long long)D, l, D);
                    vstore<G, E>(a.g_out + a.ld_out * chain, t, l, D);
                    zc_lp = CLP[cand_cur];
                    zc_lk = CLK[cand_cur];
                }
            }
            // tree = combine(treeleft, treeright) (:715): rho, the moved edge, statistics
            double rho_t[E], r_other[E], t1[E];
#pragma unroll
            for (int e = 0; e < E; ++e) rho_t[e] = r_other[e] = 0.0;
            double* edge = (v < 0) ? LEFT : RIGHT;        // the edge that moves
            const double* other = (v < 0) ? RIGHT : LEFT;
            bool uturn_extra = false;
            if (VAR && crit == 2) {
                // StrictGeneralisedNoUTurn at the top level (:579-613), T = old tree, S = new subtree:
                //   X: rho = T.rho + S.rfirst, against dH/dr(r_far),  dH/dr(S.rfirst)
                //   Y: rho = r_near + S.rho,   against dH/dr(r_near), dH/dr(r_leaf)      (r_near = the edge being replaced)
                double rhoT[E], rsf[E], rnear[E], rfar[E], tA[E], tB[E], tC[E];
#pragma unroll
                for (int e = 0; e < E; ++e) rhoT[e] = rsf[e] = rnear[e] = rfar[e] = 0.0;
                if (complete) {
                    vload_nc<G, E>(rhoT, RHO, l, D);
                    vload_nc<G, E>(rnear, edge + D, l, D);
                    vload_nc<G, E>(rfar, other + D, l, D);
                    if (jsub == 0) {
#pragma unroll
                        for (int e = 0; e < E; ++e) rsf[e] = s.r[e];
                    } else {
                        const double* P = level(jsub - 1);
                        vload_nc<G, E>(rsf, (jsub == 1) ? P + 3 * (long long)D : P + D, l, D);
                    }
                }
                me.dHdr(rfar, tA, xs, l);
                me.dHdr(rsf, tB, xs, l);
                me.dHdr(rnear, tC, xs, l);
                double x1 = 0.0, x2 = 0.0, y1 = 0.0, y2 = 0.0;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const double rx = rhoT[e] + rsf[e];
                    const double ry = rnear[e] + rho_cur[e];
                    x1 = fma(rx, tA[e], x1);
                    x2 = fma(rx, tB[e], x2);
                    y1 = fma(ry, tC[e], y1);
                    y2 = fma(ry, dr[e], y2);
                }
                x1 = Grp<G>::sum(x1);
                x2 = Grp<G>::sum(x2);
                y1 = Grp<G>::sum(y1);
                y2 = Grp<G>::sum(y2);
                uturn_extra = (x1 <= 0.0) || (x2 <= 0.0) || (y1 <= 0.0) || (y2 <= 0.0);
            }
            double th_other[E];
            if (VAR && crit == 1) {
#pragma unroll
                for (int e = 0; e < E; ++e) th_other[e] = 0.0;
                if (complete) vload_nc<G, E>(th_other, other, l, D);
            }
            if (complete) {
                vload_nc<G, E>(rho_t, RHO, l, D);
#pragma unroll
                for (int e = 0; e < E; ++e) rho_t[e] += rho_cur[e];
                vstore<G, E>(RHO, rho_t, l, D);
                vstore<G, E>(edge, s.th, l, D);
                vstore<G, E>(edge + D, s.r, l, D);
                vstore<G, E>(edge + 2 * (long long)D, s.g, l, D);
                vload_nc<G, E>(r_other, other + D, l, D);
            }
            if constexpr (is_dense_metric(METRIC)) {  // dH/dr of both edges is parked: no product at the top level
#pragma unroll
                for (int e = 0; e < E; ++e) t1[e] = 0.0;
                if (complete) {
                    vstore<G, E>((v < 0) ? LEFT_DR : RIGHT_DR, dr, l, D);
                    vload_nc<G, E>(t1, (v < 0) ? RIGHT_DR : LEFT_DR, l, D);
                }
            } else {
                me.dHdr(r_other, t1, xs, l);
            }
            double d1 = 0.0, d2 = 0.0;
            bool uturn_top;
            if (VAR && crit == 1) {  // ClassicNoUTurn on the whole tree: q = -(theta_right - theta_left)
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const double q = (v > 0) ? (th_other[e] - s.th[e]) : (s.th[e] - th_other[e]);
                    d1 = fma(q, t1[e], d1);
                    d2 = fma(q, dr[e], d2);
                }
                d1 = Grp<G>::sum(d1);
                d2 = Grp<G>::sum(d2);
                uturn_top = (d1 >= 0.0) || (d2 >= 0.0);
            } else {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    d1 = fma(rho_t[e], t1[e], d1);
                    d2 = fma(rho_t[e], dr[e], d2);
                }
                d1 = Grp<G>::sum(d1);
                d2 = Grp<G>::sum(d2);
                uturn_top = (d1 <= 0.0) || (d2 <= 0.0) || uturn_extra;
            }
            if (complete) {
                sa_tree = (v < 0) ? sa_c + sa_tree : sa_tree + sa_c;
                na_tree += (int)na_c;
                dh_tree = (v < 0) ? maxabs(dh_c, dh_tree) : maxabs(dh_tree, dh_c);
                if (VAR && samp == 1) {
                    lw_tree = lw_tree + lw_c;  // combine(zcand, s1::SliceTS, s2): n1 + n2 (:185-189)
                } else {                       // combine(zcand, sampler, sampler') (:197-200, :717) on (m, w)
                    const double dT = lw_tree - lw_c;
                    const double tT = (lw_tree == lw_c) ? 1.0 : exp(-fabs(dT));
                    if (dT >= 0.0) {
                        ww_tree = fma(ww_c, tT, ww_tree);
                    } else {
                        ww_tree = fma(ww_tree, tT, ww_c);
                        lw_tree = (lw_tree != lw_tree) ? lw_tree : lw_c;
                    }
                }
                term_dyn = term_dyn || tdyn_c || uturn_top;  // (:719-722)
                term_num = term_num || tnum_c;
                in_sub = false;
                if (term_dyn || term_num || !(j < a.max_depth)) done = true;
            }
            __syncwarp();
        }
        if (in_sub) ++i;
    }

}

#ifndef __CUDACC_RTC__
// dynamic shared memory of a NUTS launch: with `coop` (dense operators, one chain per warp, default family) the
// cooperative products' pipeline (coop_smem_doubles), otherwise the groups' operator slabs (smem_bytes); then every
// group's level scalars
template <int E>
__host__ inline size_t nuts_smem_bytes(bool coop, int model_kind, int metric_kind, int D, int G, int max_depth) {
    const int maxd = max_depth > 0 ? max_depth : 1;
    if (coop) return ((size_t)coop_smem_doubles(D, coop_kc<E>()) + (size_t)kCoopWarps * maxd * kLevelScalars) * sizeof(double);
    return smem_bytes(model_kind, metric_kind, D, G) + (size_t)(kBlockThreads / G) * maxd * kLevelScalars * sizeof(double);
}
#endif

#if !defined(AHMC_SIMT_EMULATION) && !defined(__CUDACC_RTC__)  // host launch code (skipped by the CPU SIMT emulation harness and by NVRTC)
template <int MODEL, int METRIC, int G, int E, bool VAR, int ADAPT>
static cudaError_t launch_nuts_v(const NutsArgs& a, cudaStream_t st) {
    // (a per-chain Dense metric, kMetricDenseChain, has no shared matrix: it always runs warp per chain)
    constexpr bool kDenseOps = (MODEL == AHMC_MODEL_DENSE_GAUSS || METRIC == AHMC_METRIC_DENSE) && METRIC != kMetricDenseChain;
    if constexpr (kDenseOps && G == 32 && !VAR) {
        // dense operators, one chain per warp: blocks of kCoopWarps chains share every D x D product (COOP form)
        const long long blocks = (a.N + kCoopWarps - 1) / kCoopWarps;
        const size_t sm = nuts_smem_bytes<E>(true, MODEL, METRIC, a.D, G, a.max_depth);
        if constexpr (E >= 2 && E <= 8) {
            if (a.D == G * E) return launch_kernel(nuts_kernel<MODEL, METRIC, G, E, VAR, ADAPT, true, true>, blocks, kCoopThreads, sm, st, a);
        }
        return launch_kernel(nuts_kernel<MODEL, METRIC, G, E, VAR, ADAPT, false, true>, blocks, kCoopThreads, sm, st, a);
    } else {
        const size_t sm = nuts_smem_bytes<E>(false, MODEL, METRIC, a.D, G, a.max_depth);
        if constexpr (G == 32 && E >= 2 && E <= 8) {
            if (a.D == G * E) return launch_warps(nuts_kernel<MODEL, METRIC, G, E, VAR, ADAPT, true>, a.N, G, sm, st, a);  // full tile: compile-time D
        }
        return launch_warps(nuts_kernel<MODEL, METRIC, G, E, VAR, ADAPT, false>, a.N, G, sm, st, a);
    }
}

// model x metric dispatch of one (VAR, ADAPT) family (ADAPT: 0, or the adaptor's estimator form, ahmc_chain_adapt.cuh);
// ONE_METRIC restricts the family to the metric its estimator adapts: Diag, or Dense for WelfordCov
template <bool VAR, int ADAPT, bool ONE_METRIC>
static cudaError_t nuts_dispatch(const NutsArgs& a, cudaStream_t st) {
    int G, E;
    if (!pick_layout(a.D, &G, &E)) return cudaErrorInvalidValue;
    auto run = [&](auto metrics, int metric) {
        return with_model_metric_layout(AllModels{}, metrics, a.model.kind, metric, G, E,
                                        [&](auto M, auto K, auto g, auto e) { return launch_nuts_v<M, K, g, e, VAR, ADAPT>(a, st); });
    };
    if constexpr (ONE_METRIC) {  // (compile-time: the family holds no kernels for the other metrics)
        // (WelfordCov: a Dense metric, shared or per chain, as the starting point; the launch reads the chain's own rows)
        constexpr int MK = ADAPT == AHMC_ADAPT_WELFORD_COV ? kMetricDenseChain : AHMC_METRIC_DIAG;
        if (a.metric.kind != (ADAPT == AHMC_ADAPT_WELFORD_COV ? AHMC_METRIC_DENSE : AHMC_METRIC_DIAG)) return cudaErrorInvalidValue;
        return run(Kinds<MK>{}, MK);
    } else {
        return run(AllMetrics{}, metric_form(a.metric));
    }
}

#endif  // AHMC_SIMT_EMULATION

}  // namespace ahmc
