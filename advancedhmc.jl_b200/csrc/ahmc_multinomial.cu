// ahmc_multinomial.cu -- the trajectory-sampling forms of the static path (SURVEY.md section 8f rank 1):
//
//  * trajectory_kernel : `step(lf, h, z, n; full_trajectory = Val(true))` (src/integrator.jl:229,249-261) --
//    every intermediate phase point is written out (streaming: one D x N slab per step).
//  * multinomial_kernel: static transition with `MultinomialTS` (src/trajectory.jl:344-390) --
//    n_fwd forward and n_bwd backward steps from z, the new point drawn from the WHOLE trajectory with
//    probabilities softmax(-H) by inverse CDF (`randcat`, src/utilities.jl:92-103), acceptance statistic
//    mean_i min(1, exp(H0 - H_i)).  The reference materialises all n+1 phase points (`vcat(reverse(zs_bwd)...,
//    z, zs_fwd...)`); here only the n+1 ENERGIES are kept (per-chain scratch), the index is selected, and the
//    chosen point is re-materialised by re-running that many steps from z: same arithmetic, same bits, no
//    O(n * D) trajectory storage.
#include "ahmc_kernels.cuh"
#ifndef AHMC_SIMT_EMULATION
#include "ahmc_dispatch.cuh"
#endif

namespace ahmc {

// ------------------------------------------------------------------------------------------------ full_trajectory
template <int MODEL, int METRIC, int G, int E>
__global__ void __launch_bounds__(kBlockThreads) trajectory_kernel(const TrajArgs a) {
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + grp_in_block;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = a.D;
    double* xs = smem + (size_t)grp_in_block * D;
    double eps = a.eps_chain ? __ldg(a.eps_chain + chain) : a.eps;
    eps = a.fwd ? eps : -eps;
    ModelOps<MODEL, G, E> mo;
    MetricOps<METRIC, G, E> me;
    mo.load(a.model, l, D);
    me.load(a.metric, chain, l, D);
    ChainState<E> s;
    double dr[E];
    vload_nc<G, E>(s.th, a.th_in + a.ld_in * chain, l, D);
    vload_nc<G, E>(s.r, a.r_in + a.ld_in * chain, l, D);
    vload_nc<G, E>(s.g, a.g_in + a.ld_in * chain, l, D);
    const double sa = a.temper_alpha > 0.0 ? sqrt(a.temper_alpha) : 1.0;  // (hoisted out of the step loop: not temper_muls)
    bool active = valid;
    int done = 0;
    for (int i = 1; i <= a.n_steps; ++i) {
        double t1 = 1.0, t2 = 1.0;
        if (a.temper_alpha > 0.0) {
            t1 = (2 * (i - 1) + 1 <= a.n_steps) ? sa : 1.0 / sa;
            t2 = (2 * (i - 1) + 2 <= a.n_steps) ? sa : 1.0 / sa;
        }
        const bool fin = leapfrog_step<MODEL, METRIC, G, E>(s, mo, me, eps, dr, xs, l, t1, t2);
        if (active) {  // res[i] = z (integrator.jl:249-251)
            const long long o = (long long)(i - 1) * a.step_stride + a.ld_out * chain;
            vstore<G, E>(a.th_out + o, s.th, l, D);
            vstore<G, E>(a.r_out + o, s.r, l, D);
            vstore<G, E>(a.g_out + o, s.g, l, D);
            if (a.dr_out) vstore<G, E>(a.dr_out + o, dr, l, D);
            if (l == 0) {
                a.lp_out[(long long)(i - 1) * a.N + chain] = s.lp;
                a.lk_out[(long long)(i - 1) * a.N + chain] = s.lk;
            }
            done = i;
            if (!fin) active = false;  // resize!(res, i); break (integrator.jl:252-258)
        }
        if (!__any_sync(FULL, active)) break;
    }
    if (valid && l == 0 && a.steps_done) a.steps_done[chain] = done;
}

// ------------------------------------------------------------------------------------------------ MultinomialTS static
template <int MODEL, int METRIC, int G, int E>
__global__ void __launch_bounds__(kBlockThreads) multinomial_kernel(const MultinomialArgs a) {
    extern __shared__ double smem[];
    const int l = threadIdx.x % G;
    const int grp_in_block = threadIdx.x / G;
    const long long chain0 = (long long)blockIdx.x * (kBlockThreads / G) + grp_in_block;
    const bool valid = chain0 < a.N;
    const long long chain = valid ? chain0 : a.N - 1;
    const int D = a.D;
    double* xs = smem + (size_t)grp_in_block * D;
    const double eps = a.eps_chain ? __ldg(a.eps_chain + chain) : a.eps;
    ModelOps<MODEL, G, E> mo;
    MetricOps<METRIC, G, E> me;
    mo.load(a.model, l, D);
    me.load(a.metric, chain, l, D);
    const int n_fwd = a.n_fwd, n_bwd = a.n_steps - a.n_fwd;
    double* Hs = a.energies + (long long)(a.n_steps + 1) * chain;  // [0..n_bwd): bwd step j+1; then fwd

    // z = refresh(rng, h, z) with the cached lp / gradient (hamiltonian.jl:213-220)
    double r0[E], dr[E];
    if (a.refresh) {
        draw_momentum(me, a.rng.normal_tape, a.rng.seed, a.rng.offset, chain, l, D, r0);
        if (a.rng.partial_alpha != 0.0) {
            double rp[E];
            vload_nc<G, E>(rp, a.r_in + a.ld_in * chain, l, D);
            const double al = a.rng.partial_alpha, be = sqrt(1.0 - al * al);
#pragma unroll
            for (int e = 0; e < E; ++e) r0[e] = al * rp[e] + be * r0[e];
        }
    } else {
        vload_nc<G, E>(r0, a.r_in + a.ld_in * chain, l, D);
    }
    const double lk0 = map_nonfinite(kinetic<METRIC, G, E>(me, r0, dr, xs, l));
    const double lp0 = map_nonfinite(a.lp_in[chain]);
    const double H0 = -(lp0 + lk0);

    ChainState<E> s;
    auto restart = [&]() {
        vload_nc<G, E>(s.th, a.th_in + a.ld_in * chain, l, D);
        vload_nc<G, E>(s.g, a.g_in + a.ld_in * chain, l, D);
#pragma unroll
        for (int e = 0; e < E; ++e) s.r[e] = r0[e];
        s.lp = lp0;
        s.lk = lk0;
    };
    // ---- pass 1: energies along the backward and forward sweeps (per-chain break on non-finite)
    int nb = 0, nf = 0;
    restart();
    {
        bool active = valid;
        for (int i = 1; i <= n_bwd; ++i) {
            double t1, t2;
            temper_muls(a.rng.temper_alpha, i, n_bwd, t1, t2);  // each leg is its own `step` call (trajectory.jl:374-376)
            const bool fin = leapfrog_step<MODEL, METRIC, G, E>(s, mo, me, -eps, dr, xs, l, t1, t2);
            if (active) {
                if (l == 0) Hs[i - 1] = -(s.lp + s.lk);
                nb = i;
                if (!fin) active = false;
            }
            if (!__any_sync(FULL, active)) break;
        }
    }
    restart();
    {
        bool active = valid;
        for (int i = 1; i <= n_fwd; ++i) {
            double t1, t2;
            temper_muls(a.rng.temper_alpha, i, n_fwd, t1, t2);
            const bool fin = leapfrog_step<MODEL, METRIC, G, E>(s, mo, me, eps, dr, xs, l, t1, t2);
            if (active) {
                if (l == 0) Hs[n_bwd + i - 1] = -(s.lp + s.lk);
                nf = i;
                if (!fin) active = false;
            }
            if (!__any_sync(FULL, active)) break;
        }
    }
    __syncwarp();
    // ---- selection: trajectory order = bwd[nb], ..., bwd[1], z, fwd[1], ..., fwd[nf]
    const int len = nb + 1 + nf;
    auto Hat = [&](int p) -> double {  // energy of the p-th point (0-based) in trajectory order
        if (p < nb) return Hs[nb - 1 - p];
        if (p == nb) return H0;
        return Hs[n_bwd + (p - nb - 1)];
    };
    double mx = -CUDART_INF;
    for (int p = 0; p < len; ++p) {
        const double w = -Hat(p);
        mx = (w > mx) ? w : mx;
    }
    double ssum = 0.0;
    for (int p = 0; p < len; ++p) ssum += exp(-Hat(p) - mx);
    const double lse = mx + log(ssum);  // logsumexp(unnorm_lp)
    double u;
    if (a.rng.exp_tape) u = a.rng.exp_tape[chain];
    else {
        uint32_t o[4];
        Philox::gen(a.rng.seed, (uint64_t)chain, (a.rng.offset << 24) ^ (STREAM_EXP << 60), o);
        u = Philox::u01(o[0], o[1]);
    }
    double C = 0.0, asum = 0.0;
    int cnt = 0;
    for (int p = 0; p < len; ++p) {
        const double Hp = Hat(p);
        C += exp(-Hp - lse);                   // cumsum(P) (utilities.jl:101)
        if (C < u) ++cnt;                      // count(C .< u)
        asum += exp(jl_min0(-(Hp - H0)));     // alpha_i = exp(min(0, -dH)) (trajectory.jl:386-388)
    }
    int idx = cnt;
    if (idx > len - 1) idx = len - 1;
    const double alpha = asum / (double)len;
    // ---- pass 2: re-materialise the chosen point (k steps in its direction from z)
    const int k = (idx < nb) ? (nb - idx) : (idx - nb);
    const double eps_dir = (idx < nb) ? -eps : eps;
    const int kmax = __reduce_max_sync(FULL, valid ? k : 0);
    restart();
    double* tho = a.th_out + a.ld_out * chain;
    double* ro = a.r_out + a.ld_out * chain;
    double* go = a.g_out + a.ld_out * chain;
    auto emit = [&]() {
        double nr[E];
#pragma unroll
        for (int e = 0; e < E; ++e) nr[e] = -s.r[e];  // flip (trajectory.jl:283)
        vstore<G, E>(tho, s.th, l, D);
        vstore<G, E>(ro, nr, l, D);
        vstore<G, E>(go, s.g, l, D);
        if (l == 0) {
            const double H = -(s.lp + s.lk);
            a.lp_out[chain] = s.lp;
            a.lk_out[chain] = s.lk;
            const StatsDev& st = a.st;  // (not record_stats: sharing it changes this kernel's generated code)
            if (st.n_steps) st.n_steps[chain] = a.n_steps;
            if (st.is_accept) st.is_accept[chain] = 1;
            if (st.acceptance_rate) st.acceptance_rate[chain] = alpha;
            if (st.log_density) st.log_density[chain] = s.lp;
            if (st.hamiltonian_energy) st.hamiltonian_energy[chain] = H;
            if (st.hamiltonian_energy_error) st.hamiltonian_energy_error[chain] = H - H0;
            if (st.numerical_error) st.numerical_error[chain] = finite_d(H) ? 0 : 1;
            if (st.tree_depth) st.tree_depth[chain] = idx - nb;  // signed offset of the draw from z
        }
    };
    if (valid && k == 0) emit();
    for (int i = 1; i <= kmax; ++i) {
        double t1, t2;
        temper_muls(a.rng.temper_alpha, i, (idx < nb) ? n_bwd : n_fwd, t1, t2);
        leapfrog_step<MODEL, METRIC, G, E>(s, mo, me, eps_dir, dr, xs, l, t1, t2);
        if (valid && i == k) emit();
    }
}

// ------------------------------------------------------------------------------------------------ dispatch
#ifndef AHMC_SIMT_EMULATION  // host launch code (skipped by the CPU SIMT emulation harness, tests/simt_emu/)
// f(MODEL, METRIC, G, E) for a full-trajectory or multinomial launch
template <class Args, class F>
static cudaError_t traj_dispatch(const Args& a, int* n_launches, F&& f) {
    int G, E;
    if (!pick_layout(a.D, &G, &E)) return cudaErrorInvalidValue;
    if (n_launches) *n_launches += 1;
    return with_model_metric_layout(AllModels{}, AllMetrics{}, a.model.kind, metric_form(a.metric), G, E, f);
}
cudaError_t launch_trajectory(const TrajArgs& a, cudaStream_t st, int* n_launches) {
    return traj_dispatch(a, n_launches, [&](auto M, auto K, auto g, auto e) {
        return launch_warps(trajectory_kernel<M, K, g, e>, a.N, g, smem_bytes(M, K, a.D, g), st, a);
    });
}
cudaError_t launch_multinomial(const MultinomialArgs& a, cudaStream_t st, int* n_launches) {
    return traj_dispatch(a, n_launches, [&](auto M, auto K, auto g, auto e) {
        return launch_warps(multinomial_kernel<M, K, g, e>, a.N, g, smem_bytes(M, K, a.D, g), st, a);
    });
}

#endif  // AHMC_SIMT_EMULATION

}  // namespace ahmc
