// pair_emu.cpp -- runs K1's two-chains-per-warp fast path (leapfrog_pair_kernel, ahmc_leapfrog.cu, unmodified) under the
// CPU SIMT emulator, launched as the product's launcher does for a lane-contiguous full tile: 8 chains per 128-thread
// block, one coefficient set for the pair when eps is a scalar and M^-1 is shared.  Built alone (tests/test_leapfrog_pair.py)
// or with -DRACE_PAIR -fsanitize=thread as a data-race check of the kernel source.  TEST INFRASTRUCTURE ONLY.
#include <cstdio>
#include <cstdlib>

#include "lf_emu.cpp"

template <int MODEL, int METRIC, bool SHARED>
static void pair_thunk(const void* p) { leapfrog_pair_kernel<MODEL, METRIC, 2, SHARED>(*static_cast<const LeapfrogArgs*>(p)); }

// D = 64 only (G = 32, E = 2), STD_NORMAL / Unit or DIAG_GAUSS / Diag, no tempering or exact checks (the launcher's conditions)
extern "C" int emu_leapfrog_pair(const EmuLf* q) {
    const int D = q->D;
    if (D != 64 || (q->flags & AHMC_FLAG_EXACT_CHECKS) || q->temper_alpha > 0.0) return -1;
    LeapfrogArgs a{};
    a.model = ModelDev{q->model_kind, D, q->p0, q->p1, q->c0};
    a.metric = MetricDev{q->metric_kind, q->Minv, q->minv_stride, q->cholU};
    a.D = D;
    a.N = q->N;
    a.eps = q->eps;
    a.eps_chain = q->eps_chain;
    a.n_steps = q->n_steps;
    a.fwd = q->fwd;
    a.th_in = q->th_in; a.r_in = q->r_in; a.g_in = q->g_in; a.lp_in = q->lp_in;
    a.ld_in = D;
    a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out; a.dr_out = q->dr_out;
    a.ld_out = D;
    a.status = q->status;
    a.steps_done = q->steps_done;
    a.flags = q->flags;
    const int m = q->model_kind, me = q->metric_kind;
    const bool shared = !q->eps_chain && (me != AHMC_METRIC_DIAG || q->minv_stride == 0);
    KernelFn fn = nullptr;
    if (m == AHMC_MODEL_STD_NORMAL && me == AHMC_METRIC_UNIT)
        fn = shared ? pair_thunk<AHMC_MODEL_STD_NORMAL, AHMC_METRIC_UNIT, true> : pair_thunk<AHMC_MODEL_STD_NORMAL, AHMC_METRIC_UNIT, false>;
    else if (m == AHMC_MODEL_DIAG_GAUSS && me == AHMC_METRIC_DIAG)
        fn = shared ? pair_thunk<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, true> : pair_thunk<AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, false>;
    if (!fn) return -2;
    const int chains_per_block = 2 * kBlockThreads / 32;
    emu_launch(fn, &a, (int)((q->N + chains_per_block - 1) / chains_per_block), kBlockThreads);
    return 0;
}

#ifdef RACE_PAIR
// N = 11: a ragged last block and a last warp whose B shadows chain 10; chain 4 defeats the magnitude proof (its pair
// partner stays fast), so the exact path runs inside the same warps.  Shared coefficients, then per-chain eps.
static int run(bool chain_eps) {
    const int D = 64, N = 11;
    std::vector<double> mu(D), w(D), Minv(D), th((size_t)N * D), r((size_t)N * D), g((size_t)N * D), eps(N);
    srand(9);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u(), Minv[d] = 0.7 + 0.6 * u();
    for (auto& x : eps) x = 0.08 + 0.04 * u();
    for (size_t i = 0; i < th.size(); ++i) th[i] = u() - 0.5, r[i] = u() - 0.5;
    th[(size_t)4 * D + 5] = 1e120;
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) g[(size_t)c * D + d] = (th[(size_t)c * D + d] - mu[d]) * w[d];
    std::vector<double> o((size_t)4 * N * D), lpo(N), lko(N);
    std::vector<uint32_t> st(N);
    std::vector<int32_t> done(N);
    EmuLf q{};
    q.model_kind = AHMC_MODEL_DIAG_GAUSS; q.metric_kind = AHMC_METRIC_DIAG; q.D = D; q.N = N; q.p0 = mu.data(); q.p1 = w.data();
    q.Minv = Minv.data(); q.eps = 0.1; q.eps_chain = chain_eps ? eps.data() : nullptr; q.n_steps = 10; q.fwd = 1;
    q.th_in = th.data(); q.r_in = r.data(); q.g_in = g.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D; q.dr_out = o.data() + (size_t)3 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.status = st.data(); q.steps_done = done.data();
    const int rc = emu_leapfrog_pair(&q);
    int finished = 0;
    for (int c = 0; c < N; ++c) finished += done[c] == 10 && st[c] == 0;
    std::printf("pair chain_eps %d: rc %d finished %d of %d\n", (int)chain_eps, rc, finished, N);
    return rc != 0 || finished != N;
}

int main() { return run(false) | run(true); }
#endif
