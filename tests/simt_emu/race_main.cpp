// race_main.cpp -- a data-race check for the kernel SOURCES: the emulator harnesses run under ThreadSanitizer
// (g++ -fsanitize=thread).  Every CUDA thread is a host thread and the only synchronisation is what the kernel itself
// asks for (shuffles / votes / __syncwarp -> the warp's barrier, __syncthreads -> the block's, mbarriers and atomics ->
// std::atomic_ref), so a missing barrier or fence in the kernel is a data race TSan reports -- the CPU counterpart of
// compute-sanitizer's racecheck, and it also covers the staged compile-time variants that have not run on a GPU yet.
// Build: -DRACE_NUTS, -DRACE_DENSE, -DRACE_LF, -DRACE_MN, -DRACE_ADAPT or -DRACE_GLM (plus the variant's -D knobs); the same
// mains also run under AddressSanitizer (tests/test_tensor_pipe_shapes_cpu.py).  TEST INFRASTRUCTURE ONLY (tests/test_simt_emulation.py).
#include <cstdio>
#include <cstdlib>
#include <vector>

#if defined(RACE_NUTS)
#include "nuts_emu.cpp"

static int run(int model, int metric, int D, int N, int T, int sampler, int criterion, bool adapt) {
    std::vector<double> mu(D), w(D), Minv, cholU, th((size_t)N * D), r((size_t)N * D, 0.0), g((size_t)N * D), lp(N, 0.0);
    std::vector<double> P;
    srand(7 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u();
    if (model == AHMC_MODEL_DENSE_GAUSS) {  // tridiagonal precision
        P.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            P[(size_t)d * D + d] = 1.0 + 0.1 * u();
            if (d) P[(size_t)d * D + d - 1] = P[(size_t)(d - 1) * D + d] = 0.2;
        }
    }
    if (metric == AHMC_METRIC_DIAG) {
        Minv.resize(D);
        for (auto& x : Minv) x = 0.7 + 0.6 * u();
    } else if (metric == AHMC_METRIC_DENSE) {  // diagonal matrices in dense storage: Minv and its Cholesky factor
        Minv.assign((size_t)D * D, 0.0);
        cholU.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            const double s = 0.8 + 0.4 * u();
            Minv[(size_t)d * D + d] = s * s;
            cholU[(size_t)d * D + d] = s;
        }
    }
    for (int c = 0; c < N; ++c) {
        for (int d = 0; d < D; ++d) th[(size_t)c * D + d] = u() - 0.5;
        for (int d = 0; d < D; ++d) {  // -grad log pi and log pi at theta
            double gd = 0.0;
            if (model == AHMC_MODEL_DENSE_GAUSS)
                for (int k = 0; k < D; ++k) gd += P[(size_t)k * D + d] * (th[(size_t)c * D + k] - mu[k]);
            else if (model == AHMC_MODEL_DIAG_GAUSS) gd = (th[(size_t)c * D + d] - mu[d]) * w[d];
            else gd = th[(size_t)c * D + d];
            g[(size_t)c * D + d] = gd;
            lp[c] -= 0.5 * gd * (th[(size_t)c * D + d] - (model == AHMC_MODEL_STD_NORMAL ? 0.0 : mu[d]));
        }
    }
    std::vector<double> o((size_t)3 * N * D), lpo(N), lko(N), acc((size_t)T * N), dH((size_t)T * N), dHm((size_t)T * N);
    std::vector<double> draws((size_t)T * N * D), eps_rw(N, 0.3), minv_rw((size_t)N * D, 0.0), trace((size_t)T * N);
    std::vector<int32_t> ns((size_t)T * N), td((size_t)T * N);
    std::vector<uint8_t> ne((size_t)T * N);
    EmuNuts q{};
    q.model_kind = model; q.metric_kind = metric; q.D = D; q.N = N;
    q.p0 = model == AHMC_MODEL_STD_NORMAL ? nullptr : mu.data();
    q.p1 = model == AHMC_MODEL_DENSE_GAUSS ? P.data() : (model == AHMC_MODEL_DIAG_GAUSS ? w.data() : nullptr);
    q.Minv = Minv.empty() ? nullptr : Minv.data();
    q.cholU = cholU.empty() ? nullptr : cholU.data();
    q.eps = 0.3; q.max_depth = 5; q.delta_max = 1000.0; q.sampler = sampler; q.criterion = criterion;
    q.seed = 11; q.refresh = 1;
    q.th_in = th.data(); q.r_in = r.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.n_steps = ns.data(); q.tree_depth = td.data(); q.numerical = ne.data();
    q.acc = acc.data(); q.dH = dH.data(); q.dHmax = dHm.data(); q.n_transitions = T; q.draws = draws.data();
    if (adapt) {
        q.adapt = 1; q.n_adapts = T - 2; q.init_buffer = 2; q.term_buffer = 2; q.window_size = 3;
        q.delta = 0.8; q.gamma = 0.05; q.t0 = 10.0; q.kappa = 0.75; q.adapt_metric = 1; q.n_min = 3;
        q.eps_rw = eps_rw.data(); q.minv_rw = minv_rw.data(); q.eps_trace = trace.data();
    }
    const int rc = emu_nuts(&q);
    long steps = 0;
    for (auto s : ns) steps += s;
    std::printf("nuts model %d metric %d D %d N %d sampler %d criterion %d adapt %d: rc %d, %ld leapfrog steps\n", model, metric, D, N,
                sampler, criterion, (int)adapt, rc, steps);
    return rc != 0 || steps < (long)T * N;
}

int main() {
    int bad = 0;
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 6, 9, 4, 0, 0, false);    // four chains per warp, ragged last block
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 40, 5, 3, 0, 0, false);   // one chain per warp (or the alt layouts)
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 100, 3, 2, 0, 0, false);  // the headline layout
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, 6, 5, 3, 0, 0, false);  // shared-memory operator slabs
    bad |= run(AHMC_MODEL_FUNNEL, AHMC_METRIC_DIAG, 5, 6, 3, 1, 2, false);        // SliceTS + strict criterion family
    bad |= run(AHMC_MODEL_STD_NORMAL, AHMC_METRIC_UNIT, 3, 7, 3, 0, 1, false);    // classic criterion
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, 40, 11, 2, 0, 0, false);  // COOP form: 8 chains per block share the D x D products
    // in-launch adaptation (chain workspace).  N fills its block: the idle groups of a ragged block alias the LAST chain
    // read-only (`chain = N - 1`, ahmc_nuts_kernel.cuh) and their unused load of its step size would be reported against the
    // owner's write-back of the adapted value -- a benign read, excluded here rather than suppressed.
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 6, 16, 12, 0, 0, true);
    return bad;
}

#elif defined(RACE_DENSE)
#include "dense_emu.cpp"

static int run(int D, int N, bool denseP, bool denseM, int n, int wide) {
    std::vector<double> P((size_t)D * D, 0.0), M((size_t)D * D, 0.0), w(D), md(D), mu(D, 0.1), th((size_t)N * D), r((size_t)N * D),
        g((size_t)N * D), o((size_t)4 * N * D), lp(N), lk(N);
    srand(3 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int i = 0; i < D; ++i) {
        P[(size_t)i * D + i] = 1.0 + 0.01 * i;
        M[(size_t)i * D + i] = 0.5 + 0.002 * i;
        if (i) P[(size_t)i * D + i - 1] = P[(size_t)(i - 1) * D + i] = 0.1, M[(size_t)i * D + i - 1] = M[(size_t)(i - 1) * D + i] = 0.05;
        w[i] = 0.8 + 0.4 * u();
        md[i] = 0.7 + 0.5 * u();
    }
    for (auto* v : {&th, &r, &g})
        for (auto& x : *v) x = u() - 0.5;
    std::vector<uint32_t> st(N);
    std::vector<int32_t> done(N);
    std::vector<uint8_t> need(N);
    EmuDense q{};
    q.D = D; q.N = N; q.P = denseP ? P.data() : nullptr; q.w = denseP ? nullptr : w.data(); q.mu = mu.data();
    q.Minv = denseM ? M.data() : nullptr; q.Mdiag = denseM ? nullptr : md.data(); q.eps = 0.1; q.n_steps = n; q.fwd = 1;
    q.th_in = th.data(); q.r_in = r.data(); q.g_in = g.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D; q.dr_out = o.data() + (size_t)3 * N * D;
    q.lp_out = lp.data(); q.lk_out = lk.data(); q.status = st.data(); q.steps_done = done.data(); q.need_exact = need.data();
    q.wide_tile = wide;
    const int rc = emu_dense(&q);
    std::printf("dense D %d N %d P %d M %d: rc %d lp0 %.6f need0 %d\n", D, N, (int)denseP, (int)denseM, rc, lp[0], (int)need[0]);
    return rc != 0 || need[0] != 0;
}

int main() {
    int bad = 0;
    bad |= run(40, 37, true, true, 4, 0);    // <1,4>: two products per step, ragged second tile
    bad |= run(100, 20, true, false, 3, 0);  // <2,2,2>
    bad |= run(70, 33, false, true, 3, 1);   // <2,4>
    bad |= run(130, 9, true, true, 2, 0);    // <3,2>: 12 chunks per product
    return bad;
}
#elif defined(RACE_LF)
#include "lf_emu.cpp"

static int run(int model, int metric, int D, int N, int n, int hmc) {
    std::vector<double> mu(D), w(D), P, Minv, cholU, th((size_t)N * D), r((size_t)N * D), g((size_t)N * D), lp(N, 0.0);
    srand(5 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u();
    if (model == AHMC_MODEL_DENSE_GAUSS) {
        P.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            P[(size_t)d * D + d] = 1.0 + 0.1 * u();
            if (d) P[(size_t)d * D + d - 1] = P[(size_t)(d - 1) * D + d] = 0.2;
        }
    }
    if (metric == AHMC_METRIC_DIAG) {
        Minv.resize(D);
        for (auto& x : Minv) x = 0.7 + 0.6 * u();
    } else if (metric == AHMC_METRIC_DENSE) {
        Minv.assign((size_t)D * D, 0.0);
        cholU.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            const double s = 0.8 + 0.4 * u();
            Minv[(size_t)d * D + d] = s * s;
            cholU[(size_t)d * D + d] = s;
        }
    }
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {
            th[(size_t)c * D + d] = u() - 0.5;
            r[(size_t)c * D + d] = u() - 0.5;
        }
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {
            double gd = 0.0;
            if (model == AHMC_MODEL_DENSE_GAUSS)
                for (int k = 0; k < D; ++k) gd += P[(size_t)k * D + d] * (th[(size_t)c * D + k] - mu[k]);
            else gd = (th[(size_t)c * D + d] - mu[d]) * w[d];
            g[(size_t)c * D + d] = gd;
            lp[c] -= 0.5 * gd * (th[(size_t)c * D + d] - mu[d]);
        }
    std::vector<double> o((size_t)4 * N * D), lpo(N), lko(N), acc(N), dH(N);
    std::vector<uint32_t> st(N);
    std::vector<int32_t> done(N);
    std::vector<uint8_t> isacc(N);
    EmuLf q{};
    q.model_kind = model; q.metric_kind = metric; q.D = D; q.N = N; q.p0 = mu.data();
    q.p1 = model == AHMC_MODEL_DENSE_GAUSS ? P.data() : w.data();
    q.Minv = Minv.data(); q.cholU = cholU.empty() ? nullptr : cholU.data(); q.eps = 0.1; q.n_steps = n; q.fwd = 1;
    q.th_in = th.data(); q.r_in = r.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D; q.dr_out = o.data() + (size_t)3 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.status = st.data(); q.steps_done = done.data();
    q.hmc = hmc; q.refresh = 1; q.n_transitions = 1; q.seed = 3; q.is_accept = isacc.data(); q.acc = acc.data(); q.dH = dH.data();
    const int rc = emu_leapfrog(&q);
    std::printf("lf model %d metric %d D %d N %d hmc %d: rc %d lp0 %.6f\n", model, metric, D, N, hmc, rc, lpo[0]);
    return rc != 0;
}

int main() {
    int bad = 0;
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 7, 21, 12, 0);   // K1 fused fast path, four chains per warp, ragged block
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, 6, 9, 6, 0);   // K1 exact path with the shared-memory operator slabs
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 40, 5, 8, 0);    // one chain per warp
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 7, 21, 5, 1);    // K2: refresh + trajectory + Metropolis step
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_DENSE, 6, 9, 4, 1);
    return bad;
}
#elif defined(RACE_MN)
#include "mn_emu.cpp"

static int run(int model, int metric, int D, int N, int n, int n_fwd) {
    std::vector<double> mu(D), w(D), P, Minv, cholU, th((size_t)N * D), g((size_t)N * D), lp(N, 0.0);
    std::vector<double> normals((size_t)N * D), unif(N);
    srand(9 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int d = 0; d < D; ++d) mu[d] = u() - 0.5, w[d] = 0.5 + u();
    if (model == AHMC_MODEL_DENSE_GAUSS) {
        P.assign((size_t)D * D, 0.0);
        for (int d = 0; d < D; ++d) {
            P[(size_t)d * D + d] = 1.0 + 0.1 * u();
            if (d) P[(size_t)d * D + d - 1] = P[(size_t)(d - 1) * D + d] = 0.2;
        }
    }
    if (metric == AHMC_METRIC_DIAG) {
        Minv.resize(D);
        for (auto& x : Minv) x = 0.7 + 0.6 * u();
    }
    for (int c = 0; c < N; ++c) {
        unif[c] = u();
        for (int d = 0; d < D; ++d) th[(size_t)c * D + d] = u() - 0.5, normals[(size_t)c * D + d] = 2.0 * u() - 1.0;
    }
    for (int c = 0; c < N; ++c)
        for (int d = 0; d < D; ++d) {
            double gd = 0.0;
            if (model == AHMC_MODEL_DENSE_GAUSS)
                for (int k = 0; k < D; ++k) gd += P[(size_t)k * D + d] * (th[(size_t)c * D + k] - mu[k]);
            else gd = (th[(size_t)c * D + d] - mu[d]) * w[d];
            g[(size_t)c * D + d] = gd;
            lp[c] -= 0.5 * gd * (th[(size_t)c * D + d] - mu[d]);
        }
    std::vector<double> o((size_t)3 * N * D), lpo(N), lko(N), acc(N);
    std::vector<int32_t> idx(N);
    EmuMn q{};
    q.model_kind = model; q.metric_kind = metric; q.D = D; q.N = N; q.p0 = mu.data();
    q.p1 = model == AHMC_MODEL_DENSE_GAUSS ? P.data() : w.data();
    q.Minv = Minv.empty() ? nullptr : Minv.data(); q.eps = 0.2; q.n_steps = n; q.n_fwd = n_fwd;
    q.normal_tape = normals.data(); q.unif_tape = unif.data(); q.th_in = th.data(); q.g_in = g.data(); q.lp_in = lp.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D;
    q.lp_out = lpo.data(); q.lk_out = lko.data(); q.acc = acc.data(); q.index = idx.data();
    const int rc = emu_multinomial(&q);
    std::printf("mn model %d metric %d D %d N %d: rc %d acc0 %.6f\n", model, metric, D, N, rc, acc[0]);
    return rc != 0;
}

int main() {
    int bad = 0;
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 7, 21, 7, 3);    // four chains per warp, ragged block, both directions
    bad |= run(AHMC_MODEL_DENSE_GAUSS, AHMC_METRIC_UNIT, 6, 9, 5, 5);    // shared-memory precision slab
    bad |= run(AHMC_MODEL_DIAG_GAUSS, AHMC_METRIC_DIAG, 40, 5, 6, 0);    // one chain per warp, all backward
    return bad;
}
#elif defined(RACE_ADAPT)
#include "adapt_emu.cpp"

int main() {
    const int D = 37;
    const long long N = 300;
    std::vector<double> theta((size_t)N * D), alpha(N), rec(2 + 2 * D), cov((size_t)D * D);
    srand(2);
    for (auto& x : theta) x = rand() / (double)RAND_MAX - 0.5;
    for (auto& x : alpha) x = rand() / (double)RAND_MAX;
    const int rc = emu_adapt(D, N, theta.data(), alpha.data(), rec.data(), cov.data());
    std::printf("adapt D %d N %lld: rc %d n %.0f\n", D, N, rc, rec[0]);
    return rc != 0 || rec[0] != (double)N;
}
#elif defined(RACE_GLM)
#include "glm_emu.cpp"

// K6: a 9-coordinate Bernoulli-logit target with 70 rows (two chunks, a partial last one), a ragged second tile
int main() {
    const int D = 9, n = 70, N = 17, steps = 2;
    std::vector<double> X((size_t)n * D), y(n), prec(D, 1.0), th((size_t)N * D), r((size_t)N * D), o((size_t)6 * N * D), lp(N), lk(N);
    std::vector<uint32_t> status(N);
    std::vector<int32_t> done(N);
    srand(3);
    auto u = [] { return rand() / (double)RAND_MAX - 0.5; };
    for (auto& x : X) x = u();
    for (auto& v : y) v = u() > 0.0 ? 1.0 : 0.0;
    for (auto& v : th) v = 0.3 * u();
    for (auto& v : r) v = u();
    EmuGlm e{};
    e.family = AHMC_GLM_BERNOULLI_LOGIT; e.D = D; e.n = n; e.N = N; e.X = X.data(); e.y = y.data(); e.prec = prec.data();
    e.eps = 0.05; e.n_steps = steps; e.fwd = 1; e.th_in = th.data(); e.r_in = r.data();
    double* p = o.data();
    e.th_out = p; e.r_out = p + N * D; e.g_out = p + 2 * N * D; e.dr_out = p + 3 * N * D; e.lp_out = lp.data(); e.lk_out = lk.data();
    e.status = status.data(); e.steps_done = done.data();
    const int rc = emu_glm(&e);
    int bad = rc != 0;
    for (int c = 0; c < N; ++c) bad |= status[c] != 0 || done[c] != steps || !std::isfinite(lp[c]);
    std::printf("glm D %d n %d N %d: rc %d\n", D, n, N, bad);
    return bad;
}
#else
#error "define RACE_NUTS, RACE_DENSE, RACE_LF, RACE_MN, RACE_ADAPT or RACE_GLM"
#endif
