"""CPU checks of the Dense-metric in-launch warm-up (WelfordCov, ahmc_chain_adapt.cuh) on run-time compiled targets: the
adaptive NUTS and static-HMC kernels instantiated as the run-time compiler instantiates them for a Dense warm-up
(AHMC_MODEL_USER, the per-chain Dense kind, the WelfordCov form) run a correlated Gaussian written as user source, in the
group form and the one-lane form, under the SIMT emulator (tests/simt_emu/dense_user_adapt_emu.cpp).  Every iteration is
replayed with the oracle's transition on the same Philox draws (tests/philox_ref.py), the oracle's DualAveraging and one
oracle WelfordCov(D) per chain.  The same harness runs under ThreadSanitizer, and the adaptive kernels compile under NVRTC
with the Dense kind for every source contract and for a GLMTarget's generated source.  The GPU side is
tests/test_dense_user_adapt.py."""
import concurrent.futures as cf
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ahmc_b200 as A
from oracle import oracle_c as oc
from tests import philox_ref as R
from tests.helpers import rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "simt_emu")
CSRC = os.path.join(ROOT, "advancedhmc.jl_b200", "csrc")
_vp = C.c_void_p
P = lambda a: None if a is None else a.ctypes.data_as(_vp)
WELFORD_COV = 3
UK_NUTS_ADAPT, UK_HMC_ADAPT = 5, 6


class EmuDenseUserAdapt(C.Structure):
    _fields_ = [("hmc", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("params", _vp), ("Minv0", _vp), ("cholU0", _vp),
                ("metric_stride", C.c_int64), ("eps0", C.c_double), ("max_depth", C.c_int32), ("n_steps", C.c_int32),
                ("seed", C.c_uint64), ("T", C.c_int32), ("n_adapts", C.c_int32), ("init_buffer", C.c_int32),
                ("term_buffer", C.c_int32), ("window_size", C.c_int32), ("adapt_metric", C.c_int32), ("n_min", C.c_int32),
                ("th_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp), ("r_out", _vp), ("g_out", _vp), ("lp_out", _vp),
                ("lk_out", _vp), ("draws", _vp), ("acc", _vp), ("eps_trace", _vp), ("n_steps_out", _vp), ("tree_depth", _vp),
                ("is_accept", _vp), ("numerical", _vp), ("eps_rw", _vp), ("minv_rw", _vp), ("cholu_rw", _vp)]


def _gxx(out, form, *extra):
    return ["g++", *extra, "-std=c++20", "-pthread", "-ffp-contract=off", "-w", *(["-DDENSE_USER_GROUP"] if form == "group" else []),
            "-I", os.path.join(EMU, "include"), "-I", CSRC, "-I", os.path.join(ROOT, "include"), os.path.join(EMU, "simt_emu.cpp"),
            os.path.join(EMU, "dense_user_adapt_emu.cpp"), "-o", str(out)]


@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    """the harness in the group form and the one-lane form, compiled once each (in parallel)"""
    tmp = tmp_path_factory.mktemp("simt_dense_user_adapt")

    def build(form):
        out = tmp / f"libdense_user_adapt_{form}.so"
        pr = subprocess.run(_gxx(out, form, "-O1", "-shared", "-fPIC"), capture_output=True, text=True)
        assert pr.returncode == 0, pr.stderr[-2000:]
        return form, C.CDLL(str(out))

    with cf.ThreadPoolExecutor(max_workers=2) as ex:
        return dict(ex.map(build, ("group", "one_lane")))


def _spd(rng, D, lo=-0.3, hi=0.3):
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    return (Q * np.exp(rng.uniform(lo, hi, D))) @ Q.T


def _ar1(D, rho):
    i = np.arange(D)
    return rho ** np.abs(i[:, None] - i[None, :])


def _run(lib, hmc, D, N, T, n_adapts, windows, n_min, seed, shared, eps0, max_depth, n_steps):
    rng = np.random.default_rng(seed)
    s = np.exp(rng.uniform(-0.3, 0.3, D))
    Sig = s[:, None] * _ar1(D, 0.7) * s[None, :]  # AR(1) correlations 0.7^|i-j|, scales s
    mu, Prec = rng.normal(size=D), np.linalg.inv(Sig)
    Prec = 0.5 * (Prec + Prec.T)
    params = np.ascontiguousarray(np.concatenate([mu, Prec.T.reshape(-1)]))
    M0 = np.stack([_spd(rng, D)] * N) if shared else np.stack([_spd(rng, D) for _ in range(N)])
    U0 = np.linalg.cholesky(M0).transpose(0, 2, 1)
    M0c, U0c = np.ascontiguousarray(M0.transpose(0, 2, 1)), np.ascontiguousarray(U0.transpose(0, 2, 1))
    th = mu + rng.normal(size=(N, D))
    g_in = (th - mu) @ Prec  # -grad lp (Prec symmetric)
    lp_in = -0.5 * np.sum((th - mu) * g_in, axis=1)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lp_o, lk_o = np.zeros(N), np.zeros(N)
    draws, acc, trace = np.zeros((T, N, D)), np.zeros((T, N)), np.zeros((T, N))
    ns, td = np.zeros((T, N), dtype=np.int32), np.zeros((T, N), dtype=np.int32)
    ia, ne = np.zeros((T, N), dtype=np.uint8), np.zeros((T, N), dtype=np.uint8)
    eps, minv, cholu = np.zeros(N), np.zeros((N, D, D)), np.zeros((N, D, D))
    q = EmuDenseUserAdapt(hmc=hmc, D=D, N=N, params=P(params), Minv0=P(M0c), cholU0=P(U0c), metric_stride=0 if shared else D * D,
                          eps0=eps0, max_depth=max_depth, n_steps=n_steps, seed=seed, T=T, n_adapts=n_adapts,
                          init_buffer=windows[0], term_buffer=windows[1], window_size=windows[2], adapt_metric=WELFORD_COV,
                          n_min=n_min, th_in=P(th), g_in=P(g_in), lp_in=P(lp_in), th_out=P(o["th"]), r_out=P(o["r"]),
                          g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o), draws=P(draws), acc=P(acc), eps_trace=P(trace),
                          n_steps_out=P(ns), tree_depth=P(td), is_accept=P(ia), numerical=P(ne), eps_rw=P(eps), minv_rw=P(minv),
                          cholu_rw=P(cholu))
    assert lib.emu_dense_user_adapt(C.byref(q)) == 0
    T_ = lambda a: a.transpose(0, 2, 1)  # column-major rows -> matrices
    return dict(mu=mu, Prec=Prec, th0=th, M0=M0, draws=draws, acc=acc, trace=trace, n_steps=ns, tree_depth=td, is_accept=ia,
                numerical=ne, eps=eps, minv=T_(minv), cholu=T_(cholu), th_out=o["th"])


# (kernel, D, N, shared starting metric): D = 6 puts four chains in a warp (G = 8) and leaves the last warp ragged; D = 40
# runs one chain per warp (G = 32, two coordinates per lane)
CASES = [("nuts", 6, 13, False), ("hmc", 6, 13, True), ("nuts", 40, 3, True), ("hmc", 40, 3, False)]


@pytest.mark.parametrize("form", ["group", "one_lane"])
@pytest.mark.parametrize("kernel,D,N,shared", CASES, ids=[f"{c[0]}-D{c[1]}" for c in CASES])
def test_welford_cov_user_kernels_under_emulation_equal_the_oracle_iteration_by_iteration(emus, form, kernel, D, N, shared):
    """Iteration i of the fused launch against the oracle's transition from the launch's draw i - 1, on the Philox draws of
    transition offset i - 1, with the launch's step size and the chain's metric (the starting one, then the oracle's
    window-end estimate): draws to 1e-10 with identical decisions; the step sizes against the oracle's DualAveraging fed
    the oracle's acceptance rates to 1e-9, and the chain's final M^-1 and factor against the oracle's WelfordCov estimate
    and numpy's Cholesky factor to 1e-9.  The schedule's first window (4 draws) is below n_min = 5: a reset without an
    update; the second window updates."""
    T, n_adapts, windows, n_min, seed = 24, 20, (3, 2, 4), 5, 40 + D + (kernel == "hmc")
    max_depth, n_steps = 6, 7
    eps0 = 0.3 if kernel == "nuts" else 0.15
    ws, we, splits = oc.stan_windows(n_adapts, *windows)
    assert (ws, we, list(splits)) == (4, 18, [7, 18])
    run = _run(emus[form], kernel == "hmc", D, N, T, n_adapts, windows, n_min, seed, shared, eps0, max_depth, n_steps)
    om = oc.Model(oc.DENSE_GAUSS, D, run["mu"], run["Prec"], 0.0)
    da = oc.DualAveraging(np.full(N, eps0), delta=0.8)
    new = lambda: [oc.WelfordCov(D) for _ in range(N)]
    wc = new()
    Minv, updates, resets = run["M0"].copy(), 0, 0
    prev = run["th0"]
    for i in range(1, T + 1):
        assert np.allclose(run["trace"][i - 1], da.eps, rtol=1e-9, atol=0), i
        nt = R.normal_tape(seed, i - 1, N, D)
        alpha = np.zeros(N)
        for c in range(N):
            ome = oc.Metric(oc.DENSE, Minv[c])
            z0 = oc.phasepoint(om, ome, prev[c][:, None], np.zeros((D, 1)))
            if kernel == "nuts":
                zo, so, _ = oc.nuts_transition(om, ome, float(run["trace"][i - 1, c]), z0, nt[:, c:c + 1],
                                               R.dir_tape(seed, i - 1, N, max_depth + 1)[c:c + 1],
                                               R.nuts_exp_tape(seed, i - 1, N, 1 << max_depth)[c:c + 1], max_depth=max_depth)
                assert run["tree_depth"][i - 1, c] == so.tree_depth[0], (i, c)
            else:
                zo, so = oc.hmc_transition(om, ome, float(run["trace"][i - 1, c]), n_steps, z0, nt[:, c:c + 1],
                                           R.static_exp_tape(seed, i - 1, N)[c:c + 1])
                assert run["is_accept"][i - 1, c] == so.is_accept[0], (i, c)
            assert run["n_steps"][i - 1, c] == so.n_steps[0], (i, c)
            assert run["numerical"][i - 1, c] == so.numerical_error[0], (i, c)
            assert rel_err(run["draws"][i - 1, c], zo.theta[:, 0]) < 1e-10, (i, c)
            assert abs(run["acc"][i - 1, c] - so.acceptance_rate[0]) <= 1e-9 * max(1.0, abs(so.acceptance_rate[0])), (i, c)
            alpha[c] = so.acceptance_rate[0]
        prev = run["draws"][i - 1]
        if i <= n_adapts:
            da.adapt(alpha)
            if ws <= i <= we:
                for c in range(N):
                    wc[c].push(prev[c])
                if i in splits:
                    if wc[0].n.value >= n_min:
                        Minv = np.stack([w.estimate() for w in wc])
                        updates += 1
                    else:
                        resets += 1
            if i in splits:
                da.reset()
                wc = new()
            if i == n_adapts:
                da.finalize()
    assert (updates, resets) == (1, 1)
    assert np.abs(run["minv"] - Minv).max() <= 1e-9 * np.abs(Minv).max()
    U = np.linalg.cholesky(Minv).transpose(0, 2, 1)
    assert np.abs(run["cholu"] - U).max() <= 1e-9 * np.abs(U).max()
    assert (np.tril(run["cholu"], -1) == 0).all()  # the factor is upper triangular (its scratch triangle cleared)
    assert np.allclose(run["eps"], da.eps, rtol=1e-9, atol=0)
    assert np.array_equal(run["th_out"], run["draws"][-1])
    assert len(np.unique(run["trace"][-1])) == N  # every chain adapted on its own
    if kernel == "nuts":
        assert run["tree_depth"].max() >= 2


@pytest.mark.parametrize("form", ["group", "one_lane"])
def test_welford_cov_user_kernels_are_data_race_free_under_thread_sanitizer(tmp_path, form):
    out = tmp_path / f"race_dense_user_adapt_{form}"
    pr = subprocess.run(_gxx(out, form, "-DDENSE_USER_ADAPT_RACE", "-O1", "-g", "-fsanitize=thread", "-x", "c++"),
                        capture_output=True, text=True)
    if pr.returncode != 0 and "tsan" in pr.stderr.lower():
        pytest.skip("ThreadSanitizer runtime not available to g++ here")
    assert pr.returncode == 0, pr.stderr[-2000:]
    r = subprocess.run([str(out)], capture_output=True, text=True, timeout=900)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr.strip().splitlines()[0])
    assert r.returncode == 0 and "WARNING: ThreadSanitizer" not in r.stderr, r.stdout + r.stderr[-3000:]
    assert r.stdout.count("rc 0") == 4, r.stdout


# ---- the adaptive kernels with the Dense kind under NVRTC (compile only: no GPU)
ONE_LANE = r'''
__device__ double ahmc_user_logp_grad(const double* th, double* g, int D, const double* p) {
    double s = 0.0;
    for (int i = 0; i < D; ++i) {
        double acc = 0.0;
        for (int j = 0; j < D; ++j) acc = fma(p[i + D * j], th[j], acc);
        g[i] = -acc;
        s = fma(th[i], acc, s);
    }
    return -0.5 * s;
}
'''
COORDWISE = r'''
#define AHMC_USER_COORDWISE
__device__ double ahmc_user_coord(int d, double th, const double* p, double* g) {
    const double w = p[d];
    *g = -w * th;
    return -0.5 * w * th * th;
}
'''
GROUPWISE = r'''
#define AHMC_USER_GROUPWISE
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    double s = 0.0;
    for (int i = grp.lane; i < D; i += grp.size) {
        double acc = 0.0;
        for (int j = 0; j < D; ++j) acc = fma(p[i + D * j], th[j], acc);
        g[i] = -acc;
        s = fma(th[i], acc, s);
    }
    ahmc_group_sync(grp);
    const double S = ahmc_group_sum(grp, s);
    return grp.lane == 0 ? -0.5 * S : 0.0;
}
'''


def _lib_or_skip():
    lib = A._lib.load()
    log = C.create_string_buffer(4096)
    if lib.ahmc_user_source_check(ONE_LANE.encode(), 0, 0, 3, log, 4096) == A._lib.ERR_UNSUPPORTED:
        pytest.skip("libnvrtc not available here: " + log.value.decode())
    return lib


def _check(lib, src, kernel, metric, D):
    log = C.create_string_buffer(8192)
    rc = lib.ahmc_user_source_check(src.encode(), kernel, metric, D, log, 8192)
    return rc, log.value.decode()


def test_adaptive_kernels_with_the_dense_kind_compile_for_every_source_contract_and_the_glm_source():
    """kernels 5 and 6 (adaptive NUTS, adaptive static HMC) with metric_kind = Dense compile the WelfordCov form on the
    per-chain Dense kind, for the one-lane, coordinate-wise and group forms at D = 6 (G = 8, several chains per warp) and
    D = 40 (G = 32), and for the Bernoulli-logit source a GLMTarget generates"""
    lib = _lib_or_skip()
    rng = np.random.default_rng(3)
    X = rng.normal(size=(50, 40))
    glm = A.GLMTarget(X, (rng.uniform(size=50) < 0.5).astype(float), "bernoulli_logit", prior_prec=1.0).source()
    jobs = [(src, kernel, A._lib.METRIC_DENSE, D) for D in (6, 40) for src in (ONE_LANE, COORDWISE, GROUPWISE)
            for kernel in (UK_NUTS_ADAPT, UK_HMC_ADAPT)]
    jobs += [(glm, kernel, A._lib.METRIC_DENSE, 40) for kernel in (UK_NUTS_ADAPT, UK_HMC_ADAPT)]
    with cf.ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        results = list(ex.map(lambda j: _check(lib, *j), jobs))
    for (src, kernel, metric, D), (rc, log) in zip(jobs, results):
        assert rc == 0, (kernel, metric, D, src[:40], log[-2000:])


def test_a_broken_source_checked_for_the_dense_warm_up_comes_back_with_its_log():
    lib = _lib_or_skip()
    for kernel in (UK_NUTS_ADAPT, UK_HMC_ADAPT):
        rc, log = _check(lib, GROUPWISE.replace("return grp.lane == 0", "return nope == 0"), kernel, A._lib.METRIC_DENSE, 6)
        assert rc == A._lib.ERR_INVALID and "nope" in log and "undefined" in log, log
