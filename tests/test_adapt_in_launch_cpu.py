"""CPU checks of the per-chain in-launch adaptation (ahmc_chain_adapt.cuh) in its adaptive NUTS and adaptive static-HMC
kernels: the kernel sources under the SIMT emulator (tests/simt_emu/adapt_chain_emu.cpp) replayed against the ORACLE's
vectorised adaptors, the same sources under ThreadSanitizer, the run-time compiled (NVRTC) user-target forms, and the
composed oracle NutpieVar against the 50-digit fixture.  The GPU side is tests/test_adapt_in_launch.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import oracle_c as oc
from tests import emu as E
from tests.emu import P, EmuAdaptChain


@pytest.fixture(scope="module")
def emu():
    return E.harness("adapt_chain")


def _run(lib, hmc, est, D, N, T, n_adapts, windows, n_min, seed):
    rng = np.random.default_rng(seed)
    sd, mu = np.exp(rng.uniform(-0.7, 0.7, D)), rng.normal(size=D)
    w = 1.0 / (sd * sd)
    th = rng.normal(size=(N, D))
    g_in = (th - mu) * w
    lp_in = -0.5 * np.sum((th - mu) ** 2 * w, axis=1)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lp_o, lk_o = np.zeros(N), np.zeros(N)
    draws, acc, trace = np.zeros((T, N, D)), np.zeros((T, N)), np.zeros((T, N))
    ns = np.zeros((T, N), dtype=np.int32)
    eps, minv = np.zeros(N), np.zeros((N, D))
    q = EmuAdaptChain(hmc=hmc, D=D, N=N, mu=P(mu), w=P(w), Minv=P(np.ones(D)), eps0=0.3 if not hmc else 0.15, max_depth=6, n_steps=6,
                      seed=seed, T=T, n_adapts=n_adapts, init_buffer=windows[0], term_buffer=windows[1], window_size=windows[2],
                      adapt_metric=dict(welford=1, nutpie=2)[est], n_min=n_min, th_in=P(th), g_in=P(g_in), lp_in=P(lp_in),
                      th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o), draws=P(draws),
                      acc=P(acc), eps_trace=P(trace), n_steps_out=P(ns), eps_rw=P(eps), minv_rw=P(minv))
    assert lib.emu_adapt_chain(C.byref(q)) == 0
    return dict(draws=draws, grads=(draws - mu) * w, acc=acc, trace=trace, n_steps=ns, eps=eps, minv=minv, eps0=q.eps0)


CASES = [  # (kernel, estimator, D, N): G = 8 packs four chains per warp, D = 40 is one chain per warp (G = 32, E = 2)
    ("nuts", "nutpie", 5, 9), ("hmc", "nutpie", 7, 12), ("hmc", "welford", 6, 9), ("nuts", "nutpie", 40, 3), ("hmc", "nutpie", 40, 3),
    ("nuts", "welford", 40, 2)]


@pytest.mark.parametrize("kernel,est,D,N", CASES, ids=[f"{c[0]}-{c[1]}-D{c[2]}" for c in CASES])
def test_adaptive_kernel_sources_under_emulation_equal_oracle_adaptors(emu, kernel, est, D, N):
    """Each chain's step size at every iteration and its M^-1 at every window end, from the kernel source, against the
    oracle's DualAveraging and WelfordVar((D, N)) -- two of them composed into NutpieVar -- fed the kernel's own acceptance
    rates, draws and gradients.  The schedule's first window (4 draws) is below n_min = 5: reset without an update."""
    T, n_adapts, windows, n_min = 24, 20, (3, 2, 4), 5
    ws, we, splits = oc.stan_windows(n_adapts, *windows)
    assert (ws, we, list(splits)) == (4, 18, [7, 18])
    run = _run(emu, kernel == "hmc", est, D, N, T, n_adapts, windows, n_min, seed=7 + D)
    da = oc.DualAveraging(np.full(N, run["eps0"]), delta=0.8)
    new = lambda: (oc.WelfordVar((D, N)), oc.WelfordVar((D, N)))
    wt, wg = new()
    Minv, updates = np.ones((N, D)), 0
    for i in range(1, T + 1):
        assert np.allclose(run["trace"][i - 1], da.eps, rtol=1e-10, atol=0), i
        if i <= n_adapts:
            da.adapt(run["acc"][i - 1])
            if ws <= i <= we:
                wt.push(run["draws"][i - 1].T)
                wg.push(run["grads"][i - 1].T)
                if i in splits and wt.n.value >= n_min:
                    e = wt.estimate()
                    Minv = np.ascontiguousarray((np.sqrt(e / wg.estimate()) if est == "nutpie" else e).T)
                    updates += 1
            if i in splits:
                da.reset()
                wt, wg = new()
            if i == n_adapts:
                da.finalize()
    assert updates == 1 and np.allclose(run["minv"], Minv, rtol=1e-10, atol=0)
    assert np.allclose(run["eps"], da.eps, rtol=1e-10, atol=0)
    assert (run["n_steps"] >= 1).all() and len(np.unique(run["trace"][-1])) == N  # every chain adapted on its own


def test_adaptive_kernel_sources_are_data_race_free_under_thread_sanitizer():
    r = E.sanitized("adapt_chain", "thread")
    assert r.returncode == 0 and "WARNING: ThreadSanitizer" not in r.stderr, r.stdout + r.stderr[-3000:]
    assert r.stdout.count("rc 0") == 6, r.stdout


def test_adaptive_user_target_kernels_compile_under_nvrtc():
    """ahmc_user_source_check kernels 5 (adaptive NUTS) and 6 (adaptive static HMC), both user-target contracts, Unit and
    Diag metrics, several layouts; a broken source comes back as the NVRTC log"""
    import ahmc_b200 as A

    lib = E.nvrtc_lib_or_skip()
    general = ("__device__ double ahmc_user_logp_grad(const double* th, double* g, int D, const double* p) {\n"
               "  double s = 0.0; for (int i = 0; i < D; ++i) { g[i] = -th[i] * p[0]; s += th[i] * th[i]; } return -0.5 * p[0] * s; }\n")
    coord = ("#define AHMC_USER_COORDWISE\n__device__ double ahmc_user_coord(int d, double x, const double* p, double* gd) {\n"
             "  *gd = -x * p[d]; return -0.5 * x * x * p[d]; }\n")
    for src in (general, coord):
        for kernel in (5, 6):
            for metric, D in ((0, 6), (1, 8), (1, 40), (1, 128), (0, 200)):
                rc, log = E.source_check(lib, src, kernel, metric, D)
                assert rc == 0, log
    bad = "__device__ double ahmc_user_logp_grad(const double* t, double* g, int D, const double* p) { return q; }"
    for kernel in (5, 6):
        rc, log = E.source_check(lib, bad, kernel, 1, 8)
        assert rc == A._lib.ERR_INVALID and "q" in log and "undefined" in log
    assert E.source_check(lib, general, 7, 1, 8)[0] == A._lib.ERR_INVALID


def test_composed_oracle_nutpie_var_reproduces_the_50_digit_fixture():
    """NutpieVar as the kernels build it -- two WelfordVar of positions and (minus) gradients, M^-1 = sqrt(est / est) --
    composed from the oracle's WelfordVar, against tests/golden/adapt_mp50.json"""
    with open(os.path.join(E.ROOT, "tests", "golden", "adapt_mp50.json")) as f:
        w = json.load(f)["welford"]
    xs, gs = np.array(w["xs"]), np.array(w["gs"])
    for sign in (1.0, -1.0):  # the kernels push MINUS grad log pi: the same variance
        wt, wg = oc.WelfordVar((xs.shape[1],)), oc.WelfordVar((xs.shape[1],))
        for x, g in zip(xs, gs):
            wt.push(x)
            wg.push(sign * g)
        assert np.allclose(np.sqrt(wt.estimate() / wg.estimate()), w["nutpie_estimate"], rtol=1e-10, atol=0)
