"""CPU checks of the WelfordCov form of the per-chain in-launch adaptor (ahmc_chain_adapt.cuh): the adaptive NUTS and static
HMC kernels with a per-chain Dense metric under the SIMT emulator (tests/simt_emu/dense_adapt_emu.cpp) replayed against the
oracle's DualAveraging and one WelfordCov per chain, the window-end estimate and Cholesky factorisation on their own
(including a failing factorisation), and the same sources under ThreadSanitizer.  The GPU side is
tests/test_dense_per_chain.py."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle_c as oc
from tests import emu as E
from tests.emu import P, EmuDenseAdapt, EmuEstimate

WELFORD_COV = 3


@pytest.fixture(scope="module")
def emu():
    return E.harness("dense_adapt")


def _spd(rng, D, scale=1.0):
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    return scale * (Q * np.exp(rng.uniform(-0.5, 0.5, D))) @ Q.T


def _run(lib, hmc, D, N, T, n_adapts, windows, n_min, seed):
    rng = np.random.default_rng(seed)
    sd, mu = np.exp(rng.uniform(-0.5, 0.5, D)), rng.normal(size=D)
    w = 1.0 / (sd * sd)
    M0 = np.stack([_spd(rng, D) for _ in range(N)])
    U0 = np.linalg.cholesky(M0).transpose(0, 2, 1)
    # column-major D x D per chain = each chain's matrix transposed, row-major
    M0c, U0c = np.ascontiguousarray(M0.transpose(0, 2, 1)), np.ascontiguousarray(U0.transpose(0, 2, 1))
    th = mu + sd * rng.normal(size=(N, D))
    g_in = (th - mu) * w
    lp_in = -0.5 * np.sum((th - mu) ** 2 * w, axis=1)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lp_o, lk_o = np.zeros(N), np.zeros(N)
    draws, acc, trace = np.zeros((T, N, D)), np.zeros((T, N)), np.zeros((T, N))
    ns = np.zeros((T, N), dtype=np.int32)
    eps, minv, cholu = np.zeros(N), np.zeros((N, D, D)), np.zeros((N, D, D))
    ws = np.zeros((N, D + D * D))
    q = EmuDenseAdapt(hmc=hmc, D=D, N=N, mu=P(mu), w=P(w), Minv0=P(M0c), cholU0=P(U0c), eps0=0.15 if hmc else 0.3, max_depth=5,
                      n_steps=6, seed=seed, T=T, n_adapts=n_adapts, init_buffer=windows[0], term_buffer=windows[1],
                      window_size=windows[2], adapt_metric=WELFORD_COV, n_min=n_min, th_in=P(th), g_in=P(g_in), lp_in=P(lp_in),
                      th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o), draws=P(draws),
                      acc=P(acc), eps_trace=P(trace), n_steps_out=P(ns), eps_rw=P(eps), minv_rw=P(minv), cholu_rw=P(cholu),
                      workspace=P(ws))
    assert lib.emu_dense_adapt(C.byref(q)) == 0
    T_ = lambda a: a.transpose(0, 2, 1)  # column-major rows -> matrices
    return dict(draws=draws, acc=acc, trace=trace, n_steps=ns, eps=eps, minv=T_(minv), cholu=T_(cholu), M0=M0, U0=U0,
                mean=ws[:, :D], M=T_(ws[:, D:].reshape(N, D, D)), eps0=q.eps0)


CASES = [("nuts", 7, 5), ("hmc", 7, 6), ("nuts", 33, 2), ("hmc", 33, 3), ("nuts", 64, 2), ("hmc", 64, 2)]  # G = 8, 32 (E = 2)


@pytest.mark.parametrize("kernel,D,N", CASES, ids=[f"{c[0]}-D{c[1]}" for c in CASES])
def test_welford_cov_kernel_sources_under_emulation_equal_oracle_adaptors(emu, kernel, D, N):
    """Each chain's step size at every iteration, and its M^-1 and factor at the window end, from the kernel sources,
    against the oracle's DualAveraging and one WelfordCov(D) per chain fed the kernel's own acceptance rates and draws, and
    numpy's Cholesky factor.  The schedule's first window (4 draws) is below n_min = 5: a reset without an update; the
    second window updates.  Then the estimator state (mean, M) part-way through a window against the oracle's."""
    T, n_adapts, windows, n_min = 24, 20, (3, 2, 4), 5
    ws, we, splits = oc.stan_windows(n_adapts, *windows)
    assert (ws, we, list(splits)) == (4, 18, [7, 18])
    run = _run(emu, kernel == "hmc", D, N, T, n_adapts, windows, n_min, seed=11 + D)
    da = oc.DualAveraging(np.full(N, run["eps0"]), delta=0.8)
    new = lambda: [oc.WelfordCov(D) for _ in range(N)]
    wc = new()
    Minv, U, updates, resets = run["M0"].copy(), run["U0"].copy(), 0, 0
    for i in range(1, T + 1):
        assert np.allclose(run["trace"][i - 1], da.eps, rtol=1e-10, atol=0), i
        if i <= n_adapts:
            da.adapt(run["acc"][i - 1])
            if ws <= i <= we:
                for c in range(N):
                    wc[c].push(run["draws"][i - 1, c])
                if i in splits:
                    if wc[0].n.value >= n_min:
                        Minv = np.stack([w.estimate() for w in wc])
                        U = np.linalg.cholesky(Minv).transpose(0, 2, 1)
                        updates += 1
                    else:
                        resets += 1
            if i in splits:
                da.reset()
                wc = new()
            if i == n_adapts:
                da.finalize()
    assert (updates, resets) == (1, 1)
    scale = np.abs(Minv).max()
    assert np.abs(run["minv"] - Minv).max() <= 1e-12 * scale
    assert np.abs(run["cholu"] - U).max() <= 1e-12 * np.abs(U).max()
    assert (np.tril(run["cholu"], -1) == 0).all()  # the factor row is upper triangular (its scratch triangle cleared)
    assert np.allclose(run["eps"], da.eps, rtol=1e-10, atol=0)
    assert (run["n_steps"] >= 1).all() and len(np.unique(run["trace"][-1])) == N  # every chain adapted on its own

    # part-way through the second window (draws 8..13): mean and the full matrix M, no symmetrisation
    part = _run(emu, kernel == "hmc", D, N, 13, n_adapts, windows, n_min, seed=11 + D)
    assert np.array_equal(part["draws"], run["draws"][:13])
    for c in range(N):
        w = oc.WelfordCov(D)
        for i in range(8, 14):
            w.push(run["draws"][i - 1, c])
        assert w.n.value == 6
        assert np.abs(part["mean"][c] - w.mu).max() <= 1e-12 * np.abs(w.mu).max()
        assert np.abs(part["M"][c] - w.M).max() <= 1e-12 * np.abs(w.M).max()


@pytest.mark.parametrize("D,N", [(7, 6), (33, 3), (64, 2)])
def test_window_end_estimate_and_factor_and_a_failed_factorisation(emu, D, N):
    """The estimate n/((n+5)(n-1)) M + 1e-3 * 5/(n+5) I into the chain's Minv row and the upper factor of its upper
    triangle into its cholU row; a chain whose M forces a non-positive pivot keeps its previous M^-1 and factor, without
    disturbing the chains next to it (four chains share a warp at D = 7)."""
    rng = np.random.default_rng(D)
    n = 12.0
    mean = rng.normal(size=(N, D))
    Ms = [_spd(rng, D, 3.0) for _ in range(N)]
    bad = list(range(1, N, 2))
    for c in bad:  # a negative eigenvalue: the factorisation must meet a non-positive pivot
        Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
        lam = np.exp(rng.uniform(-0.5, 0.5, D))
        lam[-1] = -50.0
        Ms[c] = (Q * lam) @ Q.T
    Ms = np.stack(Ms)
    W = np.ascontiguousarray(np.concatenate([mean, Ms.transpose(0, 2, 1).reshape(N, D * D)], axis=1))
    prev_M = np.stack([_spd(rng, D) for _ in range(N)])
    prev_U = np.linalg.cholesky(prev_M).transpose(0, 2, 1)
    minv = np.ascontiguousarray(prev_M.transpose(0, 2, 1))
    cholu = np.ascontiguousarray(prev_U.transpose(0, 2, 1))
    ok = np.full(N, -1, dtype=np.int32)
    q = EmuEstimate(D=D, N=N, n=n, W=P(W), minv=P(minv), cholu=P(cholu), ok=P(ok))
    assert emu.emu_dense_estimate(C.byref(q)) == 0
    got_M, got_U = minv.transpose(0, 2, 1), cholu.transpose(0, 2, 1)
    for c in range(N):
        if c in bad:
            assert ok[c] == 0
            assert np.array_equal(got_M[c], prev_M[c]) and np.array_equal(got_U[c], prev_U[c])
        else:
            assert ok[c] == 1
            w = oc.WelfordCov(D)
            w.n.value, w.M[...] = int(n), Ms[c]
            want = w.estimate()
            assert np.abs(got_M[c] - want).max() <= 1e-12 * np.abs(want).max()
            U = np.linalg.cholesky(want).T
            assert np.abs(got_U[c] - U).max() <= 1e-12 * np.abs(U).max()
            assert (np.tril(got_U[c], -1) == 0).all()


def test_welford_cov_kernel_sources_are_data_race_free_under_thread_sanitizer():
    r = E.sanitized("dense_adapt", "thread")
    assert r.returncode == 0 and "WARNING: ThreadSanitizer" not in r.stderr, r.stdout + r.stderr[-3000:]
    assert r.stdout.count("rc 0") == 4, r.stdout
