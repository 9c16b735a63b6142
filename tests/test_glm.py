"""GLM targets (`A.GLMTarget`: Bernoulli-logit and Poisson-log regressions with a Gaussian prior) on the GPU: the chain-tile
kernel against the float64 numpy statement of the target (tests/glm_ref.py) and against the general (run-time compiled)
form, which form a call takes, multi-transition sampling, NUTS and in-launch adaptation, a statistical pin and the life
time of the model's device memory (run with -m gpu on an H100)."""
import ctypes as C

import numpy as np
import pytest
import torch

import ahmc_b200 as A
from tests import glm_ref as R
from tests.helpers import rel_err
from tests.test_gpu_parity import DEV, F, T, make_metric

pytestmark = pytest.mark.gpu
FAMILIES = ["bernoulli_logit", "poisson_log"]


def _problem(family, D, n, N, metric, seed):
    rng = np.random.default_rng(seed)
    X, y, beta = R.data(family, n, D, seed, scale=0.3 if family == "poisson_log" else 1.0)
    prec = rng.uniform(0.5, 2.0, D)
    Minv = None if metric == "unit" else np.exp(rng.uniform(-0.5, 0.5, D if metric == "diag" else (N, D)))
    th, r = beta + 0.05 * rng.normal(size=(N, D)), rng.normal(size=(N, D))
    return X, y, prec, Minv, th, r, rng


def _metric(metric, Minv, D):
    if metric == "chain":
        return A.DiagEuclideanMetric(torch.as_tensor(Minv, device=DEV))
    return make_metric(metric, Minv, D)


def _z(zt):
    g = lambda t: t.cpu().numpy()
    return dict(th=g(zt.theta), r=g(zt.r), g=g(zt.lp.gradient), lp=g(zt.lp.value), lk=g(zt.lk.value))


def _close(z, ref, tol=1e-10, keys=("th", "r", "g", "lp", "lk")):
    for k in keys:
        assert rel_err(z[k], ref[k]) < tol, (k, rel_err(z[k], ref[k]))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("D,N,metric", [(25, 333, "unit"), (25, 4096, "diag"), (100, 200, "chain"), (100, 77, "diag")])
def test_tile_lane_matches_reference_and_general_form(family, D, N, metric):
    """phasepoint, `step` (forward, per-chain eps, with and without a cached gradient) and a static transition on tapes:
    the tile kernel agrees with the numpy statement and with the general form to 1e-10 and makes the same accept decisions;
    `ctx.launches` tells which form ran (tile: 1 launch per phasepoint / step, 4 per transition; general: 1 per transition)."""
    n = 1000
    X, y, prec, Minv, th, r, rng = _problem(family, D, n, N, metric, seed=D + N)
    tgt = A.GLMTarget(X, y, family, prior_prec=prec, c0=0.5)
    h = A.Hamiltonian(_metric(metric, Minv, D), tgt)
    ctx = A.get_context(0)
    tht, rt = torch.as_tensor(th, device=DEV), torch.as_tensor(r, device=DEV)
    l0 = ctx.launches
    z = A.phasepoint(h, tht, rt)
    assert ctx.launches - l0 == 1
    zg = A.phasepoint(h, tht, rt, flags=A.FLAG_EXACT_CHECKS)  # the general form
    z0 = R.phasepoint(family, X, y, prec, 0.5, Minv, th, r)
    _close(_z(z), z0)
    _close(_z(zg), z0)
    eps = 0.01 * np.exp(rng.uniform(-0.3, 0.3, N))
    lf = A.Leapfrog(torch.as_tensor(eps, device=DEV))
    z1, info = A.step(lf, h, z, 5, return_info=True)
    z1g = A.step(lf, h, z, 5, flags=A.FLAG_EXACT_CHECKS)
    ref, st, steps = R.leapfrog(family, X, y, prec, 0.5, Minv, eps, z0, 5)
    _close(_z(z1), ref)
    _close(_z(z1g), ref)
    assert rel_err(z1.lk.gradient.cpu().numpy(), ref["dr"]) < 1e-10
    assert (F(info.steps_done) == 5).all() and (F(info.status) == 0).all()
    z1n = A.step(lf, h, A.PhasePoint(z.theta, z.r, A.DualValue(None, None), A.DualValue(None, None)), 5)
    _close(_z(z1n), ref)
    zb = A.step(lf, h, z, -3)
    _close(_z(zb), R.leapfrog(family, X, y, prec, 0.5, Minv, eps, z0, -3)[0])
    nt, et = rng.normal(size=(N, D)), rng.exponential(size=N)
    kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.02), A.FixedNSteps(8)))
    tape = A.TapeRNG(normal=torch.as_tensor(nt, device=DEV), exp=torch.as_tensor(et, device=DEV))
    l0 = ctx.launches
    tr = A.transition(tape, h, kern, z)
    assert ctx.launches - l0 == 4  # refresh, kinetic energy, tile trajectory, select
    l0 = ctx.launches
    trg = A.transition(tape, h, kern, z, flags=A.FLAG_EXACT_CHECKS)
    assert ctx.launches - l0 == 1
    new, acc, nerr = R.transition(family, X, y, prec, 0.5, Minv, 0.02, 8, z0, nt, et)
    for t_ in (tr, trg):
        assert np.array_equal(t_.stat["is_accept"].cpu().numpy().astype(bool), acc)
        assert (t_.stat["n_steps"].cpu().numpy() == 8).all() and not t_.stat["numerical_error"].cpu().numpy().any()
        _close(_z(t_.z), new)
    assert 0.2 < acc.mean() <= 1.0


def test_calls_the_tile_kernel_does_not_serve_take_the_general_form():
    """Dense metric, host buffers and a tempered integrator run the run-time compiled kernels (one launch per call) and give
    the tile lane's numbers; a NUTS variant refused for run-time compiled targets is refused with the same code."""
    D, N = 25, 64
    X, y, prec, _, th, r, rng = _problem("bernoulli_logit", D, 300, N, "unit", seed=3)
    tgt = A.GLMTarget(X, y, prior_prec=prec)
    ctx = A.get_context(0)
    hu = A.Hamiltonian(A.UnitEuclideanMetric(D), tgt)
    hd = A.Hamiltonian(A.DenseEuclideanMetric(np.eye(D)), tgt)
    tht, rt = torch.as_tensor(th, device=DEV), torch.as_tensor(r, device=DEV)
    zu, zd = A.phasepoint(hu, tht, rt), A.phasepoint(hd, tht, rt)
    assert rel_err(zd.lp.gradient.cpu().numpy(), zu.lp.gradient.cpu().numpy()) < 1e-11
    a, b = A.step(A.Leapfrog(0.02), hu, zu, 4), A.step(A.Leapfrog(0.02), hd, zd, 4)
    _close(_z(b), _z(a), 1e-10)
    zh = A.step(A.Leapfrog(0.02), hu, A.PhasePoint(th, r, A.DualValue(None, None), A.DualValue(None, None)), 4)
    assert rel_err(zh.theta, a.theta.cpu().numpy()) < 1e-10
    kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.TemperedLeapfrog(0.02, 1.05), A.FixedNSteps(4)))
    l0 = ctx.launches
    A.transition(A.PhiloxRNG(1), hu, kern, zu)
    assert ctx.launches - l0 == 1
    with pytest.raises(A._lib.AhmcError) as e:
        A.transition(A.PhiloxRNG(1), hu, A.HMCKernel(A.Trajectory(A.SliceTS, A.Leapfrog(0.02), A.GeneralisedNoUTurn())), zu)
    assert e.value.code == A._lib.ERR_UNSUPPORTED


@pytest.mark.parametrize("family", FAMILIES)
def test_a_non_finite_chain_stops_alone(family):
    D, N = 25, 40
    X, y, prec, Minv, th, r, rng = _problem(family, D, 500, N, "diag", seed=11)
    h = A.Hamiltonian(make_metric("diag", Minv, D), A.GLMTarget(X, y, family, prior_prec=prec))
    if family == "bernoulli_logit":
        th[7] = 1e200
    else:
        r[7] = 1e5 * np.sign(X[0])
    z = A.phasepoint(h, torch.as_tensor(th, device=DEV), torch.as_tensor(r, device=DEV))
    z1, info = A.step(A.Leapfrog(0.01), h, z, 6, return_info=True)
    z0 = R.phasepoint(family, X, y, prec, 0.0, Minv, th, r)
    ref, st, steps = R.leapfrog(family, X, y, prec, 0.0, Minv, 0.01, z0, 6)
    assert np.array_equal(F(info.status), st) and np.array_equal(F(info.steps_done), steps) and st[7] == 1 and st.sum() == 1
    assert z1.lp.value[7].item() == -np.inf
    keep = np.arange(N) != 7
    _close({k: v[keep] for k, v in _z(z1).items()}, {k: v[keep] for k, v in ref.items()})


def test_sample_transitions_equals_single_transitions_bit_for_bit():
    """T transitions enqueued by one call = T calls of `transition` at Philox offsets 0..T-1: identical bits, draws row t is
    transition t, 4 launches per transition and nothing else."""
    D, N, Tn = 25, 300, 6
    X, y, prec, Minv, th, r, rng = _problem("bernoulli_logit", D, 400, N, "diag", seed=21)
    h = A.Hamiltonian(make_metric("diag", Minv, D), A.GLMTarget(X, y, prior_prec=prec))
    ctx = A.get_context(0)
    z = A.phasepoint(h, torch.as_tensor(th, device=DEV), torch.as_tensor(r, device=DEV))
    kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.03), A.FixedNSteps(5)))
    l0 = ctx.launches
    zl, draws, stats = A.sample_transitions(A.PhiloxRNG(9), h, kern, z, Tn)
    assert ctx.launches - l0 == 4 * Tn
    zc = z
    for t in range(Tn):
        rng_t = A.PhiloxRNG(9)
        rng_t.offset = t
        tr = A.transition(rng_t, h, kern, zc)
        zc = tr.z
        assert torch.equal(draws[t], zc.theta)
        assert torch.equal(stats["is_accept"][t], tr.stat["is_accept"])
        assert torch.equal(stats["hamiltonian_energy"][t], tr.stat["hamiltonian_energy"])
    assert torch.equal(zl.theta, zc.theta) and torch.equal(zl.lp.value, zc.lp.value) and torch.equal(zl.r, zc.r)
    assert 0.3 < stats["is_accept"].double().mean().item() < 1.0


@pytest.mark.parametrize("family", FAMILIES)
def test_nuts_stepsize_search_and_in_launch_adaptation_run_on_a_glm_target(family):
    """the general form: find_good_stepsize_batched, a NUTS transition, and the adaptive launches; with n_adapts = 0 the
    adaptive static launch is `sample_transitions` on the general form"""
    D, N = 10, 96
    X, y, prec, Minv, th, r, rng = _problem(family, D, 200, N, "diag", seed=31)
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), A.GLMTarget(X, y, family, prior_prec=prec))
    tht = torch.as_tensor(th, device=DEV)
    eps = A.find_good_stepsize_batched(A.PhiloxRNG(4), h, tht)
    assert torch.isfinite(eps).all() and (eps > 0).all()
    z = A.phasepoint(h, tht, torch.zeros_like(tht))
    nuts = A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.05), A.GeneralisedNoUTurn()))
    tr = A.transition(A.PhiloxRNG(5), h, nuts, z)
    lp_ref, _ = R.logp_mgrad(family, X, y, prec, 0.0, tr.z.theta.cpu().numpy())
    assert rel_err(tr.z.lp.value.cpu().numpy(), lp_ref) < 1e-10 and (tr.stat["tree_depth"] >= 1).all()
    ad = A.VectorisedStanAdaptor(delta=0.8)
    zl, draws, stats, e_ad, M_ad, _ = A.nuts_adapt_sample(A.PhiloxRNG(6), h, nuts, z, 150, 100, ad)
    assert torch.isfinite(e_ad).all() and (e_ad > 0).all() and torch.isfinite(M_ad).all() and (M_ad > 0).all()
    hmc = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.05), A.FixedNSteps(6)))
    zl, draws, stats, e_ad, M_ad, _ = A.hmc_adapt_sample(A.PhiloxRNG(7), h, hmc, z, 120, 80, A.VectorisedStanAdaptor(delta=0.8))
    assert torch.isfinite(e_ad).all() and (e_ad > 0).all() and 0.5 < stats["acceptance_rate"][80:].mean().item() <= 1.0
    z0, d0, s0, _, _, _ = A.hmc_adapt_sample(A.PhiloxRNG(8), h, hmc, z, 5, 0, A.VectorisedStanAdaptor(delta=0.8))
    z1, d1, s1 = A.sample_transitions(A.PhiloxRNG(8), h, hmc, z, 5, flags=A.FLAG_EXACT_CHECKS)
    assert torch.equal(d0, d1) and torch.equal(s0["is_accept"], s1["is_accept"])
    z2, d2, s2 = A.sample_transitions(A.PhiloxRNG(8), h, hmc, z, 5)  # the tile lane: same decisions, states to 1e-10
    assert torch.equal(s2["is_accept"], s1["is_accept"]) and rel_err(d2.cpu().numpy(), d1.cpu().numpy()) < 1e-9


def test_posterior_means_of_a_logistic_regression():
    """n = 200, D = 5, 1024 chains x 400 draws after warm-up on the tile lane; posterior means within 4 Monte-Carlo standard
    errors of a self-normalised importance-sampling estimate around the Laplace approximation (numpy, seeded)."""
    D, n, N = 5, 200, 1024
    X, y, _ = R.data("bernoulli_logit", n, D, 77)
    prec = np.ones(D)
    lpf = lambda th: R.logp_mgrad("bernoulli_logit", X, y, prec, 0.0, th)
    mode = np.zeros((1, D))
    for _ in range(50):  # Newton
        _, g = lpf(mode)
        mu = 1.0 / (1.0 + np.exp(-(mode @ X.T)))[0]
        Hm = (X * (mu * (1 - mu))[:, None]).T @ X + np.diag(prec)
        mode = mode - np.linalg.solve(Hm, g[0])[None, :]
    cov = np.linalg.inv(Hm)
    rng = np.random.default_rng(123)
    Lc = np.linalg.cholesky(cov * 1.5)
    S = 400000
    zs = rng.normal(size=(S, D))
    prop = mode + zs @ Lc.T
    logw = lpf(prop)[0] + 0.5 * (zs * zs).sum(axis=1)
    w = np.exp(logw - logw.max())
    w /= w.sum()
    ref_mean = (w[:, None] * prop).sum(axis=0)
    ess = 1.0 / (w * w).sum()
    ref_se = np.sqrt((w[:, None] ** 2 * (prop - ref_mean) ** 2).sum(axis=0))
    assert ess > 1e5
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.diag(cov).copy()), A.GLMTarget(X, y, prior_prec=prec))
    th0 = torch.as_tensor(mode + rng.normal(size=(N, D)) @ Lc.T, device=DEV)
    z = A.phasepoint(h, th0, torch.zeros_like(th0))
    kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.35), A.FixedNSteps(6)))
    z, _, _ = A.sample_transitions(A.PhiloxRNG(2024), h, kern, z, 100, keep_draws=False)
    rng2 = A.PhiloxRNG(2024)
    rng2.offset = 100
    z, draws, stats = A.sample_transitions(rng2, h, kern, z, 400)
    assert stats["is_accept"].double().mean().item() > 0.6
    d = draws.cpu().numpy()  # (T, N, D)
    chain_means = d.mean(axis=0)
    est, se = chain_means.mean(axis=0), chain_means.std(axis=0, ddof=1) / np.sqrt(N)  # chains are independent
    assert (np.abs(est - ref_mean) < 4 * np.sqrt(se ** 2 + ref_se ** 2)).all(), (est, ref_mean, se, ref_se)
    assert (se < 0.01).all()


def test_constructor_validation_and_model_memory():
    """invalid data is refused with AHMC_ERR_INVALID and a message; the padded design matrix belongs to the model: creating
    and destroying 50 models leaves this process's device memory where it was (per-process figure: the card is shared)."""
    ctx = A.get_context(0)
    X, y, _ = R.data("bernoulli_logit", 50, 4, 1)

    def bad(match, X=X, y=y, family="bernoulli_logit", **kw):
        with pytest.raises(A.InvalidArgument, match=match):
            A.GLMTarget(X, y, family, **kw).handle(ctx)

    bad("Bernoulli", y=y + 0.5)
    bad("Poisson", y=y - 1.0, family="poisson_log")
    bad("Poisson", y=y + 0.25, family="poisson_log")
    bad("not finite", X=np.where(np.arange(200).reshape(50, 4) == 7, np.inf, X))
    bad("not finite", y=np.where(np.arange(50) == 3, np.nan, y))
    bad("prior_prec", prior_prec=-1.0)
    bad("1..512", X=np.zeros((3, 513)), y=np.zeros(3))
    with pytest.raises(A.InvalidArgument):
        A.GLMTarget(X, y, "probit")
    with pytest.raises(A.InvalidArgument):
        A.GLMTarget(X, y[:-1])

    import os
    import subprocess

    def proc_mem():  # MiB this process holds on the device, as the driver accounts it
        out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True).stdout
        for line in out.splitlines():
            pid, mem = [s.strip() for s in line.split(",")]
            if int(pid) == os.getpid():
                return float(mem)
        return None

    Xb, yb, _ = R.data("bernoulli_logit", 20000, 100, 2)  # 16 MB of X and as much again padded
    lib = ctx.lib

    def cycle(k):
        for _ in range(k):
            t = A.GLMTarget(Xb, yb)
            hnd = t.handle(ctx)
            assert lib.ahmc_model_destroy(ctx.h, hnd) == 0
            t._handles.clear()

    cycle(2)
    before = proc_mem()
    cycle(50)
    after = proc_mem()
    if before is None or after is None:
        pytest.skip("the driver does not report this process's device memory here")
    assert after - before < 32, (before, after)  # 50 leaked models would be 1600 MiB
