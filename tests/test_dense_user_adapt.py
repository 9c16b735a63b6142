"""The Dense-metric in-launch warm-up (one WelfordCov per chain, ahmc_chain_adapt.cuh) on run-time compiled targets: a
group-form and a one-lane UserTarget and a GLMTarget (which adapts in its general, run-time compiled form).  A fused
warm-up must equal its iteration-by-iteration replay with single transitions, the oracle's DualAveraging and one oracle
WelfordCov(D) per chain, exactly as for the built-in targets (tests/test_dense_per_chain.py).  The CPU side is
tests/test_dense_user_adapt_cpu.py (run with -m gpu on an H100)."""
import numpy as np
import pytest
import torch

import ahmc_b200 as A
from ahmc_b200 import _lib as L
from ahmc_b200 import core as K
from oracle import oracle_c as oc
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# log pi = -(th - mu)' P (th - mu) / 2, params = [mu (D) | P (D x D, column-major)]
GAUSS_GROUP = r'''
#define AHMC_USER_GROUPWISE
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    const double* mu = p;
    const double* P = p + D;
    double s = 0.0;
    for (int i = grp.lane; i < D; i += grp.size) {
        double acc = 0.0;
        for (int j = 0; j < D; ++j) acc = fma(P[i + D * j], th[j] - mu[j], acc);
        g[i] = -acc;
        s = fma(th[i] - mu[i], acc, s);
    }
    ahmc_group_sync(grp);
    const double S = ahmc_group_sum(grp, s);
    return grp.lane == 0 ? -0.5 * S : 0.0;
}
'''
GAUSS_ONE_LANE = r'''
__device__ double ahmc_user_logp_grad(const double* th, double* g, int D, const double* p) {
    const double* mu = p;
    const double* P = p + D;
    double s = 0.0;
    for (int i = 0; i < D; ++i) {
        double acc = 0.0;
        for (int j = 0; j < D; ++j) acc = fma(P[i + D * j], th[j] - mu[j], acc);
        g[i] = -acc;
        s = fma(th[i] - mu[i], acc, s);
    }
    return -0.5 * s;
}
'''


def _spd(rng, D, lo=-0.5, hi=0.5):
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    return (Q * np.exp(rng.uniform(lo, hi, D))) @ Q.T


def _ar1(D, rho):
    i = np.arange(D)
    return rho ** np.abs(i[:, None] - i[None, :])


def _gauss(form, mu, Sig):
    P = np.linalg.inv(Sig)
    P = 0.5 * (P + P.T)
    src = GAUSS_GROUP if form == "group" else GAUSS_ONE_LANE
    return A.UserTarget(mu.size, src, np.concatenate([mu, P.T.reshape(-1)]))


def _logistic(rng, n, D, rho=0.9):
    """Bernoulli-logit regression with AR(1)-correlated predictors (corr rho^|i-j|) and a N(0, I) prior"""
    X = rng.normal(size=(n, D)) @ np.linalg.cholesky(_ar1(D, rho)).T
    beta = rng.normal(size=D) * 0.5
    y = (rng.uniform(size=n) < 1.0 / (1.0 + np.exp(-X @ beta))).astype(np.float64)
    return A.GLMTarget(X, y, "bernoulli_logit", prior_prec=1.0), beta


def _target(which, D, rng):
    """(target, a point near its mode)"""
    if which == "glm":
        tgt, beta = _logistic(rng, 200, D)
        return tgt, beta
    mu = rng.normal(size=D)
    return _gauss(which, mu, _spd(rng, D, -1.0, 1.0)), mu


def _kernel(sampler, eps):
    if sampler == "nuts":
        return A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(eps), A.GeneralisedNoUTurn(8, 1000.0)))
    return A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(eps), A.FixedNSteps(12)))


@pytest.mark.parametrize("which", ["group", "one_lane", "glm"])
@pytest.mark.parametrize("sampler", ["nuts", "hmc"])
def test_fused_welford_cov_equals_iteration_by_iteration_replay_with_oracle_adaptors(sampler, which):
    """single-transition launches on the same Philox streams with the fused launch's step sizes, the oracle's DualAveraging
    and one oracle WelfordCov(D) per chain on the host: step sizes and the window-end M^-1 / factor to 1e-9, draws to 1e-10
    with identical decisions; after the update the replay continues with the kernel's own per-chain matrices"""
    D, N, T_, n_adapts, seed = 8, 64, 60, 50, 37
    ib, tb, wsz = 10, 8, 6
    ws, we, splits = oc.stan_windows(n_adapts, ib, tb, wsz)
    assert (ws, we, list(splits)) == (11, 42, [16, 42])  # the first window holds 6 < n_min draws: reset without an update
    rng = np.random.default_rng(seed)
    target, centre = _target(which, D, rng)
    M0 = torch.as_tensor(np.stack([_spd(rng, D, -0.2, 0.2) for _ in range(N)]), device=DEV)
    if which == "glm":
        M0 = M0 * 0.05  # the posterior's scale
    h = A.Hamiltonian(A.DenseEuclideanMetric(M0), target)
    th0 = torch.as_tensor(centre + (0.1 if which == "glm" else 1.0) * rng.normal(size=(N, D)), device=DEV)
    z0 = A.phasepoint(h, th0, torch.zeros_like(th0))
    eps0 = 0.3 if sampler == "nuts" else 0.1
    ad = A.VectorisedStanAdaptor(delta=0.8, init_buffer=ib, term_buffer=tb, window_size=wsz, metric_estimator="welford_cov")
    run = A.nuts_adapt_sample if sampler == "nuts" else A.hmc_adapt_sample
    zl, draws, st, eps_f, met_f, trace = run(A.PhiloxRNG(seed), h, _kernel(sampler, eps0), z0, T_, n_adapts, ad, keep_eps_trace=True)
    assert isinstance(met_f, A.DenseEuclideanMetric) and tuple(met_f.Minv.shape) == (N, D, D) == tuple(met_f.cholU.shape)

    prng = A.PhiloxRNG(seed)
    da = oc.DualAveraging(np.full(N, eps0), delta=0.8)
    wc = [oc.WelfordCov(D) for _ in range(N)]
    metric, z, updates = h.metric, z0, 0
    for i in range(1, T_ + 1):
        assert np.allclose(trace[i - 1].cpu().numpy(), da.eps, rtol=1e-9, atol=0), i
        tr = A.transition(prng, A.Hamiltonian(metric, target), _kernel(sampler, trace[i - 1].clone()), z)
        z = tr.z
        assert rel_err(draws[i - 1].cpu().numpy(), z.theta.cpu().numpy()) < 1e-10, i
        assert torch.equal(st["n_steps"][i - 1].cpu(), tr.stat["n_steps"].cpu()), i
        key = "tree_depth" if sampler == "nuts" else "is_accept"
        assert torch.equal(st[key][i - 1].cpu(), tr.stat[key].cpu()), i
        assert torch.equal(st["numerical_error"][i - 1].cpu(), tr.stat["numerical_error"].cpu()), i
        if i <= n_adapts:
            da.adapt(tr.stat["acceptance_rate"].cpu().numpy())
            if ws <= i <= we:
                thn = z.theta.cpu().numpy()
                for c in range(N):
                    wc[c].push(thn[c])
                if i in splits and wc[0].n.value >= 10:
                    want = np.stack([w.estimate() for w in wc])
                    got = met_f.Minv.cpu().numpy()
                    assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max(), i
                    U = np.linalg.cholesky(want).transpose(0, 2, 1)
                    assert np.abs(met_f.cholU.cpu().numpy() - U).max() <= 1e-9 * np.abs(U).max(), i
                    metric = A.DenseEuclideanMetric(met_f.Minv.clone(), cholU=met_f.cholU.clone())  # the kernel's own
                    updates += 1
            if i in splits:
                da.reset()
                wc = [oc.WelfordCov(D) for _ in range(N)]
            if i == n_adapts:
                da.finalize()
    assert updates == 1
    assert np.allclose(eps_f.cpu().numpy(), da.eps, rtol=1e-9, atol=0)
    assert rel_err(zl.theta.cpu().numpy(), z.theta.cpu().numpy()) < 1e-10


@pytest.mark.parametrize("which", ["group", "glm"])
@pytest.mark.parametrize("sampler", ["nuts", "hmc"])
def test_welford_cov_without_adaptation_is_plain_sampling_bit_for_bit_and_host_equals_device(sampler, which):
    D, N, T_ = 12, 48, 10
    rng = np.random.default_rng(19)
    target, centre = _target(which, D, rng)
    scale = 0.05 if which == "glm" else 1.0
    Ms = np.stack([_spd(rng, D) for _ in range(N)]) * scale
    th = centre + np.sqrt(scale) * rng.normal(size=(N, D))
    kappa = _kernel(sampler, 0.2)
    ad = A.VectorisedStanAdaptor(metric_estimator="welford_cov")
    run = A.nuts_adapt_sample if sampler == "nuts" else A.hmc_adapt_sample
    h = A.Hamiltonian(A.DenseEuclideanMetric(torch.as_tensor(Ms, device=DEV)), target)
    z0 = A.phasepoint(h, torch.as_tensor(th, device=DEV), torch.zeros((N, D), dtype=torch.float64, device=DEV))
    za, da_, sa, ea, ma, _ = run(A.PhiloxRNG(7), h, kappa, z0, T_, 0, ad)
    zs, ds, ss = A.sample_transitions(A.PhiloxRNG(7), h, kappa, z0, T_)
    assert torch.equal(da_, ds) and torch.equal(za.theta, zs.theta) and torch.equal(za.r, zs.r)
    assert torch.equal(za.lp.value, zs.lp.value) and torch.equal(za.lk.value, zs.lk.value)
    for k in ss.keys() & sa.keys():
        if isinstance(ss[k], torch.Tensor):
            assert torch.equal(sa[k], ss[k]), k
    assert (ea.cpu().numpy() == 0.2).all()
    assert torch.equal(ma.Minv, h.metric.Minv) and torch.equal(ma.cholU, h.metric.cholU.contiguous())
    # host buffers: the same launch from numpy arrays
    hh = A.Hamiltonian(A.DenseEuclideanMetric(Ms, cholU=h.metric.cholU.cpu().numpy()), target)
    zh0 = A.phasepoint(hh, th.copy(), np.zeros((N, D)))
    zh, dh, sh, eh, mh, _ = run(A.PhiloxRNG(7), hh, kappa, zh0, T_, 0, ad)
    assert np.array_equal(dh, da_.cpu().numpy()) and np.array_equal(zh.theta, za.theta.cpu().numpy())
    assert np.array_equal(mh.Minv, ma.Minv.cpu().numpy()) and np.array_equal(mh.cholU, ma.cholU.cpu().numpy())


@pytest.mark.parametrize("sampler", ["nuts", "hmc"])
def test_step_size_only_with_a_dense_metric_moves_the_step_sizes_and_leaves_the_metric(sampler):
    D, N = 6, 32
    rng = np.random.default_rng(4)
    target, centre = _target("group", D, rng)
    Ms = torch.as_tensor(np.stack([_spd(rng, D) for _ in range(N)]), device=DEV)
    for me in (A.DenseEuclideanMetric(Ms), A.DenseEuclideanMetric(Ms[0].clone())):  # per chain and shared
        M_before = me.Minv.clone()
        h = A.Hamiltonian(me, target)
        th = torch.as_tensor(centre + rng.normal(size=(N, D)), device=DEV)
        z = A.phasepoint(h, th, torch.zeros_like(th))
        run = A.nuts_adapt_sample if sampler == "nuts" else A.hmc_adapt_sample
        zl, _, _, eps_f, met, _ = run(A.PhiloxRNG(2), h, _kernel(sampler, 0.2), z, 30, 20, A.VectorisedStanAdaptor(adapt_metric=False))
        assert met is None and torch.isfinite(zl.theta).all()
        e = eps_f.cpu().numpy()
        assert (e != 0.2).all() and len(np.unique(e)) == N
        assert torch.equal(h.metric.Minv, M_before)


def test_welford_cov_warm_up_on_a_group_form_gaussian_finds_the_covariance():
    """AR(1) correlations 0.9^|i-j| (eigenvalues 0.05..9.9) as a group-form UserTarget, D = 16, 512 chains, 1000 warm-up
    iterations with Stan's windows: the median over chains of ||M^-1 - Sigma||_F / ||Sigma||_F is below 0.15, the bound of
    the built-in dense Gaussian"""
    D, N, n_adapts, T_ = 16, 512, 1000, 1100
    rng = np.random.default_rng(2026)
    Sig = _ar1(D, 0.9)
    mu = rng.normal(size=D)
    h = A.Hamiltonian(A.DenseEuclideanMetric(D), _gauss("group", mu, Sig))
    th0 = torch.as_tensor(mu + rng.normal(size=(N, D)), device=DEV)
    z0 = A.phasepoint(h, th0, torch.zeros_like(th0))
    _, draws, _, _, met, _ = A.nuts_adapt_sample(A.PhiloxRNG(11), h, _kernel("nuts", 0.1), z0, T_, n_adapts,
                                                 A.VectorisedStanAdaptor(metric_estimator="welford_cov"))
    err = np.linalg.norm(met.Minv.cpu().numpy() - Sig, axis=(1, 2)) / np.linalg.norm(Sig)
    assert np.median(err) < 0.15, np.median(err)
    x = draws[n_adapts:].cpu().numpy().reshape(-1, D) - mu
    wz = np.linalg.solve(np.linalg.cholesky(Sig), x.T).T
    assert np.abs(wz.mean(axis=0)).max() < 0.1 and np.abs(wz.var(axis=0) - 1.0).max() < 0.05


def test_welford_cov_warm_up_on_a_correlated_logistic_regression():
    """Bernoulli-logit, AR(1)-0.9 predictors, n = 500, D = 6, 128 chains, 2000 warm-up iterations (the last window holds
    1100 draws): each chain's adapted M^-1 is within 0.2 relative Frobenius error of the covariance of all chains' pooled
    post-warm-up draws, and its sampling transitions take fewer leapfrog steps on average than those of a WelfordVar
    warm-up from the same start"""
    D, N, n_adapts, T_ = 6, 128, 2000, 2500
    rng = np.random.default_rng(77)
    target, beta = _logistic(rng, 500, D)
    th0 = torch.as_tensor(beta + 0.1 * rng.normal(size=(N, D)), device=DEV)
    kappa = _kernel("nuts", 0.05)
    hd = A.Hamiltonian(A.DenseEuclideanMetric(D), target)
    zd = A.phasepoint(hd, th0, torch.zeros_like(th0))
    _, draws, st, _, met, _ = A.nuts_adapt_sample(A.PhiloxRNG(5), hd, kappa, zd, T_, n_adapts,
                                                  A.VectorisedStanAdaptor(metric_estimator="welford_cov"))
    x = draws[n_adapts:].cpu().numpy().reshape(-1, D)
    pooled = np.cov(x.T)
    err = np.linalg.norm(met.Minv.cpu().numpy() - pooled, axis=(1, 2)) / np.linalg.norm(pooled)
    assert err.max() < 0.2, (np.median(err), err.max())
    hv = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), target)
    zv = A.phasepoint(hv, th0, torch.zeros_like(th0))
    _, _, sv, _, _, _ = A.nuts_adapt_sample(A.PhiloxRNG(5), hv, kappa, zv, T_, n_adapts,
                                            A.VectorisedStanAdaptor(metric_estimator="welford"), keep_draws=False)
    steps_dense = st["n_steps"][n_adapts:].double().mean().item()
    steps_var = sv["n_steps"][n_adapts:].double().mean().item()
    assert steps_dense < steps_var, (steps_dense, steps_var)


def test_dense_warm_up_refusals_on_user_and_callback_targets():
    """still refused with ERR_UNSUPPORTED: WelfordVar / NutpieVar with a Dense metric on a user target, a callback target
    with a Dense warm-up, NUTS variants with a Dense warm-up on a user target, and D > 512"""
    D, N = 6, 8
    rng = np.random.default_rng(1)
    target, centre = _target("group", D, rng)
    hD = A.Hamiltonian(A.DenseEuclideanMetric(torch.as_tensor(np.stack([_spd(rng, D) for _ in range(N)]), device=DEV)), target)
    th = torch.as_tensor(centre + rng.normal(size=(N, D)), device=DEV)
    zD = A.phasepoint(hD, th, torch.zeros_like(th))
    runs = ((A.nuts_adapt_sample, _kernel("nuts", 0.2)), (A.hmc_adapt_sample, _kernel("hmc", 0.1)))
    for est in ("nutpie", "welford"):
        for run, k in runs:
            with pytest.raises(A.AhmcError) as e:
                run(A.PhiloxRNG(1), hD, k, zD, 8, 6, A.VectorisedStanAdaptor(metric_estimator=est))
            assert e.value.code == L.ERR_UNSUPPORTED
    with pytest.raises(A.AhmcError) as e:
        A.nuts_adapt_sample(A.PhiloxRNG(1), hD, runs[0][1], zD, 8, 6, A.VectorisedStanAdaptor(metric_estimator="welford_cov"),
                            flags=L.FLAG_NUTS_CLASSIC)
    assert e.value.code == L.ERR_UNSUPPORTED and "MultinomialTS" in str(e.value)
    # a callback target: the target never runs (the refusal comes first)
    cb = A.CallbackTarget(D, lambda t: (torch.zeros(t.shape[0], dtype=t.dtype, device=t.device), -t))
    hc = A.Hamiltonian(A.DenseEuclideanMetric(D), cb)
    zc = K.PhasePoint(th, torch.zeros_like(th), K.DualValue(torch.zeros(N, dtype=torch.float64, device=DEV), -th.clone()),
                      K.DualValue(torch.zeros(N, dtype=torch.float64, device=DEV), None))
    for est in ("welford_cov", None):
        ad = A.VectorisedStanAdaptor(metric_estimator="welford_cov") if est else A.VectorisedStanAdaptor(adapt_metric=False)
        with pytest.raises(A.AhmcError) as e:
            A.hmc_adapt_sample(A.PhiloxRNG(1), hc, runs[1][1], zc, 8, 6, ad)
        assert e.value.code == L.ERR_UNSUPPORTED and "callback" in str(e.value)
    # D > 512: register-resident only
    D2, N2 = 600, 2
    big = A.UserTarget(D2, GAUSS_ONE_LANE, np.zeros(D2 + D2 * D2))
    h2 = A.Hamiltonian(A.DenseEuclideanMetric(D2), big)
    th2 = torch.as_tensor(rng.normal(size=(N2, D2)), device=DEV)
    z2 = K.PhasePoint(th2, torch.zeros_like(th2), K.DualValue(torch.zeros(N2, dtype=torch.float64, device=DEV), th2.clone()),
                      K.DualValue(torch.zeros(N2, dtype=torch.float64, device=DEV), None))
    for run, k in runs:
        with pytest.raises(A.AhmcError, match="register-resident"):
            run(A.PhiloxRNG(1), h2, k, z2, 4, 2, A.VectorisedStanAdaptor(metric_estimator="welford_cov"))
