"""Per-chain Dense metrics (an (N, D, D) M^-1: `DenseEuclideanMetric{..., AbstractArray{T,3}}`, metric.jl:89-103) and the
in-launch WelfordCov warm-up that adapts one per chain (ahmc_chain_adapt.cuh).  The oracle for NUTS and dense operators is
the reference's single-chain path applied to each chain: chain c of a per-chain call must equal oracle_c run on chain c's
own metric, and a fused warm-up must equal its iteration-by-iteration replay with the oracle's DualAveraging and one
WelfordCov(D) per chain.  The CPU side is tests/test_dense_adapt_cpu.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import ahmc_b200 as A
from ahmc_b200 import _lib as L
from ahmc_b200 import core as K
from oracle import oracle_c as oc
from tests.helpers import MODEL_KINDS, rel_err
from tests.test_gpu_parity import F, T, assert_pp_close, make_target

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _spd(rng, D, lo=-0.5, hi=0.5):
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    return (Q * np.exp(rng.uniform(lo, hi, D))) @ Q.T


def _problem(model, D, N, seed):
    rng = np.random.default_rng(seed)
    p0 = p1 = None
    if model == "dense_gauss":
        p0, p1 = rng.normal(size=D), np.linalg.inv(_spd(rng, D))
    Ms = np.stack([_spd(rng, D) for _ in range(N)])  # N different SPD matrices
    th = rng.normal(size=(D, N)) * (0.3 if model == "funnel" else 1.0)
    return rng, p0, p1, Ms, th


def _chain(z, c):
    """chain c of a device phase point, as the oracle's (D, 1) / (1,) arrays"""
    return dict(theta=F(z.theta)[:, c:c + 1], r=F(z.r)[:, c:c + 1], lp_gradient=F(z.lp.gradient)[:, c:c + 1],
                lp_value=F(z.lp.value)[c:c + 1], lk_value=F(z.lk.value)[c:c + 1])


def _close(got, zo, tol=1e-10):
    for f in ("theta", "r", "lp_gradient", "lp_value", "lk_value"):
        assert rel_err(got[f], getattr(zo, f)) < tol, (f, rel_err(got[f], getattr(zo, f)))


@pytest.mark.parametrize("model", ["dense_gauss", "funnel"])
@pytest.mark.parametrize("D", [5, 16, 33, 64, 200, 512])
def test_per_chain_dense_transitions_equal_oracle_on_each_chains_metric(model, D):
    """NUTS and static transitions on tapes: chain c equals oracle_c on chain c's own M^-1 (state within 1e-10, identical
    tree depths, n_steps, accept and divergence flags)"""
    N = 6 if D >= 200 else 8
    rng, p0, p1, Ms, th = _problem(model, D, N, seed=3 * D + (model == "funnel"))
    eps = {"dense_gauss": 0.25, "funnel": 0.1}[model]
    max_depth = 7 if D >= 200 else 9
    nt = rng.normal(size=(D, N))
    dirs = rng.integers(0, 2, size=(N, max_depth + 1)).astype(np.uint8)
    exps = rng.exponential(size=(N, 1 << max_depth))
    et = rng.exponential(size=N) * 0.05
    h = A.Hamiltonian(A.DenseEuclideanMetric(torch.as_tensor(Ms, device=DEV)), make_target(model, D, p0, p1, 0.0))
    z0 = A.phasepoint(h, T(th), T(np.zeros((D, N))))
    nuts = A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(eps), A.GeneralisedNoUTurn(max_depth, 1000.0)))
    tn = A.transition(A.TapeRNG(normal=T(nt), exp=torch.as_tensor(exps, device=DEV), dirs=torch.as_tensor(dirs, device=DEV)),
                      h, nuts, z0)
    L_ = 8
    stat = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(eps), A.FixedNSteps(L_)))
    ts = A.transition(A.TapeRNG(normal=T(nt), exp=torch.as_tensor(et, device=DEV)), h, stat, z0)
    om = oc.Model(MODEL_KINDS[model], D, p0, p1, 0.0)
    for c in range(N):
        ome = oc.Metric(oc.DENSE, Ms[c])
        z0o = oc.phasepoint(om, ome, th[:, c:c + 1], np.zeros((D, 1)))
        _close(_chain(z0, c), z0o)
        zo, so, _ = oc.nuts_transition(om, ome, eps, z0o, nt[:, c:c + 1], dirs[c:c + 1], exps[c:c + 1], max_depth=max_depth)
        _close(_chain(tn.z, c), zo)
        for k, v in (("tree_depth", so.tree_depth), ("n_steps", so.n_steps), ("numerical_error", so.numerical_error)):
            assert F(tn.stat[k])[c] == v[0], (c, k)
        assert rel_err(F(tn.stat["acceptance_rate"])[c:c + 1], so.acceptance_rate) < 1e-9
        z0o = oc.phasepoint(om, ome, th[:, c:c + 1], np.zeros((D, 1)))
        zs, ss = oc.hmc_transition(om, ome, eps, L_, z0o, nt[:, c:c + 1], et[c:c + 1])
        _close(_chain(ts.z, c), zs)
        assert F(ts.stat["is_accept"])[c] == ss.is_accept[0] and F(ts.stat["numerical_error"])[c] == ss.numerical_error[0]


def test_per_chain_dense_rand_momentum_phasepoint_step_and_find_good_stepsize():
    D, N = 33, 7
    rng, _, _, Ms, th = _problem("dense_gauss", D, N, seed=5)
    nt, r = rng.normal(size=(D, N)), rng.normal(size=(D, N))
    for Mi in (Ms, torch.as_tensor(Ms, device=DEV)):  # factors from numpy on the host, from torch.linalg on the device
        me = A.DenseEuclideanMetric(Mi)
        got = F(A.rand_momentum(A.TapeRNG(normal=T(nt)), me, None, T(th)))
        h = A.Hamiltonian(me, A.StdNormal(D))
        z = A.phasepoint(h, T(th), T(r))
        zl = A.step(A.Leapfrog(0.2), h, z, 5)
        om = oc.Model(oc.STD_NORMAL, D)
        for c in range(N):
            ome = oc.Metric(oc.DENSE, Ms[c])
            want = np.linalg.solve(ome.cholU, nt[:, c])  # rand_momentum: U \\ z (metric.jl:311-320)
            assert rel_err(got[:, c], want) < 1e-12
            zo = oc.phasepoint(om, ome, th[:, c:c + 1], r[:, c:c + 1])
            _close(_chain(z, c), zo)
            zlo, _, _ = oc.leapfrog(om, ome, 0.2, zo, 5)
            _close(_chain(zl, c), zlo)
    # find_good_stepsize, one search per chain in one launch, against the same search with chain c's metric alone
    h = A.Hamiltonian(A.DenseEuclideanMetric(Ms), A.StdNormal(D))
    e_all = A.find_good_stepsize_batched(A.TapeRNG(normal=T(nt)), h, T(th), 0.5).cpu().numpy()
    for c in (0, 3, N - 1):
        hc = A.Hamiltonian(A.DenseEuclideanMetric(Ms[c]), A.StdNormal(D))
        ec = A.find_good_stepsize_batched(A.TapeRNG(normal=T(nt[:, c:c + 1])), hc, T(th[:, c:c + 1]), 0.5).cpu().numpy()[0]
        assert abs(e_all[c] - ec) <= 1e-12 * ec


@pytest.mark.parametrize("D", [33, 64, 256])  # one chain per warp: the shared call runs the cooperative NUTS form
def test_same_matrix_per_chain_equals_the_shared_dense_call(D):
    """every chain given the same matrix per chain = the shared Dense call (cooperative NUTS form / tiled trajectory) to
    1e-10 with identical decisions (the summation orders differ, so bit equality is not expected)"""
    N = 40
    rng, p0, p1, Ms, th = _problem("dense_gauss", D, 1, seed=D)
    M = Ms[0]
    target = make_target("dense_gauss", D, p0, p1, 0.0)
    hs = A.Hamiltonian(A.DenseEuclideanMetric(M), target)
    hp = A.Hamiltonian(A.DenseEuclideanMetric(np.broadcast_to(M, (N, D, D)).copy()), target)
    th = rng.normal(size=(D, N))
    for kappa in (A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.2), A.GeneralisedNoUTurn(8, 1000.0))),
                  A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.2), A.FixedNSteps(10)))):
        zs, ds, ss = A.sample_transitions(A.PhiloxRNG(4), hs, kappa, A.phasepoint(hs, T(th), T(np.zeros((D, N)))), 5)
        zp, dp, sp = A.sample_transitions(A.PhiloxRNG(4), hp, kappa, A.phasepoint(hp, T(th), T(np.zeros((D, N)))), 5)
        assert rel_err(dp.cpu().numpy(), ds.cpu().numpy()) < 1e-10
        assert_pp_close(zp, dict(theta=F(zs.theta), r=F(zs.r), lp_gradient=F(zs.lp.gradient), lp_value=F(zs.lp.value),
                                 lk_value=F(zs.lk.value)))
        for k in ("n_steps", "is_accept", "numerical_error") + (("tree_depth",) if "tree_depth" in ss else ()):
            assert torch.equal(sp[k].cpu(), ss[k].cpu()), k
    # one step of the tiled trajectory form against the per-chain warp form
    z = A.phasepoint(hs, T(th), T(rng.normal(size=(D, N))))
    zp = A.phasepoint(hp, T(th), z.r.clone())
    assert_pp_close(A.step(A.Leapfrog(0.1), hp, zp, 6), _all(A.step(A.Leapfrog(0.1), hs, z, 6)))


def _all(z):
    return dict(theta=F(z.theta), r=F(z.r), lp_gradient=F(z.lp.gradient), lp_value=F(z.lp.value), lk_value=F(z.lk.value))


def _kernel(sampler, eps):
    if sampler == "nuts":
        return A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(eps), A.GeneralisedNoUTurn(8, 1000.0)))
    return A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(eps), A.FixedNSteps(12)))


@pytest.mark.parametrize("sampler", ["nuts", "hmc"])
def test_fused_welford_cov_equals_iteration_by_iteration_replay_with_oracle_adaptors(sampler):
    """single-transition launches on the same Philox streams with the fused launch's step sizes, the oracle's DualAveraging
    and one oracle WelfordCov(D) per chain on the host: step sizes and the window-end M^-1 / factor to 1e-9, draws to 1e-10
    with identical decisions; after the update the replay continues with the kernel's own per-chain matrices"""
    D, N, T_, n_adapts, seed = 8, 64, 60, 50, 31
    ib, tb, wsz = 10, 8, 6
    ws, we, splits = oc.stan_windows(n_adapts, ib, tb, wsz)
    assert (ws, we, list(splits)) == (11, 42, [16, 42])  # the first window holds 6 < n_min draws: reset without an update
    rng = np.random.default_rng(seed)
    Sig = _spd(rng, D, -1.0, 1.0)
    target = A.DenseGaussian(rng.normal(size=D), np.linalg.inv(Sig))
    M0 = torch.as_tensor(np.stack([_spd(rng, D, -0.2, 0.2) for _ in range(N)]), device=DEV)
    h = A.Hamiltonian(A.DenseEuclideanMetric(M0), target)
    th0 = torch.as_tensor(rng.normal(size=(N, D)), device=DEV)
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


@pytest.mark.parametrize("sampler", ["nuts", "hmc"])
def test_welford_cov_without_adaptation_is_plain_sampling_bit_for_bit_and_host_equals_device(sampler):
    D, N, T_ = 24, 48, 12
    rng = np.random.default_rng(9)
    Ms = np.stack([_spd(rng, D) for _ in range(N)])
    target = A.DenseGaussian(rng.normal(size=D), np.linalg.inv(_spd(rng, D)))
    th = rng.normal(size=(N, D))
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


def test_welford_cov_warm_up_finds_the_covariance_and_samples_the_target():
    """correlated Gaussian (AR(1) correlations 0.9^|i-j|: eigenvalues 0.05..9.9), D = 16, 512 chains, 1000 warm-up
    iterations with Stan's windows: the median over chains of ||M^-1 - Sigma||_F / ||Sigma||_F is below 0.15 (500 draws
    in the last window); whitened post-warm-up draws have mean 0 and variance 1"""
    D, N, n_adapts, T_ = 16, 512, 1000, 1200
    rng = np.random.default_rng(2026)
    i = np.arange(D)
    Sig = 0.9 ** np.abs(i[:, None] - i[None, :])
    mu = rng.normal(size=D)
    h = A.Hamiltonian(A.DenseEuclideanMetric(D), A.DenseGaussian(mu, np.linalg.inv(Sig)))
    th0 = torch.as_tensor(mu + rng.normal(size=(N, D)), device=DEV)
    z0 = A.phasepoint(h, th0, torch.zeros_like(th0))
    kappa = _kernel("nuts", 0.1)
    zl, draws, st, eps, met, _ = A.nuts_adapt_sample(A.PhiloxRNG(11), h, kappa, z0, T_, n_adapts,
                                                     A.VectorisedStanAdaptor(metric_estimator="welford_cov"))
    Mi = met.Minv.cpu().numpy()
    err = np.linalg.norm(Mi - Sig, axis=(1, 2)) / np.linalg.norm(Sig)
    assert np.median(err) < 0.15, np.median(err)
    Lc = np.linalg.cholesky(Sig)
    x = draws[n_adapts:].cpu().numpy().reshape(-1, D) - mu
    wz = np.linalg.solve(Lc, x.T).T
    assert np.abs(wz.mean(axis=0)).max() < 0.1
    assert np.abs(wz.var(axis=0) - 1.0).max() < 0.05


def test_per_chain_dense_and_welford_cov_errors():
    D, N = 6, 4
    rng = np.random.default_rng(1)
    ctx = A.get_context(0)
    Ms = torch.as_tensor(np.stack([_spd(rng, D) for _ in range(N)]), device=DEV)
    # 0 < chain_stride < D*D: AxesMismatch
    Mi, U = Ms.mT.contiguous(), torch.linalg.cholesky(Ms).contiguous()
    r = torch.zeros((N, D), dtype=torch.float64, device=DEV)
    rc = L.Rng(1, 0, None, None, 0, None, 0, 0.0, 0.0)
    for s in (1, D, D * D - 1):
        md = L.Metric(L.METRIC_DENSE, Mi.data_ptr(), s, U.data_ptr())
        assert ctx.lib.ahmc_rand_momentum_f64(ctx.h, C.byref(md), D, N, C.byref(rc), r.data_ptr(), D, 0) == L.ERR_INVALID
        assert b"AxesMismatch" in ctx.lib.ahmc_last_error(ctx.h)
    md = L.Metric(L.METRIC_DENSE, Mi.data_ptr(), D * D, U.data_ptr())
    assert ctx.lib.ahmc_rand_momentum_f64(ctx.h, C.byref(md), D, N, C.byref(rc), r.data_ptr(), D, 0) == 0
    target = A.StdNormal(D)
    th = torch.as_tensor(rng.normal(size=(N, D)), device=DEV)
    kern = _kernel("nuts", 0.2)
    # WelfordCov with a Diag metric: INVALID, from the Python mirror and from the C entry points
    hd = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), target)
    zd = A.phasepoint(hd, th, torch.zeros_like(th))
    runs = ((A.nuts_adapt_sample, kern), (A.hmc_adapt_sample, _kernel("hmc", 0.1)))
    for run, k in runs:
        with pytest.raises(A.InvalidArgument):
            run(A.PhiloxRNG(1), hd, k, zd, 8, 6, A.VectorisedStanAdaptor(metric_estimator="welford_cov"))
    for hmc in (False, True):
        _, _, _, out, md, keep, eps, minv, trace, cfg, rc2, draws = K._adapt_launch_args(hd, runs[hmc][1], zd, 8, 6,
                                                                                          A.VectorisedStanAdaptor(), False, False,
                                                                                          A.PhiloxRNG(1))
        cfg.adapt_metric = 3
        st, sc = K._stats_buffers(zd.theta, N, not hmc, T=8)
        zc, oc_ = zd._c(False), out._c(False)
        if hmc:
            code = ctx.lib.ahmc_hmc_adapt_sample_f64(ctx.h, hd.target.handle(ctx), C.byref(md), D, N, 12, 8, C.byref(cfg), C.byref(rc2),
                                                     C.byref(zc), C.byref(oc_), None, C.byref(sc), 0)
        else:
            code = ctx.lib.ahmc_nuts_adapt_sample_f64(ctx.h, hd.target.handle(ctx), C.byref(md), D, N, 8, 1000.0, 8, C.byref(cfg),
                                                      C.byref(rc2), C.byref(zc), C.byref(oc_), None, C.byref(sc), 0)
        assert code == L.ERR_INVALID, code
    # Dense with WelfordVar / NutpieVar: UNSUPPORTED
    hD = A.Hamiltonian(A.DenseEuclideanMetric(Ms), target)
    zD = A.phasepoint(hD, th, torch.zeros_like(th))
    for est in ("nutpie", "welford"):
        for run, k in runs:
            with pytest.raises(A.AhmcError) as e:
                run(A.PhiloxRNG(1), hD, k, zD, 8, 6, A.VectorisedStanAdaptor(metric_estimator=est))
            assert e.value.code == L.ERR_UNSUPPORTED
    # a Dense metric without its factor: refused before anything runs, even with AHMC_FLAG_NO_REFRESH (the launch copies
    # the factor into the chain's cholU_chain row)
    for hmc in (False, True):
        for est in (0, 3):
            _, _, _, out, md, keep, eps, minv, trace, cfg, rc2, draws = K._adapt_launch_args(hD, runs[hmc][1], zD, 8, 6,
                                                                                              A.VectorisedStanAdaptor(metric_estimator="welford_cov"),
                                                                                              False, False, A.PhiloxRNG(1))
            cfg.adapt_metric = est
            md.cholU = None
            st, sc = K._stats_buffers(zD.theta, N, not hmc, T=8)
            zc, oc_ = zD._c(False), out._c(False)
            fl = L.FLAG_NO_REFRESH
            if hmc:
                code = ctx.lib.ahmc_hmc_adapt_sample_f64(ctx.h, hD.target.handle(ctx), C.byref(md), D, N, 12, 8, C.byref(cfg),
                                                         C.byref(rc2), C.byref(zc), C.byref(oc_), None, C.byref(sc), fl)
            else:
                code = ctx.lib.ahmc_nuts_adapt_sample_f64(ctx.h, hD.target.handle(ctx), C.byref(md), D, N, 8, 1000.0, 8, C.byref(cfg),
                                                          C.byref(rc2), C.byref(zc), C.byref(oc_), None, C.byref(sc), fl)
            assert code == L.ERR_INVALID, (hmc, est, code)
            assert b"cholU" in ctx.lib.ahmc_last_error(ctx.h)
    # step size only with a Dense metric runs and leaves the metric alone
    zl, _, _, eps_f, met, _ = A.nuts_adapt_sample(A.PhiloxRNG(1), hD, kern, zD, 8, 6, A.VectorisedStanAdaptor(adapt_metric=False))
    assert met is None and torch.isfinite(zl.theta).all() and (eps_f != 0.2).any()
    # a Dense metric at D = 600 is still register-resident only, shared or per chain, with or without WelfordCov
    D2, N2 = 600, 2
    th2 = torch.as_tensor(rng.normal(size=(N2, D2)), device=DEV)
    for me in (A.DenseEuclideanMetric(D2), A.DenseEuclideanMetric(torch.eye(D2, dtype=torch.float64, device=DEV).expand(N2, D2, D2).contiguous())):
        h2 = A.Hamiltonian(me, A.StdNormal(D2))
        with pytest.raises(A.AhmcError, match="register-resident"):
            A.phasepoint(h2, th2, torch.zeros_like(th2))
        with pytest.raises(A.AhmcError, match="register-resident"):
            A.rand_momentum(A.PhiloxRNG(1), me, None, th2)
        z2 = K.PhasePoint(th2, torch.zeros_like(th2), K.DualValue(torch.zeros(N2, dtype=torch.float64, device=DEV), th2.clone()),
                          K.DualValue(torch.zeros(N2, dtype=torch.float64, device=DEV), None))
        with pytest.raises(A.AhmcError, match="register-resident"):
            A.hmc_adapt_sample(A.PhiloxRNG(1), h2, _kernel("hmc", 0.1), z2, 4, 2, A.VectorisedStanAdaptor(metric_estimator="welford_cov"))
