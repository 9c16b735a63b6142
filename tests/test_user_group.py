"""Run-time compiled targets in the GROUP form (`#define AHMC_USER_GROUPWISE`, `ahmc_user_logp_grad_group`): every lane of
the chain's group evaluates the user's log density and gradient together.  Checked against the built-in targets, the
recursive oracle, a float64 numpy evaluation and the one-lane form, and bit for bit against the entry points a launch must
agree with (run with -m gpu on an H100)."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import ahmc_b200 as A
from oracle import oracle_c as oc
from tests.helpers import METRIC_KINDS, rel_err
from tests.test_gpu_parity import DEV, F, T, assert_pp_close, make_metric

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Neal's funnel: lane 0 computes e^-v and broadcasts it; lane l owns the coordinates d = l + G k; the sum of th_d^2 e^-v
# is reduced across the group and lane 0 adds the v terms
GROUP_FUNNEL = r'''
#define AHMC_USER_GROUPWISE
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    const double v = th[0];
    const double ev = ahmc_group_bcast(grp, grp.lane == 0 ? exp(-v) : 0.0, 0);
    double s = 0.0;
    for (int d = grp.lane; d < D; d += grp.size) {
        if (d == 0) continue;
        const double gd = th[d] * ev;
        g[d] = -gd;
        s = fma(th[d], gd, s);
    }
    const double S = ahmc_group_sum(grp, s);
    if (grp.lane != 0) return 0.0;
    g[0] = -v / 9.0 + (S - (D - 1)) * 0.5;
    return -v * v / 18.0 - (S + (D - 1) * v) * 0.5;
}
'''
# diagonal Gaussian, p = [mean_0, 1/s_0^2, mean_1, ...]: each lane writes the gradient of its coordinates, and after a group
# sync returns the log-density share of the NEXT lane's coordinates, read back from the gradient slab
GROUP_DIAG = r'''
#define AHMC_USER_GROUPWISE
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    for (int d = grp.lane; d < D; d += grp.size) g[d] = -(th[d] - p[2 * d]) * p[2 * d + 1];
    ahmc_group_sync(grp);
    double share = 0.0;
    for (int d = (grp.lane + 1) % grp.size; d < D; d += grp.size) share = fma(0.5 * (th[d] - p[2 * d]), g[d], share);
    return share;
}
'''


def _cost_module():
    spec = importlib.util.spec_from_file_location("user_group_cost", os.path.join(ROOT, "scripts", "user_group_cost.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _pp_equal(a, b):
    return all(torch.equal(x, y) if isinstance(x, torch.Tensor) else np.array_equal(x, y)
               for x, y in ((a.theta, b.theta), (a.r, b.r), (a.lp.gradient, b.lp.gradient), (a.lp.value, b.lp.value),
                            (a.lk.value, b.lk.value)))


def _metric(metric, D, rng):
    if metric == "diag":
        return np.exp(rng.uniform(-0.5, 0.5, D))
    if metric == "dense":
        B = rng.normal(size=(D, D))
        return B @ B.T / D + 0.5 * np.eye(D)
    return None


@pytest.mark.parametrize("which,D,metric", [("funnel", 3, "unit"), ("funnel", 20, "diag"), ("funnel", 100, "unit"),
                                            ("diag", 128, "diag"), ("diag", 3, "diag"), ("diag", 7, "dense")])
def test_group_form_equals_the_builtin_target(which, D, metric):
    """phasepoint, 11 exact-path steps with and without a cached gradient (device and host buffers), a static transition on
    tapes and find_good_stepsize_batched: the group form gives the built-in target's results (same arithmetic up to
    summation order).  D = 3 puts eight chains in one warp."""
    rng = np.random.default_rng(70 + D)
    N = 77
    Minv = _metric(metric, D, rng)
    if which == "funnel":
        builtin, user = A.Funnel(D, 0.25), A.UserTarget(D, GROUP_FUNNEL, c0=0.25)
        th = rng.normal(size=(D, N)) * 0.4
    else:
        m, s = rng.normal(size=D), np.exp(rng.uniform(-0.7, 0.7, D))
        builtin = A.DiagGaussian(m, s, normalised=False)
        builtin.c0 = 0.25
        user = A.UserTarget(D, GROUP_DIAG, params=np.stack([m, 1.0 / s ** 2], axis=1), c0=0.25)
        th = rng.normal(size=(D, N))
    r = rng.normal(size=(D, N))
    hb, hu = A.Hamiltonian(make_metric(metric, Minv, D), builtin), A.Hamiltonian(make_metric(metric, Minv, D), user)
    zb, zu = A.phasepoint(hb, T(th), T(r)), A.phasepoint(hu, T(th), T(r))
    for a, b in [(zu.lp.value, zb.lp.value), (zu.lp.gradient, zb.lp.gradient), (zu.lk.value, zb.lk.value)]:
        assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-12
    z1b = A.step(A.Leapfrog(0.05), hb, zb, 11, flags=A.FLAG_EXACT_CHECKS)
    z1u, info = A.step(A.Leapfrog(0.05), hu, zu, 11, return_info=True)
    assert (F(info.steps_done) == 11).all()
    for a, b in [(z1u.theta, z1b.theta), (z1u.r, z1b.r), (z1u.lp.gradient, z1b.lp.gradient), (z1u.lp.value, z1b.lp.value),
                 (z1u.lk.value, z1b.lk.value)]:
        assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-11
    z1n = A.step(A.Leapfrog(0.05), hu, A.PhasePoint(zu.theta, zu.r, A.DualValue(None, None), A.DualValue(None, None)), 11)
    assert torch.equal(z1n.theta, z1u.theta) and torch.equal(z1n.lp.gradient, z1u.lp.gradient)
    if metric != "dense":
        zh = A.step(A.Leapfrog(0.05), hu, A.PhasePoint(np.ascontiguousarray(th.T), np.ascontiguousarray(r.T), A.DualValue(None, None),
                                                        A.DualValue(None, None)), 11)
        assert np.array_equal(zh.theta, z1u.theta.cpu().numpy())
    nt, et = T(rng.normal(size=(D, N))), torch.as_tensor(rng.exponential(size=N), device=DEV)
    kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.1), A.FixedNSteps(7)))
    tb = A.transition(A.TapeRNG(normal=nt, exp=et), hb, kern, zb, flags=A.FLAG_EXACT_CHECKS)
    tu = A.transition(A.TapeRNG(normal=nt, exp=et), hu, kern, zu)
    assert torch.equal(tu.stat["is_accept"], tb.stat["is_accept"])
    assert rel_err(tu.z.theta.cpu().numpy(), tb.z.theta.cpu().numpy()) < 1e-11
    eb = A.find_good_stepsize_batched(A.TapeRNG(normal=nt), hb, T(th))
    eu = A.find_good_stepsize_batched(A.TapeRNG(normal=nt), hu, T(th))
    assert torch.equal(eb, eu)


@pytest.mark.parametrize("D,eps,scale,metric", [(20, 0.12, 0.6, "diag"), (100, 0.1, 0.5, "diag"), (3, 0.9, 2.0, "unit"),
                                                (3, 0.5, 1.5, "diag")])
def test_nuts_on_the_group_form_matches_the_recursive_oracle_on_tapes(D, eps, scale, metric):
    """NUTS with the group-form funnel compiled into the kernel: same trees, draws and statistics as the recursive oracle
    running the built-in funnel, chain by chain.  At D = 3 eight chains share a warp and sit at different tree positions."""
    N, max_depth = 150, 10
    rng = np.random.default_rng(D * 17 + 3)
    Minv = np.exp(rng.uniform(-0.5, 0.5, D)) if metric == "diag" else None
    th, nt = rng.normal(size=(D, N)) * scale, rng.normal(size=(D, N))
    dirs = rng.integers(0, 2, size=(N, max_depth + 1)).astype(np.uint8)
    exps = rng.exponential(size=(N, 1 << max_depth))
    om, ome = oc.Model(oc.FUNNEL, D, None, None, 0.0), oc.Metric(METRIC_KINDS[metric], Minv)
    zo, so, _ = oc.nuts_transition(om, ome, eps, oc.phasepoint(om, ome, th, np.zeros((D, N))), nt, dirs, exps, max_depth=max_depth)
    h = A.Hamiltonian(make_metric(metric, Minv, D), A.UserTarget(D, GROUP_FUNNEL))
    z0 = A.phasepoint(h, T(th), T(np.zeros((D, N))))
    tau = A.Trajectory(A.MultinomialTS, A.Leapfrog(eps), A.GeneralisedNoUTurn(max_depth, 1000.0))
    tr = A.transition(A.TapeRNG(normal=T(nt), exp=torch.as_tensor(exps, device=DEV), dirs=torch.as_tensor(dirs, device=DEV)), h,
                      A.HMCKernel(tau), z0)
    st = tr.stat
    assert (F(st["tree_depth"]) == so.tree_depth).all() and (F(st["n_steps"]) == so.n_steps).all()
    assert (F(st["numerical_error"]) == so.numerical_error).all()
    assert len(set(so.tree_depth.tolist())) > 1
    assert_pp_close(tr.z, zo, tol=1e-10)
    assert rel_err(F(st["acceptance_rate"]), so.acceptance_rate) < 1e-9


@pytest.mark.parametrize("D", [7, 25])
def test_logistic_regression_group_form_against_numpy_and_the_one_lane_form(D):
    """the logistic regression of scripts/user_group_cost.py (n = 1000 rows): the group form's lp and gradient equal a float64
    numpy evaluation; under NUTS on shared tapes the group and one-lane forms build the same trees"""
    cost = _cost_module()
    n, N, max_depth, eps = 1000, 64, 8, 0.03
    params, X, y, beta = cost.logreg_data(n, D, seed=D)
    one, grp = cost.logreg_sources(n, D)
    rng = np.random.default_rng(D)
    th = beta + 0.1 * rng.normal(size=(N, D))
    hg = A.Hamiltonian(A.UnitEuclideanMetric(D), A.UserTarget(D, grp, params=params))
    h1 = A.Hamiltonian(A.UnitEuclideanMetric(D), A.UserTarget(D, one, params=params))
    zg = A.phasepoint(hg, torch.as_tensor(th, device=DEV), torch.zeros((N, D), dtype=torch.float64, device=DEV))
    lp, grad = cost.logreg_numpy(th, X, y, params[0])
    assert rel_err(zg.lp.value.cpu().numpy(), lp) < 1e-12
    assert rel_err(-zg.lp.gradient.cpu().numpy(), grad) < 1e-12
    z1 = A.phasepoint(h1, torch.as_tensor(th, device=DEV), torch.zeros((N, D), dtype=torch.float64, device=DEV))
    nt = torch.as_tensor(rng.normal(size=(N, D)), device=DEV)
    dirs = torch.as_tensor(rng.integers(0, 2, size=(N, max_depth + 1)).astype(np.uint8), device=DEV)
    exps = torch.as_tensor(rng.exponential(size=(N, 1 << max_depth)), device=DEV)
    kern = A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(eps), A.GeneralisedNoUTurn(max_depth, 1000.0)))
    tg = A.transition(A.TapeRNG(normal=nt, exp=exps, dirs=dirs), hg, kern, zg)
    t1 = A.transition(A.TapeRNG(normal=nt, exp=exps, dirs=dirs), h1, kern, z1)
    for k in ("tree_depth", "n_steps", "numerical_error"):
        assert torch.equal(tg.stat[k], t1.stat[k]), k
    assert tg.stat["n_steps"].min().item() >= 3
    for a, b in ((tg.z.theta, t1.z.theta), (tg.z.r, t1.z.r), (tg.z.lp.gradient, t1.z.lp.gradient), (tg.z.lp.value, t1.z.lp.value)):
        assert rel_err(a.cpu().numpy(), b.cpu().numpy()) < 1e-10


def _funnel_problem(D, N, seed, metric="diag"):
    rng = np.random.default_rng(seed)
    Minv = np.exp(rng.uniform(-0.3, 0.3, D)) if metric == "diag" else None
    h = A.Hamiltonian(make_metric(metric, Minv, D), A.UserTarget(D, GROUP_FUNNEL))
    th = torch.as_tensor(rng.normal(size=(N, D)) * 0.5, device=DEV)
    return h, th


@pytest.mark.parametrize("D", [3, 20])
def test_group_form_launches_agree_bit_for_bit(D):
    """a persistent launch equals the loop of single transitions (static HMC and NUTS); host buffers equal device buffers;
    the adaptive launches with n_adapts = 0 equal sample_transitions; two identical launches give identical bits"""
    N, Tn = 70, 4
    h, th = _funnel_problem(D, N, 40 + D)
    z0 = A.phasepoint(h, th, torch.zeros_like(th))
    static = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.15), A.FixedNSteps(6)))
    nuts = A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.2), A.GeneralisedNoUTurn(8, 1000.0)))
    for kern in (static, nuts):
        zl, draws, st = A.sample_transitions(A.PhiloxRNG(23), h, kern, z0, Tn)
        prng, z = A.PhiloxRNG(23), z0
        for t in range(Tn):
            tr = A.transition(prng, h, kern, z)
            z = tr.z
            assert torch.equal(draws[t], z.theta), t
            for k in ("acceptance_rate", "hamiltonian_energy", "numerical_error", "n_steps"):
                assert torch.equal(st[k][t], tr.stat[k]), (t, k)
        assert _pp_equal(zl, z)
        zl2, draws2, st2 = A.sample_transitions(A.PhiloxRNG(23), h, kern, z0, Tn)
        assert _pp_equal(zl, zl2) and torch.equal(draws, draws2) and torch.equal(st["acceptance_rate"], st2["acceptance_rate"])
        ref = A.transition(A.PhiloxRNG(17), h, kern, z0)
        zh0 = A.phasepoint(h, th.cpu().numpy(), np.zeros((N, D)))
        trh = A.transition(A.PhiloxRNG(17), h, kern, zh0)
        assert np.array_equal(trh.z.theta, ref.z.theta.cpu().numpy()) and np.array_equal(trh.z.r, ref.z.r.cpu().numpy())
        assert np.array_equal(trh.z.lp.value, ref.z.lp.value.cpu().numpy())
        run = A.nuts_adapt_sample if kern is nuts else A.hmc_adapt_sample
        for est in ("welford", "nutpie"):
            za, da, sa, _, _, _ = run(A.PhiloxRNG(23), h, kern, z0, Tn, 0, A.VectorisedStanAdaptor(metric_estimator=est))
            assert torch.equal(da, draws) and _pp_equal(za, zl)
            for k in ("n_steps", "acceptance_rate", "hamiltonian_energy", "numerical_error"):
                assert torch.equal(sa[k], st[k]), (est, k)


@pytest.mark.parametrize("sampler", ["nuts", "hmc"])
def test_warm_up_on_a_group_form_gaussian_recovers_the_variances(sampler):
    """in-launch warm-up (WelfordVar, NutpieVar) on the group-form diagonal Gaussian, D = 20, scales log-spaced over
    0.3..3: the median over chains of M^-1 / s^2 within 10 % for every coordinate"""
    D, N, Tn, n_adapts = 20, 1024, 600, 500
    s = np.exp(np.linspace(np.log(0.3), np.log(3.0), D))
    target = A.UserTarget(D, GROUP_DIAG, params=np.stack([np.zeros(D), 1.0 / s ** 2], axis=1))
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), target)
    th0 = torch.as_tensor(np.random.default_rng(8).normal(size=(N, D)) * s, device=DEV)
    z0 = A.phasepoint(h, th0, torch.zeros_like(th0))
    run = A.nuts_adapt_sample if sampler == "nuts" else A.hmc_adapt_sample
    for est in ("welford", "nutpie"):
        kern = (A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.1), A.GeneralisedNoUTurn(8, 1000.0))) if sampler == "nuts"
                else A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.05), A.FixedNSteps(16))))
        _, _, _, _, minv, _ = run(A.PhiloxRNG(12), h, kern, z0, Tn, n_adapts, A.VectorisedStanAdaptor(metric_estimator=est),
                                  keep_draws=False)
        med = np.median(minv.cpu().numpy() / s ** 2, axis=0)
        print(f"{sampler} {est}: median ratio {med.min():.3f}..{med.max():.3f}")
        assert 0.9 < med.min() and med.max() < 1.1, (est, med.min(), med.max())


def test_group_form_errors_come_back_as_messages():
    both = "#define AHMC_USER_COORDWISE\n" + GROUP_DIAG
    h = A.Hamiltonian(A.UnitEuclideanMetric(4), A.UserTarget(4, both, params=np.ones(8)))
    z = torch.zeros((3, 4), dtype=torch.float64, device=DEV)
    with pytest.raises(A.AhmcError) as e:
        A.phasepoint(h, z, z)
    assert "AHMC_USER_GROUPWISE" in str(e.value) and "AHMC_USER_COORDWISE" in str(e.value)
    bad = GROUP_FUNNEL.replace("return 0.0;", "return nope;")
    h = A.Hamiltonian(A.UnitEuclideanMetric(4), A.UserTarget(4, bad))
    with pytest.raises(A.AhmcError) as e:
        A.phasepoint(h, z, z)
    assert "nope" in str(e.value) and "undefined" in str(e.value)
