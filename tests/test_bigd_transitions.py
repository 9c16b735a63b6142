"""Sampling beyond 512 dimensions (ahmc_bigd_hmc.cu): rand_momentum, static EndPointTS transitions (one, several, with
in-launch adaptation) and find_good_stepsize in the streaming form, against the oracle and against the entry points they
must agree with bit for bit (run with -m gpu on an H100)."""
import ctypes as C

import numpy as np
import pytest
import torch

import ahmc_b200 as A
from ahmc_b200 import core as K
from oracle import oracle_c as oc
from tests.helpers import METRIC_KINDS, MODEL_KINDS, rel_err
from tests.test_adapt_in_launch import _replay
from tests.test_gpu_parity import DEV, F, T, assert_pp_close, make_metric, make_target

pytestmark = pytest.mark.gpu


def _pp_equal(a, b):
    return all(torch.equal(x, y) if isinstance(x, torch.Tensor) else np.array_equal(x, y)
               for x, y in ((a.theta, b.theta), (a.r, b.r), (a.lp.gradient, b.lp.gradient), (a.lp.value, b.lp.value),
                            (a.lk.value, b.lk.value)))


def _static(eps, L):
    return A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(eps), A.FixedNSteps(L)))


def _problem(model, metric, D, N, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    p0 = p1 = Minv = None
    if model == "diag_gauss":
        p0, p1 = rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))
    mk = "diag" if metric == "diag_perchain" else metric
    if metric == "diag":
        Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    elif metric == "diag_perchain":
        Minv = np.exp(rng.uniform(-0.5, 0.5, (D, N)))
    om, ome = oc.Model(MODEL_KINDS[model], D, p0, p1, 0.25), oc.Metric(METRIC_KINDS[mk], Minv)
    h = A.Hamiltonian(make_metric(mk, Minv, D), make_target(model, D, p0, p1, 0.25))
    th = rng.normal(size=(D, N)) * scale
    return rng, om, ome, h, th


def test_rand_momentum_beyond_512_extends_the_512_draw():
    D, N = 600, 37
    z = torch.zeros((N, D), dtype=torch.float64, device=DEV)
    r600 = A.rand_momentum(A.PhiloxRNG(5), A.UnitEuclideanMetric(D), None, z)
    r512 = A.rand_momentum(A.PhiloxRNG(5), A.UnitEuclideanMetric(512), None, z[:, :512].contiguous())
    assert torch.equal(r600[:, :512], r512)
    assert len({tuple(x) for x in r600[:, 512:].cpu().numpy()}) == N
    Minv = np.exp(np.random.default_rng(1).uniform(-1, 1, D))
    rd = A.rand_momentum(A.PhiloxRNG(5), A.DiagEuclideanMetric(Minv), None, z).cpu().numpy()
    assert rel_err(rd, r600.cpu().numpy() / np.sqrt(Minv)) < 1e-15
    xi = np.random.default_rng(2).normal(size=(D, 3))  # the tape path against the oracle's rand_momentum
    from tests.test_gpu_parity import _orc_rand_momentum

    got = F(A.rand_momentum(A.TapeRNG(normal=T(xi)), A.DiagEuclideanMetric(Minv), None, T(xi)))
    want = np.stack([_orc_rand_momentum(oc.Metric(oc.DIAG, Minv), xi[:, c]) for c in range(3)], axis=1)
    assert rel_err(got, want) < 1e-14


TAPE_CASES = [("diag_gauss", "diag", 513, 5, 0.0), ("diag_gauss", "diag_perchain", 777, 7, 0.6), ("funnel", "diag", 1500, 6, 0.0),
              ("std_normal", "unit", 5000, 3, 0.0), ("funnel", "unit", 1100, 5, -0.3)]


@pytest.mark.parametrize("model,metric,D,N,partial", TAPE_CASES, ids=[f"{c[0]}-{c[1]}-D{c[2]}" for c in TAPE_CASES])
def test_transition_beyond_512_vs_oracle_with_tapes(model, metric, D, N, partial):
    """one transition from tapes: state within 1e-10, identical decisions and step counts; chain 1 takes a step 25x too
    large and is rejected; partial momentum refreshment where `partial` != 0"""
    rng, om, ome, h, th = _problem(model, metric, D, N, D, scale=0.3 if (model == "funnel" and metric != "unit") else 1.0)
    r_prev = rng.normal(size=(D, N))
    nt, et = rng.normal(size=(D, N)), rng.exponential(size=N) * 0.05
    eps0 = {"diag_gauss": 0.15, "std_normal": 0.1, "funnel": 0.03}[model]
    eps = np.full(N, eps0)
    eps[1] *= 25.0
    L = 9
    oc.set_partial_refresh(partial)
    try:
        zo, so = oc.hmc_transition(om, ome, eps, L, oc.phasepoint(om, ome, th, r_prev), nt, et)
    finally:
        oc.set_partial_refresh(0.0)
    z0 = A.phasepoint(h, T(th), T(r_prev))
    tau = A.Trajectory(A.EndPointTS, A.Leapfrog(torch.as_tensor(eps, device=DEV)), A.FixedNSteps(L))
    kern = A.HMCKernel(tau, A.PartialMomentumRefreshment(partial)) if partial else A.HMCKernel(tau)
    tr = A.transition(A.TapeRNG(normal=T(nt), exp=torch.as_tensor(et, device=DEV)), h, kern, z0)
    acc = F(tr.stat["is_accept"]).astype(bool)
    assert not acc[1] and acc.sum() >= 1
    assert (acc == so.is_accept.astype(bool)).all()
    assert_pp_close(tr.z, zo)
    assert rel_err(F(tr.stat["acceptance_rate"]), so.acceptance_rate) < 1e-9
    assert rel_err(F(tr.stat["hamiltonian_energy"]), so.hamiltonian_energy) < 1e-10
    assert np.allclose(F(tr.stat["hamiltonian_energy_error"]), so.hamiltonian_energy_error, rtol=0, atol=1e-9 * D)
    assert (F(tr.stat["n_steps"]) == L).all() and (F(tr.stat["numerical_error"]) == so.numerical_error).all()


def test_nonfinite_start_is_rejected_and_restored_bit_for_bit():
    D, N = 700, 5
    rng, om, ome, h, th = _problem("diag_gauss", "diag", D, N, 11)
    th[3, 2] = 1e200
    z0 = A.phasepoint(h, T(th), T(np.zeros((D, N))))
    nt = rng.normal(size=(D, N))
    tr = A.transition(A.TapeRNG(normal=T(nt), exp=torch.full((N,), 0.1, dtype=torch.float64, device=DEV)), h, _static(0.1, 6), z0)
    ne, acc = F(tr.stat["numerical_error"]), F(tr.stat["is_accept"])
    assert ne[2] == 1 and acc[2] == 0 and (ne[[0, 1, 3, 4]] == 0).all()
    assert float(tr.z.lp.value[2]) == -np.inf
    assert torch.equal(tr.z.theta[2], z0.theta[2]) and torch.equal(tr.z.lp.gradient[2], z0.lp.gradient[2])
    r0 = A.rand_momentum(A.TapeRNG(normal=T(nt)), h.metric, None, z0.theta)
    assert torch.equal(tr.z.r[2], -r0[2])


def test_no_refresh_accepted_transition_is_the_flipped_step():
    D, N, L = 900, 6, 7
    rng, om, ome, h, th = _problem("diag_gauss", "diag_perchain", D, N, 4)
    z0 = A.phasepoint(h, T(th), T(rng.normal(size=(D, N))))
    tau = A.Trajectory(A.EndPointTS, A.Leapfrog(0.01), A.FixedNSteps(L))
    tr = A.transition(A.TapeRNG(exp=torch.full((N,), 50.0, dtype=torch.float64, device=DEV)), h, tau, z0)  # bare Trajectory: no refresh
    assert (tr.stat["is_accept"] == 1).all()
    z1 = A.step(A.Leapfrog(0.01), h, z0, L)
    assert torch.equal(tr.z.theta, z1.theta) and torch.equal(tr.z.r, -z1.r) and torch.equal(tr.z.lp.gradient, z1.lp.gradient)
    assert torch.equal(tr.z.lp.value, z1.lp.value) and torch.equal(tr.z.lk.value, z1.lk.value)


def _transition_into(h, z_in, z_out, eps, L, rng):
    """ahmc_hmc_transition_f64 with caller-chosen output buffers (z_out may be z_in)"""
    ctx = A.get_context(0)
    N, D = z_in._nd()
    md, keep = h.metric._desc(D, N, z_in.theta)
    e, ep, keep2 = K._eps_args(eps, z_in.theta, N)
    rc, keep3 = rng._c()
    st, sc = K._stats_buffers(z_in.theta, N, False)
    zc, oc_ = z_in._c(False), z_out._c(False)
    torch.cuda.synchronize()
    ctx.check(ctx.lib.ahmc_hmc_transition_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, e, ep, L, C.byref(rc), C.byref(zc),
                                              C.byref(oc_), C.byref(sc), 0))
    torch.cuda.synchronize()
    return st


@pytest.mark.parametrize("model", ["diag_gauss", "funnel"])
def test_in_place_and_host_buffers_equal_the_device_transition(model):
    D, N, L = 1030, 9, 8
    eps = 0.1 if model == "diag_gauss" else 0.02
    rng, om, ome, h, th = _problem(model, "diag", D, N, 6, scale=0.3 if model == "funnel" else 1.0)
    z0 = A.phasepoint(h, T(th), T(np.zeros((D, N))))
    ref = A.transition(A.PhiloxRNG(17), h, _static(eps, L), z0)
    zi = A.PhasePoint(z0.theta.clone(), z0.r.clone(), A.DualValue(z0.lp.value.clone(), z0.lp.gradient.clone()),
                      A.DualValue(z0.lk.value.clone(), None))
    st = _transition_into(h, zi, zi, eps, L, A.PhiloxRNG(17))
    assert _pp_equal(zi, ref.z) and torch.equal(st["is_accept"], ref.stat["is_accept"])
    zh0 = A.phasepoint(h, np.ascontiguousarray(th.T), np.zeros((N, D)))
    trh = A.transition(A.PhiloxRNG(17), h, _static(eps, L), zh0)
    assert np.array_equal(trh.z.theta, ref.z.theta.cpu().numpy()) and np.array_equal(trh.z.r, ref.z.r.cpu().numpy())
    assert np.array_equal(trh.z.lp.value, ref.z.lp.value.cpu().numpy())
    assert np.array_equal(trh.stat["acceptance_rate"], ref.stat["acceptance_rate"].cpu().numpy())


@pytest.mark.parametrize("partial", [0.0, 0.5])
def test_persistent_launch_equals_single_transitions(partial):
    D, N, Tn = 800, 10, 4
    rng, om, ome, h, th = _problem("diag_gauss", "diag_perchain", D, N, 8)
    z0 = A.phasepoint(h, T(th), T(np.zeros((D, N))))
    kern = _static(0.2, 6)
    if partial:
        kern = A.HMCKernel(kern.tau, A.PartialMomentumRefreshment(partial))
    zl, draws, st = A.sample_transitions(A.PhiloxRNG(23), h, kern, z0, Tn)
    prng, z = A.PhiloxRNG(23), z0
    for t in range(Tn):
        tr = A.transition(prng, h, kern, z)
        z = tr.z
        assert torch.equal(draws[t], z.theta), t
        for k in ("is_accept", "acceptance_rate", "hamiltonian_energy", "numerical_error", "n_steps"):
            assert torch.equal(st[k][t], tr.stat[k]), (t, k)
    assert _pp_equal(zl, z)
    assert st["is_accept"].any()


def test_adapt_sample_without_adaptation_is_sample_transitions():
    D, N, Tn = 640, 13, 6
    rng, om, ome, h, th = _problem("funnel", "diag", D, N, 9, scale=0.3)
    z0 = A.phasepoint(h, T(th), T(np.zeros((D, N))))
    kern = _static(0.02, 5)
    zl2, dr2, st2 = A.sample_transitions(A.PhiloxRNG(3), h, kern, z0, Tn)
    for est in ("welford", "nutpie"):
        zl, dr, st, eps, minv, tr = A.hmc_adapt_sample(A.PhiloxRNG(3), h, kern, z0, Tn, 0, A.VectorisedStanAdaptor(metric_estimator=est),
                                                        keep_eps_trace=True)
        assert torch.equal(dr, dr2) and _pp_equal(zl, zl2)
        for k in ("n_steps", "is_accept", "acceptance_rate", "log_density", "hamiltonian_energy", "hamiltonian_energy_error",
                  "numerical_error"):
            assert torch.equal(st[k], st2[k]), k
        assert torch.equal(eps, torch.full_like(eps, 0.02)) and torch.equal(tr, torch.full_like(tr, 0.02))
        assert np.array_equal(minv.cpu().numpy(), np.broadcast_to(h.metric.Minv, (N, D)))


@pytest.mark.parametrize("est", ["welford", "nutpie"])
def test_adaptation_beyond_512_equals_iteration_by_iteration_replay(est):
    _replay("hmc", est, "diag", D=600, N=22)


def test_both_estimators_recover_the_target_variances_at_1024_dimensions():
    """DiagGaussian with scales log-spaced over 0.1..10, D = 1024, 1024 chains, 1000 warm-up iterations (Stan windows): the
    median over chains of M^-1 / s^2 within 10 % for every coordinate"""
    D, N, Tn, n_adapts = 1024, 1024, 1000, 1000
    s = np.exp(np.linspace(np.log(0.1), np.log(10.0), D))
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), A.DiagGaussian(np.zeros(D), s))
    th0 = torch.as_tensor(np.random.default_rng(8).normal(size=(N, D)) * s, device=DEV)
    z0 = A.phasepoint(h, th0, torch.zeros_like(th0))
    for est in ("welford", "nutpie"):
        kern = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.01), A.FixedNSteps(32)))
        zl, _, st, eps, minv, _ = A.hmc_adapt_sample(A.PhiloxRNG(12), h, kern, z0, Tn, n_adapts,
                                                     A.VectorisedStanAdaptor(metric_estimator=est), keep_draws=False)
        med = np.median(minv.cpu().numpy() / s ** 2, axis=0)
        print(f"{est}: median ratio {med.min():.3f}..{med.max():.3f}")
        assert 0.9 < med.min() and med.max() < 1.1, (est, med.min(), med.max())


def test_find_good_stepsize_batched_equals_the_scalar_search_beyond_512():
    D, N = 700, 6
    rng, om, ome, h, th = _problem("diag_gauss", "diag", D, N, 14)
    xi = rng.normal(size=(N, D))
    eps_b = A.find_good_stepsize_batched(A.TapeRNG(normal=torch.as_tensor(xi, device=DEV)), h, T(th))
    for c in range(N):
        e1 = A.find_good_stepsize(A.TapeRNG(normal=torch.as_tensor(xi[c:c + 1], device=DEV)), h, torch.as_tensor(th[:, c], device=DEV))
        assert float(eps_b[c]) == e1, c
    # the search restated on the oracle's leapfrog for chain 0 (test_find_good_stepsize_matches_reference_logic)
    z = oc.phasepoint(om, ome, th[:, :1], A.rand_momentum(A.TapeRNG(normal=torch.as_tensor(xi[:1], device=DEV)), h.metric, None,
                                                          torch.as_tensor(th[:, :1].T.copy(), device=DEV)).cpu().numpy().T)
    H = z.energy()[0]
    Af = lambda e: oc.leapfrog(om, ome, e, z, 1)[0].energy()[0]
    e = ep = 0.1
    too_high = (H - Af(e)) > np.log(0.5)
    for _ in range(100):
        ep = 2 * e if too_high else 0.5 * e
        if too_high != ((H - Af(e)) > np.log(0.5)):
            break
        e = ep
    e, ep = min(e, ep), max(e, ep)
    for _ in range(100):
        mid = 0.5 * (e + ep)
        dH = H - Af(mid)
        if dH > np.log(0.75):
            e = mid
        elif dH < 2 * np.log(0.5):
            ep = mid
        else:
            e = mid
            break
    assert float(eps_b[0]) == pytest.approx(e, rel=1e-12)
    eps_p = A.find_good_stepsize_batched(A.PhiloxRNG(4), h, T(th))  # Philox momentum: finite, positive
    assert torch.isfinite(eps_p).all() and (eps_p > 0).all()


def test_hmcda_host_loop_and_pooled_device_adaptor_run_beyond_512():
    from ahmc_b200 import adaptation as AD

    D, N = 600, 64
    s = np.exp(np.linspace(np.log(0.5), np.log(2.0), D))
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), A.DiagGaussian(np.zeros(D), s))
    th = torch.as_tensor(np.random.default_rng(3).normal(size=(N, D)) * s, device=DEV)
    hmcda = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.1), A.FixedIntegrationTime(1.0)))
    ad = AD.StanHMCAdaptor(AD.WelfordVar(D), AD.NesterovDualAveraging(0.8, 0.1), init_buffer=5, term_buffer=5, window_size=5)
    res = AD.sample(A.PhiloxRNG(1), h, hmcda, th, 40, ad, n_adapts=30)
    assert torch.isfinite(res.theta).all() and res.leapfrog_steps > 0
    assert all(np.isfinite(x["acceptance_rate"]) for x in res.stats)
    resp = AD.sample_pooled_device(A.PhiloxRNG(2), h, _static(0.1, 8), th, 30, 20, eps0=0.1, windows=(5, 5, 5))
    assert torch.isfinite(resp.theta).all() and np.isfinite(resp.eps) and np.isfinite(resp.Minv).all()


def test_still_unsupported_beyond_512_dimensions():
    D, N = 600, 4
    h = A.Hamiltonian(A.UnitEuclideanMetric(D), A.StdNormal(D))
    z = A.phasepoint(h, torch.zeros((N, D), dtype=torch.float64, device=DEV), torch.zeros((N, D), dtype=torch.float64, device=DEV))

    def unsupported(fn, word):
        with pytest.raises(A.AhmcError) as e:
            fn()
        assert e.value.code == A._lib.ERR_UNSUPPORTED and word in str(e.value), str(e.value)

    tempered = A.HMCKernel(A.Trajectory(A.EndPointTS, A.TemperedLeapfrog(0.1, 1.05), A.FixedNSteps(4)))
    unsupported(lambda: A.transition(A.PhiloxRNG(1), h, tempered, z), "TemperedLeapfrog")
    for kern in (A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.1), A.GeneralisedNoUTurn())),
                 A.HMCKernel(A.Trajectory(A.SliceTS, A.Leapfrog(0.1), A.ClassicNoUTurn()))):
        unsupported(lambda: A.transition(A.PhiloxRNG(1), h, kern, z), "register-resident")
    unsupported(lambda: A.transition(A.TapeRNG(n_fwd=2), h, A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.1), A.FixedNSteps(4))), z),
                "register-resident")
    unsupported(lambda: A.step(A.Leapfrog(0.1), h, z, 3, full_trajectory=True), "register-resident")
    hd = A.Hamiltonian(A.DenseEuclideanMetric(np.eye(D)), A.StdNormal(D))
    unsupported(lambda: A.transition(A.PhiloxRNG(1), hd, _static(0.1, 4), z), "register-resident")
    unsupported(lambda: A.rand_momentum(A.PhiloxRNG(1), hd.metric, None, z.theta), "register-resident")
    hg = A.Hamiltonian(A.UnitEuclideanMetric(D), A.DenseGaussian(np.zeros(D), np.eye(D)))
    unsupported(lambda: A.sample_transitions(A.PhiloxRNG(1), hg, _static(0.1, 4), z, 2), "register-resident")
    user = "__device__ double ahmc_user_logp_grad(const double* th, double* g, int D, const double* p) { return 0.0; }"
    hu = A.Hamiltonian(A.UnitEuclideanMetric(D), A.UserTarget(D, user))
    unsupported(lambda: A.transition(A.PhiloxRNG(1), hu, _static(0.1, 4), z), "register-resident")
    hc = A.Hamiltonian(A.UnitEuclideanMetric(D), A.CallbackTarget(D, lambda th: (torch.zeros(th.shape[0], dtype=th.dtype, device=th.device),
                                                                                 torch.zeros_like(th))))
    unsupported(lambda: A.transition(A.PhiloxRNG(1), hc, _static(0.1, 4), z), "register-resident")
