"""Per-chain warm-up inside one launch beyond the WelfordVar + built-in NUTS case: NutpieVar (positions and gradients),
the adaptive static-HMC launch (ahmc_hmc_adapt_sample_f64) and run-time compiled (NVRTC) targets.  Each fused run is
replayed iteration by iteration -- one transition launch per iteration on the same Philox stream, with the step size and
metric the fused launch reported -- while the ORACLE's vectorised adaptors (oracle/oracle_c.py: DualAveraging, WelfordVar
((D, N)); NutpieVar = two WelfordVar((D, N)) of positions and gradients) run alongside on the replay's acceptance rates
and draws, and must reproduce the fused launch's step size at every iteration, its M^-1 at every window end and its
final step size."""
import ctypes as C

import numpy as np
import pytest
import torch

import ahmc_b200 as A
from ahmc_b200 import core as K
from tests.helpers import rel_err
from tests.test_gpu_parity import USER_DIAG, USER_FUNNEL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _target(kind, D, rng):
    if kind == "diag":
        mu, sd = rng.normal(size=D), np.exp(rng.uniform(-0.8, 0.8, D))
        return A.DiagGaussian(mu, sd), sd
    if kind == "user_diag":
        mu, sd = rng.normal(size=D), np.exp(rng.uniform(-0.8, 0.8, D))
        return A.UserTarget(D, USER_DIAG, params=np.stack([mu, 1.0 / sd ** 2], axis=1)), sd
    return A.UserTarget(D, USER_FUNNEL), None


def _kernel(sampler, eps):
    if sampler == "nuts":
        return A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(eps), A.GeneralisedNoUTurn(8, 1000.0)))
    return A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(eps), A.FixedNSteps(12)))


class _OracleMetric:
    """the oracle's WelfordVar((D, N)), or NutpieVar((D, N)) composed of two of them (massmatrix.jl:172-250)"""

    def __init__(self, est, D, N):
        from oracle import oracle_c as oc

        self.est, self.wt = est, oc.WelfordVar((D, N))
        self.wg = oc.WelfordVar((D, N)) if est == "nutpie" else None

    def push(self, z):
        self.wt.push(z.theta.cpu().numpy().T)
        if self.wg is not None:
            self.wg.push(z.lp.gradient.cpu().numpy().T)  # MINUS grad log pi: same variance

    @property
    def n(self):
        return self.wt.n.value

    def estimate(self):
        e = self.wt.estimate()
        if self.wg is not None:
            e = np.sqrt(e / self.wg.estimate())
        return np.ascontiguousarray(e.T)


def _replay(sampler, est, kind, D=8, N=96, T=60, n_adapts=50, seed=21):
    from oracle import oracle_c as oc

    ib, tb, wsz = 10, 8, 6
    ws, we, splits = oc.stan_windows(n_adapts, ib, tb, wsz)
    assert (ws, we, list(splits)) == (11, 42, [16, 42])  # the first window holds 6 < n_min draws: reset without an update
    rng = np.random.default_rng(seed)
    target, sd = _target(kind, D, rng)
    th0 = torch.as_tensor(rng.normal(size=(N, D)) * (0.4 if kind == "user_funnel" else 1.0), device=DEV)
    eps0 = 0.3 if sampler == "nuts" else 0.1
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), target)
    z0 = A.phasepoint(h, th0, torch.zeros_like(th0))
    adaptor = A.VectorisedStanAdaptor(delta=0.8, init_buffer=ib, term_buffer=tb, window_size=wsz, metric_estimator=est)
    run = A.nuts_adapt_sample if sampler == "nuts" else A.hmc_adapt_sample
    zl, draws, st, eps_f, minv_f, trace = run(A.PhiloxRNG(seed), h, _kernel(sampler, eps0), z0, T, n_adapts, adaptor,
                                              keep_eps_trace=True)

    prng = A.PhiloxRNG(seed)
    da, pc = oc.DualAveraging(np.full(N, eps0), delta=0.8), _OracleMetric(est, D, N)
    Minv_dev = torch.ones((N, D), dtype=torch.float64, device=DEV)
    z, updates = z0, 0
    for i in range(1, T + 1):
        assert np.allclose(trace[i - 1].cpu().numpy(), da.eps, rtol=1e-9, atol=0), i
        hi = A.Hamiltonian(A.DiagEuclideanMetric(Minv_dev), target)
        tr = A.transition(prng, hi, _kernel(sampler, trace[i - 1].clone()), z)
        z = tr.z
        assert rel_err(draws[i - 1].cpu().numpy(), z.theta.cpu().numpy()) < 1e-10, i
        assert torch.equal(st["n_steps"][i - 1].cpu(), tr.stat["n_steps"].cpu()), i
        if sampler == "nuts":
            assert torch.equal(st["tree_depth"][i - 1].cpu(), tr.stat["tree_depth"].cpu()), i
        else:
            assert torch.equal(st["is_accept"][i - 1].cpu(), tr.stat["is_accept"].cpu()), i
        assert np.allclose(st["acceptance_rate"][i - 1].cpu().numpy(), tr.stat["acceptance_rate"].cpu().numpy(), rtol=1e-10), i
        if i <= n_adapts:
            da.adapt(tr.stat["acceptance_rate"].cpu().numpy())
            if ws <= i <= we:
                pc.push(z)
                if i in splits and pc.n >= 10:
                    assert np.allclose(minv_f.cpu().numpy(), pc.estimate(), rtol=1e-9, atol=0), i
                    Minv_dev = minv_f.clone()
                    updates += 1
            if i in splits:
                da.reset()
                pc = _OracleMetric(est, D, N)
            if i == n_adapts:
                da.finalize()
    assert updates == 1 and not torch.allclose(Minv_dev, torch.ones_like(Minv_dev))
    assert np.allclose(eps_f.cpu().numpy(), da.eps, rtol=1e-9, atol=0)
    assert rel_err(zl.theta.cpu().numpy(), z.theta.cpu().numpy()) < 1e-10
    return h, z0, adaptor, (zl, draws, st, eps_f, minv_f, trace)


@pytest.mark.parametrize("sampler,est", [("nuts", "nutpie"), ("hmc", "welford"), ("hmc", "nutpie")])
def test_fused_adaptation_equals_iteration_by_iteration_replay_with_oracle_adaptors(sampler, est):
    _replay(sampler, est, "diag")


@pytest.mark.parametrize("sampler,est,kind", [("nuts", "welford", "user_diag"), ("nuts", "nutpie", "user_funnel"),
                                              ("hmc", "welford", "user_funnel"), ("hmc", "nutpie", "user_diag")])
def test_run_time_compiled_targets_adapt_in_launch_and_host_buffers_match(sampler, est, kind):
    """the adaptive NUTS / static-HMC kernels compiled (NVRTC) with a user target, replayed like the built-in ones; the same
    run from host (numpy) buffers is bit-identical to the device-buffer run"""
    h, z0, adaptor, (zl, draws, st, eps_f, minv_f, _) = _replay(sampler, est, kind, seed=33)
    run = A.nuts_adapt_sample if sampler == "nuts" else A.hmc_adapt_sample
    zh0 = A.phasepoint(h, z0.theta.cpu().numpy(), np.zeros(tuple(z0.theta.shape)))
    zh, dh, sh, eh, mh, _ = run(A.PhiloxRNG(33), h, _kernel(sampler, 0.3 if sampler == "nuts" else 0.1), zh0, 60, 50, adaptor)
    assert np.array_equal(dh, draws.cpu().numpy()) and np.array_equal(eh, eps_f.cpu().numpy())
    assert np.array_equal(mh, minv_f.cpu().numpy()) and np.array_equal(zh.theta, zl.theta.cpu().numpy())


@pytest.mark.parametrize("variant", ["leapfrog", "partial+tempered"])
def test_static_hmc_without_adaptation_is_the_plain_persistent_launch(variant):
    """n_adapts = 0: draws, statistics and the final phase point equal ahmc_hmc_sample_f64's bit for bit"""
    D, N, T = 13, 130, 9
    rng = np.random.default_rng(5)
    Minv = np.exp(rng.uniform(-0.3, 0.3, D))
    h = A.Hamiltonian(A.DiagEuclideanMetric(Minv),
                      A.DiagGaussian(rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))))
    lf = A.Leapfrog(0.15) if variant == "leapfrog" else A.TemperedLeapfrog(0.15, 1.05)
    kern = A.HMCKernel(A.Trajectory(A.EndPointTS, lf, A.FixedNSteps(10)))
    if variant != "leapfrog":
        kern = A.HMCKernel(kern.tau, A.PartialMomentumRefreshment(0.4))
    th = torch.as_tensor(rng.normal(size=(N, D)), device=DEV)
    z0 = A.phasepoint(h, th, torch.zeros_like(th))
    for est in ("welford", "nutpie"):
        zl, dr, st, eps, minv, tr = A.hmc_adapt_sample(A.PhiloxRNG(3), h, kern, z0, T, 0,
                                                        A.VectorisedStanAdaptor(metric_estimator=est), keep_eps_trace=True)
        zl2, dr2, st2 = A.sample_transitions(A.PhiloxRNG(3), h, kern, z0, T)
        assert torch.equal(dr, dr2)
        for a, b in ((zl.theta, zl2.theta), (zl.r, zl2.r), (zl.lp.value, zl2.lp.value), (zl.lp.gradient, zl2.lp.gradient),
                     (zl.lk.value, zl2.lk.value)):
            assert torch.equal(a, b)
        for k in ("n_steps", "is_accept", "acceptance_rate", "log_density", "hamiltonian_energy", "hamiltonian_energy_error",
                  "numerical_error"):
            assert torch.equal(st[k], st2[k]), k
        assert torch.equal(eps, torch.full_like(eps, 0.15)) and torch.equal(tr, torch.full_like(tr, 0.15))
        assert np.array_equal(minv.cpu().numpy(), np.broadcast_to(Minv, (N, D)))


@pytest.mark.parametrize("sampler", ["nuts", "hmc"])
def test_both_estimators_recover_the_target_variances_on_c3(sampler):
    """DiagGaussian with scales log-spaced over 0.1..10, D = 128, 4096 chains, 1000 warm-up iterations (Stan windows):
    for a Gaussian both NutpieVar's sqrt(var theta / var grad) and WelfordVar's var theta estimate s^2 per chain.
    Tolerances: the median over chains of M^-1 / s^2 within 10 % for every coordinate, and 95 % of all (chain, coordinate)
    ratios within a factor 1.5 (WelfordVar: the last window's ~500 correlated draws per chain) or 1.1 (NutpieVar: exact for
    a Gaussian up to the regulariser and the window's finite sample).  Dual averaging brings the mean acceptance rate within
    0.05 of delta = 0.8 over the second half of the last slow window (iterations 701..950, the DA state converged and not
    reset); after finalize! the sampling iterations run with exp(x_bar), a smaller step than the last iterates, and accept
    more (0.75..0.95)."""
    D, N, T, n_adapts = 128, 4096, 1100, 1000
    s = np.exp(np.linspace(np.log(0.1), np.log(10.0), D))
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), A.DiagGaussian(np.zeros(D), s))
    th0 = torch.as_tensor(np.random.default_rng(8).normal(size=(N, D)) * s, device=DEV)
    z0 = A.phasepoint(h, th0, torch.zeros_like(th0))
    run = A.nuts_adapt_sample if sampler == "nuts" else A.hmc_adapt_sample
    for est, band in (("welford", 1.5), ("nutpie", 1.1)):
        kern = _kernel(sampler, 0.05) if sampler == "nuts" else A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.01), A.FixedNSteps(32)))
        zl, _, st, eps, minv, _ = run(A.PhiloxRNG(12), h, kern, z0, T, n_adapts, A.VectorisedStanAdaptor(metric_estimator=est),
                                      keep_draws=False)
        ratio = minv.cpu().numpy() / s ** 2
        med = np.median(ratio, axis=0)
        within = np.mean((ratio > 1 / band) & (ratio < band))
        acc = st["acceptance_rate"][700:950].double().mean().item()
        acc_s = st["acceptance_rate"][n_adapts:].double().mean().item()
        print(f"{sampler} {est}: median ratio {med.min():.3f}..{med.max():.3f}, within x{band}: {within:.4f}, "
              f"acc warm-up {acc:.4f} sampling {acc_s:.4f}")
        assert 0.9 < med.min() and med.max() < 1.1, (est, med.min(), med.max())
        assert within > 0.95, (est, within)
        assert abs(acc - 0.8) < 0.05, (est, acc)
        assert 0.75 < acc_s < 0.95, (est, acc_s)


def test_invalid_requests_fail_loudly(monkeypatch):
    D, N = 6, 40
    rng = np.random.default_rng(2)
    target = A.DiagGaussian(rng.normal(size=D), np.ones(D))
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), target)
    th = torch.as_tensor(rng.normal(size=(N, D)), device=DEV)
    z0 = A.phasepoint(h, th, torch.zeros_like(th))
    kh, kn = _kernel("hmc", 0.1), _kernel("nuts", 0.2)
    ad = A.VectorisedStanAdaptor(init_buffer=2, term_buffer=2, window_size=3)
    # adapt_metric outside {0, 1, 2}
    monkeypatch.setitem(K._ESTIMATORS, "bogus", 3)
    for run, k in ((A.hmc_adapt_sample, kh), (A.nuts_adapt_sample, kn)):
        with pytest.raises(A.InvalidArgument):
            run(A.PhiloxRNG(1), h, k, z0, 8, 6, A.VectorisedStanAdaptor(metric_estimator="bogus"))
    # random tapes instead of the Philox streams: refused by the Python mirror, and by the C entry points themselves (what
    # the Julia shim relies on), each tape on its own
    with pytest.raises(A.InvalidArgument):
        A.hmc_adapt_sample(A.TapeRNG(normal=torch.zeros_like(th)), h, kh, z0, 8, 6, ad)
    ctx = A.get_context(0)
    tape = torch.zeros((N, 64), dtype=torch.float64, device=DEV)
    dirs = torch.zeros((N, 64), dtype=torch.uint8, device=DEV)
    for field, ptr, stride in (("normal_tape", tape.data_ptr(), None), ("exp_tape", tape.data_ptr(), "exp_stride"),
                               ("dir_tape", dirs.data_ptr(), "dir_stride")):
        for sampler in ("hmc", "nuts"):
            kern = kh if sampler == "hmc" else kn
            _, _, _, out, md, keep, eps, minv, trace, cfg, rc, draws = K._adapt_launch_args(h, kern, z0, 8, 6, ad, False, False,
                                                                                             A.PhiloxRNG(1))
            setattr(rc, field, ptr)
            if stride:
                setattr(rc, stride, 64)
            st, sc = K._stats_buffers(z0.theta, N, sampler == "nuts", T=8)
            zc, oc_ = z0._c(False), out._c(False)
            if sampler == "hmc":
                code = ctx.lib.ahmc_hmc_adapt_sample_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, 12, 8, C.byref(cfg),
                                                         C.byref(rc), C.byref(zc), C.byref(oc_), None, C.byref(sc), 0)
            else:
                code = ctx.lib.ahmc_nuts_adapt_sample_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, 8, 1000.0, 8,
                                                          C.byref(cfg), C.byref(rc), C.byref(zc), C.byref(oc_), None,
                                                          C.byref(sc), 0)
            assert code == A._lib.ERR_INVALID, (field, sampler, code)
            assert "Philox" in ctx.lib.ahmc_last_error(ctx.h).decode()
    # Unit metric
    hu = A.Hamiltonian(A.UnitEuclideanMetric(D), target)
    with pytest.raises(A.AhmcError) as e:
        A.hmc_adapt_sample(A.PhiloxRNG(1), hu, kh, A.phasepoint(hu, th, torch.zeros_like(th)), 8, 6, ad)
    assert e.value.code == A._lib.ERR_UNSUPPORTED
    # FixedIntegrationTime (HMCDA)
    kd = A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.1), A.FixedIntegrationTime(1.0)))
    with pytest.raises(A.AhmcError) as e:
        A.hmc_adapt_sample(A.PhiloxRNG(1), h, kd, z0, 8, 6, ad)
    assert e.value.code == A._lib.ERR_UNSUPPORTED
    # callback (split-step) target
    hc = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), A.CallbackTarget(D, lambda t: (-0.5 * (t * t).sum(dim=1), -t)))
    zc = A.phasepoint(hc, th, torch.zeros_like(th))
    for run, k in ((A.hmc_adapt_sample, kh), (A.nuts_adapt_sample, kn)):
        with pytest.raises(A.AhmcError) as e:
            run(A.PhiloxRNG(1), hc, k, zc, 8, 6, ad)
        assert e.value.code == A._lib.ERR_UNSUPPORTED
    # n_adapts > n_transitions
    with pytest.raises(A.InvalidArgument):
        A.hmc_adapt_sample(A.PhiloxRNG(1), h, kh, z0, 4, 5, ad)
    # user target + SliceTS: still unsupported
    hs = A.Hamiltonian(A.DiagEuclideanMetric(np.ones(D)), A.UserTarget(D, USER_FUNNEL))
    zs = A.phasepoint(hs, th * 0.3, torch.zeros_like(th))
    ks = A.HMCKernel(A.Trajectory(A.SliceTS, A.Leapfrog(0.1), A.GeneralisedNoUTurn()))
    with pytest.raises(A.AhmcError) as e:
        A.sample_transitions(A.PhiloxRNG(1), hs, ks, zs, 3)
    assert e.value.code == A._lib.ERR_UNSUPPORTED
    with pytest.raises(A.AhmcError) as e:
        A.nuts_adapt_sample(A.PhiloxRNG(1), hs, ks, zs, 8, 6, ad)
    assert e.value.code == A._lib.ERR_UNSUPPORTED
