"""The shape tables of tests/test_tensor_pipe_shapes_cpu.py on the GPU (run with -m gpu on an H100), through the public API:
K4 (`A.step` with GEMM-shaped operators), K6 (`A.GLMTarget` on the tile lane) and the cooperative NUTS form
(`A.transition` / `A.sample_transitions` with a dense target or a Dense metric) against the C oracle or tests/glm_ref.py at
1e-10, plus the limits the CPU sweep cannot reach: K4 at D = 512 with 4096 chains (its launch uses all but a few hundred
bytes of a block's shared memory), K6 at D = 256 with 1000 and 5 rows, and COOP launches of 4099 chains with several
transitions each."""
import numpy as np
import pytest
import torch

import ahmc_b200 as A
from oracle import oracle_c as oc
from tests import glm_ref as R
from tests.helpers import METRIC_KINDS, MODEL_KINDS, rel_err
from tests.test_glm import _close, _metric, _problem, _z
from tests.test_gpu_parity import DEV, F, T, TOL, _nuts_case, make_metric, make_target
from tests.test_tensor_pipe_shapes_cpu import COOP_D, K4_CASES, K6_CASES, SAMPLERS

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------- K4
def _k4(model, metric, D, N, seed, steps=(3, -2), exact_chain=None):
    rng = np.random.default_rng(seed)
    p0 = p1 = Minv = None
    if model == "diag_gauss":
        p0, p1 = rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))
    elif model == "dense_gauss":
        B = rng.normal(size=(D, D))
        p0, p1 = rng.normal(size=D), B @ B.T / D + np.eye(D)
    if metric == "diag":
        Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    elif metric == "dense":
        B = rng.normal(size=(D, D))
        Minv = B @ B.T / D + 0.5 * np.eye(D)
    th, r = rng.normal(size=(D, N)), rng.normal(size=(D, N))
    if exact_chain is not None:
        th[0, exact_chain] = 1e250  # energy overflow at step 1: that chain freezes, its tile goes to the exact kernel
    eps = 0.05 * np.exp(rng.uniform(-0.3, 0.3, N))
    om, ome = oc.Model(MODEL_KINDS[model], D, p0, p1, 0.3), oc.Metric(METRIC_KINDS[metric], Minv)
    z0o = oc.phasepoint(om, ome, th, r)
    h = A.Hamiltonian(make_metric(metric, Minv, D), make_target(model, D, p0, p1, 0.3))
    z0 = A.phasepoint(h, T(th), T(r))
    lf = A.Leapfrog(torch.as_tensor(eps, device=DEV))
    ok = np.array([c != exact_chain for c in range(N)])
    for n in steps:
        zo, st_o, dn_o = oc.leapfrog(om, ome, eps, z0o, n)
        z1, info = A.step(lf, h, z0, n, return_info=True)
        assert (F(info.steps_done) == dn_o).all() and (F(info.status) == st_o).all()
        for f, got in [("theta", z1.theta), ("r", z1.r), ("lp_gradient", z1.lp.gradient), ("lk_gradient", z1.lk.gradient)]:
            assert rel_err(F(got)[:, ok], getattr(zo, f)[:, ok]) < TOL, (f, n)
        assert rel_err(F(z1.lp.value)[ok], zo.lp_value[ok]) < TOL and rel_err(F(z1.lk.value)[ok], zo.lk_value[ok]) < TOL
    # the tile path and the exact path agree to rounding
    ze = A.step(lf, h, z0, steps[0], flags=A.FLAG_EXACT_CHECKS)
    z1 = A.step(lf, h, z0, steps[0])
    assert rel_err(F(z1.theta)[:, ok], F(ze.theta)[:, ok]) < 1e-12


@pytest.mark.parametrize("model,metric,D", [c[:3] for c in K4_CASES], ids=[f"{c[0]}-{c[1]}-D{c[2]}" for c in K4_CASES])
def test_dense_tile_kernel_shapes_vs_oracle(model, metric, D):
    N = 333 if D <= 256 else 77  # ragged last tile for 32-, 16- and 8-chain tiles
    _k4(model, metric, D, N, seed=D * 5 + 1, exact_chain=N // 2 if D in (65, 193, 321) else None)


def test_dense_tile_kernel_at_the_shared_memory_limit():
    """D = 512 (RB = 8): the launch asks for 232,240 of the 232,448 bytes a block may have; 4096 chains, 512 tiles"""
    _k4("dense_gauss", "dense", 512, 4096, seed=512, steps=(2,))


# ------------------------------------------------------------------------------------------------------------------- K6
def _k6(family, D, n, N, metric, seed):
    X, y, prec, Minv, th, r, rng = _problem(family, D, n, N, metric, seed=seed)
    tgt = A.GLMTarget(X, y, family, prior_prec=prec, c0=0.5)
    h = A.Hamiltonian(_metric(metric, Minv, D), tgt)
    tht, rt = torch.as_tensor(th, device=DEV), torch.as_tensor(r, device=DEV)
    ctx = A.get_context(0)
    l0 = ctx.launches
    z = A.phasepoint(h, tht, rt)
    assert ctx.launches - l0 == 1  # the tile kernel
    z0 = R.phasepoint(family, X, y, prec, 0.5, Minv, th, r)
    _close(_z(z), z0)
    eps = 0.01 * np.exp(rng.uniform(-0.3, 0.3, N))
    lf = A.Leapfrog(torch.as_tensor(eps, device=DEV))
    for steps in (3, -2):
        z1, info = A.step(lf, h, z, steps, return_info=True)
        ref, st, done = R.leapfrog(family, X, y, prec, 0.5, Minv, eps, z0, steps)
        _close(_z(z1), ref)
        assert rel_err(z1.lk.gradient.cpu().numpy(), ref["dr"]) < 1e-10
        assert (F(info.steps_done) == done).all() and (F(info.status) == st).all()
    # without a cached gradient
    z1n = A.step(lf, h, A.PhasePoint(z.theta, z.r, A.DualValue(None, None), A.DualValue(None, None)), 3)
    _close(_z(z1n), R.leapfrog(family, X, y, prec, 0.5, Minv, eps, z0, 3)[0])


@pytest.mark.parametrize("family,D,n,metric", [(c[0], c[1], c[2], c[4]) for c in K6_CASES],
                         ids=[f"{c[0]}-D{c[1]}-n{c[2]}-{c[4]}" for c in K6_CASES])
def test_glm_tile_kernel_shapes_vs_reference(family, D, n, metric):
    _k6(family, D, n, 37, metric, seed=D * 3 + n)


@pytest.mark.parametrize("family", ["bernoulli_logit", "poisson_log"])
@pytest.mark.parametrize("n", [1000, 5])
def test_glm_tile_kernel_at_d256(family, n):
    """32-row chunks (D = 256): many more chunks than stages, and fewer"""
    _k6(family, 256, n, 333, "chain", seed=n)


# ------------------------------------------------------------------------------------------------------------ COOP NUTS
def _nuts_vs_oracle(model, metric, D, N, max_depth, sampler="multinomial", criterion="generalised"):
    eps = 0.3 if D < 100 else 0.25
    tr, zo, so = _nuts_case(model, metric, D, N, eps, seed=D * 11 + N, max_depth=max_depth, sampler=sampler, criterion=criterion)
    st = tr.stat
    assert (F(st["tree_depth"]) == so.tree_depth).all() and (F(st["n_steps"]) == so.n_steps).all()
    assert (F(st["numerical_error"]) == so.numerical_error).all()
    for f, got in [("theta", tr.z.theta), ("r", tr.z.r), ("lp_gradient", tr.z.lp.gradient)]:
        assert rel_err(F(got), getattr(zo, f)) < TOL, f
    assert rel_err(F(tr.z.lp.value), zo.lp_value) < TOL and rel_err(F(tr.z.lk.value), zo.lk_value) < TOL
    assert rel_err(F(st["acceptance_rate"]), so.acceptance_rate) < 1e-9
    assert so.n_steps.max() >= 3


@pytest.mark.parametrize("D", COOP_D)
@pytest.mark.parametrize("N", [1, 7, 9])
def test_cooperative_nuts_shapes_vs_oracle(D, N):
    _nuts_vs_oracle("dense_gauss", "dense", D, N, 4 if D <= 256 else 3)


@pytest.mark.parametrize("model,metric,D", [("dense_gauss", "unit", 25), ("dense_gauss", "diag", 100), ("dense_gauss", "unit", 300),
                                            ("diag_gauss", "dense", 65), ("diag_gauss", "dense", 129), ("funnel", "dense", 24)])
def test_cooperative_nuts_target_metric_combinations_vs_oracle(model, metric, D):
    _nuts_vs_oracle(model, metric, D, 9, 4)


@pytest.mark.parametrize("D", [33, 129])
@pytest.mark.parametrize("sampler,criterion", SAMPLERS, ids=[f"{s}-{c}" for s, c in SAMPLERS])
def test_every_sampler_and_criterion_at_cooperative_shapes_vs_oracle(D, sampler, criterion):
    _nuts_vs_oracle("dense_gauss", "dense", D, 7, 4, sampler, criterion)


@pytest.mark.parametrize("D", [24, 100])
def test_cooperative_nuts_4099_chains_vs_oracle(D):
    _nuts_vs_oracle("dense_gauss", "dense", D, 4099, 5)


@pytest.mark.parametrize("D", [24, 100, 300, 512])
def test_cooperative_nuts_several_transitions_per_launch_equal_single_transitions(D):
    """4099 chains (a ragged last block of 3), 3 transitions in one launch: every product of every transition re-arms the
    block's pipeline; the draws, statistics and end state equal those of 3 single-transition launches bit for bit"""
    N, Tn = 4099, 3
    rng = np.random.default_rng(D)
    B = rng.normal(size=(D, D))
    P = B @ B.T / D + np.eye(D)
    B = rng.normal(size=(D, D))
    Minv = B @ B.T / D + 0.5 * np.eye(D)
    h = A.Hamiltonian(A.DenseEuclideanMetric(Minv), A.DenseGaussian(rng.normal(size=D), P, 0.0))
    th = torch.as_tensor(rng.normal(size=(N, D)), device=DEV)
    z0 = A.phasepoint(h, th, torch.zeros_like(th))
    kern = A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.25), A.GeneralisedNoUTurn(5, 1000.0)))
    zl, draws, st = A.sample_transitions(A.PhiloxRNG(7), h, kern, z0, Tn)
    rng_t = A.PhiloxRNG(7)
    z = z0
    for t in range(Tn):
        tr = A.transition(rng_t, h, kern, z)
        z = tr.z
        assert torch.equal(draws[t], z.theta), t
        for k in ("n_steps", "tree_depth", "acceptance_rate", "numerical_error"):
            assert torch.equal(st[k][t], tr.stat[k]), (k, t)
    assert torch.equal(zl.theta, z.theta) and torch.equal(zl.lp.gradient, z.lp.gradient)
    assert torch.isfinite(draws).all() and st["n_steps"].max().item() >= 3
