"""GPU checks of the on-device Philox streams (run with -m gpu on an H100): `rand_momentum` returns the normals of the host
restatement (tests/philox_ref.py) coordinate by coordinate, and Philox-mode transitions -- static EndPointTS and
MultinomialTS, NUTS in every layout family, multi-transition and in-launch adaptive launches -- equal the CPU oracle run
chain by chain on the tapes the restatement builds for each transition.  A Philox run also equals the same launch fed
those tapes, which separates the variate plumbing from the kernel's arithmetic.  The CPU side is
tests/test_philox_streams_cpu.py."""
import numpy as np
import pytest
import scipy.linalg
import torch

import ahmc_b200 as A
from oracle import oracle_c as oc
from tests import philox_ref as R
from tests.helpers import MODEL_KINDS, rel_err, rel_err_elem_scaled
from tests.test_gpu_parity import DEV, F, T, assert_pp_close, make_target

pytestmark = pytest.mark.gpu
TOL = 1e-10
SEED_HI = 2**32 + 0x5EED  # key word k1 != 0
SEED_BIG = 0xC0FFEE0123456789
OFF_HI = 2**35 + 12345
_SAMPLERS = {"multinomial": "MultinomialTS", "slice": "SliceTS"}
_CRITERIA = {"generalised": "GeneralisedNoUTurn", "classic": "ClassicNoUTurn", "strict": "StrictGeneralisedNoUTurn"}


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _spd(rng, D):
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    return (Q * np.exp(rng.uniform(-0.5, 0.5, D))) @ Q.T


# ---------------------------------------------------------------------------------------------- rand_momentum
@pytest.mark.parametrize("D", R.LAYOUT_DS + [513, 1000, 1537])
def test_rand_momentum_unit_and_diag_equal_the_restated_normals(D):
    N = 37  # ragged: not a multiple of any group count
    rng = np.random.Generator(np.random.PCG64(D))
    th = torch.zeros((N, D), dtype=torch.float64, device=DEV)
    mi = np.exp(rng.uniform(-0.7, 0.7, D))
    for seed, off in [(SEED_HI, 0), (SEED_BIG, 1), (7, OFF_HI)]:
        z = R.normals(seed, off, np.arange(N), D)
        g = A.PhiloxRNG(seed)
        g.offset = off
        r = _np(A.rand_momentum(g, A.UnitEuclideanMetric(D), None, th))
        assert g.offset == off + 1
        assert np.abs(r - z).max() < 1e-13, np.abs(r - z).max()
        r = _np(A.rand_momentum(g, A.DiagEuclideanMetric(mi), None, th))  # the next offset
        want = R.normals(seed, off + 1, np.arange(N), D) / np.sqrt(mi)
        assert np.abs(r - want).max() < 1e-13 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("D", [1, 3, 5, 17, 33, 128, 300, 512])
def test_rand_momentum_dense_shared_and_per_chain_is_the_factor_solve_of_the_restated_normals(D):
    N = 13
    rng = np.random.Generator(np.random.PCG64(100 + D))
    M = _spd(rng, D)
    Ms = np.stack([_spd(rng, D) for _ in range(N)])
    th = torch.zeros((N, D), dtype=torch.float64, device=DEV)
    seed, off = SEED_BIG, OFF_HI + D
    z = R.normals(seed, off, np.arange(N), D)
    for met, mats in [(A.DenseEuclideanMetric(M), [M] * N), (A.DenseEuclideanMetric(torch.as_tensor(Ms, device=DEV)), list(Ms))]:
        g = A.PhiloxRNG(seed)
        g.offset = off
        r = _np(A.rand_momentum(g, met, None, th))
        want = np.stack([scipy.linalg.solve_triangular(np.linalg.cholesky(Mc).T, z[c]) for c, Mc in enumerate(mats)])  # U \ z
        assert rel_err(r, want) < 1e-12, rel_err(r, want)


def test_philox_offsets_past_2_to_the_36_are_refused():
    """the counter holds the transition offset in 36 bits: a launch that would reach offset 2^36 is refused, naming the bound"""
    D, N = 5, 8
    th = torch.zeros((N, D), dtype=torch.float64, device=DEV)
    g = A.PhiloxRNG(1)
    g.offset = 2**36 - 1
    r = _np(A.rand_momentum(g, A.UnitEuclideanMetric(D), None, th))  # the last offset there is
    assert np.abs(r - R.normals(1, 2**36 - 1, np.arange(N), D)).max() < 1e-13
    with pytest.raises(A.InvalidArgument) as e:
        A.rand_momentum(g, A.UnitEuclideanMetric(D), None, th)
    assert "2^36" in str(e.value)
    h = A.Hamiltonian(A.UnitEuclideanMetric(D), A.StdNormal(D, 0.0))
    z0 = A.phasepoint(h, th, torch.zeros_like(th))
    for kern in [A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(0.1), A.FixedNSteps(3))),
                 A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(0.1), A.GeneralisedNoUTurn()))]:
        g = A.PhiloxRNG(1)
        g.offset = 2**36 - 3
        A.sample_transitions(g, h, kern, z0, 3)  # offsets 2^36 - 3 .. 2^36 - 1
        g.offset = 2**36 - 2
        with pytest.raises(A.InvalidArgument) as e:
            A.sample_transitions(g, h, kern, z0, 3)
        assert "2^36" in str(e.value)
        g.offset = 2**36
        with pytest.raises(A.InvalidArgument) as e:
            A.transition(g, h, kern, z0)


# ---------------------------------------------------------------------------------------------- transitions vs the oracle
def _problem(model, metric, D, N, seed, scale=1.0):
    rng = np.random.Generator(np.random.PCG64(seed))
    p0 = p1 = Minv = None
    if model == "diag_gauss":
        p0, p1 = rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))
    elif model == "dense_gauss":
        B = rng.normal(size=(D, D))
        p0, p1 = rng.normal(size=D), B @ B.T / D + np.eye(D)
    if metric == "diag":
        Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    elif metric == "diag_chain":
        Minv = np.exp(rng.uniform(-0.5, 0.5, (D, N)))
    elif metric == "dense":
        B = rng.normal(size=(D, D))
        Minv = B @ B.T / D + 0.5 * np.eye(D)
    elif metric == "dense_chain":
        Minv = np.stack([_spd(rng, D) for _ in range(N)])
    th = rng.normal(size=(D, N)) * scale
    return p0, p1, Minv, th


def _dev_metric(metric, Minv, D):
    if metric == "unit":
        return A.UnitEuclideanMetric(D)
    if metric == "diag":
        return A.DiagEuclideanMetric(Minv)
    if metric == "diag_chain":
        return A.DiagEuclideanMetric(np.ascontiguousarray(Minv.T))
    if metric == "dense":
        return A.DenseEuclideanMetric(Minv)
    return A.DenseEuclideanMetric(torch.as_tensor(Minv, device=DEV))


def _orc_groups(metric, Minv, N):
    """[(oracle metric, chains)]: all chains at once, or chain by chain for a per-chain Dense metric"""
    if metric == "dense_chain":
        return [(oc.Metric(oc.DENSE, Minv[c]), slice(c, c + 1)) for c in range(N)]
    kind = {"unit": oc.UNIT, "diag": oc.DIAG, "diag_chain": oc.DIAG, "dense": oc.DENSE}[metric]
    return [(oc.Metric(kind, Minv), slice(None))]


_STATS = {"hmc": ("is_accept", "acceptance_rate", "numerical_error"),
          "multinomial": ("tree_depth", "acceptance_rate", "numerical_error"),
          "nuts": ("tree_depth", "n_steps", "acceptance_rate", "numerical_error")}


def _tapes(kind, seed, off, N, D, max_depth, sampler):
    tp = dict(normal=R.normal_tape(seed, off, N, D))
    if kind == "hmc":
        tp["exp"] = R.static_exp_tape(seed, off, N)
    elif kind == "multinomial":
        tp["exp"] = R.static_unif_tape(seed, off, N)
    else:
        tp["exp"] = R.nuts_exp_tape(seed, off, N, 1 << max_depth, sampler)
        tp["dirs"] = R.dir_tape(seed, off, N, max_depth + 1)
    return tp


def _oracle(kind, model, metric, D, N, p0, p1, Minv, th, eps, seed, offset, n_tr, L=None, n_fwd=None, max_depth=10,
            sampler="multinomial", criterion="generalised"):
    """the oracle over n_tr transitions on the restated tapes of offsets offset .. offset + n_tr - 1:
    (thetas (n_tr, D, N), stats {name: (n_tr, N)}, last phase point {field: array})"""
    om = oc.Model(MODEL_KINDS[model], D, p0, p1, 0.0)
    tapes = [_tapes(kind, seed, offset + t, N, D, max_depth, sampler) for t in range(n_tr)]
    thetas = np.zeros((n_tr, D, N))
    stats = {k: np.zeros((n_tr, N)) for k in _STATS[kind]}
    last = dict(theta=np.zeros((D, N)), r=np.zeros((D, N)), lp_gradient=np.zeros((D, N)), lp_value=np.zeros(N), lk_value=np.zeros(N))
    for ome, cs in _orc_groups(metric, Minv, N):
        z = oc.phasepoint(om, ome, th[:, cs], np.zeros_like(th[:, cs]))
        for t, tp in enumerate(tapes):
            nt = tp["normal"][:, cs]
            if kind == "hmc":
                z, so = oc.hmc_transition(om, ome, eps, L, z, nt, tp["exp"][cs])
            elif kind == "multinomial":
                z, so = oc.hmc_multinomial_transition(om, ome, eps, L, n_fwd, z, nt, tp["exp"][cs])
            else:
                z, so, used = oc.nuts_transition(om, ome, eps, z, nt, tp["dirs"][cs], tp["exp"][cs], max_depth=max_depth,
                                                 sampler=sampler, criterion=criterion)
                assert (used <= tp["exp"].shape[1]).all()
            thetas[t][:, cs] = z.theta
            for k in stats:
                stats[k][t, cs] = getattr(so, k)
        for f in last:
            last[f][..., cs] = getattr(z, f)
    return thetas, stats, last, tapes


def _kernel(kind, eps, L=None, max_depth=10, sampler="multinomial", criterion="generalised"):
    if kind == "hmc":
        return A.HMCKernel(A.Trajectory(A.EndPointTS, A.Leapfrog(eps), A.FixedNSteps(L)))
    if kind == "multinomial":
        return A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(eps), A.FixedNSteps(L)))
    return A.HMCKernel(A.Trajectory(getattr(A, _SAMPLERS[sampler]), A.Leapfrog(eps), getattr(A, _CRITERIA[criterion])(max_depth, 1000.0)))


def _assert_matches(kind, thetas_got, st, z_last, ref, n_tr, N):
    thetas, so, last = ref[:3]
    for t in range(n_tr):
        assert rel_err(thetas_got[t], thetas[t]) < TOL, (t, rel_err(thetas_got[t], thetas[t]))
        assert rel_err_elem_scaled(thetas_got[t], thetas[t]) < 10 * TOL, t
    for k in _STATS[kind]:
        got = _np(st[k]).reshape(n_tr, N)
        if k == "acceptance_rate":
            assert rel_err(got, so[k]) < 1e-9, (k, rel_err(got, so[k]))
        else:
            bad = np.argwhere(got != so[k])
            assert bad.size == 0, (k, bad[:5].tolist(), got[tuple(bad[0])], so[k][tuple(bad[0])])
    assert_pp_close(z_last, last)


def _philox(seed, off):
    g = A.PhiloxRNG(seed)
    g.offset = off
    return g


def _run_case(kind, model, metric, D, N, eps, seed, off, L=None, max_depth=10, sampler="multinomial", criterion="generalised",
              scale=1.0, n_tr=3, tape_check=True):
    """transition() at `off`, its tape twin, and sample_transitions(n_tr) from `off`, each against the oracle; returns the
    oracle's stats of the multi-transition run"""
    p0, p1, Minv, th = _problem(model, metric, D, N, seed=D * 31 + N, scale=scale)
    h = A.Hamiltonian(_dev_metric(metric, Minv, D), make_target(model, D, p0, p1, 0.0))
    z0 = A.phasepoint(h, T(th), T(np.zeros((D, N))))
    kern = _kernel(kind, eps, L, max_depth, sampler, criterion)
    g = _philox(seed, off)
    tr = A.transition(g, h, kern, z0)
    assert g.offset == off + 1
    n_fwd = tr.stat.get("n_steps_fwd")
    kw = dict(L=L, n_fwd=n_fwd, max_depth=max_depth, sampler=sampler, criterion=criterion)
    ref1 = _oracle(kind, model, metric, D, N, p0, p1, Minv, th, eps, seed, off, 1, **kw)
    _assert_matches(kind, [F(tr.z.theta)], tr.stat, tr.z, ref1, 1, N)
    if tape_check:  # the same launch on the restated tapes: only the variates' source differs
        tp = ref1[3][0]
        tr_t = A.transition(A.TapeRNG(normal=T(tp["normal"]), exp=torch.as_tensor(tp["exp"], device=DEV),
                                      dirs=torch.as_tensor(tp["dirs"], device=DEV) if "dirs" in tp else None, n_fwd=n_fwd),
                            h, kern, z0)
        for f in ("theta", "r"):
            assert rel_err(F(getattr(tr_t.z, f)), F(getattr(tr.z, f))) < 1e-12, f
        assert rel_err(F(tr_t.z.lp.value), F(tr.z.lp.value)) < 1e-12
        for k in _STATS[kind]:
            if k == "acceptance_rate":
                assert rel_err(F(tr_t.stat[k]), F(tr.stat[k])) < 1e-12
            else:
                assert np.array_equal(F(tr_t.stat[k]), F(tr.stat[k])), k
    if kind == "multinomial":  # multi-transition launches run EndPointTS / NUTS only
        return ref1[1]
    g = _philox(seed, off)
    zl, draws, st = A.sample_transitions(g, h, kern, z0, n_tr)
    assert g.offset == off + n_tr
    ref = _oracle(kind, model, metric, D, N, p0, p1, Minv, th, eps, seed, off, n_tr, **kw)
    _assert_matches(kind, [F(draws[t]) for t in range(n_tr)], st, zl, ref, n_tr, N)
    return ref[1]


@pytest.mark.parametrize("model,metric,D,N,eps,L,seed,off", [
    ("std_normal", "unit", 3, 37, 0.9, 10, SEED_HI, 0),
    ("funnel", "diag", 10, 45, 0.1, 8, SEED_BIG, 1),
    ("dense_gauss", "dense", 40, 29, 0.3, 10, 5, OFF_HI),
    ("diag_gauss", "diag", 128, 301, 0.6, 10, SEED_HI, OFF_HI),        # the fused fast path
    ("diag_gauss", "diag_chain", 300, 45, 0.4, 10, SEED_BIG, 0),
    ("dense_gauss", "dense", 128, 333, 0.3, 8, SEED_HI, 1),            # the tiled (K4) trajectory for transition()
    ("diag_gauss", "diag", 700, 9, 0.45, 10, SEED_BIG, OFF_HI),        # streamed D > 512
    ("funnel", "unit", 1500, 5, 0.05, 8, SEED_HI, 1),
])
def test_static_hmc_in_philox_mode_equals_oracle_on_restated_tapes(model, metric, D, N, eps, L, seed, off):
    so = _run_case("hmc", model, metric, D, N, eps, seed, off, L=L, scale=0.3 if model == "funnel" else 1.0)
    if D == 128 and metric == "diag":
        acc = so["is_accept"].astype(bool)
        assert 0 < acc.sum() < acc.size  # the exp draw decides some transitions


@pytest.mark.parametrize("model,metric,D,N,eps,seed,off", [
    ("std_normal", "unit", 5, 61, 0.6, SEED_HI, 0),
    ("diag_gauss", "diag", 128, 211, 0.45, SEED_BIG, OFF_HI),
    ("funnel", "unit", 10, 50, 0.15, 3, 1),
])
def test_static_multinomial_in_philox_mode_equals_oracle_on_the_restated_uniform(model, metric, D, N, eps, seed, off):
    so = _run_case("multinomial", model, metric, D, N, eps, seed, off, L=11, scale=0.4 if model == "funnel" else 1.0)
    assert len(set(so["tree_depth"].ravel().tolist())) > 3  # the uniform really picks across the trajectory


@pytest.mark.parametrize("model,metric,D,N,eps,scale,sampler,criterion,seed,off", [
    ("funnel", "unit", 3, 77, 0.9, 2.0, "multinomial", "generalised", SEED_HI, 0),     # G = 4
    ("funnel", "unit", 3, 77, 0.9, 2.0, "slice", "generalised", SEED_BIG, 1),          # G = 4, SliceTS
    ("diag_gauss", "unit", 5, 70, 0.4, 1.0, "multinomial", "generalised", SEED_BIG, OFF_HI),  # G = 8
    ("diag_gauss", "diag", 5, 70, 0.4, 1.0, "slice", "generalised", SEED_HI, 1),       # G = 8, SliceTS
    ("std_normal", "unit", 10, 53, 0.3, 1.0, "multinomial", "generalised", 9, OFF_HI),  # G = 16
    ("std_normal", "unit", 10, 53, 0.3, 1.0, "multinomial", "classic", SEED_HI, 0),    # G = 16, ClassicNoUTurn
    ("funnel", "diag", 10, 53, 0.12, 0.6, "slice", "generalised", SEED_BIG, 1),
    ("diag_gauss", "diag", 40, 45, 0.15, 1.0, "multinomial", "generalised", SEED_HI, 1),   # G = 32, E = 2
    ("diag_gauss", "diag", 64, 33, 0.15, 1.0, "multinomial", "generalised", SEED_BIG, 0),  # compile-time D = 64
    ("diag_gauss", "diag", 128, 33, 0.15, 1.0, "multinomial", "generalised", SEED_HI, OFF_HI),  # compile-time D = 128
    ("diag_gauss", "diag", 128, 33, 0.15, 1.0, "slice", "generalised", SEED_BIG, 1),
    ("diag_gauss", "diag", 256, 20, 0.1, 1.0, "multinomial", "generalised", SEED_HI, 0),   # compile-time D = 256
    ("dense_gauss", "dense", 40, 11, 0.25, 1.0, "multinomial", "generalised", SEED_BIG, OFF_HI),  # cooperative: 8 + 3 chains
    ("diag_gauss", "dense", 33, 11, 0.2, 1.0, "multinomial", "generalised", SEED_HI, 1),         # cooperative, Dense metric
    ("diag_gauss", "dense_chain", 33, 8, 0.2, 1.0, "multinomial", "generalised", SEED_BIG, 0),   # per-chain Dense metric
])
def test_nuts_in_philox_mode_equals_oracle_on_restated_tapes(model, metric, D, N, eps, scale, sampler, criterion, seed, off):
    so = _run_case("nuts", model, metric, D, N, eps, seed, off, sampler=sampler, criterion=criterion, scale=scale)
    if D <= 16:  # several chains per warp with divergent tree sizes
        assert len(set(so["tree_depth"].ravel().tolist())) > 1


def test_nuts_deep_trees_cross_many_prefetch_windows_and_direction_blocks():
    """max_depth 10 with a step size small enough that trees reach it: up to 1023 exponentials per transition (128
    prefetch windows of G = 8 lanes) and 10 direction bits"""
    so = _run_case("nuts", "std_normal", "unit", 5, 29, 0.002, SEED_BIG, OFF_HI, max_depth=10)
    assert so["tree_depth"].max() == 10 and so["tree_depth"].min() >= 8


def _adapt_case(kind, model, D, N, eps, seed, off, L=None):
    p0, p1, Minv, th = _problem(model, "diag", D, N, seed=D * 17 + N)
    h = A.Hamiltonian(_dev_metric("diag", Minv, D), make_target(model, D, p0, p1, 0.0))
    z0 = A.phasepoint(h, T(th), T(np.zeros((D, N))))
    kern = _kernel(kind, eps, L)
    run = A.nuts_adapt_sample if kind == "nuts" else A.hmc_adapt_sample
    g = _philox(seed, off)
    n_tr = 3
    zl, draws, st, eps_f, minv_f, _ = run(g, h, kern, z0, n_tr, 0, A.VectorisedStanAdaptor())
    assert g.offset == off + n_tr
    ref = _oracle(kind, model, "diag", D, N, p0, p1, Minv, th, eps, seed, off, n_tr, L=L)
    _assert_matches(kind, [F(draws[t]) for t in range(n_tr)], st, zl, ref, n_tr, N)


def test_adaptive_nuts_family_with_no_adaptation_equals_oracle_on_restated_tapes():
    _adapt_case("nuts", "diag_gauss", 10, 41, 0.3, SEED_HI, OFF_HI)


def test_adaptive_static_family_with_no_adaptation_equals_oracle_on_restated_tapes():
    _adapt_case("hmc", "diag_gauss", 64, 41, 0.5, SEED_BIG, 1, L=10)
