"""Growth of the context's device buffers (ahmc_api.cu): the host-buffer staging arena and the split-step, dense (K4),
column-padded (cooperative NUTS), per-chain, multinomial energy and adapt_summary workspaces.  In a fresh context each
entry point is called at a small and then at a larger N (the column-padded metric also at a larger D), so every buffer it
uses is allocated and then grown; the same calls from host buffers (numpy, staged through the arena) must give bit for bit
what device tensors give, with the same number of kernel launches."""
import numpy as np
import pytest
import torch

import ahmc_b200 as A
from ahmc_b200 import core as K

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture
def ctx(monkeypatch):
    """a context of its own for the test (every buffer starts unallocated), destroyed at its end"""
    c = K.Context(0)
    monkeypatch.setitem(K._contexts, 0, c)
    yield c
    c.lib.ahmc_destroy(c.h)


def _np(x):
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy()
    return np.asarray(x)


def _flat(res):
    """the arrays of a result: phase points, stats dicts, tuples and lists of them"""
    if res is None or isinstance(res, (int, float)):
        return []
    if isinstance(res, K.PhasePoint):
        return _flat([res.theta, res.r, res.lp.value, res.lp.gradient, res.lk.value, res.lk.gradient])
    if isinstance(res, K.Transition):
        return _flat([res.z, res.stat])
    if isinstance(res, K.DenseEuclideanMetric):
        return _flat([res.Minv, res.cholU])
    if isinstance(res, dict):
        return _flat([res[k] for k in sorted(res)])
    if isinstance(res, (tuple, list)):
        return [a for r in res for a in _flat(r)]
    return [_np(res)]


def _problem(D, N, seed):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(N, D)), rng.normal(size=(N, D)), rng.uniform(0.2, 1.0, size=N)


def _diag_h(D):
    s = np.linspace(0.5, 2.0, D)
    return A.Hamiltonian(A.DiagEuclideanMetric(s * s), A.DiagGaussian(np.zeros(D), s))


def _dense_h(D):
    rng = np.random.default_rng(D)
    Q, _ = np.linalg.qr(rng.normal(size=(D, D)))
    M = (Q * np.exp(rng.uniform(-0.3, 0.3, D))) @ Q.T
    return A.Hamiltonian(A.DenseEuclideanMetric(M), A.DenseGaussian(rng.normal(size=D), np.linalg.inv(M)))


def _callback_h(D):
    return A.Hamiltonian(A.DiagEuclideanMetric(np.linspace(0.5, 2.0, D)),
                         A.CallbackTarget(D, lambda th: (-0.5 * (th * th).sum(dim=1), -th)))


def _static(eps, n, sampler=A.EndPointTS):
    return A.HMCKernel(A.Trajectory(sampler, A.Leapfrog(eps), A.FixedNSteps(n)))


def _nuts(eps, depth=6):
    return A.HMCKernel(A.Trajectory(A.MultinomialTS, A.Leapfrog(eps), A.GeneralisedNoUTurn(depth, 1000.0)))


def _without(tr, key):
    return K.Transition(tr.z, {k: v for k, v in tr.stat.items() if k != key})


_ADAPTOR = A.VectorisedStanAdaptor(init_buffer=4, term_buffer=3, window_size=5)

# name -> (shapes (D, N) in call order, call(h builder, x = array maker, D, N) -> result).  N = 600 in `step` takes the
# chunked host-buffer lane with one chunk (pageable buffers below N = 1024), which launches what the device call does.
CASES = {
    "phasepoint": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: A.phasepoint(_diag_h(D), x(th), x(r))),
    "step": ([(6, 16), (6, 600)], lambda D, N, x, th, r, al: A.step(A.Leapfrog(0.1), _diag_h(D),
                                                                    A.phasepoint(_diag_h(D), x(th), x(r)), 5)),
    "rand_momentum": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: A.rand_momentum(A.PhiloxRNG(3), _diag_h(D).metric,
                                                                                     None, x(th))),
    "static_transition": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: A.transition(
        A.PhiloxRNG(4), _diag_h(D), _static(0.2, 8), A.phasepoint(_diag_h(D), x(th), x(r)))),
    "static_sample_bigd": ([(600, 4), (600, 40)], lambda D, N, x, th, r, al: A.sample_transitions(
        A.PhiloxRNG(5), A.Hamiltonian(A.UnitEuclideanMetric(D), A.StdNormal(D)), _static(0.1, 4),
        A.phasepoint(A.Hamiltonian(A.UnitEuclideanMetric(D), A.StdNormal(D)), x(th), x(r)), 3)),
    # a static MultinomialTS transition does not report max_hamiltonian_energy_error (only NUTS writes it)
    "multinomial_transition": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: _without(A.transition(
        A.PhiloxRNG(6), _diag_h(D), _static(0.2, 7, A.MultinomialTS), A.phasepoint(_diag_h(D), x(th), x(r))),
        "max_hamiltonian_energy_error")),
    "nuts_sample": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: A.sample_transitions(
        A.PhiloxRNG(7), _diag_h(D), _nuts(0.3), A.phasepoint(_diag_h(D), x(th), x(r)), 3)),
    "nuts_adapt": ([(6, 16), (6, 300)], lambda D, N, x, th, r, al: A.nuts_adapt_sample(
        A.PhiloxRNG(8), _diag_h(D), _nuts(0.3), A.phasepoint(_diag_h(D), x(th), x(r)), 16, 12, _ADAPTOR,
        keep_eps_trace=True)),
    "hmc_adapt": ([(6, 16), (6, 300)], lambda D, N, x, th, r, al: A.hmc_adapt_sample(
        A.PhiloxRNG(9), _diag_h(D), _static(0.2, 6), A.phasepoint(_diag_h(D), x(th), x(r)), 16, 12, _ADAPTOR,
        keep_eps_trace=True)),
    "full_trajectory": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: A.step(
        A.Leapfrog(0.1), _diag_h(D), A.phasepoint(_diag_h(D), x(th), x(r)), 4, full_trajectory=True)),
    "find_good_stepsize": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: A.find_good_stepsize_batched(
        A.PhiloxRNG(10), _diag_h(D), x(th), 0.5, return_momentum=True)),
    "adapt_summary": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: A.adapt_summary(x(th), x(al))),
    "callback_split_step": ([(6, 16), (6, 700)], lambda D, N, x, th, r, al: [
        A.step(A.Leapfrog(0.1), _callback_h(D), A.phasepoint(_callback_h(D), x(th), x(r)), 3),
        A.transition(A.PhiloxRNG(11), _callback_h(D), _static(0.2, 3), A.phasepoint(_callback_h(D), x(th), x(r)))]),
    "dense_tile_and_coop": ([(20, 8), (40, 300)], lambda D, N, x, th, r, al: [
        A.step(A.Leapfrog(0.1), _dense_h(D), A.phasepoint(_dense_h(D), x(th), x(r)), 4),
        A.transition(A.PhiloxRNG(12), _dense_h(D), _static(0.1, 4), A.phasepoint(_dense_h(D), x(th), x(r))),
        A.transition(A.PhiloxRNG(13), _dense_h(D), _nuts(0.1, 5), A.phasepoint(_dense_h(D), x(th), x(r)))]),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_buffers_equal_device_calls_while_context_buffers_grow(ctx, name):
    shapes, call = CASES[name]
    for D, N in shapes:
        th, r, al = _problem(D, N, seed=D * 1000 + N)
        out = {}
        for where, x in (("host", np.ascontiguousarray), ("device", lambda a: torch.as_tensor(a, device=DEV))):
            before = ctx.launches
            res = call(D, N, x, th, r, al)
            out[where] = (_flat(res), ctx.launches - before)
        (host, n_host), (dev, n_dev) = out["host"], out["device"]
        assert n_host == n_dev > 0, (D, N, n_host, n_dev)
        assert len(host) == len(dev) > 0
        for i, (a, b) in enumerate(zip(host, dev)):
            assert a.shape == b.shape and np.array_equal(a, b, equal_nan=True), (D, N, i)
