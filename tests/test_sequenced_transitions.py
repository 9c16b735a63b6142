"""Static HMC transitions of callback (split-step) targets, which run one kernel per stage around the user's closure:
`sample_transitions` keeps its draw, and a transition in place (z_out = z_in) equals the out-of-place one bit for bit
(run with -m gpu on an H100)."""
import numpy as np
import pytest
import torch

import ahmc_b200 as A
from tests.test_bigd_transitions import _pp_equal, _static, _transition_into
from tests.test_gpu_parity import DEV, T, _torch_funnel, make_metric

pytestmark = pytest.mark.gpu
D, N, L = 12, 50, 6


def _callback_problem(metric, seed):
    """a funnel written in torch; chain 1 takes a step 25x too large, so that a rejection restores its start point"""
    rng = np.random.default_rng(seed)
    Minv = np.exp(rng.uniform(-0.5, 0.5, D)) if metric == "diag" else None
    h = A.Hamiltonian(make_metric(metric, Minv, D), A.CallbackTarget(D, _torch_funnel))
    z0 = A.phasepoint(h, T(rng.normal(size=(D, N)) * 0.5), T(rng.normal(size=(D, N))))
    eps = torch.full((N,), 0.1, dtype=torch.float64, device=DEV)
    eps[1] *= 25.0
    return h, z0, eps


@pytest.mark.parametrize("metric", ["unit", "diag"])
def test_callback_sample_transitions_keeps_its_draw(metric):
    h, z0, eps = _callback_problem(metric, 3)
    zl, draws, stats = A.sample_transitions(A.PhiloxRNG(8), h, _static(eps, L), z0, 1)
    assert h.target.error is None
    assert torch.equal(draws[0], zl.theta)
    tr = A.transition(A.PhiloxRNG(8), h, _static(eps, L), z0)
    assert _pp_equal(zl, tr.z) and torch.equal(stats["is_accept"][0], tr.stat["is_accept"])
    assert not stats["is_accept"][0, 1] and stats["is_accept"].sum() >= 1


@pytest.mark.parametrize("metric", ["unit", "diag"])
def test_callback_transition_in_place_equals_out_of_place(metric):
    h, z0, eps = _callback_problem(metric, 5)
    ref = A.transition(A.PhiloxRNG(17), h, _static(eps, L), z0)
    zi = A.PhasePoint(z0.theta.clone(), z0.r.clone(), A.DualValue(z0.lp.value.clone(), z0.lp.gradient.clone()),
                      A.DualValue(z0.lk.value.clone(), None))
    st = _transition_into(h, zi, zi, eps, L, A.PhiloxRNG(17))
    assert h.target.error is None
    assert _pp_equal(zi, ref.z)
    for k in ("is_accept", "acceptance_rate", "hamiltonian_energy", "hamiltonian_energy_error"):
        assert torch.equal(st[k], ref.stat[k]), k
    assert not st["is_accept"][1] and st["is_accept"].sum() >= 1
