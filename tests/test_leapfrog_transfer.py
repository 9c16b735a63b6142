"""The transfer form of K1's shared-coefficient pair kernel (`leapfrog_pair_kernel<..., SHARED=true>`): with a scalar eps and
a shared M^-1 a warp derives each coordinate's matrix P = S^(n-1) of the n - 1 merged steps once (Chebyshev form,
FastCoef::prepare_transfer), and both of its chains' end points are P applied to their entry states.  It is taken only
when the trajectory is one proof segment, n > 1 and every coordinate has 0 <= a*b <= 3; otherwise the stepwise loop runs.

Which form ran is read off the bits: the per-chain coefficient form of the same kernel (a per-chain eps array holding the
same value everywhere) always steps, so the shared run equals it bit for bit exactly when the transfer form was NOT taken.
Both runs are compared with the oracle at 1e-10.  Chain 2 (proof fails, stays finite) and chain 5 (overflows at step 1)
go to the exact path in either form.  CPU: the kernel source under the SIMT emulator at D = 64; GPU: the library at
D = 128."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle_c as oc
from tests import emu as E
from tests.emu import P, EmuLf
from tests.helpers import rel_err
from tests.test_simt_emulation import KINDS, MKINDS

EPS = 0.1
BAD = (2, 5)  # chain 2: |theta| = 1e120 defeats the proof, finite; chain 5: 1e250 overflows at step 1

# (id, n, a*b of coordinate 5 or None, transfer form expected).  s log-spaced 0.1..10 with M^-1 ~ s^2 gives
# K = (1 + max a)(1 + max b) < 128, log2 K <= 7: one proof segment up to n = 34
CASES = [("n1", 1, None, False), ("n2", 2, None, True), ("n32", 32, None, True), ("multi-segment", 40, None, False),
         ("inside-margin", 32, 2.9, True), ("outside-margin", 32, 3.1, False)]


def _system(D, N, ab5, seed):
    rng = np.random.default_rng(seed)
    s = np.exp(np.linspace(np.log(0.1), np.log(10.0), D))
    Minv = s * s * np.exp(rng.uniform(-0.05, 0.05, D))
    if ab5 is not None:  # a = b = sqrt(ab5) at coordinate 5
        q = np.sqrt(ab5) / EPS
        Minv[5], s[5] = q, 1.0 / np.sqrt(q)
    m = rng.normal(size=D)
    th, r = rng.normal(size=(N, D)) * s, rng.normal(size=(N, D)) / np.sqrt(Minv)
    th[2, 9] = 1e120
    th[5, 3] = 1e250
    return m, s, Minv, th, r


def _check(got, zo, so, do, n, status, done):
    assert list(status) == list(so) and list(done) == list(do) and done[5] == 1 and done[2] == n
    ok = [c for c in range(len(do)) if c != 5]
    for k, want in (("th", zo.theta), ("r", zo.r), ("g", zo.lp_gradient)):
        assert rel_err(got[k][ok].T, want[:, ok]) < 1e-10, k
    assert np.allclose(got["lp"][ok], zo.lp_value[ok], rtol=1e-10, atol=1e-10)
    assert np.allclose(got["lk"][ok], zo.lk_value[ok], rtol=1e-10, atol=1e-10)


def _form(shared, stepwise, transfer):
    """shared vs per-chain coefficient runs: bit-identical unless the transfer form ran; the exact-path chains always are"""
    fast = [c for c in range(len(shared["lp"])) if c not in BAD]
    same = all(np.array_equal(shared[k][fast], stepwise[k][fast]) for k in ("th", "r", "g", "lp", "lk"))
    assert same != transfer
    for k in ("th", "r", "g", "lp", "lk"):
        assert np.array_equal(shared[k][list(BAD)], stepwise[k][list(BAD)], equal_nan=True), k


@pytest.fixture(scope="module")
def emu_pair():
    return E.harness("pair")


def _emu_run(lib, D, m, s, Minv, th, r, g, lp, eps_chain, n):
    N = th.shape[0]
    w = 1.0 / (s * s)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g", "dr")}
    o["lp"], o["lk"] = np.zeros(N), np.zeros(N)
    status, done = np.zeros(N, dtype=np.uint32), np.zeros(N, dtype=np.int32)
    q = EmuLf(model_kind=KINDS["diag_gauss"], metric_kind=MKINDS["diag"], D=D, N=N, p0=P(m), p1=P(w), c0=0.0, Minv=P(Minv),
              minv_stride=0, cholU=None, eps=EPS, eps_chain=P(eps_chain) if eps_chain is not None else None, n_steps=n, fwd=1,
              temper_alpha=0.0, th_in=P(th), r_in=P(r), g_in=P(g), lp_in=P(lp), th_out=P(o["th"]), r_out=P(o["r"]),
              g_out=P(o["g"]), lp_out=P(o["lp"]), lk_out=P(o["lk"]), dr_out=P(o["dr"]), status=P(status), steps_done=P(done),
              flags=0, hmc=0)
    assert lib.emu_leapfrog_pair(C.byref(q)) == 0
    return o, status, done


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_transfer_form_under_emulation_matches_oracle(emu_pair, case):
    _, n, ab5, transfer = case
    D, N = 64, 9
    m, s, Minv, th, r = _system(D, N, ab5, 11)
    om, ome = oc.Model(oc.DIAG_GAUSS, D, m, s, 0.0), oc.Metric(oc.DIAG, Minv.copy())
    z0 = oc.phasepoint(om, ome, th.T, r.T)
    zo, so, do = oc.leapfrog(om, ome, EPS, z0, n)
    g, lp = np.ascontiguousarray(z0.lp_gradient.T), np.ascontiguousarray(z0.lp_value)
    shared, st, dn = _emu_run(emu_pair, D, m, s, Minv, th, r, g, lp, None, n)
    _check(shared, zo, so, do, n, st, dn)
    stepwise, st2, dn2 = _emu_run(emu_pair, D, m, s, Minv, th, r, g, lp, np.full(N, EPS), n)
    _check(stepwise, zo, so, do, n, st2, dn2)
    _form(shared, stepwise, transfer)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_transfer_form_on_the_gpu_matches_oracle(case):
    import torch

    import ahmc_b200 as A

    _, n, ab5, transfer = case
    D, N = 128, 9
    m, s, Minv, th, r = _system(D, N, ab5, 12)
    om, ome = oc.Model(oc.DIAG_GAUSS, D, m, s, 0.0), oc.Metric(oc.DIAG, Minv.copy())
    zo, so, do = oc.leapfrog(om, ome, EPS, oc.phasepoint(om, ome, th.T, r.T), n)
    h = A.Hamiltonian(A.DiagEuclideanMetric(Minv), A.DiagGaussian(m, s, normalised=False))
    dev = "cuda:0"
    z0 = A.phasepoint(h, torch.as_tensor(th, device=dev), torch.as_tensor(r, device=dev))
    npy = lambda t: t.detach().cpu().numpy()
    runs = []
    for eps in (EPS, torch.full((N,), EPS, dtype=torch.float64, device=dev)):
        z1, info = A.step(A.Leapfrog(eps), h, z0, n, return_info=True)
        got = {"th": npy(z1.theta), "r": npy(z1.r), "g": npy(z1.lp.gradient), "lp": npy(z1.lp.value), "lk": npy(z1.lk.value)}
        _check(got, zo, so, do, n, npy(info.status), npy(info.steps_done))
        runs.append(got)
    _form(runs[0], runs[1], transfer)
