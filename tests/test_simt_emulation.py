"""The product's NUTS kernel SOURCE (advancedhmc.jl_b200/csrc/ahmc_nuts_kernel.cuh + ahmc_device.cuh, unmodified) executed
on the CPU by a small SIMT emulator (tests/simt_emu/: one host thread per CUDA thread, the 32 threads of a warp meet at
a barrier in every shuffle / vote) and compared with the recursive C oracle on shared random tapes.  This checks the
kernel's actual code -- control flow, workspace addressing, warp-uniform predicates, every template family -- without a
GPU; the GPU parity tests (-m gpu) remain the authority for the compiled binary."""
import concurrent.futures as cf
import ctypes as C
import os

import numpy as np
import pytest

from oracle import oracle_c as oc
from tests import emu as E
from tests.emu import P, EmuDense, EmuLf, EmuMn, EmuNuts
from tests.helpers import rel_err


@pytest.fixture(scope="module")
def emu():
    """the NUTS harness (kernel source + emulator)"""
    return E.harness("nuts")


KINDS = dict(std_normal=oc.STD_NORMAL, diag_gauss=oc.DIAG_GAUSS, dense_gauss=oc.DENSE_GAUSS, funnel=oc.FUNNEL)
MKINDS = dict(unit=oc.UNIT, diag=oc.DIAG, dense=oc.DENSE)


def _case(lib, kind, mkind, D, N, eps, sampler, criterion, seed, max_depth=6, delta_max=1000.0, scale=1.0, temper=0.0, coop_padded=0):
    rng = np.random.default_rng(seed)
    p0 = p1 = Minv = cholU = None
    if kind == "diag_gauss":
        p0, p1 = rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))
    elif kind == "dense_gauss":
        B = rng.normal(size=(D, D))
        p0, p1 = rng.normal(size=D), B @ B.T / D + np.eye(D)
    if mkind == "diag":
        Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    elif mkind == "dense":
        B = rng.normal(size=(D, D))
        Minv = B @ B.T / D + 0.5 * np.eye(D)
        cholU = np.ascontiguousarray(np.linalg.cholesky(Minv).T.T)  # U column-major == U' row-major
    th, r = rng.normal(size=(N, D)) * scale, rng.normal(size=(N, D))
    dirs = rng.integers(0, 2, size=(N, max_depth + 1)).astype(np.uint8)
    var = rng.exponential(size=(N, 1 << max_depth))
    if sampler == "slice":
        var[:, 1:] = rng.uniform(size=(N, (1 << max_depth) - 1))
    model = oc.Model(KINDS[kind], D, p0, None if kind != "dense_gauss" else np.asfortranarray(p1), 0.0) if kind != "diag_gauss" \
        else oc.Model(oc.DIAG_GAUSS, D, p0, p1, 0.0)
    metric = oc.Metric(MKINDS[mkind], None if Minv is None else np.asfortranarray(Minv))
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    oc.set_tempering(temper)  # TemperedLeapfrog(eps, alpha) as the transition's integrator (0: plain)
    try:
        zo, so, used = oc.nuts_transition(model, metric, eps, z0, None, dirs, var, max_depth=max_depth, delta_max=delta_max,
                                          sampler=sampler, criterion=criterion)
    finally:
        oc.set_tempering(0.0)
    # what the device-side model holds: DIAG_GAUSS p1 = 1/s^2; DENSE_GAUSS p1 = precision (column-major == symmetric)
    dp1 = None if p1 is None else (1.0 / (p1 * p1) if kind == "diag_gauss" else np.ascontiguousarray(p1))
    g_in = np.ascontiguousarray(z0.lp_gradient.T)
    lp_in = np.ascontiguousarray(z0.lp_value)
    out = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lp_o, lk_o, acc, dH, dHm = (np.zeros(N) for _ in range(5))
    ns, td = np.zeros(N, dtype=np.int32), np.zeros(N, dtype=np.int32)
    ne = np.zeros(N, dtype=np.uint8)
    q = EmuNuts(model_kind=KINDS[kind], metric_kind=MKINDS[mkind], D=D, N=N, p0=P(p0), p1=P(dp1), c0=0.0,
                Minv=P(Minv), minv_stride=0, cholU=P(cholU), eps=eps, eps_chain=None, max_depth=max_depth, delta_max=delta_max,
                sampler=oc.SAMPLER[sampler], criterion=oc.CRITERION[criterion], seed=1, offset=0, normal_tape=None,
                exp_tape=P(var), exp_stride=var.shape[1], dir_tape=P(dirs), dir_stride=dirs.shape[1], partial_alpha=0.0,
                refresh=0, th_in=P(th), r_in=P(r), g_in=P(g_in), lp_in=P(lp_in), th_out=P(out["th"]), r_out=P(out["r"]),
                g_out=P(out["g"]), lp_out=P(lp_o), lk_out=P(lk_o), n_steps=P(ns), tree_depth=P(td), numerical=P(ne), acc=P(acc),
                dH=P(dH), dHmax=P(dHm), n_transitions=1, draws=None, adapt=0, temper_alpha=temper, coop_padded=coop_padded)
    assert lib.emu_nuts(C.byref(q)) == 0
    assert (td == so.tree_depth).all() and (ns == so.n_steps).all() and (ne == so.numerical_error).all()
    assert rel_err(out["th"].T, zo.theta) < 1e-10 and rel_err(out["r"].T, zo.r) < 1e-10
    assert rel_err(out["g"].T, zo.lp_gradient) < 1e-10
    assert np.allclose(lp_o, zo.lp_value, rtol=1e-10, atol=1e-10) and np.allclose(lk_o, zo.lk_value, rtol=1e-10, atol=1e-10)
    assert np.allclose(acc, so.acceptance_rate, rtol=1e-10)
    assert np.allclose(dHm, so.max_hamiltonian_energy_error, rtol=1e-9, atol=1e-12)
    return so


CASES = [
    ("diag_gauss", "diag", 7, 9, 0.25, "multinomial", "generalised"),   # G=8: four chains per warp at different tree positions
    ("std_normal", "unit", 3, 11, 0.35, "multinomial", "generalised"),  # G=4: eight chains per warp
    ("funnel", "diag", 6, 6, 0.25, "multinomial", "generalised"),
    ("diag_gauss", "diag", 40, 3, 0.2, "multinomial", "generalised"),   # G=32, E=2: one chain per warp
    ("dense_gauss", "dense", 6, 5, 0.3, "multinomial", "generalised"),  # shared-memory slab, cached M^-1 r_first
    ("diag_gauss", "diag", 7, 9, 0.25, "slice", "generalised"),
    ("diag_gauss", "diag", 7, 9, 0.25, "multinomial", "classic"),
    ("diag_gauss", "diag", 7, 9, 0.25, "multinomial", "strict"),
    ("dense_gauss", "dense", 6, 5, 0.3, "slice", "strict"),
    ("diag_gauss", "unit", 5, 7, 0.3, "slice", "classic"),
    ("diag_gauss", "diag", 13, 5, 0.25, "multinomial", "generalised"),  # G=16: two chains per warp
    ("diag_gauss", "diag", 128, 2, 0.12, "multinomial", "generalised"),  # G=32, E=4: the headline layout
    ("dense_gauss", "dense", 200, 1, 0.25, "multinomial", "generalised"),  # G=32, E=8: C5's layout; COOP block with 7 idle warps
    ("dense_gauss", "dense", 40, 11, 0.3, "multinomial", "generalised"),   # COOP: a full block of 8 chains + a ragged one of 3
    ("dense_gauss", "diag", 64, 9, 0.3, "multinomial", "generalised"),     # COOP, full tile (E=2), dense target only
    ("diag_gauss", "dense", 33, 5, 0.3, "multinomial", "generalised"),     # COOP, dense metric only
    ("dense_gauss", "dense", 264, 1, 0.25, "multinomial", "generalised"),  # G=32, E=16 (D in 257..512): 16-column chunks, 2 stages
]


@pytest.mark.parametrize("kind,mkind,D,N,eps,sampler,criterion", CASES,
                         ids=[f"{c[0]}-{c[1]}-D{c[2]}-{c[5]}-{c[6]}" for c in CASES])
def test_kernel_source_under_cpu_simt_emulation_matches_oracle(emu, kind, mkind, D, N, eps, sampler, criterion):
    so = _case(emu, kind, mkind, D, N, eps, sampler, criterion, seed=5 + D)
    assert so.n_steps.max() >= 7


@pytest.mark.parametrize("kind,mkind,D,N", [("dense_gauss", "dense", 40, 11), ("dense_gauss", "diag", 64, 9), ("diag_gauss", "dense", 33, 5),
                                            ("dense_gauss", "dense", 200, 1), ("dense_gauss", "dense", 264, 2)])
def test_cooperative_products_from_column_padded_matrices_match_oracle(emu, kind, mkind, D, N):
    """the cooperative NUTS form with the column-padded copies of the dense matrices the library prepares (one bulk copy
    per chunk of columns instead of one per column): same transitions as from the plain matrices"""
    so = _case(emu, kind, mkind, D, N, 0.3 if D < 100 else 0.25, "multinomial", "generalised", seed=5 + D, coop_padded=1)
    assert so.n_steps.max() >= 7


def test_kernel_source_emulated_divergent_and_max_depth(emu):
    so = _case(emu, "funnel", "diag", 4, 8, 1.5, "multinomial", "generalised", seed=3, delta_max=3.0, scale=1.5)
    assert so.numerical_error.sum() > 0
    so = _case(emu, "std_normal", "unit", 3, 6, 0.02, "multinomial", "generalised", seed=4, max_depth=4)
    assert (so.tree_depth == 4).all()


@pytest.mark.parametrize("kind,mkind,D,N,eps,sampler,criterion", [
    ("diag_gauss", "diag", 128, 3, 0.12, "multinomial", "generalised"), ("diag_gauss", "diag", 64, 4, 0.25, "multinomial", "strict"),
    ("funnel", "diag", 4, 10, 0.3, "slice", "generalised"), ("dense_gauss", "dense", 8, 5, 0.3, "multinomial", "generalised"),
    ("diag_gauss", "diag", 7, 9, 0.25, "multinomial", "generalised")],
    ids=["D128-full", "D64-full-strict", "D4-slice", "D8-dense", "D7-ragged"])
def test_full_tile_instantiation_matches_oracle(emu, kind, mkind, D, N, eps, sampler, criterion):
    """D == G * E (G = 32, E in 2..8) takes the instantiation with a compile-time D (no `d < D` guards), every other D the
    general one."""
    _case(emu, kind, mkind, D, N, eps, sampler, criterion, seed=29 + D, scale=0.5 if kind == "funnel" else 1.0)


@pytest.mark.parametrize("kind,mkind,D,N,eps,sampler,criterion,alpha", [
    ("diag_gauss", "diag", 7, 9, 0.25, "multinomial", "generalised", 1.05),
    ("funnel", "diag", 6, 6, 0.2, "slice", "strict", 0.9),
    ("dense_gauss", "dense", 40, 9, 0.3, "multinomial", "generalised", 1.1),   # COOP form
], ids=["diag", "funnel-slice-strict", "dense-coop"])
def test_nuts_with_tempered_leapfrog_under_emulation_matches_oracle(emu, kind, mkind, D, N, eps, sampler, criterion, alpha):
    """`TemperedLeapfrog(eps, alpha)` as the integrator of a NUTS transition: every leaf is `step(lf, h, z, +-1)`
    (trajectory.jl:640), i.e. r * sqrt(alpha) before the first half kick and r / sqrt(alpha) after the second
    (integrator.jl:198-209 with n_steps = 1)."""
    so = _case(emu, kind, mkind, D, N, eps, sampler, criterion, seed=77 + D, temper=alpha)
    assert so.n_steps.max() >= 3


def test_kernel_source_emulated_wild_funnel_start(emu):
    _case(emu, "funnel", "diag", 4, 8, 2.5, "multinomial", "generalised", seed=6, delta_max=1000.0, scale=3.0)


def _philox_run(lib, N, D, T, seed, n_adapts=0, adapt=False, eps0=0.3, Minv0=None, sd=None, mu=None, windows=(3, 2, 4), n_min=3,
                dense_target=False, coop_padded=0):
    """Philox-mode run of the (adaptive or plain) persistent kernel: T transitions per chain from theta = 0."""
    th = np.zeros((N, D))
    th[:] = np.linspace(-1, 1, D)
    r = np.zeros((N, D))
    w = 1.0 / (sd * sd)
    g_in = (th - mu) * w
    lp_in = -0.5 * np.sum((th - mu) ** 2 * w, axis=1)
    out = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lp_o, lk_o = np.zeros(N), np.zeros(N)
    acc, dH, dHm = (np.zeros(T * N) for _ in range(3))
    ns, td = np.zeros(T * N, dtype=np.int32), np.zeros(T * N, dtype=np.int32)
    ne = np.zeros(T * N, dtype=np.uint8)
    draws = np.zeros((T, N, D))
    eps_rw, minv_rw, trace = np.full(N, eps0), np.zeros((N, D)), np.zeros((T, N))
    Minv = np.ones(D) if Minv0 is None else Minv0
    Pm = np.ascontiguousarray(np.diag(w))  # the same target written as a dense-precision Gaussian (the cooperative form)
    q = EmuNuts(model_kind=oc.DENSE_GAUSS if dense_target else oc.DIAG_GAUSS, metric_kind=oc.DIAG, D=D, N=N, p0=P(mu),
                p1=P(Pm) if dense_target else P(w), c0=0.0, Minv=P(Minv),
                minv_stride=0 if Minv.ndim == 1 else D, cholU=None, eps=eps0, eps_chain=None, max_depth=6, delta_max=1000.0,
                sampler=0, criterion=0, seed=seed, offset=0, normal_tape=None, exp_tape=None, exp_stride=0, dir_tape=None,
                dir_stride=0, partial_alpha=0.0, refresh=1, th_in=P(th), r_in=P(r), g_in=P(g_in), lp_in=P(lp_in),
                th_out=P(out["th"]), r_out=P(out["r"]), g_out=P(out["g"]), lp_out=P(lp_o), lk_out=P(lk_o), n_steps=P(ns),
                tree_depth=P(td), numerical=P(ne), acc=P(acc), dH=P(dH), dHmax=P(dHm), n_transitions=T, draws=P(draws),
                adapt=1 if adapt else 0, n_adapts=n_adapts, init_buffer=windows[0], term_buffer=windows[1], window_size=windows[2],
                delta=0.8, gamma=0.05, t0=10.0, kappa=0.75, adapt_metric=1, n_min=n_min, eps_rw=P(eps_rw), minv_rw=P(minv_rw),
                eps_trace=P(trace), coop_padded=coop_padded)
    assert lib.emu_nuts(C.byref(q)) == 0
    return dict(draws=draws, acc=acc.reshape(T, N), n_steps=ns.reshape(T, N), eps=eps_rw, minv=minv_rw, trace=trace, theta=out["th"])


def test_in_launch_adaptation_under_emulation_equals_oracle_adaptors(emu):
    """The adaptive kernel family (per-chain NesterovDualAveraging + windowed WelfordVar inside the persistent launch)
    executed by the emulator, replayed iteration by iteration with the ORACLE's adaptors fed by the kernel's own
    acceptance rates and draws: step-size trace, window update of M^-1, reset and finalize! must agree."""
    rng = np.random.default_rng(3)
    D, N, T, n_adapts = 5, 6, 24, 20
    ib, tb, wsz = 3, 2, 4
    ws, we, splits = oc.stan_windows(n_adapts, ib, tb, wsz)
    sd, mu = np.exp(rng.uniform(-0.7, 0.7, D)), rng.normal(size=D)
    run = _philox_run(emu, N, D, T, seed=5, n_adapts=n_adapts, adapt=True, sd=sd, mu=mu, windows=(ib, tb, wsz), n_min=3)
    da, wv = oc.DualAveraging(np.full(N, 0.3), delta=0.8), oc.WelfordVar((D, N))
    Minv = np.ones((N, D))
    updates = 0
    for i in range(1, T + 1):
        assert np.allclose(run["trace"][i - 1], da.eps, rtol=1e-10), i
        if i <= n_adapts:
            da.adapt(run["acc"][i - 1])
            if ws <= i <= we:
                wv.push(run["draws"][i - 1].T)
                if i in splits and wv.n.value >= 3:
                    Minv = np.ascontiguousarray(wv.estimate().T)
                    updates += 1
            if i in splits:
                da.reset()
                wv = oc.WelfordVar((D, N))
            if i == n_adapts:
                da.finalize()
    assert updates >= 1 and np.allclose(run["minv"], Minv, rtol=1e-9)
    assert np.allclose(run["eps"], da.eps, rtol=1e-10)
    # n_adapts = 0: the adaptive family is the plain persistent launch
    p0 = _philox_run(emu, N, D, 6, seed=9, sd=sd, mu=mu)
    p1 = _philox_run(emu, N, D, 6, seed=9, n_adapts=0, adapt=True, sd=sd, mu=mu)
    assert np.array_equal(p0["draws"], p1["draws"]) and np.array_equal(p1["trace"], np.full((6, N), 0.3))


# ------------------------------------------------------------------------------------------------ K1 / K2 under emulation
@pytest.fixture(scope="module")
def emu_lf():
    return E.harness("lf")


def _lf_system(kind, mkind, D, rng):
    p0 = p1 = Minv = cholU = None
    if kind == "diag_gauss":
        p0, p1 = rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))
    elif kind == "dense_gauss":
        B = rng.normal(size=(D, D))
        p0, p1 = rng.normal(size=D), B @ B.T / D + np.eye(D)
    if mkind == "diag":
        Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    elif mkind == "dense":
        B = rng.normal(size=(D, D))
        Minv = B @ B.T / D + 0.5 * np.eye(D)
        cholU = np.ascontiguousarray(np.linalg.cholesky(Minv))  # U column-major == (U')' = L row-major
    model = oc.Model(KINDS[kind], D, p0, p1 if kind != "dense_gauss" else np.asfortranarray(p1), 0.0)
    metric = oc.Metric(MKINDS[mkind], None if Minv is None else np.asfortranarray(Minv))
    dp1 = None if p1 is None else (1.0 / (p1 * p1) if kind == "diag_gauss" else np.ascontiguousarray(p1))
    return model, metric, p0, dp1, Minv, cholU


LF_CASES = [("diag_gauss", "diag", 7, 9, 0.1, 20, 1),    # fused fast path, 4 chains per warp
            ("std_normal", "unit", 3, 13, 0.2, 11, 1),   # fast path, 8 chains per warp
            ("funnel", "diag", 6, 7, 0.05, 12, 1),       # exact per-step path
            ("dense_gauss", "dense", 6, 5, 0.1, 9, 1),   # exact path with the shared-memory slab matvec
            ("diag_gauss", "diag", 40, 3, 0.1, 16, 0),   # backward, one chain per warp (E = 2)
            ("diag_gauss", "diag", 64, 3, 0.1, 32, 1),   # full tile: lane-contiguous 128-bit layout of the fast path
            ("std_normal", "unit", 64, 2, 0.2, 7, 0),    # same, unit coefficients, backward
            ("diag_gauss", "diag", 5, 9, 0.1, 300, 1)]   # n * log2(K) > 240: periodic magnitude tests instead of one


@pytest.mark.parametrize("with_g", [True, False], ids=["cached-grad", "no-grad"])
@pytest.mark.parametrize("kind,mkind,D,N,eps,n,fwd", LF_CASES, ids=[f"{c[0]}-{c[1]}-D{c[2]}-n{c[5]}" for c in LF_CASES])
def test_trajectory_kernel_source_under_emulation_matches_oracle(emu_lf, kind, mkind, D, N, eps, n, fwd, with_g):
    """K1 (`leapfrog_kernel`, fast and exact paths of ahmc_traj.cuh) executed by the emulator vs the oracle's `step`;
    `no-grad`: z_in.lp_gradient == NULL, the kernel recomputes dH/dtheta at the start point."""
    rng = np.random.default_rng(11 + D)
    model, metric, p0, dp1, Minv, cholU = _lf_system(kind, mkind, D, rng)
    th, r = rng.normal(size=(N, D)) * (0.5 if kind == "funnel" else 1.0), rng.normal(size=(N, D))
    eps_chain = eps * np.exp(rng.uniform(-0.3, 0.3, N))
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    zo = oc.leapfrog(model, metric, eps_chain, z0, n if fwd else -n)[0]
    g_in, lp_in = np.ascontiguousarray(z0.lp_gradient.T), np.ascontiguousarray(z0.lp_value)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g", "dr")}
    lp_o, lk_o = np.zeros(N), np.zeros(N)
    status, done = np.zeros(N, dtype=np.uint32), np.zeros(N, dtype=np.int32)
    q = EmuLf(model_kind=KINDS[kind], metric_kind=MKINDS[mkind], D=D, N=N, p0=P(p0), p1=P(dp1), c0=0.0, Minv=P(Minv),
              minv_stride=0, cholU=P(cholU), eps=eps, eps_chain=P(eps_chain), n_steps=n, fwd=fwd, temper_alpha=0.0,
              th_in=P(th), r_in=P(r), g_in=P(g_in) if with_g else None, lp_in=P(lp_in), th_out=P(o["th"]), r_out=P(o["r"]),
              g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o), dr_out=P(o["dr"]), status=P(status), steps_done=P(done), flags=0,
              hmc=0)
    assert emu_lf.emu_leapfrog(C.byref(q)) == 0
    assert (done == n).all() and (status == 0).all()
    assert rel_err(o["th"].T, zo.theta) < 1e-10 and rel_err(o["r"].T, zo.r) < 1e-10 and rel_err(o["g"].T, zo.lp_gradient) < 1e-10
    assert np.allclose(lp_o, zo.lp_value, rtol=1e-10, atol=1e-10) and np.allclose(lk_o, zo.lk_value, rtol=1e-10, atol=1e-10)
    assert rel_err(o["dr"].T, zo.lk_gradient) < 1e-10


@pytest.mark.parametrize("kind,mkind,D,N,eps,n,alpha", [("diag_gauss", "diag", 7, 9, 0.6, 6, 0.0), ("funnel", "diag", 5, 10, 0.45, 6, 0.0),
                                                        ("dense_gauss", "dense", 6, 6, 0.7, 5, 0.0), ("diag_gauss", "diag", 7, 9, 0.6, 7, 1.1),
                                                        ("funnel", "diag", 5, 10, 0.45, 6, 0.93)],
                         ids=["diag-fast", "funnel-exact", "dense", "diag-tempered", "funnel-tempered"])
def test_hmc_transition_kernel_source_under_emulation_matches_oracle(emu_lf, kind, mkind, D, N, eps, n, alpha):
    """K2 (`hmc_kernel`: momentum refresh from a normal tape, trajectory, Metropolis step, revert, flip) vs the oracle;
    alpha > 0: the trajectory is integrated by `TemperedLeapfrog(eps, alpha)` (odd and even n: the middle step of an odd
    trajectory multiplies before and divides after, integrator.jl:198-209)."""
    rng = np.random.default_rng(21 + D)
    model, metric, p0, dp1, Minv, cholU = _lf_system(kind, mkind, D, rng)
    th = rng.normal(size=(N, D)) * (1.5 if kind == "funnel" else 1.0)
    nt, et = rng.normal(size=(N, D)), rng.exponential(size=N)
    z0 = oc.phasepoint(model, metric, th.T, np.zeros((D, N)))
    oc.set_tempering(alpha)
    try:
        zo, so = oc.hmc_transition(model, metric, eps, n, z0, nt.T, et)
    finally:
        oc.set_tempering(0.0)
    g_in, lp_in = np.ascontiguousarray(z0.lp_gradient.T), np.ascontiguousarray(z0.lp_value)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lp_o, lk_o, acc, dH = (np.zeros(N) for _ in range(4))
    isacc = np.zeros(N, dtype=np.uint8)
    r0 = np.zeros((N, D))
    q = EmuLf(model_kind=KINDS[kind], metric_kind=MKINDS[mkind], D=D, N=N, p0=P(p0), p1=P(dp1), c0=0.0, Minv=P(Minv),
              minv_stride=0, cholU=P(cholU), eps=eps, eps_chain=None, n_steps=n, fwd=1, temper_alpha=alpha, th_in=P(th), r_in=P(r0),
              g_in=P(g_in), lp_in=P(lp_in), th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o),
              dr_out=None, status=None, steps_done=None, flags=0, hmc=1, refresh=1, n_transitions=1, seed=1, offset=0,
              normal_tape=P(nt), exp_tape=P(et), is_accept=P(isacc), acc=P(acc), dH=P(dH), draws=None)
    assert emu_lf.emu_leapfrog(C.byref(q)) == 0
    assert (isacc == so.is_accept).all()
    assert rel_err(o["th"].T, zo.theta) < 1e-10 and rel_err(o["r"].T, zo.r) < 1e-10
    assert np.allclose(acc, so.acceptance_rate, rtol=1e-10) and np.allclose(lp_o, zo.lp_value, rtol=1e-10, atol=1e-10)


def test_in_launch_adaptation_in_the_cooperative_form_equals_the_diagonal_run(emu):
    """A dense-precision Gaussian with the Diag metric runs the adaptive family in the block-cooperative form (8 chains
    share the precision product).  Written with a DIAGONAL precision it is the same target as the diagonal Gaussian: step
    size traces, adapted M^-1 and draws of the two kernels agree (products sum in a different order: 1e-7 after 8
    transitions), from plain and from column-padded matrices."""
    rng = np.random.default_rng(31)
    D, N, T, n_adapts = 40, 8, 8, 6
    sd, mu = np.exp(rng.uniform(-0.4, 0.4, D)), rng.normal(size=D) * 0.3
    kw = dict(seed=4, n_adapts=n_adapts, adapt=True, eps0=0.2, sd=sd, mu=mu, windows=(2, 1, 3), n_min=2)
    ref = _philox_run(emu, N, D, T, **kw)
    for padded in (0, 1):
        got = _philox_run(emu, N, D, T, dense_target=True, coop_padded=padded, **kw)
        assert (got["n_steps"] == ref["n_steps"]).all()
        assert np.allclose(got["trace"], ref["trace"], rtol=1e-7) and np.allclose(got["eps"], ref["eps"], rtol=1e-7)
        assert np.allclose(got["minv"], ref["minv"], rtol=1e-6) and np.allclose(got["draws"], ref["draws"], atol=1e-6)
    assert ref["n_steps"].max() >= 7 and not np.allclose(ref["minv"], 1.0)


def test_kernel_source_emulated_randomised_configurations(emu):
    """A small fuzz over (target, metric, dimension / layout, chains per warp, step size, depth limit, divergence threshold,
    sampler, criterion) of the emulated kernel source against the recursive oracle."""
    rng = np.random.default_rng(123)
    combos = [("std_normal", "unit"), ("diag_gauss", "diag"), ("funnel", "diag"), ("dense_gauss", "dense"), ("diag_gauss", "unit")]
    for cfg in range(12):
        kind, mkind = combos[int(rng.integers(0, len(combos)))]
        D = int([3, 4, 6, 8, 11, 16, 40][int(rng.integers(0, 7))])
        if kind == "funnel":
            D = max(D, 2)
        N = int(rng.integers(1, 10))
        eps = float(np.exp(rng.uniform(np.log(0.08), np.log(0.6))))
        sampler = ["multinomial", "slice"][int(rng.integers(0, 2))]
        criterion = ["generalised", "classic", "strict"][int(rng.integers(0, 3))]
        _case(emu, kind, mkind, D, N, eps, sampler, criterion, seed=1000 + cfg, max_depth=int(rng.integers(2, 7)),
              delta_max=[1000.0, 2.5][int(rng.integers(0, 2))], scale=0.6 if kind == "funnel" else 1.3)


# ------------------------------------------------------------------------------------------------ MultinomialTS static kernel
@pytest.fixture(scope="module")
def emu_mn():
    return E.harness("mn")


def test_multinomial_static_kernel_source_under_emulation_matches_mp50_fixtures(emu_mn):
    """`multinomial_kernel` (energy pass, inverse-CDF draw, re-materialisation of the drawn point) executed by the emulator
    on the 50-digit MultinomialTS fixtures of tests/golden/hmc_mp50.json (mixed, all-forward and all-backward splits, and one
    integrated by TemperedLeapfrog)."""
    from tests.helpers import hmc_golden_cases

    done = 0
    for case in hmc_golden_cases():
        if case["sampler"] != "multinomial":
            continue
        D, N = case["D"], case["N"]
        kind, mkind = case["model"], case["metric"]
        p0 = None if case["p0"] is None else np.array(case["p0"])
        p1 = None if case["p1"] is None else np.array(case["p1"])
        Minv = None if case["Minv"] is None else np.array(case["Minv"])
        cholU = None if mkind != "dense" else np.ascontiguousarray(np.linalg.cholesky(Minv))
        dp1 = None if p1 is None else (1.0 / (p1 * p1) if kind == "diag_gauss" else np.ascontiguousarray(p1))
        model = oc.Model(KINDS[kind], D, p0, p1 if kind != "dense_gauss" else np.asfortranarray(p1), 0.0)
        metric = oc.Metric(MKINDS[mkind], None if Minv is None else np.asfortranarray(Minv))
        th = np.array(case["theta0"])
        z0 = oc.phasepoint(model, metric, th.T, np.zeros((D, N)))
        g_in, lp_in = np.ascontiguousarray(z0.lp_gradient.T), np.ascontiguousarray(z0.lp_value)
        nt, ut = np.array(case["normals"]), np.array(case["variates"])
        o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
        lp_o, lk_o, acc = np.zeros(N), np.zeros(N), np.zeros(N)
        idx = np.zeros(N, dtype=np.int32)
        q = EmuMn(model_kind=KINDS[kind], metric_kind=MKINDS[mkind], D=D, N=N, p0=P(p0), p1=P(dp1), Minv=P(Minv), cholU=P(cholU),
                  eps=case["eps"], n_steps=case["n_steps"], n_fwd=case["n_fwd"], normal_tape=P(nt), unif_tape=P(ut), th_in=P(th),
                  g_in=P(g_in), lp_in=P(lp_in), th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o),
                  acc=P(acc), index=P(idx), temper_alpha=case.get("temper_alpha", 0.0))
        assert emu_mn.emu_multinomial(C.byref(q)) == 0, case["name"]
        e = case["expect"]
        if "index" in e:
            assert (idx == np.array(e["index"])).all(), case["name"]
        assert rel_err(o["th"], np.array(e["theta"])) < 1e-10 and rel_err(o["r"], np.array(e["r"])) < 1e-10
        assert np.allclose(acc, e["acceptance_rate"], rtol=1e-10)
        assert np.allclose(lp_o, e["lp_value"], rtol=1e-10, atol=1e-10) and np.allclose(lk_o, e["lk_value"], rtol=1e-10, atol=1e-10)
        done += 1
    assert done == 4  # mixed, all-forward, all-backward, and a tempered one


@pytest.mark.parametrize("n,n_fwd", [(7, 3), (6, 6), (5, 0)])
def test_multinomial_static_with_tempered_leapfrog_under_emulation_matches_oracle(emu_mn, n, n_fwd):
    """MultinomialTS static transition integrated by `TemperedLeapfrog`: the forward and the backward leg are separate
    `step` calls (trajectory.jl:374-376), each tempering by its OWN number of steps -- also in the replay that
    re-materialises the drawn point."""
    rng = np.random.default_rng(500 + n)
    D, N, eps, alpha = 7, 9, 0.35, 1.08
    p0, p1 = rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))
    Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    model, metric = oc.Model(oc.DIAG_GAUSS, D, p0, p1, 0.0), oc.Metric(oc.DIAG, Minv)
    th, nt, ut = rng.normal(size=(N, D)), rng.normal(size=(N, D)), rng.uniform(size=N)
    z0 = oc.phasepoint(model, metric, th.T, np.zeros((D, N)))
    oc.set_tempering(alpha)
    try:
        zo, so = oc.hmc_multinomial_transition(model, metric, eps, n, n_fwd, z0, nt.T, ut)
    finally:
        oc.set_tempering(0.0)
    g_in, lp_in = np.ascontiguousarray(z0.lp_gradient.T), np.ascontiguousarray(z0.lp_value)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lp_o, lk_o, acc = np.zeros(N), np.zeros(N), np.zeros(N)
    idx = np.zeros(N, dtype=np.int32)
    q = EmuMn(model_kind=oc.DIAG_GAUSS, metric_kind=oc.DIAG, D=D, N=N, p0=P(p0), p1=P(1.0 / (p1 * p1)), Minv=P(Minv), cholU=None,
              eps=eps, n_steps=n, n_fwd=n_fwd, normal_tape=P(nt), unif_tape=P(ut), th_in=P(th), g_in=P(g_in), lp_in=P(lp_in),
              th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o), acc=P(acc), index=P(idx),
              temper_alpha=alpha)
    assert emu_mn.emu_multinomial(C.byref(q)) == 0
    assert rel_err(o["th"].T, zo.theta) < 1e-10 and rel_err(o["r"].T, zo.r) < 1e-10
    assert np.allclose(acc, so.acceptance_rate, rtol=1e-10)
    assert np.allclose(lp_o, zo.lp_value, rtol=1e-10, atol=1e-10) and np.allclose(lk_o, zo.lk_value, rtol=1e-10, atol=1e-10)
    # tempering is not volume preserving: the energies along the legs differ visibly from the untempered ones
    zu, su = oc.hmc_multinomial_transition(model, metric, eps, n, n_fwd, z0, nt.T, ut)
    assert not np.allclose(su.acceptance_rate, so.acceptance_rate, rtol=1e-6)


def test_adaptor_statistics_kernel_sources_under_emulation():
    """K5 (`adapt_kernel`: per-block partials, last-block reduction through a device counter) and K5b (`adapt_cov_kernel`:
    tiled second moment) executed by the emulator (block barriers, static shared variables) vs numpy."""
    lib = E.harness("adapt")
    rng = np.random.default_rng(8)
    for D, N in ((7, 33), (40, 13), (33, 3)):
        Lm = rng.normal(size=(D, D)) / np.sqrt(D)
        th = rng.normal(size=(N, D)) @ Lm + rng.normal(size=D)
        al = rng.uniform(0, 1.4, N)
        rec, cov = np.zeros(2 + 2 * D), np.zeros((D, D))
        assert lib.emu_adapt(D, C.c_longlong(N), P(th), P(al), P(rec), P(cov)) == 0
        mu = th.mean(axis=0)
        c = th - mu
        assert rec[0] == N and rec[1] == pytest.approx(np.minimum(1, al).sum(), rel=1e-13)
        assert np.allclose(rec[2:2 + D], mu, rtol=1e-12) and np.allclose(rec[2 + D:], (c ** 2).sum(axis=0), rtol=1e-11)
        want = c.T @ c
        assert np.allclose(cov, want, rtol=1e-11, atol=1e-11 * np.abs(want).max()) and np.array_equal(cov, cov.T)


@pytest.mark.parametrize("R,adapt_metric", [(1, 1), (2, 1), (5, 1), (3, 0)])
def test_pooled_adaptor_kernel_source_under_emulation_equals_host_adaptors(R, adapt_metric):
    """The device-side exchange's arithmetic (`pooled_update_kernel`, ahmc_pooled.cu: rank-ordered Chan merge of R per-rank
    records, NesterovDualAveraging, WelfordVar, Stan windows, reset / finalize) executed by the CPU emulator on the records R
    ranks would all-gather, against the host-side pooled adaptors of adaptation.py fed with the merged record -- the N > 1
    path of the exchange without a GPU or NCCL (the GPU suite repeats it over a real 2-rank communicator)."""
    from ahmc_b200 import adaptation as ad

    lib = E.harness("pooled")
    lib.emu_pooled_create.restype = C.c_void_p
    lib.emu_pooled_create.argtypes = [C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int]
    lib.emu_pooled_update.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.emu_pooled_destroy.argtypes = [C.c_void_p]
    D, n_adapts, windows = 13, 40, (5, 4, 6)
    rng = np.random.default_rng(17 + R)
    chains = [50 + 7 * r for r in range(R)]  # ragged shards
    h = lib.emu_pooled_create(D, chains[0], n_adapts, *windows, 0.21, 0.8, adapt_metric, 3)
    assert h
    pc = ad.WelfordVar(D, n_min=3) if adapt_metric else ad.UnitMassMatrix()
    host = ad.StanHMCAdaptor(pc, ad.NesterovDualAveraging(0.8, 0.21), *windows)
    host.initialize(n_adapts)
    scale = np.exp(rng.uniform(-1, 1, D))
    for i in range(1, n_adapts + 1):
        recs = []
        for r in range(R):
            th = rng.normal(size=(chains[r], D)) * scale + 0.2 * r
            al = rng.uniform(0.1, 1.5, chains[r])
            mu = th.mean(axis=0)
            recs.append(np.concatenate([[chains[r], np.minimum(1.0, al).sum()], mu, ((th - mu) ** 2).sum(axis=0)]))
        gathered = np.ascontiguousarray(np.stack(recs))
        eps, minv, merged = C.c_double(), np.zeros(D), np.zeros(2 + 2 * D)
        it = lib.emu_pooled_update(h, P(gathered), R, C.byref(eps), P(minv), P(merged))
        assert it == i
        want = ad.merge_records(recs)
        assert np.allclose(merged, want, rtol=1e-13, atol=0)
        host.adapt(want)
        if i == n_adapts:
            host.finalize()
        assert abs(eps.value - host.eps) <= 1e-13 * host.eps, (i, eps.value, host.eps)
        if adapt_metric:
            assert np.allclose(minv, host.Minv, rtol=1e-12, atol=0), i
        else:
            assert (minv == 1.0).all()
    lib.emu_pooled_destroy(h)


def test_trajectory_kernel_emulated_nonfinite_freeze_tempering_and_fast_path_fallback(emu_lf):
    """K1 under emulation on the awkward inputs: a chain that overflows freezes on its own at the break step with -Inf
    energies while its warp-mates finish (integrator.jl:252-258, hamiltonian.jl:95-104); tempering (exact path,
    integrator.jl:198-209); a chain whose magnitude defeats the fast path's proof is redone by the exact path in-launch."""
    rng = np.random.default_rng(31)
    # (a) per-chain freeze, std-normal / unit (fast-path kernel with in-launch exact fallback)
    D, N, n = 3, 6, 5
    model, metric = oc.Model(oc.STD_NORMAL, D), oc.Metric(oc.UNIT)
    th, r = np.ones((N, D)), np.ones((N, D))
    th[2] = 1e200
    th[4] = 1e120  # large but finite throughout: defeats the magnitude proof, must equal the exact result
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    zo, so, do = oc.leapfrog(model, metric, 0.1, z0, n)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g", "dr")}
    lp_o, lk_o = np.zeros(N), np.zeros(N)
    status, done = np.zeros(N, dtype=np.uint32), np.zeros(N, dtype=np.int32)
    g_in, lp_in = np.ascontiguousarray(z0.lp_gradient.T), np.ascontiguousarray(z0.lp_value)
    q = EmuLf(model_kind=oc.STD_NORMAL, metric_kind=oc.UNIT, D=D, N=N, p0=None, p1=None, c0=0.0, Minv=None, minv_stride=0, cholU=None,
              eps=0.1, eps_chain=None, n_steps=n, fwd=1, temper_alpha=0.0, th_in=P(th), r_in=P(r), g_in=P(g_in), lp_in=P(lp_in),
              th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o), dr_out=P(o["dr"]),
              status=P(status), steps_done=P(done), flags=0, hmc=0)
    assert emu_lf.emu_leapfrog(C.byref(q)) == 0
    assert list(status) == list(so) and list(done) == list(do) and done[2] == 1 and status[2] == 1
    ok = status == 0
    assert rel_err(o["th"][ok].T, zo.theta[:, ok]) < 1e-10 and np.allclose(lp_o[ok], zo.lp_value[ok], rtol=1e-10)
    assert lp_o[2] == -np.inf and zo.lp_value[2] == -np.inf
    # (b) tempering on a diagonal Gaussian (exact path)
    D, N, n = 6, 5, 8
    model, metric, p0, dp1, Minv, cholU = _lf_system("diag_gauss", "diag", D, rng)
    th, r = rng.normal(size=(N, D)), rng.normal(size=(N, D))
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    zo, so, do = oc.leapfrog(model, metric, 0.1, z0, n, temper_alpha=1.05)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g", "dr")}
    lp_o, lk_o = np.zeros(N), np.zeros(N)
    g_in, lp_in = np.ascontiguousarray(z0.lp_gradient.T), np.ascontiguousarray(z0.lp_value)
    q = EmuLf(model_kind=oc.DIAG_GAUSS, metric_kind=oc.DIAG, D=D, N=N, p0=P(p0), p1=P(dp1), c0=0.0, Minv=P(Minv), minv_stride=0,
              cholU=None, eps=0.1, eps_chain=None, n_steps=n, fwd=1, temper_alpha=1.05, th_in=P(th), r_in=P(r), g_in=P(g_in),
              lp_in=P(lp_in), th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o), dr_out=P(o["dr"]),
              status=None, steps_done=None, flags=0, hmc=0)
    assert emu_lf.emu_leapfrog(C.byref(q)) == 0
    assert rel_err(o["th"].T, zo.theta) < 1e-10 and rel_err(o["r"].T, zo.r) < 1e-10
    assert np.allclose(lk_o, zo.lk_value, rtol=1e-10, atol=1e-10)


# ---------------------------------------------------------------------------------------------------------------- K4
@pytest.fixture(scope="module")
def emu_dense():
    lib = E.harness("dense")
    assert lib.emu_dense_stages() == 3
    return lib


def _dense_run(lib, kind, mkind, D, N, eps, n, fwd, seed, per_chain_eps=True, wide=0, poison=None):
    rng = np.random.default_rng(seed)
    model, metric, p0, dp1, Minv, _ = _lf_system(kind, mkind, D, rng)
    th, r = rng.normal(size=(N, D)), rng.normal(size=(N, D))
    eps_chain = eps * np.exp(rng.uniform(-0.3, 0.3, N)) if per_chain_eps else None
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    zo = oc.leapfrog(model, metric, eps_chain if per_chain_eps else eps, z0, n if fwd else -n)[0]
    g_in = np.ascontiguousarray(z0.lp_gradient.T)
    if poison is not None:
        th[poison, 0] = 1e250  # beyond the magnitude proof: the whole tile must be handed to the exact kernel
    o = {k: np.full((N, D), np.nan) for k in ("th", "r", "g", "dr")}
    lp_o, lk_o = np.full(N, np.nan), np.full(N, np.nan)
    status, done, need = np.full(N, 7, dtype=np.uint32), np.zeros(N, dtype=np.int32), np.full(N, 9, dtype=np.uint8)
    Pm = np.asfortranarray(dp1) if kind == "dense_gauss" else None
    w = dp1 if kind == "diag_gauss" else None
    Mm = np.asfortranarray(Minv) if mkind == "dense" else None
    Md = Minv if mkind == "diag" else None
    q = EmuDense(D=D, N=N, P=P(Pm), w=P(w), mu=P(p0), c0=0.0, Minv=P(Mm), Mdiag=P(Md), eps=eps, eps_chain=P(eps_chain), n_steps=n,
                 fwd=fwd, th_in=P(th), r_in=P(r), g_in=P(g_in), th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]),
                 dr_out=P(o["dr"]), lp_out=P(lp_o), lk_out=P(lk_o), status=P(status), steps_done=P(done), need_exact=P(need),
                 wide_tile=wide)
    assert lib.emu_dense(C.byref(q)) == 0
    nM = np.abs(Minv).sum(axis=1).max() if mkind == "dense" else (np.abs(Minv).max() if mkind == "diag" else 1.0)
    nP = np.abs(dp1).sum(axis=1).max() if kind == "dense_gauss" else (np.abs(dp1).max() if kind == "diag_gauss" else 1.0)
    assert np.isclose(q.norms_out[0], nM, rtol=1e-13) and np.isclose(q.norms_out[1], nP, rtol=1e-13)
    return zo, o, lp_o, lk_o, status, done, need


DENSE_CASES = [("dense_gauss", "dense", 40, 37, 0.1, 5, 1, True, 0),    # Dp = 64: <1,4>, two ragged 32-chain tiles
               ("dense_gauss", "diag", 100, 20, 0.08, 4, 0, True, 0),   # Dp = 128: default <2,2,2>, backward
               ("diag_gauss", "dense", 70, 33, 0.12, 3, 1, False, 1),   # Dp = 128: the 32-chain form, shared eps
               ("dense_gauss", "dense", 130, 17, 0.05, 2, 1, True, 0),  # Dp = 192: <3,2>
               ("dense_gauss", "unit", 64, 8, 0.1, 1, 1, False, 0)]     # D == Dp, a single step (half kicks only)


@pytest.mark.parametrize("kind,mkind,D,N,eps,n,fwd,pce,wide", DENSE_CASES, ids=[f"{c[0]}-{c[1]}-D{c[2]}" for c in DENSE_CASES])
def test_dense_tile_kernel_source_under_emulation_matches_oracle(emu_dense, kind, mkind, D, N, eps, n, fwd, pce, wide):
    """K4 (`dense_traj_kernel`: bulk-copy pipeline on mbarriers, DMMA fragment layout, tile staging, padding, ragged tiles,
    energy reduction) executed by the emulator vs the oracle's `step`; `pad_norm_kernel` / `vec_norm_kernel` too."""
    zo, o, lp_o, lk_o, status, done, need = _dense_run(emu_dense, kind, mkind, D, N, eps, n, fwd, seed=100 + D, per_chain_eps=pce,
                                                       wide=wide)
    assert (need == 0).all() and (done == n).all() and (status == 0).all()
    assert rel_err(o["th"].T, zo.theta) < 1e-10 and rel_err(o["r"].T, zo.r) < 1e-10 and rel_err(o["g"].T, zo.lp_gradient) < 1e-10
    assert np.allclose(lp_o, zo.lp_value, rtol=1e-10, atol=1e-10) and np.allclose(lk_o, zo.lk_value, rtol=1e-10, atol=1e-10)
    assert rel_err(o["dr"].T, zo.lk_gradient) < 1e-10


def test_dense_tile_kernel_emulated_hands_a_suspect_tile_to_the_exact_kernel(emu_dense):
    """a magnitude beyond the linear-dynamics proof flags the WHOLE tile (`need_exact`), writes nothing for it, and leaves
    the other tile's results intact"""
    N, D = 37, 40
    zo, o, lp_o, lk_o, status, done, need = _dense_run(emu_dense, "dense_gauss", "dense", D, N, 0.1, 3, 1, seed=5, poison=34)
    assert (need[:32] == 0).all() and (need[32:] == 1).all()
    assert np.isnan(o["th"][32:]).all() and np.isnan(lp_o[32:]).all() and (status[32:] == 7).all()
    assert rel_err(o["th"][:32].T, zo.theta[:, :32]) < 1e-10 and np.allclose(lk_o[:32], zo.lk_value[:32], rtol=1e-10)


# ------------------------------------------------------------------------------- data-race check of the kernel sources
_RACE_HARNESS = {"nuts": "nuts", "lf": "lf", "multinomial": "mn", "adapt": "adapt", "dense": "dense",
                 "dense-mutant": "dense"}  # with a copy of ahmc_dense.cu with one barrier removed: the detector must fire


@pytest.fixture(scope="module")
def _race_runs(tmp_path_factory):
    """each program's outcome (the run, or the skip), all built and run at once"""
    mut = tmp_path_factory.mktemp("mutant")
    src = open(os.path.join(E.CSRC, "ahmc_dense.cu")).read()
    barrier = "= v[rb][cb][j];\n    __syncthreads();"  # tile_to_smem: publish the staged vectors to the other warps
    assert src.count(barrier) == 1
    (mut / "ahmc_dense.cu").write_text(src.replace(barrier, "= v[rb][cb][j];"))
    with cf.ThreadPoolExecutor(max_workers=len(_RACE_HARNESS)) as ex:
        return {name: ex.submit(E.sanitized, h, "thread", include_first=str(mut) if name == "dense-mutant" else None, timeout=600)
                for name, h in _RACE_HARNESS.items()}


@pytest.mark.parametrize("name", list(_RACE_HARNESS))
def test_kernel_sources_are_data_race_free_under_thread_sanitizer(_race_runs, name):
    """Every CUDA thread is a host thread whose only synchronisation is what the kernel asks for, so ThreadSanitizer sees a
    missing __syncwarp / __syncthreads / mbarrier wait as a data race: the shipped NUTS, trajectory / HMC, MultinomialTS, adaptor-statistics
    and dense-tile sources must be clean, and a copy of the dense kernel with one barrier removed must be reported."""
    r = _race_runs[name].result()
    races = r.stderr.count("WARNING: ThreadSanitizer: data race")
    if name == "dense-mutant":
        assert races > 0 and "dense_traj_kernel" in r.stderr
    else:
        assert races == 0 and r.returncode == 0, r.stderr[-3000:] + r.stdout[-500:]
        assert r.stdout.count("rc 0") == {"nuts": 8, "lf": 5, "dense": 4, "multinomial": 3, "adapt": 1}[name.split("-")[0]]


def test_host_window_schedule_of_the_in_launch_adaptation_equals_the_oracle(emu):
    """`stan_window_schedule` (ahmc_kernels.cuh: the host code `ahmc_nuts_adapt_sample_f64` runs before the launch) against
    the oracle's `initialize!` restatement for every n_adapts up to 1300 and several buffer settings; the reference's own
    expectation for n_adapts = 1000 (test/adaptation.jl:131-151); more splits than the device struct holds is refused."""
    ws, we, sp = C.c_int(), C.c_int(), (C.c_int * 16)()
    n = emu.emu_window_schedule(75, 50, 25, 1000, C.byref(ws), C.byref(we), sp)
    assert (ws.value, we.value, list(sp[:n])) == (76, 950, [100, 150, 250, 450, 950])
    for ib, tb, wsz in ((75, 50, 25), (3, 2, 4), (0, 0, 1), (10, 0, 7), (100, 100, 50)):
        for n_adapts in range(0, 1301):
            n = emu.emu_window_schedule(ib, tb, wsz, n_adapts, C.byref(ws), C.byref(we), sp)
            ows, owe, osp = oc.stan_windows(n_adapts, ib, tb, wsz)
            if len(osp) > 12:
                assert n == -1
                continue
            assert (ws.value, we.value, list(sp[:n])) == (ows, owe, osp), (ib, tb, wsz, n_adapts)
    assert emu.emu_window_schedule(0, 0, 1, 100000, C.byref(ws), C.byref(we), sp) == -1
