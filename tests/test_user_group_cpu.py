"""CPU tests of the group form of run-time compiled targets (`#define AHMC_USER_GROUPWISE`, ahmc_user_logp_grad_group):
the library's embedded kernel sources compile under NVRTC with group-form targets for every kernel, metric and layout, broken
sources come back with their logs, and the unmodified kernel sources run a group-form funnel under the CPU SIMT emulator
(tests/simt_emu/) with the results of the C oracle's built-in funnel."""
import concurrent.futures as cf
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

import ahmc_b200 as A
from oracle import oracle_c as oc
from tests.helpers import rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_vp = C.c_void_p
P = lambda a: None if a is None else a.ctypes.data_as(_vp)

FUNNEL = r'''
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
    ahmc_group_sync(grp);
    const double S = ahmc_group_sum(grp, s);
    if (grp.lane != 0) return 0.0;
    g[0] = -v / 9.0 + (S - (D - 1)) * 0.5;
    return -v * v / 18.0 - (S + (D - 1) * v) * 0.5;
}
'''


def _lib_or_skip():
    lib = A._lib.load()
    log = C.create_string_buffer(4096)
    if lib.ahmc_user_source_check(FUNNEL.encode(), 0, 0, 3, log, 4096) == A._lib.ERR_UNSUPPORTED:
        pytest.skip("libnvrtc not available here: " + log.value.decode())
    return lib


def _check(lib, src, kernel, metric, D):
    log = C.create_string_buffer(8192)
    rc = lib.ahmc_user_source_check(src.encode(), kernel, metric, D, log, 8192)
    return rc, log.value.decode()


def test_group_form_sources_compile_for_every_kernel_metric_and_layout():
    """kernels 0..6 (phasepoint, trajectory, static HMC, NUTS, find_good_stepsize, adaptive NUTS, adaptive static HMC) x
    Unit / Diag / Dense x D in {3, 10, 128, 512} (G = 4, 16, 32, 32), for the funnel and the logistic regression"""
    lib = _lib_or_skip()
    spec = importlib.util.spec_from_file_location("user_group_cost", os.path.join(ROOT, "scripts", "user_group_cost.py"))
    cost = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cost)
    jobs = [(src, kernel, metric, D) for D in (3, 10, 128, 512) for src in (FUNNEL, cost.logreg_sources(1000, D)[1])
            for kernel in range(7) for metric in (0, 1, 2)]
    with cf.ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        results = list(ex.map(lambda j: _check(lib, *j), jobs))
    for (src, kernel, metric, D), (rc, log) in zip(jobs, results):
        assert rc == 0, (kernel, metric, D, log[-2000:])


def test_group_form_sources_that_do_not_compile_come_back_with_their_logs():
    lib = _lib_or_skip()
    both = "#define AHMC_USER_COORDWISE\n" + FUNNEL
    rc, log = _check(lib, both, 1, 1, 10)
    assert rc == A._lib.ERR_INVALID and "AHMC_USER_COORDWISE" in log and "AHMC_USER_GROUPWISE" in log, log
    rc, log = _check(lib, FUNNEL.replace("return 0.0;", "return nope;"), 3, 1, 10)
    assert rc == A._lib.ERR_INVALID and "nope" in log and "undefined" in log, log
    with pytest.raises(A.InvalidArgument):
        A.UserTarget.check_source(both, 10)
    A.UserTarget.check_source(FUNNEL, 10)


class EmuUser(C.Structure):
    _fields_ = [("op", C.c_int32), ("metric_kind", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("c0", C.c_double),
                ("Minv", _vp), ("cholU", _vp), ("eps", C.c_double), ("n_steps", C.c_int32), ("max_depth", C.c_int32),
                ("exp_tape", _vp), ("exp_stride", C.c_int64), ("dir_tape", _vp), ("dir_stride", C.c_int64),
                ("th_in", _vp), ("r_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp), ("r_out", _vp), ("g_out", _vp),
                ("lp_out", _vp), ("lk_out", _vp), ("steps", _vp), ("tree_depth", _vp), ("numerical", _vp), ("acc", _vp)]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the group-form harness (kernel sources + emulator + the funnel as a C++ definition), compiled once"""
    tmp = tmp_path_factory.mktemp("simt_user_group")
    d = os.path.join(ROOT, "tests", "simt_emu")
    out = tmp / "libuser_group_emu.so"
    cmd = ["g++", "-O1", "-std=c++20", "-shared", "-fPIC", "-pthread", "-ffp-contract=off", "-I", os.path.join(d, "include"),
           "-I", os.path.join(ROOT, "advancedhmc.jl_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
           os.path.join(d, "simt_emu.cpp"), os.path.join(d, "user_group_emu.cpp"), "-o", str(out)]
    pr = subprocess.run(cmd, capture_output=True, text=True)
    assert pr.returncode == 0, pr.stderr[-2000:]
    return C.CDLL(str(out))


MKINDS = dict(unit=oc.UNIT, diag=oc.DIAG, dense=oc.DENSE)


def _metric(mkind, D, rng):
    Minv = cholU = None
    if mkind == "diag":
        Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    elif mkind == "dense":
        B = rng.normal(size=(D, D))
        Minv = B @ B.T / D + 0.5 * np.eye(D)
        cholU = np.ascontiguousarray(np.linalg.cholesky(Minv).T.T)
    return Minv, cholU, oc.Metric(MKINDS[mkind], None if Minv is None else np.asfortranarray(Minv))


def _run(lib, **kw):
    q = EmuUser(**kw)
    assert lib.emu_user_group(C.byref(q)) == 0


@pytest.mark.parametrize("mkind,D,N", [("unit", 3, 11), ("diag", 3, 9), ("dense", 3, 5), ("diag", 20, 3), ("dense", 40, 2),
                                       ("unit", 40, 3)])
def test_emulated_phasepoint_and_trajectory_match_the_oracle(emu, mkind, D, N):
    """phasepoint and 9 exact-path steps (with and without a cached gradient) of the group-form funnel: G = 4 (eight chains
    per warp, a ragged last warp) and G = 32"""
    rng = np.random.default_rng(100 + D + N)
    Minv, cholU, ome = _metric(mkind, D, rng)
    om = oc.Model(oc.FUNNEL, D, None, None, 0.5)
    th, r = rng.normal(size=(N, D)) * 0.5, rng.normal(size=(N, D))
    z0 = oc.phasepoint(om, ome, th.T, r.T)
    lp, lk, g = np.zeros(N), np.zeros(N), np.zeros((N, D))
    _run(emu, op=0, metric_kind=MKINDS[mkind], D=D, N=N, c0=0.5, Minv=P(Minv), cholU=P(cholU), th_in=P(th), r_in=P(r),
         g_out=P(g), lp_out=P(lp), lk_out=P(lk))
    assert rel_err(lp, z0.lp_value) < 1e-13 and rel_err(lk, z0.lk_value) < 1e-13 and rel_err(g.T, z0.lp_gradient) < 1e-13
    zo, _, done = oc.leapfrog(om, ome, 0.1, z0, 9)
    g_in, lp_in = g, lp  # the kernel's own phasepoint: the recomputed start gradient must then give identical bits
    outs = []
    for cached in (True, False):
        o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
        lpo, lko, steps = np.zeros(N), np.zeros(N), np.zeros(N, dtype=np.int32)
        _run(emu, op=1, metric_kind=MKINDS[mkind], D=D, N=N, c0=0.5, Minv=P(Minv), cholU=P(cholU), eps=0.1, n_steps=9, th_in=P(th),
             r_in=P(r), g_in=P(g_in) if cached else None, lp_in=P(lp_in), th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]),
             lp_out=P(lpo), lk_out=P(lko), steps=P(steps))
        assert (steps == done).all()
        assert rel_err(o["th"].T, zo.theta) < 1e-11 and rel_err(o["r"].T, zo.r) < 1e-11 and rel_err(o["g"].T, zo.lp_gradient) < 1e-11
        assert rel_err(lpo, zo.lp_value) < 1e-11 and rel_err(lko, zo.lk_value) < 1e-11
        outs.append(o["th"])
    assert np.array_equal(outs[0], outs[1])


def test_emulated_trajectory_of_a_chain_that_stops_on_a_nonfinite_step(emu):
    """one chain of a warp of eight blows up and stops; its warp keeps evaluating the model for the others"""
    D, N = 3, 8
    rng = np.random.default_rng(7)
    om, ome = oc.Model(oc.FUNNEL, D, None, None, 0.0), oc.Metric(oc.UNIT, None)
    th, r = rng.normal(size=(N, D)) * 0.5, rng.normal(size=(N, D))
    th[5, 0] = -700.0  # e^-v overflows within a step
    z0 = oc.phasepoint(om, ome, th.T, r.T)
    zo, _, done = oc.leapfrog(om, ome, 0.1, z0, 6)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lpo, lko, steps = np.zeros(N), np.zeros(N), np.zeros(N, dtype=np.int32)
    _run(emu, op=1, metric_kind=oc.UNIT, D=D, N=N, eps=0.1, n_steps=6, th_in=P(th), r_in=P(r), g_in=None,
         lp_in=P(np.ascontiguousarray(z0.lp_value)), th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lpo),
         lk_out=P(lko), steps=P(steps))
    assert (steps == done).all() and done[5] < 6 and (np.delete(done, 5) == 6).all()
    keep = np.arange(N) != 5
    assert rel_err(o["th"][keep].T, zo.theta[:, keep]) < 1e-11 and lpo[5] == -np.inf


@pytest.mark.parametrize("mkind,D,N,eps,scale", [("unit", 3, 11, 0.9, 2.0), ("diag", 3, 9, 0.5, 1.5), ("diag", 20, 3, 0.12, 0.6),
                                                 ("dense", 40, 2, 0.1, 0.5)])
def test_emulated_nuts_transition_matches_the_oracle(emu, mkind, D, N, eps, scale):
    """one NUTS transition (MultinomialTS + GeneralisedNoUTurn) on shared tapes: identical trees, states within 1e-10; at
    G = 4 the chains of a warp sit at different tree positions"""
    max_depth = 8
    rng = np.random.default_rng(200 + D + N)
    Minv, cholU, ome = _metric(mkind, D, rng)
    om = oc.Model(oc.FUNNEL, D, None, None, 0.0)
    th = rng.normal(size=(N, D)) * scale
    r = rng.normal(size=(N, D))
    dirs = rng.integers(0, 2, size=(N, max_depth + 1)).astype(np.uint8)
    exps = rng.exponential(size=(N, 1 << max_depth))
    z0 = oc.phasepoint(om, ome, th.T, r.T)
    zo, so, _ = oc.nuts_transition(om, ome, eps, z0, None, dirs, exps, max_depth=max_depth)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
    lpo, lko, acc = np.zeros(N), np.zeros(N), np.zeros(N)
    ns, td, ne = np.zeros(N, dtype=np.int32), np.zeros(N, dtype=np.int32), np.zeros(N, dtype=np.uint8)
    _run(emu, op=2, metric_kind=MKINDS[mkind], D=D, N=N, Minv=P(Minv), cholU=P(cholU), eps=eps, max_depth=max_depth,
         exp_tape=P(exps), exp_stride=exps.shape[1], dir_tape=P(dirs), dir_stride=dirs.shape[1], th_in=P(th), r_in=P(r),
         g_in=P(np.ascontiguousarray(z0.lp_gradient.T)), lp_in=P(np.ascontiguousarray(z0.lp_value)), th_out=P(o["th"]),
         r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lpo), lk_out=P(lko), steps=P(ns), tree_depth=P(td), numerical=P(ne), acc=P(acc))
    assert (td == so.tree_depth).all() and (ns == so.n_steps).all() and (ne == so.numerical_error).all()
    assert rel_err(o["th"].T, zo.theta) < 1e-10 and rel_err(o["r"].T, zo.r) < 1e-10 and rel_err(o["g"].T, zo.lp_gradient) < 1e-10
    assert np.allclose(lpo, zo.lp_value, rtol=1e-10, atol=1e-10) and np.allclose(acc, so.acceptance_rate, rtol=1e-10)
    assert ns.max() >= 3
