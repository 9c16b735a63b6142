"""CPU tests of the GLM targets: the chain-tile kernel source (ahmc_glm.cu, unmodified) under the SIMT emulator against the
float64 numpy statement of the target (tests/glm_ref.py), the stable link-function branches against 50-digit values, and
the generated group-form source through the compile-only check."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ahmc_b200 as A
from tests import glm_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_vp = C.c_void_p
FAM = {"bernoulli_logit": 0, "poisson_log": 1}


class EmuGlm(C.Structure):
    _fields_ = [("family", C.c_int32), ("D", C.c_int32), ("n", C.c_int32), ("N", C.c_int64), ("X", _vp), ("y", _vp), ("prec", _vp),
                ("c0", C.c_double), ("Minv", _vp), ("chain_stride", C.c_int64), ("eps", C.c_double), ("eps_chain", _vp),
                ("n_steps", C.c_int32), ("fwd", C.c_int32), ("th_in", _vp), ("r_in", _vp), ("g_in", _vp), ("th_out", _vp),
                ("r_out", _vp), ("g_out", _vp), ("dr_out", _vp), ("lp_out", _vp), ("lk_out", _vp), ("status", _vp),
                ("steps_done", _vp), ("nc_out", C.c_int32), ("stages_out", C.c_int32)]


def P(a):
    return None if a is None else a.ctypes.data_as(_vp)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("simt_glm")
    d = os.path.join(ROOT, "tests", "simt_emu")
    out = tmp / "libglm_emu.so"
    cmd = ["g++", "-O1", "-std=c++20", "-shared", "-fPIC", "-pthread", "-ffp-contract=off", "-x", "c++",
           "-I", os.path.join(d, "include"), "-I", os.path.join(ROOT, "advancedhmc.jl_b200", "csrc"),
           "-I", os.path.join(ROOT, "include"), os.path.join(d, "simt_emu.cpp"), os.path.join(d, "glm_emu.cpp"), "-o", str(out)]
    pr = subprocess.run(cmd, capture_output=True, text=True)
    assert pr.returncode == 0, pr.stderr[-3000:]
    return C.CDLL(str(out))


def run_emu(lib, family, X, y, prec, c0, Minv, eps, n_steps, th, r, g, in_place=False):
    N, D = th.shape
    th, r = np.ascontiguousarray(th), np.ascontiguousarray(r)
    o = {k: np.full((N, D), np.nan) for k in ("th", "r", "g", "dr")}
    if in_place:
        o["th"], o["r"] = th, r
    o["lp"], o["lk"] = np.full(N, np.nan), np.full(N, np.nan)
    status, steps = np.full(N, 7, dtype=np.uint32), np.full(N, -1, dtype=np.int32)
    eps_chain = None if np.isscalar(eps) else np.ascontiguousarray(eps)
    Mv = None if Minv is None else np.ascontiguousarray(Minv)
    q = EmuGlm(family=FAM[family], D=D, n=len(y), N=N, X=P(X), y=P(y), prec=P(prec), c0=c0, Minv=P(Mv),
               chain_stride=0 if Mv is None or Mv.ndim == 1 else D, eps=eps if eps_chain is None else 0.0,
               eps_chain=P(eps_chain), n_steps=abs(n_steps), fwd=1 if n_steps >= 0 else 0, th_in=P(th), r_in=P(r), g_in=P(g),
               th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), dr_out=P(o["dr"]), lp_out=P(o["lp"]), lk_out=P(o["lk"]),
               status=P(status), steps_done=P(steps))
    assert lib.emu_glm(C.byref(q)) == 0
    return o, status, steps, (q.nc_out, q.stages_out)


def close(a, b, tol=1e-10):
    a, b = np.asarray(a), np.asarray(b)
    assert (np.isfinite(a) == np.isfinite(b)).all()
    m = np.isfinite(a)
    assert np.abs(a[m] - b[m]).max(initial=0.0) <= tol * (1.0 + np.abs(b[m]).max(initial=0.0))
    assert np.array_equal(a[~m], b[~m], equal_nan=True)


def assert_z(o, z, tol=1e-10):
    for k in ("th", "r", "g", "dr", "lp", "lk"):
        close(o[k], z[k], tol)


# (family, D, n, N, n_steps, metric, per-chain eps, cached gradient): the tile shapes RB = 1..3, one and several chunks, a
# chunk boundary at n = 63 / 64 / 65, ragged tiles, backward, a shared and a per-chain Diag metric, no cached gradient
CASES = [("bernoulli_logit", 1, 1, 3, 2, "unit", False, True),
         ("poisson_log", 7, 63, 17, 3, "diag", True, True),
         ("bernoulli_logit", 8, 64, 16, -2, "chain", True, True),
         ("poisson_log", 25, 65, 21, 2, "diag", False, False),
         ("bernoulli_logit", 100, 200, 19, 2, "chain", True, False),
         ("poisson_log", 130, 70, 5, -1, "unit", True, True)]


def _setup(family, D, n, N, metric, pce, seed):
    rng = np.random.default_rng(seed)
    X, y, beta = R.data(family, n, D, seed, scale=0.5)
    prec = rng.uniform(0.5, 2.0, D)
    Minv = None if metric == "unit" else rng.uniform(0.5, 2.0, D if metric == "diag" else (N, D))
    th, r = beta + 0.1 * rng.normal(size=(N, D)), rng.normal(size=(N, D))
    eps = 0.02 * np.exp(rng.uniform(-0.3, 0.3, N)) if pce else 0.02
    return X, y, prec, Minv, th, r, eps


@pytest.mark.parametrize("family,D,n,N,n_steps,metric,pce,cached", CASES, ids=[f"{c[0]}-D{c[1]}-n{c[2]}" for c in CASES])
def test_tile_kernel_source_under_emulation_matches_reference(emu, family, D, n, N, n_steps, metric, pce, cached):
    X, y, prec, Minv, th, r, eps = _setup(family, D, n, N, metric, pce, seed=D + n)
    z0 = R.phasepoint(family, X, y, prec, 0.25, Minv, th, r)
    o, status, steps, _ = run_emu(emu, family, X, y, prec, 0.25 - (0 if family == "bernoulli_logit" else R.gammaln(y + 1).sum()),
                                  Minv, 0.0, 0, th, r, None)  # phasepoint: energies, gradient, dH/dr
    for k in ("g", "dr", "lp", "lk"):
        close(o[k], z0[k])
    zo, st_ref, steps_ref = R.leapfrog(family, X, y, prec, 0.25, Minv, eps, z0, n_steps)
    c0 = 0.25 - (0 if family == "bernoulli_logit" else R.gammaln(y + 1).sum())
    o, status, steps, _ = run_emu(emu, family, X, y, prec, c0, Minv, eps, n_steps, th.copy(), r.copy(),
                                  np.ascontiguousarray(z0["g"]) if cached else None, in_place=True)
    assert_z(o, zo)
    assert (status == st_ref).all() and (steps == steps_ref).all() and (status == 0).all()


@pytest.mark.parametrize("family", ["bernoulli_logit", "poisson_log"])
def test_a_non_finite_chain_stops_alone_and_leaves_its_tile_untouched(emu, family):
    """Chain 3 goes non-finite (log pi = -Inf from a 1e200 start; a Poisson exp that overflows): it stops at that step with
    AHMC_STATUS_NONFINITE, and every other chain of its tile is bit for bit what it is in a run without the bad chain."""
    D, n, N, steps_n = 9, 40, 13, 3
    X, y, prec, Minv, th, r, eps = _setup(family, D, n, N, "diag", True, seed=5)
    c0 = 0.0 - (0 if family == "bernoulli_logit" else R.gammaln(y + 1).sum())
    g = R.phasepoint(family, X, y, prec, 0.0, Minv, th, r)["g"]
    good, st_g, _, _ = run_emu(emu, family, X, y, prec, c0, Minv, eps, steps_n, th, r, g)
    bad_th, bad_r = th.copy(), r.copy()
    if family == "bernoulli_logit":
        bad_th[3] = 1e200
    else:
        bad_r[3] = 4e4 * np.sign(X[0])  # drives eta of row 0 past 709 within the first step
    gb = R.phasepoint(family, X, y, prec, 0.0, Minv, bad_th, bad_r)["g"]
    o, status, steps, _ = run_emu(emu, family, X, y, prec, c0, Minv, eps, steps_n, bad_th, bad_r, gb)
    zo, st_ref, steps_ref = R.leapfrog(family, X, y, prec, 0.0, Minv, eps,
                                       dict(R.phasepoint(family, X, y, prec, 0.0, Minv, bad_th, bad_r)), steps_n)
    assert status[3] == 1 and steps[3] == steps_ref[3] < steps_n and o["lp"][3] == -np.inf
    assert (status == st_ref).all() and (steps == steps_ref).all()
    keep = np.arange(N) != 3
    for k in ("th", "r", "g", "dr", "lp", "lk"):
        assert np.array_equal(o[k][keep], good[k][keep])


def test_stable_link_branches_match_50_digit_values():
    """tests/golden/glm_mp50.json (gen_glm_mp.py): log pi and its gradient for rows with eta = +-40 and +-750, where a naive
    softplus / sigmoid overflows; Poisson at eta = 750 is non-finite."""
    import json

    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "glm_mp50.json")))
    for case in gold["cases"]:
        X, y, th = np.array(case["X"]), np.array(case["y"]), np.array(case["theta"])[None, :]
        prec = np.array(case["prec"])
        lp, g = R.logp_mgrad(case["family"], X, y, prec, 0.0, th)
        if case["lp"] is None:
            assert not np.isfinite(lp[0])
            continue
        assert abs(lp[0] - float(case["lp"])) <= 1e-13 * (1 + abs(float(case["lp"])))
        ref = -np.array([float(v) for v in case["grad"]])
        assert np.abs(g[0] - ref).max() <= 1e-13 * (1 + np.abs(ref).max())


def test_emulated_kernel_matches_50_digit_values(emu):
    import json

    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "glm_mp50.json")))
    for case in gold["cases"]:
        X, y, th = np.array(case["X"]), np.array(case["y"]), np.array(case["theta"])[None, :]
        c0 = 0.0 - (0 if case["family"] == "bernoulli_logit" else R.gammaln(y + 1).sum())
        o, _, _, _ = run_emu(emu, case["family"], X, y, np.array(case["prec"]), c0, None, 0.0, 0, th, np.zeros_like(th), None)
        if case["lp"] is None:
            assert o["lp"][0] == -np.inf
            continue
        assert abs(o["lp"][0] - float(case["lp"])) <= 1e-10 * (1 + abs(float(case["lp"])))
        ref = -np.array([float(v) for v in case["grad"]])
        assert np.abs(o["g"][0] - ref).max() <= 1e-10 * (1 + np.abs(ref).max())


def test_tile_shapes_fit_shared_memory(emu):
    """D <= 128 streams 64-row chunks; the shape shrinks the chunk beyond that and is refused beyond 256"""
    rng = np.random.default_rng(0)
    for D, want_nc in ((25, 64), (100, 64), (128, 64), (256, 32)):
        X, y, _ = R.data("bernoulli_logit", 8, D, 1)
        th = rng.normal(size=(1, D)) * 0.01
        _, _, _, (nc, stages) = run_emu(emu, "bernoulli_logit", X, y, np.ones(D), 0.0, None, 0.0, 0, th, th, None)
        assert nc == want_nc and stages in (2, 3)


@pytest.mark.parametrize("family", ["bernoulli_logit", "poisson_log"])
@pytest.mark.parametrize("D", [3, 25, 100, 300])
def test_generated_group_source_compiles(family, D):
    """the source a GLM target runs as on the run-time compiled kernels passes the compile-only check (needs NVRTC, no GPU)"""
    lib = A._lib.load()
    log = C.create_string_buffer(4096)
    probe = "__device__ double ahmc_user_logp_grad(const double* t, double* g, int D, const double* p) { return 0.0; }"
    if lib.ahmc_user_source_check(probe.encode(), 1, 1, 4, log, 4096) == A._lib.ERR_UNSUPPORTED:
        pytest.skip("NVRTC is not available: " + log.value.decode())
    n = lib.ahmc_glm_source(FAM[family], D, 1000, None, 0)
    buf = C.create_string_buffer(n + 1)
    assert lib.ahmc_glm_source(FAM[family], D, 1000, buf, n + 1) == n
    src = buf.value
    assert b"AHMC_USER_GROUPWISE" in src and f"GLM_D {D}".encode() in src
    for kernel, metric in ((1, 0), (2, 1), (3, 2)):
        assert lib.ahmc_user_source_check(src, kernel, metric, D, log, 4096) == 0, log.value.decode()
