"""The trajectory kernels' addressing at a leading dimension ld > D, on the CPU: each kernel source runs under the SIMT
emulator (tests/simt_emu) on buffers whose padding rows D..ld-1 and a guard tail after the last chain hold a NaN canary,
with z_in.ld != z_out.ld.  Every run must return the ld = D run's D x N blocks and scalars bit for bit, leave every canary
and every input as it was, and agree with the oracle to 1e-10.  The pair kernel is called directly, so it also runs at an
ld the launcher's alignment test would send to the one-chain kernel."""
import ctypes as C

import numpy as np
import pytest
from scipy.special import gammaln

from oracle import oracle_c as oc
from tests import emu as E
from tests import glm_ref as R
from tests.emu import P, EmuDense, EmuGlm, EmuLf, EmuMn, EmuNuts
from tests.helpers import rel_err
from tests.test_simt_emulation import KINDS, MKINDS, _lf_system

TOL = 1e-10
GUARD = 3
CANARY = np.array([0x7FF8DEADBEEF0001], dtype="<i8").view(np.float64)[0]


def pad(a, ld):
    """(N, D) rows -> a flat buffer of ld * N + GUARD doubles holding them at leading dimension ld, the rest the canary"""
    N, D = a.shape
    b = np.full(ld * N + GUARD, CANARY)
    b[: ld * N].reshape(N, ld)[:, :D] = a
    return b


def block(b, N, D, ld):
    return b[: ld * N].reshape(N, ld)[:, :D].copy()


def canaries_intact(b, N, D, ld):
    keep = np.ones(b.size, bool)
    keep[: ld * N].reshape(N, ld)[:, :D] = False
    return np.array_equal(b[keep].view(np.int64), np.full(keep.sum(), CANARY).view(np.int64))


def run(fn, cls, make, ins, outs, N, D, ld_in, ld_out):
    """one harness call: `ins` ((N, D) arrays) padded at ld_in, `outs` (names) at ld_out; `make()` gives the request's other
    fields and the scalar outputs it points at.  -> (the D x N outputs, the scalar outputs)"""
    bufs = {f: pad(a, ld_in) for f, a in ins.items()}
    bufs.update({f: pad(np.zeros((N, D)), ld_out) for f in outs})
    kw, scalars = make()
    q = cls(**kw, **{f: P(b) for f, b in bufs.items()}, ld_in=ld_in, ld_out=ld_out)
    assert fn(C.byref(q)) == 0
    for f, b in bufs.items():
        ld = ld_in if f in ins else ld_out
        assert canaries_intact(b, N, D, ld), (f, ld_in, ld_out, "padding or guard written")
    for f, a in ins.items():
        assert np.array_equal(block(bufs[f], N, D, ld_in), a), (f, "input changed")
    return {f: block(bufs[f], N, D, ld_out) for f in outs}, scalars


def same_as_ld_d(fn, cls, make, ins, outs, N, D, lds):
    """runs at ld = D and at each (ld_in, ld_out) of `lds`; every output bit-identical to the ld = D run's"""
    ref, ref_s = run(fn, cls, make, ins, outs, N, D, D, D)
    for ld_in, ld_out in lds:
        got, got_s = run(fn, cls, make, ins, outs, N, D, ld_in, ld_out)
        for f in outs:
            assert got[f].tobytes() == ref[f].tobytes(), (f, ld_in, ld_out)
        for f in ref_s:
            assert got_s[f].tobytes() == ref_s[f].tobytes(), (f, ld_in, ld_out)
    return ref, ref_s


def _lf_problem(kind, mkind, D, N, seed, n):
    rng = np.random.default_rng(seed)
    model, metric, p0, dp1, Minv, cholU = _lf_system(kind, mkind, D, rng)
    th, r = rng.normal(size=(N, D)), rng.normal(size=(N, D))
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    g = np.ascontiguousarray(z0.lp_gradient.T)
    return model, metric, p0, dp1, Minv, cholU, th, r, g, z0, rng


def _lf_make(kind, mkind, D, N, p0, dp1, Minv, cholU, n, lp_in, **extra):
    def make():
        s = dict(lp_out=np.zeros(N), lk_out=np.zeros(N), status=np.zeros(N, np.uint32), steps_done=np.zeros(N, np.int32))
        kw = dict(model_kind=KINDS[kind], metric_kind=MKINDS[mkind], D=D, N=N, p0=P(p0), p1=P(dp1), c0=0.0, Minv=P(Minv),
                  minv_stride=0, cholU=P(cholU), eps=0.1, eps_chain=None, n_steps=n, fwd=1, temper_alpha=0.0, lp_in=P(lp_in),
                  lp_out=P(s["lp_out"]), lk_out=P(s["lk_out"]), status=P(s["status"]), steps_done=P(s["steps_done"]), flags=0,
                  hmc=0)
        for k, v in extra.items():
            if isinstance(v, np.ndarray):
                s[k] = v.copy()
                kw[k] = P(s[k])
            else:
                kw[k] = v
        return kw, s
    return make


def _assert_leapfrog(got, s, zo):
    for f, want in (("th_out", zo.theta), ("r_out", zo.r), ("g_out", zo.lp_gradient), ("dr_out", zo.lk_gradient)):
        assert rel_err(got[f].T, want) < TOL, f
    assert rel_err(s["lp_out"], zo.lp_value) < TOL and rel_err(s["lk_out"], zo.lk_value) < TOL


LF_OUTS = ("th_out", "r_out", "g_out", "dr_out")


@pytest.mark.parametrize("lds", [[(66, 68), (68, 66)], [(66, 66), (68, 68)]], ids=["in-ne-out", "in-eq-out"])
def test_pair_kernel_at_padded_leading_dimensions(lds):
    """D = 64, N = 7: three pairs and a shadowed last B; chain 2 past the magnitude proof (re-run exactly inside its warp)"""
    D, N, n = 64, 7, 10
    model, metric, p0, dp1, Minv, cholU, th, r, g, z0, rng = _lf_problem("diag_gauss", "diag", D, N, 3, n)
    th[2, 9] = 1e120
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    g = np.ascontiguousarray(z0.lp_gradient.T)
    zo = oc.leapfrog(model, metric, 0.1, z0, n)[0]
    lib = E.harness("pair")
    make = _lf_make("diag_gauss", "diag", D, N, p0, dp1, Minv, cholU, n, z0.lp_value)
    got, s = same_as_ld_d(lib.emu_leapfrog_pair, EmuLf, make, dict(th_in=th, r_in=r, g_in=g), LF_OUTS, N, D, lds)
    _assert_leapfrog(got, s, zo)


@pytest.mark.parametrize("kind,mkind,D,N", [("diag_gauss", "diag", 7, 9), ("funnel", "diag", 6, 7), ("dense_gauss", "dense", 6, 5),
                                            ("diag_gauss", "diag", 40, 3), ("std_normal", "unit", 64, 3)])
def test_one_chain_kernel_at_odd_leading_dimensions(kind, mkind, D, N):
    """K1's one-chain (and grouped) kernel: fast, exact and dense-slab paths; at D = 64 the harness's lane-contiguous form"""
    n = 8
    model, metric, p0, dp1, Minv, cholU, th, r, g, z0, rng = _lf_problem(kind, mkind, D, N, D, n)
    zo = oc.leapfrog(model, metric, 0.1, z0, n)[0]
    make = _lf_make(kind, mkind, D, N, p0, dp1, Minv, cholU, n, z0.lp_value)
    got, s = same_as_ld_d(E.harness("lf").emu_leapfrog, EmuLf, make, dict(th_in=th, r_in=r, g_in=g), LF_OUTS, N, D,
                          [(D + 1, 2 * D + 3), (2 * D + 3, D + 1), (D + 1, D + 1)])
    _assert_leapfrog(got, s, zo)


def test_multi_transition_hmc_kernel_reads_later_transitions_at_ld_out():
    """K2 with three transitions (Philox refresh): transition 0 starts at ld_in, later ones at ld_out"""
    D, N, n, T = 7, 9, 6, 3
    model, metric, p0, dp1, Minv, cholU, th, r, g, z0, rng = _lf_problem("diag_gauss", "diag", D, N, 9, n)
    make = _lf_make("diag_gauss", "diag", D, N, p0, dp1, Minv, cholU, n, z0.lp_value, hmc=1, refresh=1, n_transitions=T, seed=5,
                    offset=0, is_accept=np.zeros(N * T, np.uint8), acc=np.zeros(N * T), dH=np.zeros(N * T),
                    draws=np.zeros(D * N * T))
    got, s = same_as_ld_d(E.harness("lf").emu_leapfrog, EmuLf, make, dict(th_in=th, r_in=r, g_in=g), ("th_out", "r_out", "g_out"),
                          N, D, [(D + 1, 2 * D + 3), (2 * D + 3, D + 1)])
    assert s["is_accept"].any() and np.array_equal(s["draws"][-D * N:].reshape(N, D), got["th_out"])


def _nuts_make(kind, mkind, D, N, p0, dp1, Minv, cholU, lp_in, dirs, var, T, seed=0):
    def make():
        s = {k: np.zeros(N * T) for k in ("lp_out", "lk_out", "acc", "dH", "dHmax")}
        s.update(n_steps=np.zeros(N * T, np.int32), tree_depth=np.zeros(N * T, np.int32), numerical=np.zeros(N * T, np.uint8),
                 draws=np.zeros(D * N * T))
        kw = dict(model_kind=KINDS[kind], metric_kind=MKINDS[mkind], D=D, N=N, p0=P(p0), p1=P(dp1), c0=0.0, Minv=P(Minv),
                  minv_stride=0, cholU=P(cholU), eps=0.25, eps_chain=None, max_depth=5, delta_max=1000.0, sampler=0, criterion=0,
                  seed=seed, offset=0, normal_tape=None, exp_tape=P(var), exp_stride=0 if var is None else var.shape[1],
                  dir_tape=P(dirs), dir_stride=0 if dirs is None else dirs.shape[1], partial_alpha=0.0, refresh=int(T > 1),
                  lp_in=P(lp_in), n_transitions=T, adapt=0, temper_alpha=0.0, coop_padded=0,
                  **{k: P(v) for k, v in s.items()})
        return kw, s
    return make


@pytest.mark.parametrize("kind,mkind,D,N", [("diag_gauss", "diag", 7, 9), ("dense_gauss", "dense", 40, 11)], ids=["warp", "cooperative"])
def test_nuts_with_different_input_and_output_leading_dimensions(kind, mkind, D, N):
    """one transition on tapes against the oracle; three Philox transitions (later ones start from z_out) bit for bit"""
    rng = np.random.default_rng(D)
    model, metric, p0, dp1, Minv, cholU = _lf_system(kind, mkind, D, rng)
    th, r = rng.normal(size=(N, D)), rng.normal(size=(N, D))
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    g = np.ascontiguousarray(z0.lp_gradient.T)
    dirs, var = rng.integers(0, 2, size=(N, 6)).astype(np.uint8), rng.exponential(size=(N, 32))
    zo, so, _ = oc.nuts_transition(model, metric, 0.25, z0, None, dirs, var, max_depth=5)
    lib = E.harness("nuts")
    lds = [(D + 1, 2 * D + 3), (2 * D + 3, D + 1)]
    ins = dict(th_in=th, r_in=r, g_in=g)
    got, s = same_as_ld_d(lib.emu_nuts, EmuNuts, _nuts_make(kind, mkind, D, N, p0, dp1, Minv, cholU, z0.lp_value, dirs, var, 1),
                          ins, ("th_out", "r_out", "g_out"), N, D, lds)
    assert rel_err(got["th_out"].T, zo.theta) < TOL and rel_err(got["r_out"].T, zo.r) < TOL
    assert rel_err(got["g_out"].T, zo.lp_gradient) < TOL and rel_err(s["lp_out"], zo.lp_value) < TOL
    assert (s["tree_depth"] == so.tree_depth).all() and (s["n_steps"] == so.n_steps).all()
    same_as_ld_d(lib.emu_nuts, EmuNuts, _nuts_make(kind, mkind, D, N, p0, dp1, Minv, cholU, z0.lp_value, None, None, 3, seed=4),
                 ins, ("th_out", "r_out", "g_out"), N, D, lds)


def test_multinomial_with_different_input_and_output_leading_dimensions():
    D, N, n, n_fwd = 7, 9, 6, 2
    rng = np.random.default_rng(2)
    model, metric, p0, dp1, Minv, cholU = _lf_system("diag_gauss", "diag", D, rng)
    th = rng.normal(size=(N, D))
    z0 = oc.phasepoint(model, metric, th.T, np.zeros((D, N)))
    g = np.ascontiguousarray(z0.lp_gradient.T)
    nt, ut = rng.normal(size=(N, D)), rng.uniform(size=N)
    zo, so = oc.hmc_multinomial_transition(model, metric, 0.3, n, n_fwd, z0, nt.T, ut)

    def make():
        s = dict(lp_out=np.zeros(N), lk_out=np.zeros(N), acc=np.zeros(N), index=np.zeros(N, np.int32))
        kw = dict(model_kind=KINDS["diag_gauss"], metric_kind=MKINDS["diag"], D=D, N=N, p0=P(p0), p1=P(dp1), Minv=P(Minv),
                  cholU=None, eps=0.3, n_steps=n, n_fwd=n_fwd, normal_tape=P(nt), unif_tape=P(ut), lp_in=P(z0.lp_value),
                  temper_alpha=0.0, **{k: P(v) for k, v in s.items()})
        return kw, s

    got, s = same_as_ld_d(E.harness("mn").emu_multinomial, EmuMn, make, dict(th_in=th, g_in=g), ("th_out", "r_out", "g_out"), N, D,
                          [(D + 1, 2 * D + 3), (2 * D + 3, D + 1)])
    assert rel_err(got["th_out"].T, zo.theta) < TOL and rel_err(got["r_out"].T, zo.r) < TOL
    assert (s["index"] == so.tree_depth).all() and rel_err(s["lp_out"], zo.lp_value) < TOL


@pytest.mark.parametrize("kind,mkind,D,N", [("dense_gauss", "dense", 40, 37), ("diag_gauss", "dense", 70, 33)])
def test_dense_tile_at_padded_leading_dimensions(kind, mkind, D, N):
    """K4: the tile kernel stages chains from and to ld_in / ld_out"""
    n = 4
    rng = np.random.default_rng(D)
    model, metric, p0, dp1, Minv, _ = _lf_system(kind, mkind, D, rng)
    th, r = rng.normal(size=(N, D)), rng.normal(size=(N, D))
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    g = np.ascontiguousarray(z0.lp_gradient.T)
    zo = oc.leapfrog(model, metric, 0.1, z0, n)[0]
    Pm = np.asfortranarray(dp1) if kind == "dense_gauss" else None
    w = dp1 if kind == "diag_gauss" else None

    def make():
        s = dict(lp_out=np.zeros(N), lk_out=np.zeros(N), status=np.zeros(N, np.uint32), steps_done=np.zeros(N, np.int32),
                 need_exact=np.zeros(N, np.uint8))
        kw = dict(D=D, N=N, P=P(Pm), w=P(w), mu=P(p0), c0=0.0, Minv=P(np.asfortranarray(Minv)), Mdiag=None, eps=0.1, eps_chain=None,
                  n_steps=n, fwd=1, wide_tile=0, **{k: P(v) for k, v in s.items()})
        return kw, s

    got, s = same_as_ld_d(E.harness("dense").emu_dense, EmuDense, make, dict(th_in=th, r_in=r, g_in=g), LF_OUTS, N, D,
                          [(D + 1, 2 * D + 3), (2 * D + 3, D + 1)])
    _assert_leapfrog(got, s, zo)


@pytest.mark.parametrize("family", ["bernoulli_logit", "poisson_log"])
def test_glm_tile_at_padded_leading_dimensions(family):
    """K6: the GLM tile kernel against the float64 numpy statement of the model (tests/glm_ref.py)"""
    D, n, N, steps = 25, 65, 21, 3
    rng = np.random.default_rng(6)
    X, y, beta = R.data(family, n, D, 6, scale=0.5)
    prec, Minv = rng.uniform(0.5, 2.0, D), rng.uniform(0.5, 2.0, D)
    th, r = beta + 0.1 * rng.normal(size=(N, D)), rng.normal(size=(N, D))
    z0 = R.phasepoint(family, X, y, prec, 0.0, Minv, th, r)
    ref = R.leapfrog(family, X, y, prec, 0.0, Minv, 0.02, z0, steps)[0]
    c0 = -gammaln(y + 1.0).sum() if family == "poisson_log" else 0.0  # the library folds the log(y!) terms into c0

    def make():
        s = dict(lp_out=np.zeros(N), lk_out=np.zeros(N), status=np.zeros(N, np.uint32), steps_done=np.zeros(N, np.int32))
        kw = dict(family=0 if family == "bernoulli_logit" else 1, D=D, n=n, N=N, X=P(X), y=P(y), prec=P(prec), c0=c0, Minv=P(Minv),
                  chain_stride=0, eps=0.02, eps_chain=None, n_steps=steps, fwd=1, **{k: P(v) for k, v in s.items()})
        return kw, s

    got, s = same_as_ld_d(E.harness("glm").emu_glm, EmuGlm, make, dict(th_in=th, r_in=r, g_in=np.ascontiguousarray(z0["g"])),
                          LF_OUTS, N, D, [(D + 1, 2 * D + 3), (2 * D + 3, D + 1)])
    for f, k in (("th_out", "th"), ("r_out", "r"), ("g_out", "g"), ("dr_out", "dr")):
        assert rel_err(got[f], ref[k]) < TOL, f
    assert rel_err(s["lp_out"], ref["lp"]) < TOL and rel_err(s["lk_out"], ref["lk"]) < TOL
