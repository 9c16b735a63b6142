"""CPU checks of the D > 512 sampling kernels (ahmc_bigd_hmc.cu) under the SIMT emulator (tests/simt_emu/bigd_emu.cpp):
tape-driven static transitions against the ORACLE, a persistent run against single transitions, the adaptive form
replayed against the oracle's adaptors, find_good_stepsize against the search restated on the oracle's leapfrog, and
the same sources under ThreadSanitizer.  The GPU side is tests/test_bigd_transitions.py."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle_c as oc
from tests import emu as E
from tests.emu import P, EmuBigd
from tests.helpers import rel_err

UNIT, DIAG = 0, 1
MODELS = {"std_normal": oc.STD_NORMAL, "diag_gauss": oc.DIAG_GAUSS, "funnel": oc.FUNNEL}


@pytest.fixture(scope="module")
def emu():
    return E.harness("bigd")


class _Problem:
    def __init__(self, model, metric, D, N, seed, scale=1.0):
        rng = self.rng = np.random.default_rng(seed)
        self.model, self.D, self.N = model, D, N
        self.p0 = self.p1 = None
        s = None
        if model == "diag_gauss":
            self.p0, s = rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))
            self.p1 = 1.0 / (s * s)
        self.metric = UNIT if metric == "unit" else DIAG
        self.Minv = None if metric == "unit" else np.exp(rng.uniform(-0.5, 0.5, (D, N) if metric == "diag_perchain" else D))
        self.om = oc.Model(MODELS[model], D, self.p0, s, 0.25)
        self.ome = oc.Metric(oc.UNIT if metric == "unit" else oc.DIAG, self.Minv)
        self.th = rng.normal(size=(D, N)) * scale

    def run(self, lib, z0, eps, L, T=1, normal=None, exp=None, partial=0.0, refresh=1, seed=0, offset=0, adapt=None):
        D, N = self.D, self.N
        f = lambda a: np.ascontiguousarray(np.asarray(a).T)  # (D, N) -> (N, D) rows
        th_in, r_in, g_in, lp_in = f(z0.theta), f(z0.r), f(z0.lp_gradient), z0.lp_value.copy()
        o = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
        lp, lk = np.zeros(N), np.zeros(N)
        draws, acc, H, dH = np.zeros((T, N, D)), np.zeros((T, N)), np.zeros((T, N)), np.zeros((T, N))
        ia, ne = np.zeros((T, N), np.uint8), np.zeros((T, N), np.uint8)
        minv = None if self.Minv is None else (f(self.Minv) if self.Minv.ndim == 2 else self.Minv)
        eps = np.full(N, float(eps)) if np.ndim(eps) == 0 else np.asarray(eps, dtype=np.float64)
        nt = None if normal is None else f(normal)
        ad = adapt or {}
        eps_rw, minv_rw, trace = eps.copy(), np.zeros((N, D)), np.zeros((T, N))
        q = EmuBigd(model=MODELS[self.model], metric=self.metric, D=D, N=N, p0=P(self.p0), p1=P(self.p1), c0=0.25, Minv=P(minv),
                    minv_stride=D if (minv is not None and minv.ndim == 2) else 0, eps=P(eps), n_steps=L, T=T, refresh=refresh, seed=seed, offset=offset,
                    partial_alpha=partial, normal_tape=P(nt), exp_tape=P(exp), th_in=P(th_in),
                    r_in=P(r_in), g_in=P(g_in), lp_in=P(lp_in), th_out=P(o["th"]), r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp),
                    lk_out=P(lk), draws=P(draws), acc=P(acc), H=P(H), dH=P(dH), is_accept=P(ia), numerical_error=P(ne),
                    adapt_metric=ad.get("adapt_metric", -1), n_adapts=ad.get("n_adapts", 0), init_buffer=ad.get("init_buffer", 0),
                    term_buffer=ad.get("term_buffer", 0), window_size=ad.get("window_size", 1), n_min=ad.get("n_min", 10),
                    eps_rw=P(eps_rw), minv_rw=P(minv_rw), eps_trace=P(trace))
        keep = (nt, exp, th_in, r_in, g_in, lp_in, minv, eps)
        assert lib.emu_bigd_hmc(C.byref(q)) == 0
        del keep
        return dict(theta=o["th"].T, r=o["r"].T, lp_gradient=o["g"].T, lp_value=lp, lk_value=lk, draws=draws, acc=acc, H=H, dH=dH,
                    is_accept=ia, numerical_error=ne, eps=eps_rw, minv=minv_rw, trace=trace)


CASES = [(m, me, D) for D in (513, 700, 1100) for m in ("std_normal", "diag_gauss", "funnel") for me in ("unit", "diag", "diag_perchain")]


@pytest.mark.parametrize("model,metric,D", CASES, ids=[f"{c[0]}-{c[1]}-D{c[2]}" for c in CASES])
def test_streamed_transition_source_equals_oracle_with_tapes(emu, model, metric, D):
    """N = 5 (a ragged block), partial refreshment on the per-chain Diag cases, chain 1 with a step 25x too large
    (rejected), chain 4 started at 1e200 (non-finite: numerical_error, -Inf energy, restored start)"""
    N, L = 5, 6
    pr = _Problem(model, metric, D, N, D + len(metric), scale=0.3 if model == "funnel" else 1.0)
    pr.th[1, 4] = 1e200
    partial = 0.5 if metric == "diag_perchain" else 0.0
    r_prev = pr.rng.normal(size=(D, N))
    nt, et = pr.rng.normal(size=(D, N)), pr.rng.exponential(size=N) * 0.05
    eps = np.full(N, {"diag_gauss": 0.12, "std_normal": 0.1, "funnel": 0.03}[model])
    eps[1] *= 25.0
    z0 = oc.phasepoint(pr.om, pr.ome, pr.th, r_prev)
    oc.set_partial_refresh(partial)
    try:
        zo, so = oc.hmc_transition(pr.om, pr.ome, eps, L, z0, nt, et)
    finally:
        oc.set_partial_refresh(0.0)
    got = pr.run(emu, z0, eps, L, normal=nt, exp=et, partial=partial)
    assert (got["is_accept"][0] == so.is_accept).all() and (got["numerical_error"][0] == so.numerical_error).all()
    assert got["is_accept"][0][1] == 0 and got["numerical_error"][0][4] == 1 and got["lp_value"][4] == -np.inf
    ok = [0, 1, 2, 3]
    for f in ("theta", "r", "lp_gradient"):
        assert rel_err(got[f][:, ok], getattr(zo, f)[:, ok]) < 1e-10, f
    for f in ("lp_value", "lk_value"):
        assert rel_err(got[f][ok], getattr(zo, f)[ok]) < 1e-10, f
    assert np.array_equal(got["theta"][:, 4], z0.theta[:, 4]) and np.array_equal(got["lp_gradient"][:, 4], z0.lp_gradient[:, 4])
    assert rel_err(got["acc"][0][ok], so.acceptance_rate[ok]) < 1e-9


def test_persistent_run_equals_single_transitions(emu):
    """a 3-transition launch against 3 one-transition launches at Philox offsets 0, 1, 2, each from the last one's output"""
    D, N, T, L = 600, 6, 3, 5
    pr = _Problem("diag_gauss", "diag", D, N, 3)
    z = oc.phasepoint(pr.om, pr.ome, pr.th, pr.rng.normal(size=(D, N)))
    full = pr.run(emu, z, 0.1, L, T=T, seed=11, partial=0.3)
    for t in range(T):
        one = pr.run(emu, z, 0.1, L, T=1, seed=11, offset=t, partial=0.3)
        assert np.array_equal(one["draws"][0], full["draws"][t]), t
        assert np.array_equal(one["is_accept"][0], full["is_accept"][t]) and np.array_equal(one["acc"][0], full["acc"][t])
        z = oc.PhasePoint(D, N, one["theta"], one["r"])
        z.lp_gradient[...] = one["lp_gradient"]
        z.lp_value[...] = one["lp_value"]
    assert np.array_equal(full["theta"], z.theta) and np.array_equal(full["r"], z.r)
    assert 0 < full["is_accept"].sum()


def test_adaptive_source_equals_oracle_adaptors(emu):
    D, N, T, n_adapts = 530, 5, 24, 20
    windows, n_min = (3, 2, 4), 5
    ws, we, splits = oc.stan_windows(n_adapts, *windows)
    for est, am in (("welford", 1), ("nutpie", 2)):
        pr = _Problem("diag_gauss", "diag", D, N, 21)
        pr.Minv = np.ones(D)
        pr.ome = oc.Metric(oc.DIAG, pr.Minv)
        z = oc.phasepoint(pr.om, pr.ome, pr.th, np.zeros((D, N)))
        run = pr.run(emu, z, 0.15, 6, T=T, seed=7, adapt=dict(adapt_metric=am, n_adapts=n_adapts, init_buffer=windows[0],
                                                              term_buffer=windows[1], window_size=windows[2], n_min=n_min))
        grads = np.stack([(run["draws"][t] - pr.p0) * pr.p1 for t in range(T)])
        da = oc.DualAveraging(np.full(N, 0.15), delta=0.8)
        wt, wg = oc.WelfordVar((D, N)), oc.WelfordVar((D, N))
        Minv, updates = np.ones((N, D)), 0
        for i in range(1, T + 1):
            assert np.allclose(run["trace"][i - 1], da.eps, rtol=1e-10, atol=0), (est, i)
            if i <= n_adapts:
                da.adapt(run["acc"][i - 1])
                if ws <= i <= we:
                    wt.push(run["draws"][i - 1].T)
                    wg.push(grads[i - 1].T)
                    if i in splits and wt.n.value >= n_min:
                        e = wt.estimate()
                        Minv = np.ascontiguousarray((np.sqrt(e / wg.estimate()) if est == "nutpie" else e).T)
                        updates += 1
                if i in splits:
                    da.reset()
                    wt, wg = oc.WelfordVar((D, N)), oc.WelfordVar((D, N))
                if i == n_adapts:
                    da.finalize()
        assert updates == 1 and np.allclose(run["minv"], Minv, rtol=1e-10, atol=0), est
        assert np.allclose(run["eps"], da.eps, rtol=1e-10, atol=0), est


def test_find_good_stepsize_source_equals_the_search_on_the_oracle(emu):
    D, N = 700, 5
    pr = _Problem("diag_gauss", "diag", D, N, 5)
    xi = pr.rng.normal(size=(D, N))
    z = oc.phasepoint(pr.om, pr.ome, pr.th, np.zeros((D, N)))
    eps_out, r_out = np.zeros(N), np.zeros((N, D))
    f = lambda a: np.ascontiguousarray(np.asarray(a).T)
    th, g, nt = f(z.theta), f(z.lp_gradient), f(xi)
    assert emu.emu_bigd_find_eps(oc.DIAG_GAUSS, DIAG, D, C.c_int64(N), P(pr.p0), P(pr.p1), C.c_double(0.25), P(pr.Minv), C.c_int64(0),
                                 P(th), P(g), P(z.lp_value), P(nt), C.c_double(0.1), 100, P(eps_out), P(r_out)) == 0
    for c in range(N):
        r = xi[:, c] / np.sqrt(pr.Minv)
        assert rel_err(r_out[c], r) < 1e-15
        zc = oc.phasepoint(pr.om, pr.ome, pr.th[:, c:c + 1], r[:, None])
        H = zc.energy()[0]
        Af = lambda e: oc.leapfrog(pr.om, pr.ome, e, zc, 1)[0].energy()[0]
        e = ep = 0.1
        too_high = (H - Af(e)) > np.log(0.5)
        for _ in range(100):
            ep = 2 * e if too_high else 0.5 * e
            if too_high != ((H - Af(e)) > np.log(0.5)):
                break
            e = ep
        e, ep = min(e, ep), max(e, ep)
        for _ in range(100):
            mid = 0.5 * (e + ep)
            dH = H - Af(mid)
            if dH > np.log(0.75):
                e = mid
            elif dH < 2 * np.log(0.5):
                ep = mid
            else:
                e = mid
                break
        assert eps_out[c] == pytest.approx(e, rel=1e-12), c


def test_streamed_sampling_sources_are_data_race_free_under_thread_sanitizer():
    r = E.sanitized("bigd", "thread")
    assert r.returncode == 0 and "WARNING: ThreadSanitizer" not in r.stderr, r.stdout + r.stderr[-3000:]
    assert r.stdout.count("rc 0 0") == 4, r.stdout
