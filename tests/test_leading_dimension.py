"""Phase points whose leading dimension ld exceeds D (element (d, chain c) at d + ld*c, include/ahmc_b200.h): every entry
point, through the raw C ABI, on device, page-locked and pageable buffers whose padding rows D..ld-1 and a guard tail
after the last chain hold a NaN canary.  Each call must (1) return the D x N blocks of the ld = D call bit for bit (or,
where ld takes K1 off its two-chains-per-warp kernel, agree with the oracle to 1e-10), (2) leave every canary in every
buffer as it was, (3) leave its inputs untouched when out of place, (4) agree with the oracle where tapes define the
result, and (5) make as many launches as the ld = D call with the same residency (run with -m gpu on an H100)."""
import ctypes as C

import numpy as np
import pytest
import torch

import ahmc_b200 as A
from ahmc_b200 import _lib as L
from oracle import oracle_c as oc
from tests import glm_ref as R
from tests.helpers import METRIC_KINDS, MODEL_KINDS, rel_err
from tests.test_gpu_parity import DEV, TOL, make_metric, make_target

pytestmark = pytest.mark.gpu

# a quiet NaN with a payload: a padding double that the library copies, sums or overwrites shows at once
CANARY = np.frombuffer(np.array([0x7FF8DEADBEEF0001], dtype="<i8").tobytes(), dtype=np.uint8)
GUARD = 3  # canaried elements after the last chain's padding
PP_FIELDS = ("theta", "r", "lp_value", "lp_gradient", "lk_value", "lk_gradient")
VEC_FIELDS = ("theta", "r", "lp_gradient", "lk_gradient")


def ld_of(D, k):
    return {"D": D, "D+1": D + 1, "D+4": D + 4, "2D+3": 2 * D + 3}[k]


# (residency, z_in.ld, z_out.ld or None for z_out = z_in).  D+1 is odd (alternate chains not 16-byte aligned), D+4 keeps
# the vector width of K1's lane-contiguous layout, 2D+3 leaves more padding than data
LAYOUTS = [("dev", "D+1", "D+1"), ("dev", "D+4", "D+4"), ("dev", "2D+3", "2D+3"), ("dev", "D+1", "2D+3"), ("dev", "D+4", None),
           ("dev", "2D+3", None), ("pinned", "D+1", "2D+3"), ("pinned", "D+4", None), ("pageable", "2D+3", "D+1"),
           ("pageable", "D+1", None)]
DEV_LAYOUTS = [l for l in LAYOUTS if l[0] == "dev"]
OUT_OF_PLACE = [l for l in LAYOUTS if l[2] is not None]
# entry points with one D x N phase point or array (phasepoint, rand_momentum, find_good_stepsize, adaptor statistics)
ONE_LD = [("dev", "D+1", None), ("dev", "D+4", None), ("dev", "2D+3", None), ("pinned", "D+4", None), ("pinned", "2D+3", None),
          ("pageable", "D+1", None), ("pageable", "2D+3", None)]


class Buf:
    """`cols` columns of `rows` elements at leading dimension `ld`, then GUARD elements; everything outside the block is
    the canary.  Held on the device, in page-locked or in pageable host memory."""

    def __init__(self, name, where, rows, cols=1, ld=None, dtype=np.float64, data=None):
        self.name, self.rows, self.cols, self.dt = name, rows, cols, np.dtype(dtype)
        self.ld = rows if ld is None else ld
        init = np.resize(CANARY, (self.ld * cols + GUARD) * self.dt.itemsize)
        if data is not None:
            self._block(init)[...] = np.asarray(data, self.dt).reshape(cols, rows)
        self.init = init.copy()
        t = torch.from_numpy(init)
        self.t = t.to(DEV) if where == "dev" else t.pin_memory() if where == "pinned" else t
        self.ptr = self.t.data_ptr()

    def _block(self, raw):
        return raw[: self.ld * self.cols * self.dt.itemsize].view(self.dt).reshape(self.cols, self.ld)[:, : self.rows]

    def raw(self):
        torch.cuda.synchronize()
        return self.t.cpu().numpy().copy()

    def value(self):
        """the block as (cols, rows); a single column as (rows,)"""
        v = self._block(self.raw()).copy()
        return v[0] if self.cols == 1 else v

    def canaries_intact(self):
        keep = np.ones(self.init.size, bool)
        keep[: self.ld * self.cols * self.dt.itemsize].reshape(self.cols, -1)[:, : self.rows * self.dt.itemsize] = False
        return np.array_equal(self.raw()[keep], self.init[keep])

    def unchanged(self):
        return np.array_equal(self.raw(), self.init)


def bits(a):
    return np.ascontiguousarray(a).tobytes()


class PP:
    """an ahmc_phasepoint over canaried buffers; `start` ((N, D) / (N,) arrays) fills them, else they are outputs"""

    def __init__(self, tag, where, D, N, ld, start=None, dr=True):
        s = start or {}
        self.f = {}
        for k in PP_FIELDS:
            if k == "lk_gradient" and not dr:
                continue
            if k in VEC_FIELDS:
                self.f[k] = Buf(f"{tag}.{k}", where, D, N, ld, data=s.get(k))
            else:
                self.f[k] = Buf(f"{tag}.{k}", where, N, data=s.get(k))
        self.c = L.PhasePoint(*(self.f[k].ptr if k in self.f else None for k in PP_FIELDS), ld)


class Run:
    """the buffers of one raw call: z_in / z_out, plus inputs (`inp`, must stay bit for bit) and outputs (`out`)"""

    def __init__(self, where, D, N, kin, kout, start, dr, pp=True):
        self.where, self.D, self.N = where, D, N
        self.ld_in, self.ld_out = ld_of(D, kin), ld_of(D, kout or kin)
        self.flags = 0 if where == "dev" else L.FLAG_HOST_BUFFERS
        self.like = torch.empty(0, device=DEV) if where == "dev" else np.empty(0)
        self.ins, self.outs, self.bufs = [], {}, []
        if pp:
            self.zin = PP("z_in", where, D, N, self.ld_in, start, dr)
            self.zout = self.zin if kout is None else PP("z_out", where, D, N, self.ld_out, None, dr)
            self.bufs += list(self.zin.f.values()) + ([] if kout is None else list(self.zout.f.values()))
            if kout is not None:
                self.ins += list(self.zin.f.values())
            self.outs.update({"z." + k: b for k, b in self.zout.f.items()})

    def inp(self, name, rows, cols=1, ld=None, dtype=np.float64, data=None):
        b = Buf(name, self.where, rows, cols, ld, dtype, data)
        self.ins.append(b)
        self.bufs.append(b)
        return b

    def out(self, name, rows, cols=1, ld=None, dtype=np.float64):
        b = Buf(name, self.where, rows, cols, ld, dtype)
        self.outs[name] = b
        self.bufs.append(b)
        return b

    def stats(self, T=1):
        """every statistics array: one an entry point does not fill (max_hamiltonian_energy_error outside NUTS) keeps its canary"""
        f = [("n_steps", np.int32), ("is_accept", np.uint8), ("acceptance_rate", np.float64), ("log_density", np.float64),
             ("hamiltonian_energy", np.float64), ("hamiltonian_energy_error", np.float64),
             ("max_hamiltonian_energy_error", np.float64), ("tree_depth", np.int32), ("numerical_error", np.uint8)]
        return L.Stats(*(self.out("st." + k, self.N * T, dtype=dt).ptr for k, dt in f))

    def tape_rng(self, nt, et=None):
        """tapes in this call's residency: normal (N, D), exponential (N,)"""
        n = self.inp("normal_tape", self.D, self.N, data=nt)
        e = None if et is None else self.inp("exp_tape", self.N, data=et)
        return L.Rng(0, 0, n.ptr, None if e is None else e.ptr, 1, None, 0, 0.0, 0.0)


def check(D, N, start, call, layouts=LAYOUTS, dr=True, pp=True, oracle=None, same_kernel=lambda ld_in, ld_out: True,
          count_launches=True):
    """`call(run)` makes the raw call on a Run; runs it at ld = D (the reference) and at every layout, checking (1)-(5)"""
    ctx = A.get_context(0)

    def go(where, kin, kout):
        run = Run(where, D, N, kin, kout, start, dr, pp)
        l0 = ctx.launches
        call(run)
        torch.cuda.synchronize()
        n = ctx.launches - l0
        for b in run.bufs:
            assert b.canaries_intact(), (where, kin, kout, b.name, "padding or guard written")
        for b in run.ins:
            assert b.unchanged(), (where, kin, kout, b.name, "input changed")
        vals = {k: b.value() for k, b in run.outs.items()}
        if oracle:
            oracle(vals, run)
        return vals, n

    ref_out = None if all(l[2] is None for l in layouts) else "D"  # in place when every layout is
    ref, n_ref = go("dev", "D", ref_out)
    launches = {"dev": n_ref}
    for where in sorted({l[0] for l in layouts} - {"dev"}):
        vals, launches[where] = go(where, "D", ref_out)
        for k in ref:
            assert bits(vals[k]) == bits(ref[k]), (where, k)
    for where, kin, kout in layouts:
        vals, n = go(where, kin, kout)
        if same_kernel(ld_of(D, kin), ld_of(D, kout or kin)):
            for k in ref:
                assert bits(vals[k]) == bits(ref[k]), (where, kin, kout, k)
        assert n == launches[where] or not count_launches, (where, kin, kout, n, launches[where])
    return ref


def close_to(vals, zo, fields=("theta", "r", "lp_gradient", "lp_value", "lk_value"), cols=None, tol=TOL):
    for f in fields:
        got, want = vals["z." + f], getattr(zo, f) if not isinstance(zo, dict) else zo[f]
        got = got.T if got.ndim == 2 else got
        if cols is not None:
            got, want = got[..., cols], want[..., cols]
        assert rel_err(got, want) < tol, (f, rel_err(got, want))


def problem(model, metric, D, N, seed, scale=1.0):
    """target, metric and start point: (h, om, ome, th (D, N), r (D, N))"""
    rng = np.random.default_rng(seed)
    p0 = p1 = Minv = None
    if model == "diag_gauss":
        p0, p1 = rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))
    elif model == "dense_gauss":
        B = rng.normal(size=(D, D))
        p0, p1 = rng.normal(size=D), B @ B.T / D + np.eye(D)
    mk = "diag" if metric == "diag_perchain" else metric
    if metric == "diag":
        Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    elif metric == "diag_perchain":
        Minv = np.exp(rng.uniform(-0.5, 0.5, (D, N)))
    elif metric == "dense":
        B = rng.normal(size=(D, D))
        Minv = B @ B.T / D + 0.5 * np.eye(D)
    h = A.Hamiltonian(make_metric(mk, Minv, D), make_target(model, D, p0, p1, 0.25))
    om = oc.Model(MODEL_KINDS[model], D, p0, p1, 0.25)
    ome = oc.Metric(METRIC_KINDS[mk], Minv)
    return h, om, ome, rng.normal(size=(D, N)) * scale, rng.normal(size=(D, N)), rng


def start_of(h, th, r):
    """the cached phase point at (th, r) as (N, D) / (N,) host arrays"""
    z = A.phasepoint(h, torch.as_tensor(np.ascontiguousarray(th.T), device=DEV), torch.as_tensor(np.ascontiguousarray(r.T), device=DEV))
    g = lambda t: t.cpu().numpy()
    return dict(theta=g(z.theta), r=g(z.r), lp_value=g(z.lp.value), lp_gradient=g(z.lp.gradient), lk_value=g(z.lk.value),
                lk_gradient=g(z.lk.gradient))


def eps_arg(run, eps):
    if np.ndim(eps) == 0:
        return float(eps), None
    return 0.0, run.inp("eps_chain", run.N, data=eps).ptr


def leapfrog_call(h, eps, n, flags=0, status=True):
    def call(run):
        ctx = A.get_context(0)
        md, keep = h.metric._desc(run.D, run.N, run.like)
        e, ep = eps_arg(run, eps)
        st = run.out("status", run.N, dtype=np.uint32).ptr if status else None
        sd = run.out("steps_done", run.N, dtype=np.int32).ptr if status else None
        ctx.check(ctx.lib.ahmc_leapfrog_f64(ctx.h, h.target.handle(ctx), C.byref(md), run.D, run.N, e, ep, n, 0.0,
                                            C.byref(run.zin.c), C.byref(run.zout.c), st, sd, run.flags | flags))
    return call


def pair_kernel_kept(D):
    """K1's two-chains-per-warp kernel needs D = 32 E and every ld a multiple of its vector width (4)"""
    return lambda ld_in, ld_out: D not in (64, 128) or (ld_in % 4 == 0 and ld_out % 4 == 0)


# ------------------------------------------------------------------------------------------------ K1
K1_CASES = [(m, mt, D) for D in (5, 64, 128, 300) for m, mt in (("diag_gauss", "diag"), ("std_normal", "unit"), ("funnel", "diag"))]


@pytest.mark.parametrize("model,metric,D", K1_CASES, ids=[f"{m}-{mt}-D{D}" for m, mt, D in K1_CASES])
def test_leapfrog_k1(model, metric, D):
    N, n = 7, 9
    h, om, ome, th, r, _ = problem(model, metric, D, N, D, scale=0.3 if model == "funnel" else 1.0)
    zo, st_o, dn_o = oc.leapfrog(om, ome, 0.05, oc.phasepoint(om, ome, th, r), n)

    def oracle(vals, run):
        close_to(vals, zo, fields=("theta", "r", "lp_gradient", "lp_value", "lk_value", "lk_gradient"))
        assert (vals["status"] == st_o).all() and (vals["steps_done"] == dn_o).all()

    check(D, N, start_of(h, th, r), leapfrog_call(h, 0.05, n), oracle=oracle, same_kernel=pair_kernel_kept(D))


@pytest.mark.parametrize("variant", ["per_chain_backward", "exact_checks", "huge_chain", "compat_break_all"])
@pytest.mark.parametrize("D", [5, 64, 128, 300])
def test_leapfrog_k1_variants(variant, D):
    """per-chain eps and per-chain Diag M^-1 (chain_stride = D) with n < 0; EXACT_CHECKS; one chain past the fast path's
    magnitude proof (the exact fallback inside the launch); COMPAT_BREAK_ALL with a chain that turns non-finite (the
    re-run; out of place, which COMPAT mode requires)"""
    N, n = 9, 8
    metric = "diag_perchain" if variant == "per_chain_backward" else "diag"
    h, om, ome, th, r, rng = problem("diag_gauss", metric, D, N, 100 + D)
    eps, flags, compat, layouts = 0.05, 0, False, LAYOUTS
    if variant == "per_chain_backward":
        eps, n = 0.05 * np.exp(rng.uniform(-0.3, 0.3, N)), -n
    elif variant == "exact_checks":
        flags = A.FLAG_EXACT_CHECKS
    elif variant == "huge_chain":
        th[min(5, D - 1), 3] = 1e120  # finite energies throughout, outside the magnitude proof
    else:
        th[min(5, D - 1), 3] = 1e250  # its square overflows: non-finite at step 1, every chain stops there
        flags, compat, layouts = A.FLAG_COMPAT_BREAK_ALL, True, OUT_OF_PLACE
    zo, st_o, dn_o = oc.leapfrog(om, ome, eps, oc.phasepoint(om, ome, th, r), n, compat_break_all=compat)
    ok = [c for c in range(N) if not (compat and c == 3)]

    def oracle(vals, run):
        close_to(vals, zo, cols=ok)
        assert (vals["status"] == st_o).all() and (vals["steps_done"] == dn_o).all()

    check(D, N, start_of(h, th, r), leapfrog_call(h, eps, n, flags), layouts=layouts, oracle=oracle, same_kernel=pair_kernel_kept(D))


# ------------------------------------------------------------------------------------------------ phasepoint, rand_momentum
def _metric_cases(D, N, rng):
    B = rng.normal(size=(D, D))
    M = B @ B.T / D + 0.5 * np.eye(D)
    Mpc = np.stack([M + 0.1 * k * np.eye(D) for k in range(N)])
    return {"unit": A.UnitEuclideanMetric(D), "diag": A.DiagEuclideanMetric(np.exp(rng.uniform(-0.5, 0.5, D))),
            "diag_perchain": A.DiagEuclideanMetric(np.exp(rng.uniform(-0.5, 0.5, (N, D)))), "dense": A.DenseEuclideanMetric(M),
            "dense_perchain": A.DenseEuclideanMetric(Mpc)}


@pytest.mark.parametrize("metric", ["unit", "diag", "diag_perchain", "dense", "dense_perchain"])
@pytest.mark.parametrize("D", [5, 33, 64])
def test_phasepoint_and_rand_momentum(metric, D):
    N = 6
    rng = np.random.default_rng(D)
    met = _metric_cases(D, N, rng)[metric]
    h = A.Hamiltonian(met, A.DiagGaussian(rng.normal(size=D), np.exp(rng.uniform(-0.5, 0.5, D))))
    th, r = rng.normal(size=(N, D)), rng.normal(size=(N, D))

    def pp_call(run):  # theta and r in, the rest out, all in one phase point
        ctx = A.get_context(0)
        run.ins += [run.zin.f["theta"], run.zin.f["r"]]
        md, keep = h.metric._desc(D, N, run.like)
        ctx.check(ctx.lib.ahmc_phasepoint_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, C.byref(run.zin.c), run.flags))

    check(D, N, dict(theta=th, r=r), pp_call, layouts=ONE_LD)
    nt = rng.normal(size=(N, D))
    if metric in ("diag", "diag_perchain"):
        Mi = met.Minv if met.Minv.ndim == 2 else np.broadcast_to(met.Minv, (N, D))
        want = nt / np.sqrt(Mi)
    elif metric == "unit":
        want = nt
    else:
        want = None

    def rm_call(run):
        ctx = A.get_context(0)
        md, keep = met._desc(D, N, run.like)
        rc = run.tape_rng(nt)
        r_out = run.out("r", D, N, run.ld_in)
        ctx.check(ctx.lib.ahmc_rand_momentum_f64(ctx.h, C.byref(md), D, N, C.byref(rc), r_out.ptr, run.ld_in, run.flags))

    def oracle(vals, run):
        if want is not None:
            assert rel_err(vals["r"], want) < 1e-14

    check(D, N, None, rm_call, layouts=ONE_LD, pp=False, oracle=oracle)


# ------------------------------------------------------------------------------------------------ trajectories, multinomial
def test_full_trajectory_and_multinomial_transition():
    D, N, n = 12, 5, 4
    h, om, ome, th, r, rng = problem("diag_gauss", "diag", D, N, 3)
    s0 = start_of(h, th, r)
    traj_o, dn_o = oc.leapfrog_trajectory(om, ome, 0.1, oc.phasepoint(om, ome, th, r), n)

    def traj_call(run):  # one spare chain slot per step: step_stride = ld * (N + 1) > ld * N
        ctx = A.get_context(0)
        ld = run.ld_out
        md, keep = h.metric._desc(D, N, run.like)
        f = {k: run.out("traj." + k, D, (N + 1) * n, ld) for k in VEC_FIELDS}
        f.update({k: run.out("traj." + k, N * n) for k in ("lp_value", "lk_value")})
        tc = L.PhasePoint(*(f[k].ptr for k in PP_FIELDS), ld)
        sd = run.out("steps_done", N, dtype=np.int32)
        ctx.check(ctx.lib.ahmc_leapfrog_trajectory_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, 0.1, None, n, 0.0,
                                                       C.byref(run.zin.c), C.byref(tc), ld * (N + 1), sd.ptr, run.flags))

    def traj_oracle(vals, run):
        for k in VEC_FIELDS:
            v = vals["traj." + k].reshape(n, N + 1, D)
            assert bits(v[:, N]) == bits(np.resize(CANARY, v[:, N].nbytes)), (k, "the gap between steps was written")
            assert rel_err(v[:, :N].transpose(2, 1, 0), traj_o[k]) < TOL, k
        for k in ("lp_value", "lk_value"):
            assert rel_err(vals["traj." + k].reshape(n, N).T, traj_o[k]) < TOL, k
        assert (vals["steps_done"] == dn_o).all()

    check(D, N, s0, traj_call, layouts=OUT_OF_PLACE, dr=False, oracle=traj_oracle)
    nt, ut = rng.normal(size=(N, D)), rng.uniform(size=N)
    zo, so = oc.hmc_multinomial_transition(om, ome, 0.1, 6, 2, oc.phasepoint(om, ome, th, r), nt.T, ut)

    def mn_call(run):
        ctx = A.get_context(0)
        md, keep = h.metric._desc(D, N, run.like)
        rc = run.tape_rng(nt, ut)
        ctx.check(ctx.lib.ahmc_hmc_multinomial_transition_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, 0.1, None, 6, 2,
                                                              C.byref(rc), C.byref(run.zin.c), C.byref(run.zout.c),
                                                              C.byref(run.stats()), run.flags))

    def mn_oracle(vals, run):
        close_to(vals, zo)
        assert (vals["st.is_accept"] == so.is_accept).all()

    check(D, N, s0, mn_call, dr=False, oracle=mn_oracle)


# ------------------------------------------------------------------------------------------------ static transitions
def hmc_call(h, eps, L_, T=1, draws=False, tapes=None, seed=7, cfg=None):
    def call(run):
        ctx = A.get_context(0)
        D, N = run.D, run.N
        md, keep = h.metric._desc(D, N, run.like)
        rc = run.tape_rng(*tapes) if tapes else L.Rng(seed, 0, None, None, 0, None, 0, 0.0, 0.0)
        st = run.stats(T)
        dr = run.out("draws", D, N * T).ptr if draws else None
        if cfg is not None:
            c = cfg(run)
            ctx.check(ctx.lib.ahmc_hmc_adapt_sample_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, L_, T, C.byref(c),
                                                        C.byref(rc), C.byref(run.zin.c), C.byref(run.zout.c), dr, C.byref(st),
                                                        run.flags))
        elif T == 1 and not draws:
            e, ep = eps_arg(run, eps)
            ctx.check(ctx.lib.ahmc_hmc_transition_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, e, ep, L_, C.byref(rc),
                                                      C.byref(run.zin.c), C.byref(run.zout.c), C.byref(st), run.flags))
        else:
            e, ep = eps_arg(run, eps)
            ctx.check(ctx.lib.ahmc_hmc_sample_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, e, ep, L_, T, C.byref(rc),
                                                  C.byref(run.zin.c), C.byref(run.zout.c), dr, C.byref(st), run.flags))
    return call


def transition_oracle(om, ome, eps, L_, th, nt, et):
    zo, so = oc.hmc_transition(om, ome, eps, L_, oc.phasepoint(om, ome, th, np.zeros_like(th)), nt.T, et)

    def oracle(vals, run):
        close_to(vals, zo)
        assert (vals["st.is_accept"] == so.is_accept).all()
        assert rel_err(vals["st.hamiltonian_energy"], so.hamiltonian_energy) < TOL
    return oracle


def adapt_cfg(D, est, eps0, dense=False):
    """an in-launch warm-up (ahmc_adapt_cfg): per-chain eps (in and out), adapted M^-1 and step-size trace as outputs"""
    def cfg(run):
        N = run.N
        eps = Buf("cfg.eps", run.where, N, data=np.full(N, eps0))  # in and out
        run.outs["cfg.eps"] = eps
        run.bufs.append(eps)
        minv = run.out("cfg.Minv", D * D if dense else D, N)
        cholu = run.out("cfg.cholU", D * D, N).ptr if dense else None
        trace = run.out("cfg.eps_trace", N * 4)
        return L.AdaptCfg(3, 1, 1, 1, 0.8, 0.05, 10.0, 0.75, est, 2, eps.ptr, minv.ptr, trace.ptr, cholu)
    return cfg


@pytest.mark.parametrize("model,metric,D", [("diag_gauss", "diag", 20), ("funnel", "diag_perchain", 64), ("std_normal", "unit", 128)])
def test_hmc_kernel_transitions(model, metric, D):
    """hmc_kernel: one transition on tapes against the oracle; three transitions with draws; the in-launch warm-up"""
    N, L_, eps = 9, 7, 0.1 if model != "funnel" else 0.03
    h, om, ome, th, r, rng = problem(model, metric, D, N, 40 + D, scale=0.3 if model == "funnel" else 1.0)
    s0 = start_of(h, th, np.zeros_like(th))
    nt, et = rng.normal(size=(N, D)), rng.exponential(size=N) * 0.05
    check(D, N, s0, hmc_call(h, eps, L_, tapes=(nt, et)), dr=False, oracle=transition_oracle(om, ome, eps, L_, th, nt, et))
    check(D, N, s0, hmc_call(h, eps, L_, T=3, draws=True), dr=False)
    if metric != "unit":
        check(D, N, s0, hmc_call(h, eps, L_, T=4, draws=True, cfg=adapt_cfg(D, 1, eps)), dr=False)


@pytest.mark.parametrize("model,D", [("diag_gauss", 700), ("funnel", 1030)])
def test_streaming_beyond_512(model, D):
    """the D > 512 streaming form: step, phasepoint, rand_momentum, one transition on tapes, hmc_sample (T = 3) and the
    in-launch warm-up"""
    N, L_, eps = 4, 5, 0.1 if model != "funnel" else 0.02
    h, om, ome, th, r, rng = problem(model, "diag", D, N, D, scale=0.3 if model == "funnel" else 1.0)
    s0 = start_of(h, th, r)
    zo, st_o, dn_o = oc.leapfrog(om, ome, eps, oc.phasepoint(om, ome, th, r), L_)
    check(D, N, s0, leapfrog_call(h, eps, L_), oracle=lambda vals, run: close_to(vals, zo))

    def pp_call(run):
        ctx = A.get_context(0)
        run.ins += [run.zin.f["theta"], run.zin.f["r"]]
        md, keep = h.metric._desc(D, N, run.like)
        ctx.check(ctx.lib.ahmc_phasepoint_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, C.byref(run.zin.c), run.flags))

    check(D, N, dict(theta=th.T, r=r.T), pp_call, layouts=ONE_LD)
    nt = rng.normal(size=(N, D))

    def rm_call(run):
        ctx = A.get_context(0)
        md, keep = h.metric._desc(D, N, run.like)
        rc = run.tape_rng(nt)
        r_out = run.out("r", D, N, run.ld_in)
        ctx.check(ctx.lib.ahmc_rand_momentum_f64(ctx.h, C.byref(md), D, N, C.byref(rc), r_out.ptr, run.ld_in, run.flags))

    check(D, N, None, rm_call, layouts=ONE_LD, pp=False)
    s00 = start_of(h, th, np.zeros_like(th))
    et = rng.exponential(size=N) * 0.05
    check(D, N, s00, hmc_call(h, eps, L_, tapes=(nt, et)), dr=False, oracle=transition_oracle(om, ome, eps, L_, th, nt, et))
    check(D, N, s00, hmc_call(h, eps, L_, T=3, draws=True), dr=False)
    check(D, N, s00, hmc_call(h, eps, L_, T=4, draws=True, cfg=adapt_cfg(D, 1, eps)), dr=False)


@pytest.mark.parametrize("model,metric,D", [("dense_gauss", "diag", 40), ("diag_gauss", "dense", 40), ("dense_gauss", "diag", 128),
                                            ("diag_gauss", "dense", 128)])
def test_dense_tile_k4(model, metric, D):
    """K4 (tiled fp64 MMA): leapfrog, and one transition into a separate z_out -- with z_in.ld != D this is the sequenced
    transition that starts its trajectory from a copy of the start point in z_out"""
    N, L_, eps = 37, 8, 0.05
    h, om, ome, th, r, rng = problem(model, metric, D, N, 7 + D)
    zo, _, _ = oc.leapfrog(om, ome, eps, oc.phasepoint(om, ome, th, r), L_)
    check(D, N, start_of(h, th, r), leapfrog_call(h, eps, L_), oracle=lambda vals, run: close_to(vals, zo))
    nt, et = rng.normal(size=(N, D)), rng.exponential(size=N) * 0.05
    check(D, N, start_of(h, th, np.zeros_like(th)), hmc_call(h, eps, L_, tapes=(nt, et)), layouts=OUT_OF_PLACE, dr=False,
          oracle=transition_oracle(om, ome, eps, L_, th, nt, et))


@pytest.mark.parametrize("family", ["bernoulli_logit", "poisson_log"])
def test_glm_tile_k6(family):
    """K6 (GLM tile kernel, device buffers): leapfrog, one transition, three with draws; in place and z_in.ld != z_out.ld"""
    D, N, n = 25, 11, 400
    rng = np.random.default_rng(3)
    X = rng.normal(size=(n, D)) / np.sqrt(D)
    y = (rng.uniform(size=n) < 0.5).astype(float) if family == "bernoulli_logit" else rng.poisson(1.0, size=n).astype(float)
    Minv = np.exp(rng.uniform(-0.3, 0.3, D))
    h = A.Hamiltonian(A.DiagEuclideanMetric(Minv), A.GLMTarget(X, y, family, prior_prec=1.0))
    th, r = rng.normal(size=(D, N)) * 0.3, rng.normal(size=(D, N))
    prec = np.ones(D)
    ref, _, _ = R.leapfrog(family, X, y, prec, 0.0, Minv, 0.02, R.phasepoint(family, X, y, prec, 0.0, Minv, th.T, r.T), 6)

    def oracle(vals, run):  # the float64 numpy statement of the model (tests/glm_ref.py)
        for k, f in (("th", "theta"), ("r", "r"), ("g", "lp_gradient"), ("lp", "lp_value"), ("lk", "lk_value")):
            assert rel_err(vals["z." + f], ref[k]) < TOL, (f, rel_err(vals["z." + f], ref[k]))

    check(D, N, start_of(h, th, r), leapfrog_call(h, 0.02, 6), layouts=DEV_LAYOUTS, oracle=oracle)
    s0 = start_of(h, th, np.zeros_like(th))
    check(D, N, s0, hmc_call(h, 0.02, 6), layouts=DEV_LAYOUTS, dr=False)
    check(D, N, s0, hmc_call(h, 0.02, 6, T=3, draws=True), layouts=DEV_LAYOUTS, dr=False)


def _callback_std_normal(th):
    x = th.contiguous()  # the closure sees the (N, ld) buffer's first D columns
    return -0.5 * (x * x).sum(1), -x


def test_callback_target():
    """split-step engine: leapfrog, one transition (out of place and in place) on tapes against the oracle"""
    D, N, eps, L_ = 10, 6, 0.1, 5
    h = A.Hamiltonian(A.UnitEuclideanMetric(D), A.CallbackTarget(D, _callback_std_normal))
    rng = np.random.default_rng(2)
    th, r = rng.normal(size=(D, N)), rng.normal(size=(D, N))
    om, ome = oc.Model(oc.STD_NORMAL, D), oc.Metric(oc.UNIT)
    zo, _, _ = oc.leapfrog(om, ome, eps, oc.phasepoint(om, ome, th, r), L_)
    check(D, N, start_of(h, th, r), leapfrog_call(h, eps, L_), oracle=lambda vals, run: close_to(vals, zo))
    nt, et = rng.normal(size=(N, D)), rng.exponential(size=N) * 0.05
    check(D, N, start_of(h, th, np.zeros_like(th)), hmc_call(h, eps, L_, tapes=(nt, et)), dr=False,
          oracle=transition_oracle(om, ome, eps, L_, th, nt, et))


# ------------------------------------------------------------------------------------------------ NUTS, run-time compiled
def nuts_call(h, eps, T=1, draws=False, seed=11, cfg=None, max_depth=6):
    def call(run):
        ctx = A.get_context(0)
        D, N = run.D, run.N
        md, keep = h.metric._desc(D, N, run.like)
        rc = L.Rng(seed, 0, None, None, 0, None, 0, 0.0, 0.0)
        st = run.stats(T)
        dr = run.out("draws", D, N * T).ptr if draws else None
        if cfg is not None:
            c = cfg(run)
            ctx.check(ctx.lib.ahmc_nuts_adapt_sample_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, max_depth, 1000.0, T,
                                                         C.byref(c), C.byref(rc), C.byref(run.zin.c), C.byref(run.zout.c), dr,
                                                         C.byref(st), run.flags))
        elif T == 1 and not draws:
            ctx.check(ctx.lib.ahmc_nuts_transition_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, eps, None, max_depth,
                                                       1000.0, C.byref(rc), C.byref(run.zin.c), C.byref(run.zout.c),
                                                       C.byref(st), run.flags))
        else:
            ctx.check(ctx.lib.ahmc_nuts_sample_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, eps, None, max_depth, 1000.0,
                                                   T, C.byref(rc), C.byref(run.zin.c), C.byref(run.zout.c), dr, C.byref(st),
                                                   run.flags))
    return call


def test_nuts_builtin_and_adaptive():
    D, N = 17, 9
    h, om, ome, th, r, rng = problem("diag_gauss", "diag", D, N, 5)
    s0 = start_of(h, th, np.zeros_like(th))
    check(D, N, s0, nuts_call(h, 0.2), dr=False)
    check(D, N, s0, nuts_call(h, 0.2, T=3, draws=True), dr=False)
    check(D, N, s0, nuts_call(h, 0.2, T=4, draws=True, cfg=adapt_cfg(D, 1, 0.2)), dr=False)
    hd = A.Hamiltonian(A.DenseEuclideanMetric(np.eye(D) * 0.8), h.target)
    check(D, N, s0, nuts_call(hd, 0.2, T=4, draws=True, cfg=adapt_cfg(D, 3, 0.2, dense=True)), dr=False)


@pytest.mark.parametrize("D", [33, 129])
def test_nuts_cooperative_dense(D):
    N = 9
    h, om, ome, th, r, rng = problem("dense_gauss", "dense", D, N, D)
    check(D, N, start_of(h, th, np.zeros_like(th)), nuts_call(h, 0.1), dr=False)


USER_ONE_LANE = r'''
__device__ double ahmc_user_logp_grad(const double* th, double* g, int D, const double* p) {
    double s = 0.0;
    for (int d = 0; d < D; ++d) { g[d] = -th[d]; s = fma(th[d], th[d], s); }
    return -0.5 * s;
}
'''
USER_GROUP = r'''
#define AHMC_USER_GROUPWISE
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    double s = 0.0;
    for (int d = grp.lane; d < D; d += grp.size) { g[d] = -th[d]; s = fma(th[d], th[d], s); }
    return -0.5 * s;
}
'''


@pytest.mark.parametrize("form", ["one_lane", "group"])
def test_run_time_compiled_target(form):
    D, N, eps, L_ = 24, 7, 0.1, 6
    rng = np.random.default_rng(4)
    Minv = np.exp(rng.uniform(-0.5, 0.5, D))
    h = A.Hamiltonian(A.DiagEuclideanMetric(Minv), A.UserTarget(D, USER_ONE_LANE if form == "one_lane" else USER_GROUP))
    th, r = rng.normal(size=(D, N)), rng.normal(size=(D, N))
    om, ome = oc.Model(oc.STD_NORMAL, D), oc.Metric(oc.DIAG, Minv)
    zo, _, _ = oc.leapfrog(om, ome, eps, oc.phasepoint(om, ome, th, r), L_)
    check(D, N, start_of(h, th, r), leapfrog_call(h, eps, L_), oracle=lambda vals, run: close_to(vals, zo))
    check(D, N, start_of(h, th, np.zeros_like(th)), nuts_call(h, 0.3), dr=False)


# ------------------------------------------------------------------------------------------------ find_good_stepsize, adaptor stats
@pytest.mark.parametrize("D", [12, 600])
def test_find_good_stepsize_with_momentum(D):
    N = 5
    h, om, ome, th, r, rng = problem("diag_gauss", "diag", D, N, D)
    nt = rng.normal(size=(N, D))

    def call(run):
        ctx = A.get_context(0)
        run.ins += [run.zin.f[k] for k in ("theta", "lp_gradient", "lp_value")]
        md, keep = h.metric._desc(D, N, run.like)
        rc = run.tape_rng(nt)
        eps = run.out("eps", N)
        r_out = run.out("r_out", D, N, run.ld_in)
        ctx.check(ctx.lib.ahmc_find_good_stepsize_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, C.byref(run.zin.c),
                                                      C.byref(rc), 0.1, 100, eps.ptr, r_out.ptr, run.flags))

    check(D, N, start_of(h, th, r), call, layouts=ONE_LD)


@pytest.mark.parametrize("D,N", [(7, 5), (40, 33)])
def test_adapt_summary_and_cov_against_numpy(D, N):
    rng = np.random.default_rng(D)
    th, alpha = rng.normal(size=(N, D)), rng.uniform(0.2, 1.5, N)
    mean = th.mean(0)

    def summary(run):
        ctx = A.get_context(0)
        t = run.inp("theta", D, N, run.ld_in, data=th)
        a = run.inp("alpha", N, data=alpha)
        ctx.check(ctx.lib.ahmc_adapt_summary_f64(ctx.h, D, N, t.ptr, run.ld_in, a.ptr, run.out("out", 2 + 2 * D).ptr, run.flags))

    def summary_np(vals, run):
        o = vals["out"]
        assert o[0] == N and abs(o[1] - np.minimum(alpha, 1).sum()) < 1e-12 * N
        assert rel_err(o[2:2 + D], mean) < 1e-11 and rel_err(o[2 + D:], ((th - mean) ** 2).sum(0)) < 1e-11

    def cov(run):
        ctx = A.get_context(0)
        t = run.inp("theta", D, N, run.ld_in, data=th)
        m = run.inp("mean", D, data=mean)
        ctx.check(ctx.lib.ahmc_adapt_cov_f64(ctx.h, D, N, t.ptr, run.ld_in, m.ptr, run.out("out", D * D).ptr, run.flags))

    def cov_np(vals, run):
        assert rel_err(vals["out"].reshape(D, D), (th - mean).T @ (th - mean)) < 1e-11

    check(D, N, None, summary, layouts=ONE_LD, pp=False, oracle=summary_np)
    check(D, N, None, cov, layouts=ONE_LD, pp=False, oracle=cov_np)


# ------------------------------------------------------------------------------------------------ host buffers
def test_host_buffer_transitions_and_nuts():
    """the staged host path of the static transition and of NUTS writes D rows per chain back"""
    D, N = 30, 8
    h, om, ome, th, r, rng = problem("diag_gauss", "diag", D, N, 9)
    s0 = start_of(h, th, np.zeros_like(th))
    check(D, N, s0, hmc_call(h, 0.1, 6), dr=False)
    check(D, N, s0, nuts_call(h, 0.2), dr=False)


@pytest.mark.parametrize("N", [300, 4099])
def test_pipelined_host_lane(N):
    """host-buffer leapfrog calls with N >= 256 take the chunked lane: with copy-engine downloads (staged) and with the
    kernel's own stores to page-locked memory (direct); with everything page-locked from 1024 chains on, the first calls of
    a shape try each transport in turn"""
    D = 64
    h, om, ome, th, r, rng = problem("diag_gauss", "diag", D, N, N)  # a shared M^-1: page-locked calls are page-locked throughout
    eps = 0.05 * np.exp(rng.uniform(-0.3, 0.3, N))
    s0 = start_of(h, th, r)
    seen = []
    call = leapfrog_call(h, eps, 9)

    def traced(run):
        call(run)
        if run.where != "dev":
            seen.append(A.get_context(0).last_transport())

    layouts = [("pinned", "D+1", "2D+3"), ("pageable", "2D+3", "D+1"), ("pinned", "D+4", "D+4"), ("pageable", "D+1", None)]
    if N >= 1024:  # enough page-locked calls of one shape to walk through every candidate transport
        layouts += [("pinned", "D+1", "2D+3")] * 4
    # at D = 64 an odd ld moves K1 off its pair kernel: the launch count stays 1 per chunk, and the oracle decides
    zo, _, _ = oc.leapfrog(om, ome, eps, oc.phasepoint(om, ome, th, r), 9)
    # the transports cut the chains into different numbers of chunks (one launch each): counted from the transport below
    check(D, N, s0, traced, layouts=layouts, oracle=lambda vals, run: close_to(vals, zo), same_kernel=pair_kernel_kept(D),
          count_launches=N < 1024)
    assert any("down=ce" in t for t in seen) and any("down=direct" in t for t in seen), seen


def test_host_buffers_read_no_further_than_the_last_chains_rows():
    """a D x N host argument needs ld * (N - 1) + D doubles: theta and r end where an inaccessible page begins, so an upload
    that reads the last chain's padding faults the (separate) process instead of passing unnoticed.  The staged lane
    (N = 3) and the pipelined copy-engine lane (N = 300) both return the device call's bytes."""
    import os
    import subprocess
    import sys

    code = r'''
import ctypes as C, mmap, numpy as np, torch, ahmc_b200 as A
from ahmc_b200 import _lib as L
libc = C.CDLL(None)
libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
PAGE, keep = mmap.PAGESIZE, []

def tail_array(values):
    """`values` in the last bytes before a PROT_NONE page"""
    nb = values.size * 8
    pages = (nb + PAGE - 1) // PAGE + 1
    m = mmap.mmap(-1, pages * PAGE)
    base = C.addressof(C.c_char.from_buffer(m))
    assert libc.mprotect(base + (pages - 1) * PAGE, PAGE, 0) == 0
    addr = base + (pages - 1) * PAGE - nb
    C.memmove(addr, values.ctypes.data, nb)
    keep.append(m)
    return addr

for D, N in ((5, 3), (64, 300)):
    ld = 2 * D + 4  # a multiple of 4: at D = 64 K1 keeps the pair kernel of the device call it is compared with
    rng = np.random.default_rng(N)
    h = A.Hamiltonian(A.DiagEuclideanMetric(np.exp(rng.uniform(-0.5, 0.5, D))), A.DiagGaussian(rng.normal(size=D), np.ones(D)))
    th, r = rng.normal(size=(N, D)), rng.normal(size=(N, D))
    zd = A.step(A.Leapfrog(0.1), h, A.phasepoint(h, torch.as_tensor(th, device="cuda"), torch.as_tensor(r, device="cuda")), 7)
    pad = lambda a: np.concatenate([a, np.zeros((N, ld - D))], 1).ravel()[: ld * (N - 1) + D].copy()
    ctx = A.get_context(0)
    md, _ = h.metric._desc(D, N, np.empty(0))
    outs = [np.zeros(ld * N) for _ in range(4)] + [np.zeros(N), np.zeros(N)]
    zi = L.PhasePoint(tail_array(pad(th)), tail_array(pad(r)), None, None, None, None, ld)
    zo = L.PhasePoint(outs[0].ctypes.data, outs[1].ctypes.data, outs[4].ctypes.data, outs[2].ctypes.data, outs[5].ctypes.data,
                      outs[3].ctypes.data, ld)
    ctx.check(ctx.lib.ahmc_leapfrog_f64(ctx.h, h.target.handle(ctx), C.byref(md), D, N, 0.1, None, 7, 0.0, C.byref(zi), C.byref(zo),
                                        None, None, A.FLAG_HOST_BUFFERS))
    got = outs[0].reshape(N, ld)[:, :D]
    assert np.array_equal(got, zd.theta.cpu().numpy()) and np.array_equal(outs[4], zd.lp.value.cpu().numpy()), (D, N)
print("ok")
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pr = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root, timeout=300)
    assert pr.returncode == 0 and "ok" in pr.stdout, (pr.returncode, pr.stderr[-2000:])
