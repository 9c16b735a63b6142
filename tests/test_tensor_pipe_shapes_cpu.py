"""Shape sweep of the three kernels that stream matrices through shared memory with bulk copies behind mbarriers and multiply
on the fp64 tensor pipe -- K4 (`dense_traj_kernel`), K6 (`glm_traj_kernel`) and the cooperative NUTS products
(`matvec_coop` / `upper_solve_coop`, the COOP form of `nuts_kernel`) -- under the strict CPU SIMT emulator
(tests/simt_emu/: exact, poisoned and guarded shared memory per launch; bulk-copy and mbarrier rules checked), against the
C oracle or tests/glm_ref.py at 1e-10, with status, steps and tree statistics compared exactly.

The shapes are the ones where these kernels can go wrong: every row-block count RB of K4 and K6 and both sides of each
64-row boundary, ragged chain tiles, fewer / exactly / more chunks than pipeline stages and a partial last chunk, every
COOP layout E with its chunk width and stage count, odd D (whose unpadded matrices take the `__ldg` staging), and idle
warps.  Each emulated run happens in a forked child, so a contract violation (the emulator aborts with a message naming
it) fails the one test instead of ending the session."""
import ctypes as C
import os
import sys
import traceback

import numpy as np
import pytest

from oracle import oracle_c as oc
from tests import emu as E
from tests import glm_ref as R
from tests.emu import P, EmuNuts
from tests.helpers import rel_err
from tests.test_glm_cpu import _setup as _glm_setup, assert_z, close, run_emu as _glm_run
from tests.test_simt_emulation import _case as _nuts_case, _dense_run

POISON_NAN, POISON_HUGE = 0, 1


@pytest.fixture(scope="module")
def libs():
    """the K4, K6 and NUTS harnesses on the strict emulator"""
    return dict(zip(("dense", "glm", "nuts"), E.harnesses("dense", "glm", "nuts")))


def isolated(lib, poison, fn, *args, **kw):
    """run fn in a forked child with the emulator's poison set; a failed comparison or an emulator abort fails the test"""
    sys.stdout.flush()
    sys.stderr.flush()
    pid = os.fork()
    if pid == 0:
        code = 0
        try:
            lib.emu_set_poison(poison)
            fn(*args, **kw)
        except BaseException:
            traceback.print_exc()
            code = 1
        finally:
            sys.stderr.flush()
            os._exit(code)
    _, st = os.waitpid(pid, 0)
    if os.WIFSIGNALED(st):
        pytest.fail(f"the emulated kernel was stopped by signal {os.WTERMSIG(st)} (a contract violation: see the captured stderr)")
    assert os.WEXITSTATUS(st) == 0, "the emulated run disagrees with the reference (traceback in the captured stderr)"


# ------------------------------------------------------------------------------------------------------------------- K4
def _dense_check(lib, kind, mkind, D, N, eps, n, fwd, exact_chain=None):
    zo, o, lp_o, lk_o, status, done, need = _dense_run(lib, kind, mkind, D, N, eps, n, fwd, seed=300 + D + N, per_chain_eps=True,
                                                       poison=exact_chain)
    Dp = -(-D // 64) * 64
    CT = 8 * (4 if Dp <= 64 else (2 if Dp <= 256 else 1))
    ok = np.ones(N, dtype=bool)
    if exact_chain is not None:  # its whole tile is handed to the exact kernel, untouched here
        t0 = exact_chain // CT * CT
        ok[t0:t0 + CT] = False
        assert (need[~ok] == 1).all() and np.isnan(o["th"][~ok]).all() and (status[~ok] == 7).all()
    assert (need[ok] == 0).all() and (done[ok] == n).all() and (status[ok] == 0).all()
    for k, ref in (("th", zo.theta), ("r", zo.r), ("g", zo.lp_gradient), ("dr", zo.lk_gradient)):
        assert rel_err(o[k][ok].T, ref[:, ok]) < 1e-10, k
    assert np.allclose(lp_o[ok], zo.lp_value[ok], rtol=1e-10, atol=1e-10)
    assert np.allclose(lk_o[ok], zo.lk_value[ok], rtol=1e-10, atol=1e-10)


_K4_COMBOS = [("dense_gauss", "dense"), ("dense_gauss", "diag"), ("dense_gauss", "unit"), ("diag_gauss", "dense"),
              ("std_normal", "dense")]
# every RB (= ceil(D / 64)) from 1 to 8 and both sides of each 64-boundary; N leaves a ragged last tile (tiles of 32, 16
# and 8 chains for RB 1-2, 2-4 and 5-8); the five target x metric combinations rotate over D, all five at D = 65 and 321
K4_CASES = []
for i, D in enumerate((1, 63, 64, 65, 129, 192, 193, 320, 321, 448, 512)):
    N = 37 if D <= 128 else (19 if D <= 256 else 9)
    for kind, mkind in (_K4_COMBOS if D in (65, 321) else [_K4_COMBOS[i % 5]]):
        K4_CASES.append((kind, mkind, D, N, 0.1 if D < 300 else 0.06, 3 if D <= 256 else 2, i % 2))


@pytest.mark.parametrize("kind,mkind,D,N,eps,n,fwd", K4_CASES, ids=[f"{c[0]}-{c[1]}-D{c[2]}-N{c[3]}" for c in K4_CASES])
def test_dense_tile_kernel_shapes_match_oracle(libs, kind, mkind, D, N, eps, n, fwd):
    isolated(libs["dense"], POISON_NAN, _dense_check, libs["dense"], kind, mkind, D, N, eps, n, fwd)


@pytest.mark.parametrize("D,N,chain", [(40, 37, 34), (193, 19, 3), (321, 9, 8)])
def test_dense_tile_kernel_hands_one_chains_tile_to_the_exact_path(libs, D, N, chain):
    """a start beyond the linear-dynamics proof flags its tile only; the other tiles' results stand"""
    isolated(libs["dense"], POISON_NAN, _dense_check, libs["dense"], "dense_gauss", "dense", D, N, 0.08, 2, 1, exact_chain=chain)


# ------------------------------------------------------------------------------------------------------------------- K6
def glm_shape(D):
    """(chunk rows nc, stages S) as glm_tile_shape (ahmc_glm.cu) picks them: the largest chunk, then the most stages, that
    fit 227 KB of shared memory"""
    lds = -(-D // 8) * 8 + 4
    for c in (64, 32, 16, 8):
        for s in (3, 2):
            if (s * c * lds + 16 * lds + 2 * 16 * (c + 4) + 8 * 16 * 3) * 8 + 3 * 8 <= 227 * 1024:
                return c, s
    raise AssertionError(D)


def _glm_check(lib, family, D, n, N, metric, pce, cached, steps):
    X, y, prec, Minv, th, r, eps = _glm_setup(family, D, n, N, metric, pce, seed=7 * D + n)
    c0 = 0.25 - (0 if family == "bernoulli_logit" else R.gammaln(y + 1).sum())
    z0 = R.phasepoint(family, X, y, prec, 0.25, Minv, th, r)
    o, status, done, shape = _glm_run(lib, family, X, y, prec, c0, Minv, 0.0, 0, th, r, None)  # phasepoint
    assert shape == glm_shape(D)
    for k in ("g", "dr", "lp", "lk"):
        close(o[k], z0[k])
    zo, st_ref, steps_ref = R.leapfrog(family, X, y, prec, 0.25, Minv, eps, z0, steps)
    o, status, done, _ = _glm_run(lib, family, X, y, prec, c0, Minv, eps, steps, th.copy(), r.copy(),
                                  np.ascontiguousarray(z0["g"]) if cached else None)
    assert_z(o, zo)
    assert (status == st_ref).all() and (done == steps_ref).all() and (status == 0).all()


def _glm_rows(D):
    nc, S = glm_shape(D)
    return sorted({1, 7, 8, 9, nc - 1, nc, nc + 1, S * nc, S * nc + 1})


# RB = 1..4 (D 1..256; D = 256 streams 32-row chunks); rows: fewer chunks than stages, exactly S, more, a partial last chunk.
# Every row count at D = 9, 129 and 256; at the other D the row counts around the chunk and the stage boundary.
K6_CASES = []
_metrics = ("unit", "diag", "chain")
for i, D in enumerate((1, 8, 9, 64, 65, 129, 192, 193, 256)):
    nc, S = glm_shape(D)
    rows = _glm_rows(D) if D in (9, 129, 256) else [7, nc, S * nc + 1]
    for j, n in enumerate(rows):
        k = i + j
        K6_CASES.append(("bernoulli_logit" if k % 2 == 0 else "poisson_log", D, n, 17 if D <= 128 else 9, _metrics[k % 3],
                         k % 2 == 1, k % 4 != 3, 2 if k % 3 else -2))


@pytest.mark.parametrize("family,D,n,N,metric,pce,cached,steps", K6_CASES,
                         ids=[f"{c[0]}-D{c[1]}-n{c[2]}-{c[4]}{'-nog' if not c[6] else ''}" for c in K6_CASES])
def test_glm_tile_kernel_shapes_match_reference(libs, family, D, n, N, metric, pce, cached, steps):
    isolated(libs["glm"], POISON_NAN, _glm_check, libs["glm"], family, D, n, N, metric, pce, cached, steps)


def test_glm_tile_shape_streams_32_row_chunks_at_d256():
    """the shapes the sweep relies on (the harness checks glm_tile_shape against glm_shape at every case): three stages of
    64 rows at D = 64, two at D = 129, 32-row chunks from D = 192 on"""
    assert glm_shape(64) == (64, 3) and glm_shape(129) == (64, 2) and glm_shape(192)[0] == glm_shape(256)[0] == 32


# ------------------------------------------------------------------------------------------------------------ COOP NUTS
# every layout E (1, 2, 4, 8, 16), chunk width KC 24 (E <= 8) and 16 (E = 16), stage counts 3 (D <= 256) and 2, ragged last
# chunks and odd D; N = 1, 7 or 9 leaves warps of a block idle; plain and column-padded matrices
COOP_D = (17, 24, 25, 32, 33, 64, 65, 100, 128, 129, 200, 256, 257, 300, 512)
COOP_CASES = []
for i, D in enumerate(COOP_D):
    N = (1, 7, 9)[i % 3]
    for padded in (0, 1):
        COOP_CASES.append(("dense_gauss", "dense", D, N, padded, 4 if D <= 256 else 3))


def _nuts_check(lib, kind, mkind, D, N, padded, depth, sampler="multinomial", criterion="generalised", temper=0.0, eps=None):
    if eps is None:
        eps = 0.3 if D < 100 else 0.25
    so = _nuts_case(lib, kind, mkind, D, N, eps, sampler, criterion, seed=11 + D + N, max_depth=depth, coop_padded=padded,
                    temper=temper)
    assert so.n_steps.max() >= 3


@pytest.mark.parametrize("kind,mkind,D,N,padded,depth", COOP_CASES,
                         ids=[f"D{c[2]}-N{c[3]}-{'padded' if c[4] else 'plain'}" for c in COOP_CASES])
def test_cooperative_nuts_shapes_match_oracle(libs, kind, mkind, D, N, padded, depth):
    isolated(libs["nuts"], POISON_NAN, _nuts_check, libs["nuts"], kind, mkind, D, N, padded, depth)


COOP_COMBOS = [("dense_gauss", "unit", 25, 7), ("dense_gauss", "diag", 100, 9), ("dense_gauss", "unit", 300, 7),
               ("dense_gauss", "diag", 257, 1), ("diag_gauss", "dense", 65, 9), ("diag_gauss", "dense", 129, 7),
               ("funnel", "dense", 24, 9), ("funnel", "dense", 200, 7)]


@pytest.mark.parametrize("kind,mkind,D,N", COOP_COMBOS, ids=[f"{c[0]}-{c[1]}-D{c[2]}" for c in COOP_COMBOS])
def test_cooperative_nuts_target_metric_combinations_match_oracle(libs, kind, mkind, D, N):
    """the products for only one of the two operators: a dense target with a Unit or Diag metric, a Dense metric with a
    separable target"""
    isolated(libs["nuts"], POISON_NAN, _nuts_check, libs["nuts"], kind, mkind, D, N, D % 2, 4, eps=0.2 if kind == "funnel" else None)


SAMPLERS = [(s, c) for s in ("multinomial", "slice") for c in ("generalised", "classic", "strict")]


@pytest.mark.parametrize("D", [33, 129])
@pytest.mark.parametrize("sampler,criterion", SAMPLERS, ids=[f"{s}-{c}" for s, c in SAMPLERS])
def test_every_sampler_and_criterion_at_cooperative_shapes_match_oracle(libs, D, sampler, criterion):
    """the default family runs COOP; SliceTS and the Classic / Strict criteria run the warp form at the same shapes"""
    isolated(libs["nuts"], POISON_NAN, _nuts_check, libs["nuts"], "dense_gauss", "dense", D, 7, 0, 4, sampler, criterion)


def test_cooperative_nuts_tempered_leaf_matches_oracle(libs):
    isolated(libs["nuts"], POISON_NAN, _nuts_check, libs["nuts"], "dense_gauss", "dense", 65, 9, 1, 4, temper=1.05)


def _coop_multi(lib, D, N, T, padded):
    """T transitions in one launch (the pipeline's barriers re-armed at every product of every transition) equal T
    single-transition launches at Philox offsets 0 .. T-1, each started from the previous one's draw"""
    rng = np.random.default_rng(D)
    B = rng.normal(size=(D, D))
    Pm, mu = np.ascontiguousarray(B @ B.T / D + np.eye(D)), rng.normal(size=D)
    B = rng.normal(size=(D, D))
    Minv = np.ascontiguousarray(B @ B.T / D + 0.5 * np.eye(D))
    cholU = np.ascontiguousarray(np.linalg.cholesky(Minv))

    def run(th, T_, offset):
        th = np.ascontiguousarray(th)
        g_in = np.ascontiguousarray((th - mu) @ Pm)
        lp_in = np.ascontiguousarray(-0.5 * np.einsum("nd,nd->n", th - mu, g_in))
        r = np.zeros((N, D))
        out = {k: np.zeros((N, D)) for k in ("th", "r", "g")}
        lp_o, lk_o = np.zeros(N), np.zeros(N)
        acc, dH, dHm = (np.zeros(T_ * N) for _ in range(3))
        ns, td, ne = np.zeros(T_ * N, dtype=np.int32), np.zeros(T_ * N, dtype=np.int32), np.zeros(T_ * N, dtype=np.uint8)
        draws = np.zeros((T_, N, D))
        q = EmuNuts(model_kind=oc.DENSE_GAUSS, metric_kind=oc.DENSE, D=D, N=N, p0=P(mu), p1=P(Pm), c0=0.0, Minv=P(Minv),
                    minv_stride=0, cholU=P(cholU), eps=0.25, eps_chain=None, max_depth=4, delta_max=1000.0, sampler=0, criterion=0,
                    seed=17, offset=offset, normal_tape=None, exp_tape=None, exp_stride=0, dir_tape=None, dir_stride=0,
                    partial_alpha=0.0, refresh=1, th_in=P(th), r_in=P(r), g_in=P(g_in), lp_in=P(lp_in), th_out=P(out["th"]),
                    r_out=P(out["r"]), g_out=P(out["g"]), lp_out=P(lp_o), lk_out=P(lk_o), n_steps=P(ns), tree_depth=P(td),
                    numerical=P(ne), acc=P(acc), dH=P(dH), dHmax=P(dHm), n_transitions=T_, draws=P(draws), adapt=0,
                    temper_alpha=0.0, coop_padded=padded)
        assert lib.emu_nuts(C.byref(q)) == 0
        return draws, ns.reshape(T_, N), td.reshape(T_, N)

    th0 = np.tile(np.linspace(-1, 1, D), (N, 1))
    draws, ns, td = run(th0, T, 0)
    th = th0
    for t in range(T):
        d1, ns1, td1 = run(th, 1, t)
        assert (ns1[0] == ns[t]).all() and (td1[0] == td[t]).all(), t
        assert rel_err(d1[0], draws[t]) < 1e-10, t
        th = d1[0]
    assert ns.max() >= 3


@pytest.mark.parametrize("D,N,padded", [(40, 9, 0), (129, 7, 1), (300, 1, 0)])
def test_cooperative_nuts_several_transitions_per_launch_equal_single_launches(libs, D, N, padded):
    isolated(libs["nuts"], POISON_NAN, _coop_multi, libs["nuts"], D, N, 3, padded)


# ------------------------------------------------------------------------------------------------- +-1e300 poison pass
# NaN poison can hide behind fmax or a comparison; a huge finite value instead trips the magnitude proofs and the energies
@pytest.mark.parametrize("case", ["k4-D65", "k4-D512", "k6-D9-n1", "k6-D256-n33", "coop-D33", "coop-D300-padded"])
def test_huge_finite_poison_subset(libs, case):
    if case == "k4-D65":
        isolated(libs["dense"], POISON_HUGE, _dense_check, libs["dense"], "dense_gauss", "dense", 65, 37, 0.1, 3, 1)
    elif case == "k4-D512":
        isolated(libs["dense"], POISON_HUGE, _dense_check, libs["dense"], "diag_gauss", "dense", 512, 9, 0.06, 2, 0)
    elif case == "k6-D9-n1":
        isolated(libs["glm"], POISON_HUGE, _glm_check, libs["glm"], "bernoulli_logit", 9, 1, 17, "diag", True, False, 2)
    elif case == "k6-D256-n33":
        isolated(libs["glm"], POISON_HUGE, _glm_check, libs["glm"], "poisson_log", 256, 33, 9, "chain", False, True, -2)
    elif case == "coop-D33":
        isolated(libs["nuts"], POISON_HUGE, _nuts_check, libs["nuts"], "dense_gauss", "dense", 33, 9, 0, 4)
    else:
        isolated(libs["nuts"], POISON_HUGE, _nuts_check, libs["nuts"], "dense_gauss", "dense", 300, 7, 1, 3)


# ------------------------------------------------------------------------------------------ AddressSanitizer builds
ASAN = {"nuts": 8, "lf": 5, "dense": 4, "glm": 1}


@pytest.mark.parametrize("name", list(ASAN))
def test_harnesses_are_clean_under_address_sanitizer(name):
    """The four tensor-pipe harnesses' small cases (their RACE_<NAME> mains) under AddressSanitizer: host
    buffers, the emulator's arenas and the kernels' global-memory accesses stay in bounds (the strict emulator already
    guards shared memory itself)"""
    r = E.sanitized(name, "address")
    assert "ERROR: AddressSanitizer" not in r.stderr and r.returncode == 0, r.stderr[-3000:] + r.stdout[-500:]
    assert r.stdout.count("rc 0") == ASAN[name]
