"""K1's two-chains-per-warp fast path (`leapfrog_pair_kernel`, lane-contiguous full tiles D = 64, 128): both coefficient
forms (one set shared by the pair; per-chain eps and M^-1), ragged N, and pairs where one chain fails the magnitude proof
and is re-run alone by the exact path.  The CPU tests run the kernel source under the SIMT emulator at D = 64
(tests/simt_emu/pair_emu.cpp), against the oracle and under ThreadSanitizer; the GPU test runs the library at D = 128."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle_c as oc
from tests.helpers import rel_err
from tests.test_simt_emulation import KINDS, MKINDS, EmuLf, P, _lf_system

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "simt_emu")
INCLUDES = ["-I", os.path.join(EMU, "include"), "-I", os.path.join(ROOT, "advancedhmc.jl_b200", "csrc"), "-I", os.path.join(ROOT, "include")]


@pytest.fixture(scope="module")
def emu_pair(tmp_path_factory):
    out = tmp_path_factory.mktemp("simt_pair") / "libpair_emu.so"
    subprocess.run(["g++", "-O1", "-std=c++20", "-shared", "-fPIC", "-pthread", "-ffp-contract=off", "-x", "c++", *INCLUDES,
                    os.path.join(EMU, "simt_emu.cpp"), os.path.join(EMU, "pair_emu.cpp"), "-o", str(out)], check=True)
    return C.CDLL(str(out))


@pytest.mark.parametrize("per_chain_eps", [False, True], ids=["shared-coef", "chain-eps"])
@pytest.mark.parametrize("with_g", [True, False], ids=["cached-grad", "no-grad"])
def test_pair_kernel_under_emulation_matches_oracle(emu_pair, per_chain_eps, with_g):
    """N = 7: three full pairs and a last warp whose B shadows chain 6; chain 2 (A of its pair) is large enough to defeat the
    proof but stays finite, chain 5 (B of its pair) overflows at step 1; their partners stay on the fast path."""
    D, N, n = 64, 7, 12
    rng = np.random.default_rng(5)
    model, metric, p0, dp1, Minv, cholU = _lf_system("diag_gauss", "diag", D, rng)
    th, r = rng.normal(size=(N, D)), rng.normal(size=(N, D))
    th[2, 9] = 1e120
    th[5, 3] = 1e250
    eps_chain = 0.1 * np.exp(rng.uniform(-0.3, 0.3, N)) if per_chain_eps else None
    z0 = oc.phasepoint(model, metric, th.T, r.T)
    zo, so, do = oc.leapfrog(model, metric, eps_chain if per_chain_eps else 0.1, z0, n)
    g_in, lp_in = np.ascontiguousarray(z0.lp_gradient.T), np.ascontiguousarray(z0.lp_value)
    o = {k: np.zeros((N, D)) for k in ("th", "r", "g", "dr")}
    lp_o, lk_o = np.zeros(N), np.zeros(N)
    status, done = np.zeros(N, dtype=np.uint32), np.zeros(N, dtype=np.int32)
    q = EmuLf(model_kind=KINDS["diag_gauss"], metric_kind=MKINDS["diag"], D=D, N=N, p0=P(p0), p1=P(dp1), c0=0.0, Minv=P(Minv),
              minv_stride=0, cholU=None, eps=0.1, eps_chain=P(eps_chain) if per_chain_eps else None, n_steps=n, fwd=1,
              temper_alpha=0.0, th_in=P(th), r_in=P(r), g_in=P(g_in) if with_g else None, lp_in=P(lp_in), th_out=P(o["th"]),
              r_out=P(o["r"]), g_out=P(o["g"]), lp_out=P(lp_o), lk_out=P(lk_o), dr_out=P(o["dr"]), status=P(status),
              steps_done=P(done), flags=0, hmc=0)
    assert emu_pair.emu_leapfrog_pair(C.byref(q)) == 0
    assert list(status) == list(so) and list(done) == list(do) and done[5] == 1 and done[2] == n
    ok = [c for c in range(N) if c != 5]
    for k, want in (("th", zo.theta), ("r", zo.r), ("g", zo.lp_gradient), ("dr", zo.lk_gradient)):
        assert rel_err(o[k][ok].T, want[:, ok]) < 1e-10, k
    assert np.allclose(lp_o[ok], zo.lp_value[ok], rtol=1e-10, atol=1e-10) and np.allclose(lk_o[ok], zo.lk_value[ok], rtol=1e-10, atol=1e-10)
    assert lp_o[5] == -np.inf


def test_pair_kernel_source_is_data_race_free_under_thread_sanitizer(tmp_path):
    """Every CUDA thread is a host thread whose only synchronisation is what the kernel asks for: a missing __syncwarp
    between A's and B's use of the warp (votes, reductions, the exact path's shared-memory slab) is a reported race."""
    exe = tmp_path / "race_pair"
    b = subprocess.run(["g++", "-DPAIR_RACE_MAIN", "-w", "-O1", "-g", "-std=c++20", "-pthread", "-fsanitize=thread", "-ffp-contract=off",
                        "-x", "c++", *INCLUDES, os.path.join(EMU, "simt_emu.cpp"), os.path.join(EMU, "pair_emu.cpp"), "-o", str(exe)],
                       capture_output=True, text=True)
    if b.returncode != 0 and ("tsan" in b.stderr.lower() or "sanitize" in b.stderr.lower()):
        pytest.skip("ThreadSanitizer runtime not available to g++ here")
    assert b.returncode == 0, b.stderr[-2000:]
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr.strip().splitlines()[0])
    assert r.stderr.count("WARNING: ThreadSanitizer: data race") == 0 and r.returncode == 0, r.stderr[-3000:] + r.stdout[-500:]
    assert r.stdout.count("rc 0 finished 11 of 11") == 2


@pytest.mark.gpu
def test_pair_kernel_per_chain_eps_and_minv_matches_oracle():
    """D = 128 with a per-chain step size and a per-chain Diag M^-1 (the pair's per-chain coefficient form), ragged N = 9,
    chain 6 outside the proof's range (re-run exactly, partner 7 fast): every chain equals the oracle run on it alone."""
    import torch

    import ahmc_b200 as A

    D, N, n = 128, 9, 20
    rng = np.random.default_rng(9)
    s = np.exp(np.linspace(np.log(0.1), np.log(10.0), D))
    m = rng.normal(size=D)
    th, r = rng.normal(size=(N, D)) * s, rng.normal(size=(N, D)) / s
    th[6, 4] = 1e120
    Minv = (s * s)[None, :] * np.exp(rng.uniform(-0.3, 0.3, (N, D)))
    eps = 0.1 * np.exp(rng.uniform(-0.3, 0.3, N))
    h = A.Hamiltonian(A.DiagEuclideanMetric(Minv), A.DiagGaussian(m, s, normalised=False))
    dev = "cuda:0"
    z1, info = A.step(A.Leapfrog(eps), h, A.phasepoint(h, torch.as_tensor(th, device=dev), torch.as_tensor(r, device=dev)), n,
                      return_info=True)
    npy = lambda t: t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    assert (npy(info.status) == 0).all() and (npy(info.steps_done) == n).all()
    got = {k: npy(v) for k, v in (("th", z1.theta), ("r", z1.r), ("g", z1.lp.gradient))}
    lp, lk = npy(z1.lp.value), npy(z1.lk.value)
    om = oc.Model(oc.DIAG_GAUSS, D, m, s)
    for c in range(N):
        ome = oc.Metric(oc.DIAG, Minv[c].copy())
        zo = oc.leapfrog(om, ome, float(eps[c]), oc.phasepoint(om, ome, th[c:c + 1].T, r[c:c + 1].T), n)[0]
        assert rel_err(got["th"][c], zo.theta[:, 0]) < 1e-10 and rel_err(got["r"][c], zo.r[:, 0]) < 1e-10, c
        assert rel_err(got["g"][c], zo.lp_gradient[:, 0]) < 1e-10, c
        assert abs(lp[c] - zo.lp_value[0]) <= 1e-10 * abs(zo.lp_value[0]) and abs(lk[c] - zo.lk_value[0]) <= 1e-10 * abs(zo.lk_value[0]), c
