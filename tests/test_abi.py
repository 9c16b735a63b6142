"""CPU tests: the C-ABI library loads and exports every symbol include/ahmc_b200.h declares, and the
host-side mirror of the reference's integrator interface behaves like test/integrator.jl:34-106."""
import ctypes
import os
import re

import numpy as np
import pytest

import ahmc_b200 as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "ahmc_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ahmc_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(os.path.join(ROOT, "advancedhmc.jl_b200", "libahmc_b200.so"))
    names = _declared_symbols()
    assert len(names) >= 14
    for n in names:
        assert hasattr(lib, n), n
    assert set(names) == set(A._lib.PROTOTYPES), set(names) ^ set(A._lib.PROTOTYPES)
    lib.ahmc_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.ahmc_version()


def test_no_cpu_fallback_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        A.get_context(0)


def test_product_package_never_imports_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "advancedhmc.jl_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(root, f)).read()
                assert "oracle_c" not in txt and "oracle_np" not in txt and "ahmc_oracle" not in txt, f


def test_jitter_and_update_nom_step_size():
    """test/integrator.jl:34-87."""
    rng = np.random.default_rng(0)
    lf = A.Leapfrog(0.1)
    assert A.nom_step_size(lf) == 0.1 and A.step_size(lf) == 0.1
    assert A.jitter(rng, lf) is lf
    lj = A.JitteredLeapfrog(0.1, 0.5)
    assert lj.eps0 == 0.1 and lj.eps == 0.1 and A.nom_step_size(lj) == 0.1
    lj2 = A.jitter(rng, lj)
    assert lj2.eps0 == 0.1 and lj2.eps != 0.1 and A.step_size(lj2) == lj2.eps
    assert abs(lj2.eps - 0.1) <= 0.05 + 1e-15
    lf2 = A.update_nom_step_size(lf, 0.5)
    assert lf2 is not lf and A.nom_step_size(lf2) == 0.5 and A.step_size(lf2) == 0.5
    lj3 = A.update_nom_step_size(lj, 0.2)
    assert A.nom_step_size(lj3) == 0.2 and A.step_size(lj3) == 0.1
    ljv = A.jitter(rng, A.JitteredLeapfrog(np.full(5, 0.1), 1.0))
    assert ljv.eps.shape == (5,) and np.all(ljv.eps >= 0) and np.all(ljv.eps <= 0.2) and len(set(ljv.eps)) == 5


def test_temper_schedule():
    """test/integrator.jl:89-106."""
    lf = A.TemperedLeapfrog(0.01, 4.0)
    r = np.ones(5)
    got = [A.temper(lf, r, (i, half), 3)[0] for i in (1, 2, 3) for half in (True, False)]
    assert got == [2.0, 2.0, 2.0, 0.5, 0.5, 0.5]
    with pytest.raises(IndexError):
        A.temper(lf, r, (4, False), 3)


def test_nsteps():
    """trajectory.jl:240-243."""
    assert A.nsteps(A.Trajectory(A.EndPointTS, A.Leapfrog(0.1), A.FixedNSteps(7))) == 7
    assert A.nsteps(A.Trajectory(A.EndPointTS, A.Leapfrog(0.1), A.FixedIntegrationTime(1.0))) == 10
    assert A.nsteps(A.Trajectory(A.EndPointTS, A.Leapfrog(3.0), A.FixedIntegrationTime(1.0))) == 1
    with pytest.raises(ValueError):
        A.nsteps(A.Trajectory(A.EndPointTS, A.Leapfrog(np.full(3, 0.1)), A.FixedIntegrationTime(1.0)))


def test_ctypes_mirror_matches_the_header(tmp_path):
    """The Python binding restates the header's constants and struct layouts by hand: compile a tiny C program against
    include/ahmc_b200.h (gcc, no CUDA needed) that prints every flag / kind value and sizeof / offsetof of every struct,
    and compare with advancedhmc.jl_b200/_lib.py."""
    import subprocess

    from ahmc_b200 import _lib as L

    src = tmp_path / "abi_probe.c"
    src.write_text(r'''
#include <stddef.h>
#include <stdio.h>
#include "ahmc_b200.h"
#define P(name, v) printf("%s %lld\n", name, (long long)(v))
int main(void) {
    P("FLAG_HOST_BUFFERS", AHMC_FLAG_HOST_BUFFERS); P("FLAG_COMPAT_BREAK_ALL", AHMC_FLAG_COMPAT_BREAK_ALL);
    P("FLAG_ASYNC", AHMC_FLAG_ASYNC); P("FLAG_EXACT_CHECKS", AHMC_FLAG_EXACT_CHECKS); P("FLAG_NO_REFRESH", AHMC_FLAG_NO_REFRESH);
    P("FLAG_NUTS_SLICE_TS", AHMC_FLAG_NUTS_SLICE_TS); P("FLAG_NUTS_CLASSIC", AHMC_FLAG_NUTS_CLASSIC);
    P("FLAG_NUTS_STRICT", AHMC_FLAG_NUTS_STRICT); P("STATUS_NONFINITE", AHMC_STATUS_NONFINITE);
    P("sizeof_metric", sizeof(ahmc_metric)); P("metric.Minv", offsetof(ahmc_metric, Minv));
    P("metric.chain_stride", offsetof(ahmc_metric, chain_stride)); P("metric.cholU", offsetof(ahmc_metric, cholU));
    P("sizeof_phasepoint", sizeof(ahmc_phasepoint)); P("phasepoint.lk_gradient", offsetof(ahmc_phasepoint, lk_gradient));
    P("phasepoint.ld", offsetof(ahmc_phasepoint, ld));
    P("sizeof_stats", sizeof(ahmc_stats)); P("stats.numerical_error", offsetof(ahmc_stats, numerical_error));
    P("sizeof_rng", sizeof(ahmc_rng)); P("rng.exp_stride", offsetof(ahmc_rng, exp_stride));
    P("rng.partial_refresh_alpha", offsetof(ahmc_rng, partial_refresh_alpha));
    P("rng.temper_alpha", offsetof(ahmc_rng, temper_alpha));
    P("sizeof_adapt_cfg", sizeof(ahmc_adapt_cfg)); P("adapt_cfg.delta", offsetof(ahmc_adapt_cfg, delta));
    P("adapt_cfg.adapt_metric", offsetof(ahmc_adapt_cfg, adapt_metric)); P("adapt_cfg.eps_chain", offsetof(ahmc_adapt_cfg, eps_chain));
    P("adapt_cfg.eps_trace", offsetof(ahmc_adapt_cfg, eps_trace));
    return 0;
}
''')
    exe = tmp_path / "abi_probe"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    got = {k: int(v) for k, v in got.items()}
    for name in ("FLAG_HOST_BUFFERS", "FLAG_COMPAT_BREAK_ALL", "FLAG_ASYNC", "FLAG_EXACT_CHECKS", "FLAG_NO_REFRESH",
                 "FLAG_NUTS_SLICE_TS", "FLAG_NUTS_CLASSIC", "FLAG_NUTS_STRICT", "STATUS_NONFINITE"):
        assert getattr(L, name) == got[name], name
    for cname, cls in (("metric", L.Metric), ("phasepoint", L.PhasePoint), ("stats", L.Stats), ("rng", L.Rng),
                       ("adapt_cfg", L.AdaptCfg)):
        assert ctypes.sizeof(cls) == got["sizeof_" + cname], cname
        for key, off in got.items():
            if key.startswith(cname + "."):
                assert getattr(cls, key.split(".")[1]).offset == off, key


def _split_top(s):
    out, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += ch
    if cur.strip():
        out.append(cur.strip())
    return out


def test_julia_shim_ccall_arity_matches_the_header():
    """julia/AdvancedHMCB200Ext.jl cannot be executed here (no julia binary); at least every `ccall` in it must name an
    exported entry point and pass exactly as many argument types -- and values -- as the C prototype has parameters."""
    import re

    hdr = open(os.path.join(ROOT, "include", "ahmc_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = {m.group(1): (0 if m.group(2).strip() == "void" else len(_split_top(m.group(2))))
              for m in re.finditer(r"\b(ahmc_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", hdr, flags=re.S)}
    jl = open(os.path.join(ROOT, "julia", "AdvancedHMCB200Ext.jl")).read()
    seen = 0
    bound = set()
    for m in re.finditer(r"ccall\(\(:(ahmc_[a-z0-9_]+),\s*libahmc\),\s*([\w{}]+),\s*\(", jl):
        name = m.group(1)
        assert name in protos, name
        # the type tuple starts at m.end() - 1
        i, depth = m.end() - 1, 0
        j = i
        while True:
            depth += jl[j] == "("
            depth -= jl[j] == ")"
            if depth == 0:
                break
            j += 1
        types = [t for t in _split_top(jl[i + 1:j]) if t]
        # the values follow up to the ccall's closing parenthesis
        k, depth = j + 1, 1
        while depth:
            depth += jl[k] == "("
            depth -= jl[k] == ")"
            k += 1
        values = [v for v in _split_top(jl[j + 1:k - 1].lstrip(", \n")) if v]
        assert len(types) == protos[name], (name, len(types), protos[name])
        assert len(values) == protos[name], (name, len(values), protos[name])
        bound.add(name)
        seen += 1
    # EVERY entry point the header declares is bound by the shim
    assert bound == set(protos), sorted(set(protos) - bound)
    # device pointers enter the C structs as plain Ptr (pointer(::CuArray) is a CuPtr): through dptr()
    assert "reinterpret(Ptr{T}, pointer(x))" in jl and "pointer(z.θ), pointer(z.r), pointer(z.ℓπ.value)" not in jl


def test_julia_shim_struct_field_counts_match_the_c_structs():
    import re

    from ahmc_b200 import _lib as L

    jl = open(os.path.join(ROOT, "julia", "AdvancedHMCB200Ext.jl")).read()
    want = {"CMetric": L.Metric, "CPhasePoint": L.PhasePoint, "CStats": L.Stats, "CRng": L.Rng, "CAdaptCfg": L.AdaptCfg,
            "CPooledCfg": L.PooledCfg}
    for name, cls in want.items():
        m = re.search(r"struct " + name + r"\n(.*?)\nend", jl, flags=re.S)
        assert m, name
        fields = [f for line in m.group(1).splitlines() for f in line.split("#")[0].split(";") if "::" in f]
        assert len(fields) == len(cls._fields_), (name, len(fields), len(cls._fields_))


def test_user_target_sources_compile_under_nvrtc_without_a_gpu():
    """ahmc_user_source_check: the library's embedded kernel sources + a user device function compile for sm_90a (NVRTC needs
    no device), for every kernel a user target can run in and for both contracts; a broken source returns the NVRTC log."""
    import ctypes as C

    import ahmc_b200 as A

    lib = A._lib.load()
    general = ("__device__ double ahmc_user_logp_grad(const double* th, double* g, int D, const double* p) {\n"
               "  double s = 0.0; for (int i = 0; i < D; ++i) { g[i] = -th[i] * p[0]; s += th[i] * th[i]; } return -0.5 * p[0] * s; }\n")
    coord = ("#define AHMC_USER_COORDWISE\n__device__ double ahmc_user_coord(int d, double x, const double* p, double* gd) {\n"
             "  *gd = -x * p[d]; return -0.5 * x * x * p[d]; }\n")
    log = C.create_string_buffer(4096)
    rc0 = lib.ahmc_user_source_check(general.encode(), 1, 1, 100, log, 4096)
    if rc0 == A._lib.ERR_UNSUPPORTED:
        pytest.skip("libnvrtc not available here: " + log.value.decode())
    for src in (general, coord):
        for kernel in range(5):
            for metric, D in ((0, 10), (1, 128), (2, 40)):
                assert lib.ahmc_user_source_check(src.encode(), kernel, metric, D, log, 4096) == 0, log.value.decode()
    assert lib.ahmc_user_source_check(b"__device__ double ahmc_user_logp_grad(const double* t, double* g, int D, const double* p) { return q; }",
                                      3, 1, 8, log, 4096) == A._lib.ERR_INVALID
    assert b"q" in log.value and b"undefined" in log.value
    with pytest.raises(A.InvalidArgument):
        A.UserTarget.check_source("__device__ double ahmc_user_logp_grad(const double* t, double* g, int D, const double* p) { return q; }", 8)
