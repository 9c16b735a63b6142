"""Building and loading the SIMT-emulator harnesses (tests/simt_emu/<name>_emu.cpp: the product's kernel sources, unmodified,
on the CPU emulator simt_emu.cpp), the ctypes mirrors of their request structs, and the compile-only NVRTC check.

A harness is compiled once per pytest process and (name, defines), whichever module asks first; the libraries live in a
temporary directory removed at exit.  Every struct below is compared on load with the harness's `emu_sizeof_<Struct>()`
(EMU_EXPORT_SIZEOF, tests/simt_emu/include/emu_harness.h): a field added on one side only would shift every later
pointer, and the emulator would read the wrong buffer without failing."""
import atexit
import concurrent.futures as cf
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "simt_emu")
CSRC = os.path.join(ROOT, "advancedhmc.jl_b200", "csrc")
_vp = C.c_void_p


def P(a):
    """a numpy array's data pointer, None for None"""
    return None if a is None else a.ctypes.data_as(_vp)


# ------------------------------------------------------------------------------------------------ request structs
# the last fields of the trajectory harnesses' requests: leading dimensions of the D x N inputs and outputs (0: D)
_LD = [("ld_in", C.c_int64), ("ld_out", C.c_int64)]


class EmuNuts(C.Structure):
    _fields_ = [("model_kind", C.c_int32), ("metric_kind", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("p0", _vp), ("p1", _vp),
                ("c0", C.c_double), ("Minv", _vp), ("minv_stride", C.c_int64), ("cholU", _vp), ("eps", C.c_double),
                ("eps_chain", _vp), ("max_depth", C.c_int32), ("delta_max", C.c_double), ("sampler", C.c_int32),
                ("criterion", C.c_int32), ("seed", C.c_uint64), ("offset", C.c_uint64), ("normal_tape", _vp), ("exp_tape", _vp),
                ("exp_stride", C.c_int64), ("dir_tape", _vp), ("dir_stride", C.c_int64), ("partial_alpha", C.c_double),
                ("refresh", C.c_int32), ("th_in", _vp), ("r_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp),
                ("r_out", _vp), ("g_out", _vp), ("lp_out", _vp), ("lk_out", _vp), ("n_steps", _vp), ("tree_depth", _vp),
                ("numerical", _vp), ("acc", _vp), ("dH", _vp), ("dHmax", _vp), ("n_transitions", C.c_int32), ("draws", _vp),
                ("adapt", C.c_int32), ("n_adapts", C.c_int32), ("init_buffer", C.c_int32), ("term_buffer", C.c_int32),
                ("window_size", C.c_int32), ("delta", C.c_double), ("gamma", C.c_double), ("t0", C.c_double), ("kappa", C.c_double),
                ("adapt_metric", C.c_int32), ("n_min", C.c_int32), ("eps_rw", _vp), ("minv_rw", _vp), ("eps_trace", _vp),
                ("temper_alpha", C.c_double), ("coop_padded", C.c_int32), *_LD]


class EmuLf(C.Structure):
    _fields_ = [("model_kind", C.c_int32), ("metric_kind", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("p0", _vp), ("p1", _vp),
                ("c0", C.c_double), ("Minv", _vp), ("minv_stride", C.c_int64), ("cholU", _vp), ("eps", C.c_double),
                ("eps_chain", _vp), ("n_steps", C.c_int32), ("fwd", C.c_int32), ("temper_alpha", C.c_double), ("th_in", _vp),
                ("r_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp), ("r_out", _vp), ("g_out", _vp), ("lp_out", _vp),
                ("lk_out", _vp), ("dr_out", _vp), ("status", _vp), ("steps_done", _vp), ("flags", C.c_uint32), ("hmc", C.c_int32),
                ("refresh", C.c_int32), ("n_transitions", C.c_int32), ("seed", C.c_uint64), ("offset", C.c_uint64),
                ("normal_tape", _vp), ("exp_tape", _vp), ("is_accept", _vp), ("acc", _vp), ("dH", _vp), ("draws", _vp), *_LD]


class EmuMn(C.Structure):
    _fields_ = [("model_kind", C.c_int32), ("metric_kind", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("p0", _vp), ("p1", _vp),
                ("Minv", _vp), ("cholU", _vp), ("eps", C.c_double), ("n_steps", C.c_int32), ("n_fwd", C.c_int32),
                ("normal_tape", _vp), ("unif_tape", _vp), ("th_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp),
                ("r_out", _vp), ("g_out", _vp), ("lp_out", _vp), ("lk_out", _vp), ("acc", _vp), ("index", _vp), ("temper_alpha", C.c_double), *_LD]


class EmuDense(C.Structure):
    _fields_ = [("D", C.c_int32), ("N", C.c_int64), ("P", _vp), ("w", _vp), ("mu", _vp), ("c0", C.c_double), ("Minv", _vp),
                ("Mdiag", _vp), ("eps", C.c_double), ("eps_chain", _vp), ("n_steps", C.c_int32), ("fwd", C.c_int32),
                ("th_in", _vp), ("r_in", _vp), ("g_in", _vp), ("th_out", _vp), ("r_out", _vp), ("g_out", _vp), ("dr_out", _vp),
                ("lp_out", _vp), ("lk_out", _vp), ("status", _vp), ("steps_done", _vp), ("need_exact", _vp),
                ("wide_tile", C.c_int32), ("norms_out", C.c_double * 2), *_LD]


class EmuGlm(C.Structure):
    _fields_ = [("family", C.c_int32), ("D", C.c_int32), ("n", C.c_int32), ("N", C.c_int64), ("X", _vp), ("y", _vp), ("prec", _vp),
                ("c0", C.c_double), ("Minv", _vp), ("chain_stride", C.c_int64), ("eps", C.c_double), ("eps_chain", _vp),
                ("n_steps", C.c_int32), ("fwd", C.c_int32), ("th_in", _vp), ("r_in", _vp), ("g_in", _vp), ("th_out", _vp),
                ("r_out", _vp), ("g_out", _vp), ("dr_out", _vp), ("lp_out", _vp), ("lk_out", _vp), ("status", _vp),
                ("steps_done", _vp), ("nc_out", C.c_int32), ("stages_out", C.c_int32), *_LD]


class EmuBigd(C.Structure):
    _fields_ = [("model", C.c_int32), ("metric", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("p0", _vp), ("p1", _vp),
                ("c0", C.c_double), ("Minv", _vp), ("minv_stride", C.c_int64), ("eps", _vp), ("n_steps", C.c_int32), ("T", C.c_int32),
                ("refresh", C.c_int32), ("seed", C.c_uint64), ("offset", C.c_uint64), ("partial_alpha", C.c_double), ("normal_tape", _vp), ("exp_tape", _vp),
                ("th_in", _vp), ("r_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp), ("r_out", _vp), ("g_out", _vp),
                ("lp_out", _vp), ("lk_out", _vp), ("draws", _vp), ("acc", _vp), ("H", _vp), ("dH", _vp), ("is_accept", _vp),
                ("numerical_error", _vp), ("adapt_metric", C.c_int32), ("n_adapts", C.c_int32), ("init_buffer", C.c_int32),
                ("term_buffer", C.c_int32), ("window_size", C.c_int32), ("n_min", C.c_int32), ("eps_rw", _vp), ("minv_rw", _vp),
                ("eps_trace", _vp)]


class EmuAdaptChain(C.Structure):
    _fields_ = [("hmc", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("mu", _vp), ("w", _vp), ("Minv", _vp), ("eps0", C.c_double),
                ("max_depth", C.c_int32), ("n_steps", C.c_int32), ("seed", C.c_uint64), ("T", C.c_int32), ("n_adapts", C.c_int32),
                ("init_buffer", C.c_int32), ("term_buffer", C.c_int32), ("window_size", C.c_int32), ("adapt_metric", C.c_int32),
                ("n_min", C.c_int32), ("th_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp), ("r_out", _vp), ("g_out", _vp),
                ("lp_out", _vp), ("lk_out", _vp), ("draws", _vp), ("acc", _vp), ("eps_trace", _vp), ("n_steps_out", _vp),
                ("eps_rw", _vp), ("minv_rw", _vp)]


class EmuDenseAdapt(C.Structure):
    _fields_ = [("hmc", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("mu", _vp), ("w", _vp), ("Minv0", _vp), ("cholU0", _vp),
                ("eps0", C.c_double), ("max_depth", C.c_int32), ("n_steps", C.c_int32), ("seed", C.c_uint64), ("T", C.c_int32),
                ("n_adapts", C.c_int32), ("init_buffer", C.c_int32), ("term_buffer", C.c_int32), ("window_size", C.c_int32),
                ("adapt_metric", C.c_int32), ("n_min", C.c_int32), ("th_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp),
                ("r_out", _vp), ("g_out", _vp), ("lp_out", _vp), ("lk_out", _vp), ("draws", _vp), ("acc", _vp), ("eps_trace", _vp),
                ("n_steps_out", _vp), ("eps_rw", _vp), ("minv_rw", _vp), ("cholu_rw", _vp), ("workspace", _vp)]


class EmuEstimate(C.Structure):
    _fields_ = [("D", C.c_int32), ("N", C.c_int64), ("n", C.c_double), ("W", _vp), ("minv", _vp), ("cholu", _vp), ("ok", _vp)]


class EmuDenseUserAdapt(C.Structure):
    _fields_ = [("hmc", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("params", _vp), ("Minv0", _vp), ("cholU0", _vp),
                ("metric_stride", C.c_int64), ("eps0", C.c_double), ("max_depth", C.c_int32), ("n_steps", C.c_int32),
                ("seed", C.c_uint64), ("T", C.c_int32), ("n_adapts", C.c_int32), ("init_buffer", C.c_int32),
                ("term_buffer", C.c_int32), ("window_size", C.c_int32), ("adapt_metric", C.c_int32), ("n_min", C.c_int32),
                ("th_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp), ("r_out", _vp), ("g_out", _vp), ("lp_out", _vp),
                ("lk_out", _vp), ("draws", _vp), ("acc", _vp), ("eps_trace", _vp), ("n_steps_out", _vp), ("tree_depth", _vp),
                ("is_accept", _vp), ("numerical", _vp), ("eps_rw", _vp), ("minv_rw", _vp), ("cholu_rw", _vp)]


class EmuUser(C.Structure):
    _fields_ = [("op", C.c_int32), ("metric_kind", C.c_int32), ("D", C.c_int32), ("N", C.c_int64), ("c0", C.c_double),
                ("Minv", _vp), ("cholU", _vp), ("eps", C.c_double), ("n_steps", C.c_int32), ("max_depth", C.c_int32),
                ("exp_tape", _vp), ("exp_stride", C.c_int64), ("dir_tape", _vp), ("dir_stride", C.c_int64),
                ("th_in", _vp), ("r_in", _vp), ("g_in", _vp), ("lp_in", _vp), ("th_out", _vp), ("r_out", _vp), ("g_out", _vp),
                ("lp_out", _vp), ("lk_out", _vp), ("steps", _vp), ("tree_depth", _vp), ("numerical", _vp), ("acc", _vp)]


_STRUCTS = {"nuts": [EmuNuts], "lf": [EmuLf], "pair": [EmuLf], "mn": [EmuMn], "dense": [EmuDense], "glm": [EmuGlm],
            "bigd": [EmuBigd], "adapt_chain": [EmuAdaptChain], "dense_adapt": [EmuDenseAdapt, EmuEstimate],
            "dense_user_adapt": [EmuDenseUserAdapt], "user_group": [EmuUser]}


# ------------------------------------------------------------------------------------------------ building
# -O1 and -ffp-contract=off are what the emulated arithmetic is compared at: no fused multiply-adds the kernels do not ask for
_FLAGS = ["-O1", "-std=c++20", "-pthread", "-ffp-contract=off", "-w"]
_libs = {}
_tmp = None


def _tmpdir():
    global _tmp
    if _tmp is None:
        _tmp = tempfile.mkdtemp(prefix="simt_emu_")
        atexit.register(shutil.rmtree, _tmp, True)
    return _tmp


def _gxx(name, out, flags, include_first=None):
    return subprocess.run(["g++", *_FLAGS, *flags, *(["-I", include_first] if include_first else []), "-I", os.path.join(EMU, "include"),
                           "-I", CSRC, "-I", os.path.join(ROOT, "include"), os.path.join(EMU, "simt_emu.cpp"),
                           os.path.join(EMU, f"{name}_emu.cpp"), "-o", out], capture_output=True, text=True)


def harnesses(*specs):
    """the harnesses `specs` (a name, or a tuple (name, *defines)) as loaded libraries, the uncached ones compiled concurrently"""
    keys = [spec if isinstance(spec, tuple) else (spec,) for spec in specs]
    todo = {k: os.path.join(_tmpdir(), f"lib{'-'.join(k)}.so") for k in keys if k not in _libs}
    with cf.ThreadPoolExecutor(max_workers=len(todo) or 1) as ex:
        built = ex.map(lambda k: _gxx(k[0], todo[k], ["-shared", "-fPIC", *(f"-D{d}" for d in k[1:])]), todo)
    for key, pr in zip(todo, built):
        assert pr.returncode == 0, pr.stderr[-3000:]
        lib = C.CDLL(todo[key])
        for S in _STRUCTS.get(key[0], []):
            size = getattr(lib, f"emu_sizeof_{S.__name__}")
            size.restype = C.c_size_t
            assert C.sizeof(S) == size(), f"{S.__name__}: {C.sizeof(S)} bytes in tests/emu.py, {size()} in {key[0]}_emu.cpp"
        _libs[key] = lib
    return [_libs[k] for k in keys]


def harness(name, *defines):
    """the harness tests/simt_emu/<name>_emu.cpp (with -D<define> for each of `defines`) as a loaded library"""
    return harnesses((name, *defines))[0]


def sanitized(name, sanitizer, *defines, include_first=None, timeout=900):
    """Builds the harness as its own program (its `main` under -DRACE_<NAME>) with -fsanitize=<sanitizer> ("thread" or
    "address") and runs it.  Skips when the compiler has no runtime for the sanitizer or the runtime cannot start here;
    `include_first` is a directory searched ahead of the product sources (a mutated copy of one of them)."""
    tag = {"thread": "tsan", "address": "asan"}[sanitizer]
    exe = os.path.join(tempfile.mkdtemp(dir=_tmpdir()), f"{tag}_{name}")
    flags = [f"-DRACE_{name.upper()}", *(f"-D{d}" for d in defines), "-g", f"-fsanitize={sanitizer}"]
    pr = _gxx(name, exe, flags + (["-fno-omit-frame-pointer"] if sanitizer == "address" else []), include_first)
    if pr.returncode != 0 and (tag in pr.stderr.lower() or "sanitize" in pr.stderr.lower()):
        pytest.skip(f"the {sanitizer} sanitizer runtime is not available to g++ here")
    assert pr.returncode == 0, pr.stderr[-3000:]
    env = {**os.environ, "ASAN_OPTIONS": "detect_leaks=0"} if sanitizer == "address" else None
    r = subprocess.run([exe], capture_output=True, text=True, timeout=timeout, env=env)
    refused = ("FATAL: ThreadSanitizer" in r.stderr if sanitizer == "thread"
               else "AddressSanitizer" in r.stderr and "ERROR: AddressSanitizer" not in r.stderr)
    if refused:
        pytest.skip(f"the {sanitizer} sanitizer cannot run in this environment: " + r.stderr.strip().splitlines()[0])
    return r


# ------------------------------------------------------------------------------------------------ NVRTC (compile only)
_PROBE = "__device__ double ahmc_user_logp_grad(const double* t, double* g, int D, const double* p) { return 0.0; }"


def source_check(lib, src, kernel, metric, D):
    """ahmc_user_source_check: (return code, NVRTC log)"""
    log = C.create_string_buffer(8192)
    rc = lib.ahmc_user_source_check(src.encode() if isinstance(src, str) else src, kernel, metric, D, log, 8192)
    return rc, log.value.decode()


def nvrtc_lib_or_skip():
    """the product library, or a skip when it cannot load NVRTC (the compile-only checks need no GPU)"""
    import ahmc_b200 as A

    lib = A._lib.load()
    rc, log = source_check(lib, _PROBE, 0, 0, 3)
    if rc == A._lib.ERR_UNSUPPORTED:
        pytest.skip("NVRTC is not available: " + log)
    return lib
