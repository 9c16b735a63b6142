// ahmc_user.cu -- user-supplied grad log pi INSIDE the fused kernels (AHMC_MODEL_USER, src/hamiltonian.jl:45-48).
//
// The reference calls an arbitrary Julia closure per leapfrog step; a persistent CUDA loop cannot call back into the host.
// A target expressible as a CUDA device function is therefore compiled at run time TOGETHER with the kernel sources
// (NVRTC; the sources are embedded in the library at build time, ahmc_embedded_sources.cu) and the resulting kernels --
// phasepoint, the fused trajectory (K1), the static transition (K2), NUTS (K3, default family), find_good_stepsize and the
// adaptive forms of K2 and K3 (in-launch warm-up, ahmc_chain_adapt.cuh) -- are the same code as the built-in targets with ModelOps<AHMC_MODEL_USER>::eval calling the user's function.  One instantiation
// (kernel x metric x layout) is compiled on first use and cached in the model.  The source picks its contract
// (ahmc_device.cuh): the one-lane function, AHMC_USER_COORDWISE or AHMC_USER_GROUPWISE; the translation unit defines the
// macro the source names, so a source naming both meets the #error there.  NVRTC and the driver API are bound with
// dlopen: the library loads without them and fails loudly (AHMC_ERR_UNSUPPORTED) when a user target is requested.
#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "ahmc_kernels.cuh"

namespace ahmc {

// generated at build time (advancedhmc.jl_b200/build.py): name / source pairs of the headers NVRTC needs
extern const char* const kEmbeddedNames[];
extern const char* const kEmbeddedSources[];
extern const int kEmbeddedCount;

namespace {
struct Rtc {
    void* nvrtc = nullptr;
    void* cuda = nullptr;
    int (*CreateProgram)(void**, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
    int (*DestroyProgram)(void**) = nullptr;
    int (*CompileProgram)(void*, int, const char* const*) = nullptr;
    int (*GetProgramLogSize)(void*, size_t*) = nullptr;
    int (*GetProgramLog)(void*, char*) = nullptr;
    int (*GetCUBINSize)(void*, size_t*) = nullptr;
    int (*GetCUBIN)(void*, char*) = nullptr;
    int (*AddNameExpression)(void*, const char*) = nullptr;
    int (*GetLoweredName)(void*, const char*, const char**) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    int (*cuModuleLoadData)(void**, const void*) = nullptr;
    int (*cuModuleUnload)(void*) = nullptr;
    int (*cuModuleGetFunction)(void**, void*, const char*) = nullptr;
    int (*cuLaunchKernel)(void*, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, void*, void**, void**) = nullptr;
    int (*cuFuncSetAttribute)(void*, int, int) = nullptr;
    int (*cuGetErrorString)(int, const char**) = nullptr;
    char why[256] = {0};
    bool tried = false, ok = false;
};
Rtc g_rtc;
std::mutex g_rtc_mutex;  // contexts of different host threads may bind / compile concurrently

template <class F>
bool sym(void* lib, const char* name, F& f) {
    f = (F)dlsym(lib, name);
    return f != nullptr;
}

const char* rtc_bind() {
    std::lock_guard<std::mutex> lock(g_rtc_mutex);
    if (g_rtc.ok) return nullptr;
    if (g_rtc.tried) return g_rtc.why;
    g_rtc.tried = true;
    const char* env = getenv("AHMC_NVRTC_LIB");
    const char* names[] = {env, "libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"};
    for (const char* n : names) {
        if (!n) continue;
        g_rtc.nvrtc = dlopen(n, RTLD_NOW);
        if (g_rtc.nvrtc) break;
    }
    if (!g_rtc.nvrtc) {
        snprintf(g_rtc.why, sizeof g_rtc.why, "libnvrtc not found (set AHMC_NVRTC_LIB): %s", dlerror());
        return g_rtc.why;
    }
    bool ok = sym(g_rtc.nvrtc, "nvrtcCreateProgram", g_rtc.CreateProgram) && sym(g_rtc.nvrtc, "nvrtcDestroyProgram", g_rtc.DestroyProgram) &&
              sym(g_rtc.nvrtc, "nvrtcCompileProgram", g_rtc.CompileProgram) && sym(g_rtc.nvrtc, "nvrtcGetProgramLogSize", g_rtc.GetProgramLogSize) &&
              sym(g_rtc.nvrtc, "nvrtcGetProgramLog", g_rtc.GetProgramLog) && sym(g_rtc.nvrtc, "nvrtcGetCUBINSize", g_rtc.GetCUBINSize) &&
              sym(g_rtc.nvrtc, "nvrtcGetCUBIN", g_rtc.GetCUBIN) && sym(g_rtc.nvrtc, "nvrtcAddNameExpression", g_rtc.AddNameExpression) &&
              sym(g_rtc.nvrtc, "nvrtcGetLoweredName", g_rtc.GetLoweredName) && sym(g_rtc.nvrtc, "nvrtcGetErrorString", g_rtc.GetErrorString);
    if (!ok) {
        snprintf(g_rtc.why, sizeof g_rtc.why, "the NVRTC library lacks a required symbol");
        return g_rtc.why;
    }
    g_rtc.ok = true;
    return nullptr;
}

const char* driver_bind() {  // the driver API, needed to load and launch (not to compile)
    std::lock_guard<std::mutex> lock(g_rtc_mutex);
    if (g_rtc.cuda) return nullptr;
    g_rtc.cuda = dlopen("libcuda.so.1", RTLD_NOW);
    if (!g_rtc.cuda) {
        snprintf(g_rtc.why, sizeof g_rtc.why, "libcuda.so.1 not found: %s", dlerror());
        return g_rtc.why;
    }
    bool ok = sym(g_rtc.cuda, "cuModuleLoadData", g_rtc.cuModuleLoadData) && sym(g_rtc.cuda, "cuModuleUnload", g_rtc.cuModuleUnload) &&
              sym(g_rtc.cuda, "cuModuleGetFunction", g_rtc.cuModuleGetFunction) && sym(g_rtc.cuda, "cuLaunchKernel", g_rtc.cuLaunchKernel) &&
              sym(g_rtc.cuda, "cuFuncSetAttribute", g_rtc.cuFuncSetAttribute) && sym(g_rtc.cuda, "cuGetErrorString", g_rtc.cuGetErrorString);
    if (!ok) {
        g_rtc.cuda = nullptr;
        snprintf(g_rtc.why, sizeof g_rtc.why, "the driver library lacks a required symbol");
        return g_rtc.why;
    }
    return nullptr;
}
}  // namespace

struct UserModule {
    std::string src;
    std::string err;
    struct Fn {
        void* module = nullptr;
        void* fn = nullptr;
        size_t smem_set = 0;
    };
    std::map<long long, Fn> fns;  // key = which | metric << 4 | G << 8 | E << 16 | form << 24
};

UserModule* user_module_create(const char* cuda_src, char* err, size_t err_len) {
    const char* why = rtc_bind();
    if (!why) why = driver_bind();
    if (why) {
        snprintf(err, err_len, "%s", why);
        return nullptr;
    }
    UserModule* m = new UserModule;
    m->src = cuda_src;
    return m;
}
void user_module_destroy(UserModule* m) {
    if (!m) return;
    for (auto& kv : m->fns)
        if (kv.second.module) g_rtc.cuModuleUnload(kv.second.module);
    delete m;
}
const char* user_last_error(const UserModule* m) { return m ? m->err.c_str() : "no user module"; }
static thread_local std::string t_user_err;
const char* user_thread_error() { return t_user_err.c_str(); }
void user_thread_error_clear() { t_user_err.clear(); }

// compile kernel `which` of the user target; load it when `out` is given (needs a device), else only check that it compiles
static bool compile(UserModule* m, int which, int metric, int G, int E, int form, UserModule::Fn* out) {
    char expr[160];
    const char* unit = "ahmc_leapfrog.cu";
    switch (which) {
        case UK_PHASEPOINT: snprintf(expr, sizeof expr, "ahmc::phasepoint_kernel<%d, %d, %d, %d>", AHMC_MODEL_USER, metric, G, E); break;
        case UK_LEAPFROG: snprintf(expr, sizeof expr, "ahmc::leapfrog_kernel<%d, %d, %d, %d, false>", AHMC_MODEL_USER, metric, G, E); break;
        case UK_HMC: snprintf(expr, sizeof expr, "ahmc::hmc_kernel<%d, %d, %d, %d>", AHMC_MODEL_USER, metric, G, E); break;
        case UK_FIND_EPS: snprintf(expr, sizeof expr, "ahmc::find_eps_kernel<%d, %d, %d, %d>", AHMC_MODEL_USER, metric, G, E); break;
        case UK_HMC_ADAPT: snprintf(expr, sizeof expr, "ahmc::hmc_kernel<%d, %d, %d, %d, %d>", AHMC_MODEL_USER, metric, G, E, form); break;
        case UK_NUTS:
        case UK_NUTS_ADAPT:
            snprintf(expr, sizeof expr, "ahmc::nuts_kernel<%d, %d, %d, %d, false, %d, false>", AHMC_MODEL_USER, metric, G, E,
                     which == UK_NUTS_ADAPT ? form : 0);
            unit = "ahmc_nuts_kernel.cuh";
            break;
        default: m->err = "unknown kernel"; return false;
    }
    // translation unit: the kernel sources see the prototypes of the user's functions (ahmc_device.cuh), the user's
    // definitions follow
    std::string tu = "#define AHMC_NVRTC_USER_MODEL 1\n";
    if (m->src.find("AHMC_USER_COORDWISE") != std::string::npos) tu += "#define AHMC_USER_COORDWISE 1\n";
    if (m->src.find("AHMC_USER_GROUPWISE") != std::string::npos) tu += "#define AHMC_USER_GROUPWISE 1\n";
    tu += std::string("#include \"") + unit + "\"\n#line 1 \"user_target.cu\"\n" + m->src + "\n";
    void* prog = nullptr;
    int rc = g_rtc.CreateProgram(&prog, tu.c_str(), "ahmc_user_tu.cu", kEmbeddedCount, kEmbeddedSources, kEmbeddedNames);
    if (rc) {
        m->err = std::string("nvrtcCreateProgram: ") + g_rtc.GetErrorString(rc);
        return false;
    }
    g_rtc.AddNameExpression(prog, expr);
    const char* opts[] = {"--gpu-architecture=sm_90a", "--std=c++17", "-default-device", "--fmad=true", "-lineinfo"};
    rc = g_rtc.CompileProgram(prog, 5, opts);
    if (rc) {
        size_t n = 0;
        g_rtc.GetProgramLogSize(prog, &n);
        std::string log(n, '\0');
        if (n) g_rtc.GetProgramLog(prog, &log[0]);
        if (log.size() > 3000) log.resize(3000);
        m->err = std::string("NVRTC could not compile the user target (") + g_rtc.GetErrorString(rc) + "):\n" + log;
        g_rtc.DestroyProgram(&prog);
        return false;
    }
    const char* lowered = nullptr;
    rc = g_rtc.GetLoweredName(prog, expr, &lowered);
    size_t sz = 0;
    if (!rc) rc = g_rtc.GetCUBINSize(prog, &sz);
    std::vector<char> cubin(sz);
    if (!rc) rc = g_rtc.GetCUBIN(prog, cubin.data());
    if (rc || !lowered) {
        m->err = std::string("NVRTC: ") + g_rtc.GetErrorString(rc);
        g_rtc.DestroyProgram(&prog);
        return false;
    }
    if (!out) {
        g_rtc.DestroyProgram(&prog);
        return true;
    }
    int drc = g_rtc.cuModuleLoadData(&out->module, cubin.data());
    if (!drc) drc = g_rtc.cuModuleGetFunction(&out->fn, out->module, lowered);
    g_rtc.DestroyProgram(&prog);
    if (drc) {
        const char* es = nullptr;
        g_rtc.cuGetErrorString(drc, &es);
        m->err = std::string("loading the compiled user kernels failed: ") + (es ? es : "?");
        return false;
    }
    return true;
}

cudaError_t user_launch(UserModule* m, int which, int metric_kind, int G, int E, const void* args, unsigned blocks, size_t smem,
                        cudaStream_t st, int form) {
    if (!m) {  // a target created without NVRTC (ahmc_model_create_glm): the general form is unavailable
        t_user_err = "run-time compilation is unavailable: libnvrtc or the driver library could not be bound (set AHMC_NVRTC_LIB)";
        return cudaErrorInvalidValue;
    }
    const long long key =
        (long long)which | ((long long)metric_kind << 4) | ((long long)G << 8) | ((long long)E << 16) | ((long long)form << 24);
    auto it = m->fns.find(key);
    if (it == m->fns.end()) {
        UserModule::Fn f;
        if (!compile(m, which, metric_kind, G, E, form, &f)) {
            t_user_err = m->err;
            return cudaErrorInvalidSource;
        }
        it = m->fns.emplace(key, f).first;
    }
    UserModule::Fn& f = it->second;
    if (smem > 48 * 1024 && smem > f.smem_set) {
        if (g_rtc.cuFuncSetAttribute(f.fn, 8 /* CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES */, (int)smem)) return cudaErrorInvalidValue;
        f.smem_set = smem;
    }
    void* params[] = {const_cast<void*>(args)};
    int drc = g_rtc.cuLaunchKernel(f.fn, blocks, 1, 1, kBlockThreads, 1, 1, (unsigned)smem, (void*)st, params, nullptr);
    if (drc) {
        const char* es = nullptr;
        g_rtc.cuGetErrorString(drc, &es);
        m->err = std::string("cuLaunchKernel: ") + (es ? es : "?");
        t_user_err = m->err;
        return cudaErrorLaunchFailure;
    }
    return cudaSuccess;
}

// compile-only check (no device needed): 0 = compiles, else the NVRTC log
int user_source_check(const char* cuda_src, int which, int metric_kind, int D, char* log, size_t log_len) {
    if (log && log_len) log[0] = 0;
    if (const char* why = rtc_bind()) {
        if (log) snprintf(log, log_len, "%s", why);
        return -3;
    }
    int G, E;
    if (!pick_layout(D, &G, &E)) return -1;
    UserModule m;
    m.src = cuda_src;
    // the adaptive kernels: every instantiation a launch with this metric can pick (adapt_kernel) -- for a Diag metric both
    // estimator forms, for a Dense one the WelfordCov form on the chain's own rows
    const bool adaptive = which == UK_NUTS_ADAPT || which == UK_HMC_ADAPT;
    std::vector<AdaptKernel> kernels{{metric_kind, 0}};
    if (adaptive) {
        AdaptDev ad{};
        const MetricDev md{metric_kind};
        kernels.clear();
        for (int est : {AHMC_ADAPT_WELFORD, AHMC_ADAPT_NUTPIE}) {
            ad.adapt_metric = est;
            const AdaptKernel k = adapt_kernel(ad, md);
            if (kernels.empty() || kernels.back().form != k.form) kernels.push_back(k);
        }
    }
    for (const AdaptKernel& k : kernels) {
        if (!compile(&m, which, k.metric_kind, G, E, k.form, nullptr)) {
            if (log) snprintf(log, log_len, "%s", m.err.c_str());
            return -1;
        }
    }
    return 0;
}

}  // namespace ahmc
