// ahmc_api.cu -- the C ABI of libahmc_b200 (include/ahmc_b200.h): context, models, argument
// validation, host-buffer staging and kernel dispatch.  No torch types, no exceptions across the ABI.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <chrono>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "ahmc_chain_adapt.cuh"
#include "ahmc_glm.cuh"
#include "ahmc_kernels.cuh"

using namespace ahmc;

// How the host-buffer lane (leapfrog_host_pipelined) moves a call's buffers.  A direct side has the kernel read or
// write page-locked host memory itself; such a launch has its residency capped at one CTA per SM, so the grid runs in
// staggered waves and uploads overlap downloads.  Otherwise that side goes through the copy engines.
struct PipeTransport {
    bool up_direct;    // the kernel loads theta / r / gradient / eps / Minv from host memory (else: copy-engine upload)
    bool down_direct;  // the kernel stores its results to host memory (else: copy-engine download)
    int chunks;        // pieces of the chain axis
};
// the autotune candidates, in the order they are tried
constexpr PipeTransport kPipeCands[] = {{true, true, 1}, {false, false, 2}, {false, false, 4}, {false, true, 4}};
constexpr int kPipeNCand = sizeof kPipeCands / sizeof kPipeCands[0];
constexpr int kMaxPipeChunks = 4;  // the context keeps two events per chunk
static_assert([] {
    for (const PipeTransport& t : kPipeCands)
        if (t.chunks > kMaxPipeChunks) return false;
    return true;
}(), "a candidate transport uses more chunks than kMaxPipeChunks");

// a grow-only device buffer of the context (see ensure)
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
};

struct ahmc_ctx {
    int device = 0;
    int sm_count = 0;  // streaming multiprocessors of the device (grid size of the one-wave reductions)
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;
    int64_t launches = 0;
    int* d_min_break = nullptr;   // device int for COMPAT_BREAK_ALL
    DevBuf arena;         // HOST_BUFFERS staging
    DevBuf chain_ws;      // per-chain workspace: NUTS trees, in-launch adaptors' estimators, D > 512 start points
    DevBuf summary_ws;    // adapt_summary: block partials and the completion counter
    DevBuf energy_ws;     // multinomial-static per-chain energy tape
    DevBuf dense_ws;      // K4: padded Minv, norms, per-chain fallback mask
    DevBuf coop_ws;       // cooperative NUTS products: Minv and cholU with padded columns (coop_lds)
    DevBuf split_ws;      // split-step (callback) mode and sequenced transitions (SplitWork)
    // host-buffer pipeline: upload stream, compute stream (= stream), download stream; per chunk an upload-done and a
    // kernel-done event, and one event that joins the downloads back into the compute stream
    cudaStream_t pipe[2] = {};  // upload, download
    cudaEvent_t ev_a = nullptr, ev_down = nullptr, ev_in[kMaxPipeChunks] = {}, ev_k[kMaxPipeChunks] = {};
    // transport choice of the host-buffer lane, measured per problem shape on its first calls (leapfrog_host_pipelined)
    struct PipeTune {
        int64_t N;
        int32_t D;
        int key;       // has_g | has_dr << 1 | per-chain eps << 2 | per-chain Minv << 3
        int calls;     // trial calls made so far
        int chosen;    // -1 while measuring
        double best_ms[kPipeNCand];
    };
    std::vector<PipeTune> tune;
    std::string transport = "none";  // what the last host-buffer call used (ahmc_last_transport)
};

struct ahmc_model {
    int kind = 0;
    int D = 0;
    double* d_p0 = nullptr;
    double* d_p1 = nullptr;
    double* d_p1_pad = nullptr;  // DENSE_GAUSS: precision zero-padded to Dp x Dp (K4), followed by |P|_inf
    double* d_p1_coop = nullptr; // DENSE_GAUSS: precision with columns padded to coop_lds(D) (cooperative NUTS products)
    int Dp = 0;
    double c0 = 0.0;
    ahmc_logp_grad_fn fn = nullptr;
    void* user = nullptr;
    UserModule* rtc = nullptr;  // AHMC_MODEL_USER: run-time compiled kernels
    // ahmc_model_create_glm: kind is AHMC_MODEL_USER (d_p0 = [prior_prec | X | y], the generated group-form source); the
    // tile kernel (K6) reads prior_prec and y from there and X from the padded copy
    int glm_family = -1;  // AHMC_GLM_*, -1: not a GLM target
    int glm_n = 0;
    double* d_glm_X = nullptr;  // glm_padded_doubles(D, n)
};

namespace {

int fail(ahmc_ctx* ctx, int code, const char* fmt, ...) {
    if (ctx) {
        char buf[4096];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof buf, fmt, ap);
        va_end(ap);
        ctx->err = buf;
    }
    return code;
}

#define CU(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e__ = (call);                                                                      \
        if (e__ != cudaSuccess) {                                                                      \
            std::string ue__ = user_thread_error();                                                    \
            user_thread_error_clear();                                                                 \
            return fail(ctx, AHMC_ERR_CUDA, "%s failed: %s (%s:%d)%s%s", #call, cudaGetErrorString(e__), __FILE__, \
                        __LINE__, ue__.empty() ? "" : " -- ", ue__.c_str());                           \
        }                                                                                              \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
        cudaGetLastError();  // a stale error left by another library on this thread must not be blamed on our launches
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// grows `b` to at least `need` bytes; the old contents are not kept.  Work already enqueued may still use the old
// allocation, so the context's streams are drained first (the pipeline streams are idle between calls).
int ensure(ahmc_ctx* ctx, DevBuf& b, size_t need, const char* what) {
    if (need <= b.bytes) return AHMC_OK;
    CU(cudaStreamSynchronize(ctx->stream));
    for (cudaStream_t s : ctx->pipe)
        if (s) CU(cudaStreamSynchronize(s));
    CU(cudaFree(b.p));
    b.p = nullptr;
    b.bytes = 0;
    cudaError_t e = cudaMalloc(&b.p, need);
    if (e != cudaSuccess) {
        b.p = nullptr;
        return fail(ctx, AHMC_ERR_NOMEM, "cudaMalloc(%zu) for %s failed: %s", need, what, cudaGetErrorString(e));
    }
    b.bytes = need;
    return AHMC_OK;
}
// the staging arena keeps 25 % headroom, so that a run of slowly growing calls does not reallocate every time
int ensure_arena(ahmc_ctx* ctx, size_t need) {
    return need > ctx->arena.bytes ? ensure(ctx, ctx->arena, need + need / 4, "staging") : AHMC_OK;
}

// Lays arrays out back to back, each on a 256-byte boundary.  Over base == nullptr it only measures (every pointer it
// hands out is nullptr), so one layout function gives both the size of a buffer and its pointers.
struct Carver {
    char* base = nullptr;
    size_t off = 0;
    template <class T>
    T* take(size_t count, bool want = true) {  // `want` false: nullptr, nothing taken
        if (!want) return nullptr;
        T* p = base ? (T*)(base + off) : nullptr;
        off += (count * sizeof(T) + 255) & ~(size_t)255;
        return p;
    }
};
// grows `b` to the size of `layout` (a function of Carver&) and runs it over `b`
template <class Layout>
int carve(ahmc_ctx* ctx, DevBuf& b, const char* what, Layout&& layout) {
    Carver m;
    layout(m);
    int rc = ensure(ctx, b, m.off, what);
    if (rc) return rc;
    Carver c{(char*)b.p};
    layout(c);
    return AHMC_OK;
}

// `rows` rows of `width` bytes, `pitch` bytes apart (the D rows of each of N chains at leading dimension ld): one
// contiguous copy when there is no gap between rows, else a 2-D copy that leaves the bytes between rows alone
cudaError_t copy_rows(void* dst, const void* src, size_t width, size_t pitch, size_t rows, cudaMemcpyKind kind,
                      cudaStream_t s) {
    if (width == pitch || rows == 1) return cudaMemcpyAsync(dst, src, width + pitch * (rows - 1), kind, s);
    return cudaMemcpy2DAsync(dst, pitch, src, pitch, width, rows, kind, s);
}

// Maps caller arrays to device arrays.  An entry point describes its arrays once, in a bind function (of Stager&) that
// calls in / out / inout for each (in2d / out2d for a D x N field) and that neither launches kernels nor reads staged
// data; stage() runs it.  Device-pointer mode: one pass, the identity.  HOST_BUFFERS mode: a first pass only measures
// the arrays, the context arena grows to fit, and a second pass carves them out of it and enqueues the uploads on the
// context stream; finish() enqueues the downloads.  The first failed copy is kept and returned by stage().
class Stager {
public:
    Stager(ahmc_ctx* c, bool host) : ctx_(c), host_(host) {}
    template <class Bind>
    int stage(Bind&& bind) {
        if (!host_) {
            bind(*this);
            return AHMC_OK;
        }
        sizing_ = true;
        carver_ = Carver{};
        bind(*this);
        sizing_ = false;
        int rc = ensure_arena(ctx_, carver_.off);
        if (rc) return rc;
        carver_ = Carver{(char*)ctx_->arena.p};
        bind(*this);
        return rc_;
    }
    template <class T>
    void in(const T* h, size_t count, const T** d) {
        *d = map(h, Span::flat(count), true, false);
    }
    template <class T>
    void out(T* h, size_t count, T** d) {
        *d = map(h, Span::flat(count), false, true);
    }
    template <class T>
    void inout(T* h, size_t count, T** d) {  // copied in now, copied back at finish
        *d = map(h, Span::flat(count), true, true);
    }
    // a D x N field at leading dimension ld (out2d: `blocks` of them, `block_stride` doubles apart -- a trajectory's
    // steps).  The device copy keeps the caller's layout and only rows d < D are copied: the caller's padding rows
    // D..ld-1 are neither read nor written, and the array needs no more than ld * (N - 1) + D doubles
    void in2d(const double* h, int32_t D, int64_t ld, int64_t N, const double** d) {
        *d = map(h, Span::matrix(D, ld, N, 1, 0), true, false);
    }
    void out2d(double* h, int32_t D, int64_t ld, int64_t N, double** d, int64_t blocks = 1, int64_t block_stride = 0) {
        *d = map(h, Span::matrix(D, ld, N, blocks, block_stride), false, true);
    }
    int finish() {
        for (auto& o : outs_)
            if (int rc = copy(o.h, o.d, o.span, o.elem, cudaMemcpyDeviceToHost)) return rc;
        return AHMC_OK;
    }
    bool host() const { return host_; }

private:
    // `blocks` blocks `block_stride` elements apart, each `rows` rows of `width` elements `pitch` apart
    struct Span {
        size_t width, pitch, rows, blocks, block_stride;
        static Span flat(size_t count) { return {count, count, 1, 1, 0}; }
        static Span matrix(int32_t D, int64_t ld, int64_t N, int64_t blocks, int64_t block_stride) {
            if (N <= 0 || blocks <= 0) return flat(0);
            if (ld != D) return {(size_t)D, (size_t)ld, (size_t)N, (size_t)blocks, (size_t)block_stride};
            const size_t n = (size_t)D * N;  // no padding: each block is contiguous, and so are back-to-back blocks
            return blocks == 1 || (size_t)block_stride == n ? flat(n * blocks) : Span{n, n, 1, (size_t)blocks, (size_t)block_stride};
        }
        size_t extent() const {
            return blocks && rows ? block_stride * (blocks - 1) + pitch * (rows - 1) + width : 0;
        }
    };
    struct Out { void* h; void* d; Span span; size_t elem; };
    int copy(void* dst, const void* src, const Span& s, size_t elem, cudaMemcpyKind kind) {
        ahmc_ctx* ctx = ctx_;
        if (!s.extent()) return AHMC_OK;
        for (size_t b = 0; b < s.blocks; ++b) {
            const size_t off = b * s.block_stride * elem;
            CU(copy_rows((char*)dst + off, (const char*)src + off, s.width * elem, s.pitch * elem, s.rows, kind, ctx->stream));
        }
        return AHMC_OK;
    }
    template <class T>
    T* map(T* h, const Span& s, bool upload, bool download) {
        if (!h || !host_) return h;
        T* p = (T*)carver_.take<T>(s.extent());
        if (sizing_) return p;
        if (upload && !rc_) rc_ = copy((void*)p, h, s, sizeof(T), cudaMemcpyHostToDevice);
        if (download) outs_.push_back({(void*)h, (void*)p, s, sizeof(T)});
        return p;
    }
    ahmc_ctx* ctx_;
    bool host_;
    bool sizing_ = false;
    Carver carver_;
    int rc_ = AHMC_OK;
    std::vector<Out> outs_;
};

int check_common(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N, bool streaming_ok = false) {
    if (!ctx) return AHMC_ERR_INVALID;
    if (D < 1) return fail(ctx, AHMC_ERR_INVALID, "D must be >= 1 (got %d)", D);
    if (N < 0) return fail(ctx, AHMC_ERR_INVALID, "N must be >= 0 (got %lld)", (long long)N);
    if (model) {
        if (model->D != D)
            return fail(ctx, AHMC_ERR_INVALID, "AxesMismatch: model has dimension %d but theta has %d rows", model->D, D);
    }
    if (metric) {
        if (metric->kind < AHMC_METRIC_UNIT || metric->kind > AHMC_METRIC_DENSE)
            return fail(ctx, AHMC_ERR_INVALID, "unknown metric kind %d", metric->kind);
        if (metric->kind != AHMC_METRIC_UNIT && !metric->Minv)
            return fail(ctx, AHMC_ERR_INVALID, "metric.Minv is NULL for a Diag/Dense metric");
        if (metric->kind == AHMC_METRIC_DIAG && metric->chain_stride != 0 && metric->chain_stride < D)
            return fail(ctx, AHMC_ERR_INVALID, "AxesMismatch: per-chain Minv stride %lld < D=%d (hamiltonian.jl:53-57)",
                        (long long)metric->chain_stride, D);
        if (metric->kind == AHMC_METRIC_DENSE && metric->chain_stride != 0 && metric->chain_stride < (int64_t)D * D)
            return fail(ctx, AHMC_ERR_INVALID, "AxesMismatch: per-chain dense Minv / cholU stride %lld < D*D=%lld (metric.jl:89-103)",
                        (long long)metric->chain_stride, (long long)D * D);
    }
    int G, E;
    if (!pick_layout(D, &G, &E)) {
        // D > 512: the streaming form (ahmc_bigd.cu, ahmc_bigd_hmc.cu) runs `step`, `phasepoint`, `rand_momentum`, static
        // EndPointTS transitions (one, several, with in-launch adaptation) and `find_good_stepsize` for the separable
        // targets and the funnel with Unit / Diag metrics; everything else is register-resident and stops at 512
        // (rand_momentum passes no model: any Unit / Diag metric streams)
        if (streaming_ok && metric && bigd_supported(model ? model->kind : AHMC_MODEL_STD_NORMAL, metric->kind)) return AHMC_OK;
        return fail(ctx, AHMC_ERR_UNSUPPORTED,
                    "D=%d: this entry point / target / metric combination is register-resident (D <= 512); D > 512 is supported by "
                    "step, phasepoint, rand_momentum, static EndPointTS transitions, sampling and in-launch adaptation, and "
                    "find_good_stepsize, for std-normal, diagonal-Gaussian and funnel targets with Unit / Diag metrics (not NUTS, "
                    "MultinomialTS static transitions, full trajectories, Dense metrics, dense-Gaussian, run-time compiled or "
                    "callback targets)", D);
    }
    return AHMC_OK;
}

// the Philox momentum draw at D > 512 indexes its blocks up to D/2 in the 24 counter bits that `offset << 24` leaves free
int check_philox_d(ahmc_ctx* ctx, int32_t D) {
    if (D >= (1 << 25)) return fail(ctx, AHMC_ERR_INVALID, "D=%d: Philox momentum draws need D < 2^25", D);
    return AHMC_OK;
}
// the transition offset fills bits 24..59 of the counter's high word, below the stream id: a launch that draws from the
// Philox streams at offsets offset .. offset + n_transitions - 1 must stay below 2^36, or its counters are another
// stream's (the normals at offset 3 * 2^36 would be the exponentials at offset 0)
static int check_philox_offset(ahmc_ctx* ctx, uint64_t offset, int64_t n_transitions) {
    constexpr uint64_t kOffsets = 1ull << 36;
    if (offset > kOffsets || (uint64_t)n_transitions > kOffsets - offset)
        return fail(ctx, AHMC_ERR_INVALID, "Philox offset %llu + %lld transitions passes 2^36: the counter holds offsets below 2^36",
                    (unsigned long long)offset, (long long)n_transitions);
    return AHMC_OK;
}

int check_pp(ahmc_ctx* ctx, const ahmc_phasepoint* z, int32_t D, const char* name, bool need_cache, int64_t N) {
    if (!z) return fail(ctx, AHMC_ERR_INVALID, "%s is NULL", name);
    if (N == 0) return AHMC_OK;  // empty batch: nothing is dereferenced
    if (!z->theta || !z->r) return fail(ctx, AHMC_ERR_INVALID, "%s.theta / %s.r is NULL", name, name);
    if (need_cache && (!z->lp_value || !z->lp_gradient || !z->lk_value))
        return fail(ctx, AHMC_ERR_INVALID, "%s.lp_value / lp_gradient / lk_value is NULL", name);
    if (z->ld < D)
        return fail(ctx, AHMC_ERR_INVALID, "%s.ld=%lld < D=%d: length(theta)==length(r)==length(gradient) violated (hamiltonian.jl:94)",
                    name, (long long)z->ld, D);
    return AHMC_OK;
}

size_t metric_minv_count(const ahmc_metric* m, int32_t D, int64_t N) {
    if (m->kind == AHMC_METRIC_DIAG) return m->chain_stride ? (size_t)m->chain_stride * (size_t)N : (size_t)D;
    if (m->kind == AHMC_METRIC_DENSE)  // per chain: chain c's matrix at chain_stride * c (the last one D*D long)
        return m->chain_stride && N > 0 ? (size_t)m->chain_stride * (size_t)(N - 1) + (size_t)D * D : (size_t)D * D;
    return 0;
}
bool per_chain_dense(const ahmc_metric* m) { return m->kind == AHMC_METRIC_DENSE && m->chain_stride != 0; }

ModelDev model_dev(const ahmc_model* m) { return ModelDev{m->kind, m->D, m->d_p0, m->d_p1, m->c0, m->rtc, m->d_p1_coop}; }

// stage the metric descriptor (device or host pointers) into a MetricDev
void stage_metric(Stager& st, const ahmc_metric* m, int32_t D, int64_t N, MetricDev* out) {
    out->kind = m->kind;
    out->chain_stride = m->kind != AHMC_METRIC_UNIT ? m->chain_stride : 0;
    out->Minv_coop = nullptr;
    out->cholU_coop = nullptr;
    st.in(m->Minv, metric_minv_count(m, D, N), &out->Minv);
    // a Dense factor has the layout of its M^-1 (shared, or per chain at the same stride)
    st.in(m->kind == AHMC_METRIC_DENSE ? m->cholU : (const double*)nullptr, metric_minv_count(m, D, N), &out->cholU);
}

// the phase-point fields the argument blocks share by name.  In: theta, r, -grad lp[, lp] of z (N chains).
template <class Args>
void stage_pp_in(Stager& st, const ahmc_phasepoint* z, int32_t D, int64_t N, Args& a, const double** lp_in = nullptr) {
    a.ld_in = z->ld;
    st.in2d((const double*)z->theta, D, z->ld, N, &a.th_in);
    st.in2d((const double*)z->r, D, z->ld, N, &a.r_in);
    st.in2d((const double*)z->lp_gradient, D, z->ld, N, &a.g_in);
    if (lp_in) st.in((const double*)z->lp_value, (size_t)N, lp_in);
}
// Out: every vector field D x N at z->ld, the energies N[, dH/dr from lk_gradient]; a trajectory has `steps` of each,
// its vector fields `step_stride` doubles apart and its energies N apart
template <class Args>
void stage_pp_out(Stager& st, const ahmc_phasepoint* z, int32_t D, int64_t N, Args& a, double** dr_out = nullptr,
                  int64_t steps = 1, int64_t step_stride = 0) {
    a.ld_out = z->ld;
    st.out2d(z->theta, D, z->ld, N, &a.th_out, steps, step_stride);
    st.out2d(z->r, D, z->ld, N, &a.r_out, steps, step_stride);
    st.out2d(z->lp_gradient, D, z->ld, N, &a.g_out, steps, step_stride);
    if (dr_out) st.out2d(z->lk_gradient, D, z->ld, N, dr_out, steps, step_stride);
    st.out(z->lp_value, (size_t)N * steps, &a.lp_out);
    st.out(z->lk_value, (size_t)N * steps, &a.lk_out);
}

int finish_call(ahmc_ctx* ctx, Stager& st, uint32_t flags) {
    int rc = st.finish();
    if (rc) return rc;
    if (!(flags & AHMC_FLAG_ASYNC) || st.host()) CU(cudaStreamSynchronize(ctx->stream));
    return AHMC_OK;
}


// D x N doubles from src (leading dimension lds) to dst (ldd) on the context stream; nothing if they are the same array
cudaError_t copy_chains(ahmc_ctx* ctx, double* dst, int64_t ldd, const double* src, int64_t lds, int32_t D, int64_t N) {
    if (dst == src) return cudaSuccess;
    return cudaMemcpy2DAsync(dst, (size_t)ldd * 8, src, (size_t)lds * 8, (size_t)D * 8, (size_t)N, cudaMemcpyDeviceToDevice,
                             ctx->stream);
}

// ---- split-step (callback) mode and sequenced transitions ------------------------------------------------------
struct SplitWork {
    double* cb_lp;           // the callback's outputs: lp[N], grad[ld x N]
    double* cb_grad;
    double* r0;              // a transition's refreshed momentum (D x N) and its kinetic energy
    double* lk0;
    uint32_t* status;        // per-chain status of a trajectory whose caller passes none
    int* flag;               // set when a chain turns non-finite in a step (COMPAT_BREAK_ALL)
    double *th0, *g0, *lp0;  // a transition's start point (D x N), when it is copied aside (`start`), else nullptr
};

int split_workspace(ahmc_ctx* ctx, int32_t D, int64_t N, int64_t ld, bool start, SplitWork* w) {
    return carve(ctx, ctx->split_ws, "the split-step workspace", [&](Carver& c) {
        w->cb_lp = c.take<double>((size_t)N);
        w->cb_grad = c.take<double>((size_t)ld * N);
        w->r0 = c.take<double>((size_t)D * N);
        w->lk0 = c.take<double>((size_t)N);
        w->status = c.take<uint32_t>((size_t)N);
        w->flag = c.take<int>(1);
        w->th0 = c.take<double>((size_t)D * N, start);
        w->g0 = c.take<double>((size_t)D * N, start);
        w->lp0 = c.take<double>((size_t)N, start);
    });
}

// user closure on the context stream: lp[N], grad[D x N] <- theta
int call_user(ahmc_ctx* ctx, const ahmc_model* model, const double* th, double* lp, double* grad, int32_t D, int64_t N,
              int64_t ld) {
    int rc = model->fn(model->user, th, lp, grad, D, N, ld, (void*)ctx->stream);
    if (rc != 0) return fail(ctx, AHMC_ERR_CALLBACK, "user gradient callback returned %d", rc);
    return AHMC_OK;
}

// lf.n_steps leapfrog steps in split mode (DEVICE pointers; w from split_workspace at lf.ld_out): the work state is the
// output phase point, which starts as a copy of the input one.  Per step a kick_drift kernel, the user closure and a
// kick_energy kernel.
int split_trajectory(ahmc_ctx* ctx, const ahmc_model* model, const LeapfrogArgs& lf, const SplitWork& w, bool compat, int* nl) {
    const int D = lf.D, n = lf.n_steps;
    const long long N = lf.N, ld = lf.ld_out;
    CU(copy_chains(ctx, lf.th_out, ld, lf.th_in, lf.ld_in, D, N));
    CU(copy_chains(ctx, lf.r_out, ld, lf.r_in, lf.ld_in, D, N));
    CU(copy_chains(ctx, lf.g_out, ld, lf.g_in, lf.ld_in, D, N));
    uint32_t* status = lf.status ? lf.status : w.status;
    CU(cudaMemsetAsync(status, 0, (size_t)N * 4, ctx->stream));
    if (lf.steps_done) CU(cudaMemsetAsync(lf.steps_done, 0, (size_t)N * 4, ctx->stream));
    CU(cudaMemsetAsync(w.flag, 0, sizeof(int), ctx->stream));
    const double ta = lf.temper_alpha;
    const double sa = ta > 0.0 ? sqrt(ta) : 1.0;
    for (int i = 1; i <= n; ++i) {
        SplitArgs a{};
        a.metric = lf.metric;
        a.D = D;
        a.N = N;
        a.eps = lf.eps;
        a.eps_chain = lf.eps_chain;
        a.fwd = lf.fwd;
        a.mul = ta > 0.0 ? ((2 * (i - 1) + 1 <= n) ? sa : 1.0 / sa) : 1.0;
        a.step_index = i;
        a.th = lf.th_out; a.r = lf.r_out; a.g = lf.g_out; a.lp = lf.lp_out; a.lk = lf.lk_out; a.dr = lf.dr_out;
        a.cb_lp = w.cb_lp; a.cb_grad = w.cb_grad;
        a.ld = ld;
        a.status = status; a.steps_done = lf.steps_done; a.any_nonfinite = w.flag;
        CU(launch_kick_drift(a, ctx->stream, nl));
        int rc = call_user(ctx, model, lf.th_out, w.cb_lp, w.cb_grad, D, N, ld);
        if (rc) return rc;
        a.mul = ta > 0.0 ? ((2 * (i - 1) + 2 <= n) ? sa : 1.0 / sa) : 1.0;
        CU(launch_kick_energy(a, ctx->stream, nl));
        if (compat) {  // reference quirk Q1: first non-finite chain stops everyone (hamiltonian.jl:141-142)
            int f = 0;
            CU(cudaMemcpyAsync(&f, w.flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
            CU(cudaStreamSynchronize(ctx->stream));
            if (f) break;
        }
    }
    return AHMC_OK;
}

// can the tiled DMMA trajectory (K4) run this target and metric?  A Gaussian target with a GEMM-shaped operator (dense
// metric and/or dense-Gaussian target), one M^-1 shared by all chains, no EXACT_CHECKS / COMPAT_BREAK_ALL, and a tile
// shape for D
bool dense_tile_eligible(const ahmc_model* model, const MetricDev& metric, uint32_t flags) {
    const bool gauss = model->kind == AHMC_MODEL_STD_NORMAL || model->kind == AHMC_MODEL_DIAG_GAUSS ||
                       model->kind == AHMC_MODEL_DENSE_GAUSS;
    const bool has_dense = model->kind == AHMC_MODEL_DENSE_GAUSS || metric.kind == AHMC_METRIC_DENSE;
    int Dp, RB, CB;
    return gauss && has_dense && metric.chain_stride == 0 && !(flags & (AHMC_FLAG_EXACT_CHECKS | AHMC_FLAG_COMPAT_BREAK_ALL)) &&
           dense_tile_shape(model->D, &Dp, &RB, &CB) && (model->kind != AHMC_MODEL_DENSE_GAUSS || model->d_p1_pad);
}

// K4: GEMM-shaped operators (dense metric and/or dense-Gaussian target) -> tiled DMMA kernel; chains of tiles it declines
// (magnitude proof not met) are redone by the exact warp-per-chain kernel from the untouched inputs.  DEVICE pointers.
int dense_trajectory(ahmc_ctx* ctx, const ahmc_model* model, const LeapfrogArgs& a, int* nl) {
    const int D = a.D;
    const long long N = a.N;
    int Dp, RB, CB;
    dense_tile_shape(D, &Dp, &RB, &CB);
    double *Mpad, *norms;
    uint8_t* mask;
    int rc = carve(ctx, ctx->dense_ws, "the dense workspace", [&](Carver& c) {
        Mpad = c.take<double>(dense_mat_doubles(Dp));
        norms = c.take<double>(2);
        mask = c.take<uint8_t>((size_t)N);
    });
    if (rc) return rc;
    DenseTrajHost h{};
    h.D = D; h.Dp = Dp; h.N = N; h.c0 = model->c0;
    h.mu = (model->kind == AHMC_MODEL_STD_NORMAL) ? nullptr : model->d_p0;
    if (model->kind == AHMC_MODEL_DENSE_GAUSS) {
        h.P = model->d_p1_pad;
        CU(cudaMemcpyAsync(norms + 1, model->d_p1_pad + dense_mat_doubles(Dp), 8, cudaMemcpyDeviceToDevice, ctx->stream));
    } else {
        h.w = (model->kind == AHMC_MODEL_DIAG_GAUSS) ? model->d_p1 : nullptr;
        CU(launch_vec_norm(h.w, D, norms + 1, ctx->stream));
        *nl += 1;
    }
    if (a.metric.kind == AHMC_METRIC_DENSE) {
        CU(launch_pad_norm(a.metric.Minv, D, Dp, Mpad, norms, ctx->stream));
        h.Minv = Mpad;
    } else {
        h.Mdiag = (a.metric.kind == AHMC_METRIC_DIAG) ? a.metric.Minv : nullptr;
        CU(launch_vec_norm(h.Mdiag, D, norms, ctx->stream));
    }
    *nl += 1;
    h.norms = norms;
    h.eps = a.eps; h.eps_chain = a.eps_chain; h.n_steps = a.n_steps; h.fwd = a.fwd;
    h.th_in = a.th_in; h.r_in = a.r_in; h.g_in = a.g_in; h.ld_in = a.ld_in;
    h.th_out = a.th_out; h.r_out = a.r_out; h.g_out = a.g_out; h.dr_out = a.dr_out;
    h.lp_out = a.lp_out; h.lk_out = a.lk_out; h.ld_out = a.ld_out;
    h.status = a.status; h.steps_done = a.steps_done; h.need_exact = mask;
    CU(launch_dense_traj(h, ctx->stream, nl));
    LeapfrogArgs b = a;
    b.only_mask = mask;
    CU(launch_leapfrog(b, ctx->stream, nl));
    return AHMC_OK;
}

// can the chain-tile kernel (K6) run this call?  A GLM target, device buffers, a Unit or Diag metric (shared or per
// chain), no EXACT_CHECKS / COMPAT_BREAK_ALL, and a tile shape for (D, n)
bool glm_tile_eligible(const ahmc_model* model, const MetricDev& metric, uint32_t flags) {
    int RB, CB, nc, stages;
    size_t sm;
    return model->glm_family >= 0 && metric.kind != AHMC_METRIC_DENSE &&
           !(flags & (AHMC_FLAG_EXACT_CHECKS | AHMC_FLAG_HOST_BUFFERS | AHMC_FLAG_COMPAT_BREAK_ALL)) &&
           glm_tile_shape(model->D, model->glm_n, &RB, &CB, &nc, &stages, &sm);
}
// the model and metric half of K6's argument block
GlmArgs glm_args(const ahmc_model* model, const MetricDev& metric, int64_t N) {
    GlmArgs g{};
    g.family = model->glm_family; g.D = model->D; g.n = model->glm_n; g.N = N;
    g.Xp = model->d_glm_X; g.prec = model->d_p0; g.y = model->d_p0 + model->D + (size_t)model->glm_n * model->D;
    g.c0 = model->c0;
    g.Minv = metric.kind == AHMC_METRIC_DIAG ? metric.Minv : nullptr;
    g.chain_stride = metric.chain_stride;
    return g;
}
// K6: the GLM target's trajectory on the chain-tile kernel.  DEVICE pointers.
int glm_trajectory(ahmc_ctx* ctx, const ahmc_model* model, const LeapfrogArgs& a, int* nl) {
    GlmArgs g = glm_args(model, a.metric, a.N);
    g.eps = a.eps; g.eps_chain = a.eps_chain; g.n_steps = a.n_steps; g.fwd = a.fwd;
    g.th_in = a.th_in; g.r_in = a.r_in; g.g_in = a.g_in; g.ld_in = a.ld_in;
    g.th_out = a.th_out; g.r_out = a.r_out; g.g_out = a.g_out; g.dr_out = a.dr_out;
    g.lp_out = a.lp_out; g.lk_out = a.lk_out; g.ld_out = a.ld_out;
    g.status = a.status; g.steps_done = a.steps_done;
    CU(launch_glm_traj(g, ctx->stream, nl));
    return AHMC_OK;
}

// The engine that integrates a call's trajectory, for ahmc_leapfrog_f64 and the static HMC transitions (hmc_impl adds
// conditions of its own before K4 or K6 runs a transition).
enum class Engine {
    Dense,  // K4, dense_trajectory
    Glm,    // K6, glm_trajectory
    Split,  // callback target, split_trajectory
    Fused,  // the register-resident kernels (K1 leapfrog, hmc_kernel), D > 512 and run-time compiled forms included
};
Engine trajectory_engine(const ahmc_model* model, const MetricDev& metric, uint32_t flags, double temper_alpha, bool has_grad) {
    if (model->kind == AHMC_MODEL_CALLBACK) return Engine::Split;
    if (temper_alpha > 0.0) return Engine::Fused;  // K4 and K6 integrate plain Leapfrog
    if (dense_tile_eligible(model, metric, flags) && has_grad) return Engine::Dense;  // K4 reads the start point's gradient
    if (glm_tile_eligible(model, metric, flags)) return Engine::Glm;
    return Engine::Fused;
}
// the trajectory of engine `e` (not Fused) from lf's inputs to its outputs; `w` serves the split-step engine
int run_trajectory(ahmc_ctx* ctx, const ahmc_model* model, Engine e, const LeapfrogArgs& lf, const SplitWork& w, bool compat,
                   int* nl) {
    if (e == Engine::Dense) return dense_trajectory(ctx, model, lf, nl);
    if (e == Engine::Glm) return glm_trajectory(ctx, model, lf, nl);
    return split_trajectory(ctx, model, lf, w, compat, nl);
}

// row `off` / N of statistics arrays that hold N entries per transition
StatsDev stats_row(StatsDev s, size_t off) {
    auto at = [off](auto* p) { return p ? p + off : p; };
    s.n_steps = at(s.n_steps);
    s.is_accept = at(s.is_accept);
    s.acceptance_rate = at(s.acceptance_rate);
    s.log_density = at(s.log_density);
    s.hamiltonian_energy = at(s.hamiltonian_energy);
    s.hamiltonian_energy_error = at(s.hamiltonian_energy_error);
    s.max_hamiltonian_energy_error = at(s.max_hamiltonian_energy_error);
    s.tree_depth = at(s.tree_depth);
    s.numerical_error = at(s.numerical_error);
    return s;
}

// hmc_kernel's static transitions, one kernel per stage, for the engines it cannot fuse (K4, K6, split-step): per
// transition refresh -> kinetic energy -> trajectory from the start point into z_out -> MH select, enqueued back to back
// (only a callback target's closure may synchronise).  Transition t draws at Philox offset offset + t, starts from z_in
// (t = 0) or from transition t - 1's z_out, and writes row t of `draws` and of the statistics.  `h`: DEVICE pointers.
int sequenced_transitions(ahmc_ctx* ctx, const ahmc_model* model, Engine e, const HmcArgs& h, int* nl) {
    const LeapfrogArgs& a = h.lf;
    const int D = a.D;
    const long long N = a.N;
    const bool alias = a.th_out == a.th_in;
    SplitWork w;
    int rc = split_workspace(ctx, D, N, a.ld_out, h.n_transitions > 1 || alias, &w);
    if (rc) return rc;
    for (int t = 0; t < h.n_transitions; ++t) {
        const double *th0 = t ? a.th_out : a.th_in, *g0 = t ? a.g_out : a.g_in, *lp0 = t ? a.lp_out : a.lp_in;
        long long ld0 = t ? a.ld_out : a.ld_in;
        RngDev rng = h.rng;
        rng.offset += (uint64_t)t;
        if (h.refresh) {
            MomentumArgs ma{};
            ma.metric = a.metric; ma.D = D; ma.N = N; ma.seed = rng.seed; ma.offset = rng.offset;
            ma.normal_tape = rng.normal_tape; ma.r = w.r0; ma.ld = D;
            CU(launch_rand_momentum(ma, ctx->stream, nl));
        } else {
            CU(copy_chains(ctx, w.r0, D, t ? a.r_out : a.r_in, ld0, D, N));
        }
        SplitArgs k0{};  // lk0 = neg kinetic energy of the refreshed momentum
        k0.metric = a.metric; k0.D = D; k0.N = N; k0.fwd = 1; k0.mul = 1.0; k0.no_kick = 1;
        k0.r = w.r0; k0.lk = w.lk0; k0.ld = D;
        CU(launch_kick_energy(k0, ctx->stream, nl));
        // MH select re-reads the start point after the trajectory has written z_out: when z_out holds it (t > 0) or
        // aliases it, it is copied aside first
        if (t || alias) {
            CU(copy_chains(ctx, w.th0, D, th0, ld0, D, N));
            CU(copy_chains(ctx, w.g0, D, g0, ld0, D, N));
            CU(cudaMemcpyAsync(w.lp0, lp0, (size_t)N * 8, cudaMemcpyDeviceToDevice, ctx->stream));
            th0 = w.th0; g0 = w.g0; lp0 = w.lp0; ld0 = D;
        }
        LeapfrogArgs lf = a;
        lf.temper_alpha = h.rng.temper_alpha;
        if (ld0 == D) {
            lf.th_in = th0; lf.r_in = w.r0; lf.g_in = g0; lf.ld_in = D;
        } else {  // the trajectory reads theta, r and -grad at one leading dimension, and r0's is D: it starts from a
                  // copy of the start point in z_out
            CU(copy_chains(ctx, a.th_out, a.ld_out, th0, ld0, D, N));
            CU(copy_chains(ctx, a.g_out, a.ld_out, g0, ld0, D, N));
            CU(copy_chains(ctx, a.r_out, a.ld_out, w.r0, D, D, N));
            lf.th_in = a.th_out; lf.r_in = a.r_out; lf.g_in = a.g_out; lf.ld_in = a.ld_out;
        }
        if ((rc = run_trajectory(ctx, model, e, lf, w, false, nl))) return rc;
        MhArgs m{};
        m.D = D; m.N = N; m.n_steps = a.n_steps;
        m.th0 = th0; m.g0 = g0; m.lp0 = lp0; m.ld0 = ld0;
        m.r0 = w.r0; m.lk0 = w.lk0;
        m.th = a.th_out; m.r = a.r_out; m.g = a.g_out; m.lp = a.lp_out; m.lk = a.lk_out; m.ld = a.ld_out;
        m.rng = rng;
        const size_t row = (size_t)t * N;
        m.st = stats_row(h.st, row);
        CU(launch_mh_select(m, ctx->stream, nl));
        if (h.draws) CU(copy_chains(ctx, h.draws + row * D, D, a.th_out, a.ld_out, D, N));
    }
    return AHMC_OK;
}
}  // namespace

// =================================================================================================
extern "C" {

const char* ahmc_version(void) { return "ahmc_b200 0.1.0 (sm_90a)"; }

int ahmc_create(ahmc_ctx** out, int32_t device, void* cuda_stream) {
    if (!out) return AHMC_ERR_INVALID;
    *out = nullptr;
    ahmc_ctx* ctx = new (std::nothrow) ahmc_ctx();
    if (!ctx) return AHMC_ERR_NOMEM;
    ctx->device = device;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || device < 0 || device >= ndev) {
        // no silent CPU fallback: the product path needs the GPU
        fprintf(stderr, "ahmc_create: no usable CUDA device %d (%s)\n", device, e != cudaSuccess ? cudaGetErrorString(e) : "out of range");
        delete ctx;
        return AHMC_ERR_CUDA;
    }
    int cc_major = 0, cc_minor = 0;
    cudaDeviceGetAttribute(&cc_major, cudaDevAttrComputeCapabilityMajor, device);
    cudaDeviceGetAttribute(&cc_minor, cudaDevAttrComputeCapabilityMinor, device);
    if (cc_major != 9 || cc_minor != 0) {
        // the library holds sm_90a code only, which runs on compute capability 9.0 (H100 / H200) and nothing else
        fprintf(stderr, "ahmc_create: device %d has compute capability %d.%d; libahmc_b200 is built for sm_90a (9.0)\n", device,
                cc_major, cc_minor);
        delete ctx;
        return AHMC_ERR_UNSUPPORTED;
    }
    cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
    DeviceGuard g(device);
    if (cuda_stream) {
        ctx->stream = (cudaStream_t)cuda_stream;
    } else {
        if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
            delete ctx;
            return AHMC_ERR_CUDA;
        }
        ctx->own_stream = true;
    }
    if (cudaMalloc((void**)&ctx->d_min_break, sizeof(int)) != cudaSuccess) {
        if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
        delete ctx;
        return AHMC_ERR_NOMEM;
    }
    *out = ctx;
    return AHMC_OK;
}

int ahmc_destroy(ahmc_ctx* ctx) {
    if (!ctx) return AHMC_OK;
    DeviceGuard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaFree(ctx->d_min_break);
    for (DevBuf* b : {&ctx->arena, &ctx->chain_ws, &ctx->summary_ws, &ctx->energy_ws, &ctx->dense_ws, &ctx->coop_ws, &ctx->split_ws})
        cudaFree(b->p);
    for (cudaStream_t s : ctx->pipe)
        if (s) cudaStreamDestroy(s);
    for (int i = 0; i < kMaxPipeChunks; ++i) {
        if (ctx->ev_in[i]) cudaEventDestroy(ctx->ev_in[i]);
        if (ctx->ev_k[i]) cudaEventDestroy(ctx->ev_k[i]);
    }
    if (ctx->ev_a) cudaEventDestroy(ctx->ev_a);
    if (ctx->ev_down) cudaEventDestroy(ctx->ev_down);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return AHMC_OK;
}

const char* ahmc_last_error(const ahmc_ctx* ctx) { return ctx ? ctx->err.c_str() : "ahmc: NULL context"; }

int ahmc_synchronize(ahmc_ctx* ctx) {
    if (!ctx) return AHMC_ERR_INVALID;
    DeviceGuard g(ctx->device);
    CU(cudaStreamSynchronize(ctx->stream));
    return AHMC_OK;
}

void* ahmc_stream(const ahmc_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int64_t ahmc_launch_count(const ahmc_ctx* ctx) { return ctx ? ctx->launches : 0; }
const char* ahmc_last_transport(const ahmc_ctx* ctx) { return ctx ? ctx->transport.c_str() : "none"; }

// ---------------------------------------------------------------------------------------------- models
int ahmc_model_create(ahmc_ctx* ctx, int32_t kind, int32_t D, const double* p0, const double* p1, double c0,
                      ahmc_model** out) {
    if (!ctx || !out) return AHMC_ERR_INVALID;
    *out = nullptr;
    if (D < 1) return fail(ctx, AHMC_ERR_INVALID, "model dimension must be >= 1");
    if (kind < AHMC_MODEL_STD_NORMAL || kind > AHMC_MODEL_FUNNEL)
        return fail(ctx, AHMC_ERR_INVALID, "unknown built-in model kind %d", kind);
    if ((kind == AHMC_MODEL_DIAG_GAUSS || kind == AHMC_MODEL_DENSE_GAUSS) && (!p0 || !p1))
        return fail(ctx, AHMC_ERR_INVALID, "model kind %d needs p0 and p1", kind);
    DeviceGuard g(ctx->device);
    ahmc_model* m = new (std::nothrow) ahmc_model();
    if (!m) return AHMC_ERR_NOMEM;
    m->kind = kind;
    m->D = D;
    m->c0 = c0;
    if (kind == AHMC_MODEL_DIAG_GAUSS) {
        std::vector<double> w((size_t)D);
        for (int d = 0; d < D; ++d) w[d] = 1.0 / (p1[d] * p1[d]);  // 1/s^2
        if (cudaMalloc((void**)&m->d_p0, sizeof(double) * D) != cudaSuccess ||
            cudaMalloc((void**)&m->d_p1, sizeof(double) * D) != cudaSuccess) {
            ahmc_model_destroy(ctx, m);
            return fail(ctx, AHMC_ERR_NOMEM, "cudaMalloc for model parameters failed");
        }
        cudaMemcpy(m->d_p0, p0, sizeof(double) * D, cudaMemcpyHostToDevice);
        cudaMemcpy(m->d_p1, w.data(), sizeof(double) * D, cudaMemcpyHostToDevice);
    } else if (kind == AHMC_MODEL_DENSE_GAUSS) {
        if (cudaMalloc((void**)&m->d_p0, sizeof(double) * D) != cudaSuccess ||
            cudaMalloc((void**)&m->d_p1, sizeof(double) * (size_t)D * D) != cudaSuccess) {
            ahmc_model_destroy(ctx, m);
            return fail(ctx, AHMC_ERR_NOMEM, "cudaMalloc for model parameters failed");
        }
        cudaMemcpy(m->d_p0, p0, sizeof(double) * D, cudaMemcpyHostToDevice);
        cudaMemcpy(m->d_p1, p1, sizeof(double) * (size_t)D * D, cudaMemcpyHostToDevice);
        int RB, CB;
        if (dense_tile_shape(D, &m->Dp, &RB, &CB)) {  // padded copy + infinity norm for the tiled DMMA kernel
            if (cudaMalloc((void**)&m->d_p1_pad, sizeof(double) * (dense_mat_doubles(m->Dp) + 2)) != cudaSuccess) {
                ahmc_model_destroy(ctx, m);
                return fail(ctx, AHMC_ERR_NOMEM, "cudaMalloc for the padded precision failed");
            }
            launch_pad_norm(m->d_p1, D, m->Dp, m->d_p1_pad, m->d_p1_pad + dense_mat_doubles(m->Dp), ctx->stream);
            cudaStreamSynchronize(ctx->stream);
        }
        if (D > 16 && D <= 512) {  // the layouts the cooperative NUTS form runs on (one chain per warp)
            if (cudaMalloc((void**)&m->d_p1_coop, sizeof(double) * coop_padded_doubles(D)) != cudaSuccess) {
                ahmc_model_destroy(ctx, m);
                return fail(ctx, AHMC_ERR_NOMEM, "cudaMalloc for the column-padded precision failed");
            }
            launch_pad_columns(m->d_p1, D, m->d_p1_coop, ctx->stream);
            cudaStreamSynchronize(ctx->stream);
        }
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        ahmc_model_destroy(ctx, m);
        return fail(ctx, AHMC_ERR_CUDA, "copying model parameters failed: %s", cudaGetErrorString(e));
    }
    *out = m;
    return AHMC_OK;
}

int ahmc_model_create_callback(ahmc_ctx* ctx, int32_t D, ahmc_logp_grad_fn fn, void* user, ahmc_model** out) {
    if (!ctx || !out) return AHMC_ERR_INVALID;
    *out = nullptr;
    if (D < 1 || !fn) return fail(ctx, AHMC_ERR_INVALID, "callback model needs D >= 1 and a function");
    ahmc_model* m = new (std::nothrow) ahmc_model();
    if (!m) return AHMC_ERR_NOMEM;
    m->kind = AHMC_MODEL_CALLBACK;
    m->D = D;
    m->fn = fn;
    m->user = user;
    *out = m;
    return AHMC_OK;
}

int ahmc_model_create_user(ahmc_ctx* ctx, int32_t D, const char* cuda_src, const double* params, int32_t n_params, double c0,
                           ahmc_model** out) {
    if (!ctx || !cuda_src || !out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/source/out");
    if (D < 1 || n_params < 0 || (n_params > 0 && !params)) return fail(ctx, AHMC_ERR_INVALID, "need D >= 1 and params for n_params > 0");
    if (!strstr(cuda_src, "ahmc_user_logp_grad") && !strstr(cuda_src, "ahmc_user_coord"))
        return fail(ctx, AHMC_ERR_INVALID, "the source must define ahmc_user_logp_grad(theta, grad, D, params) or, with "
                                           "#define AHMC_USER_COORDWISE, ahmc_user_coord(d, theta_d, params, grad_d)");
    DeviceGuard g(ctx->device);
    char why[256];
    UserModule* um = user_module_create(cuda_src, why, sizeof why);
    if (!um) return fail(ctx, AHMC_ERR_UNSUPPORTED, "run-time compilation is unavailable: %s", why);
    ahmc_model* m = new (std::nothrow) ahmc_model;
    if (!m) {
        user_module_destroy(um);
        return fail(ctx, AHMC_ERR_NOMEM, "out of host memory");
    }
    m->kind = AHMC_MODEL_USER;
    m->D = D;
    m->c0 = c0;
    m->rtc = um;
    if (n_params > 0) {
        if (cudaMalloc((void**)&m->d_p0, (size_t)n_params * 8) != cudaSuccess) {
            user_module_destroy(um);
            delete m;
            return fail(ctx, AHMC_ERR_NOMEM, "cudaMalloc for the user parameters failed");
        }
        CU(cudaMemcpy(m->d_p0, params, (size_t)n_params * 8, cudaMemcpyHostToDevice));
    }
    *out = m;
    return AHMC_OK;
}

int ahmc_user_source_check(const char* cuda_src, int32_t kernel, int32_t metric_kind, int32_t D, char* log, int64_t log_len) {
    if (!cuda_src || kernel < 0 || kernel > UK_HMC_ADAPT || metric_kind < 0 || metric_kind > 2 || D < 1) return AHMC_ERR_INVALID;
    int rc = user_source_check(cuda_src, kernel, metric_kind, D, log, log_len > 0 ? (size_t)log_len : 0);
    return rc == 0 ? AHMC_OK : (rc == -3 ? AHMC_ERR_UNSUPPORTED : AHMC_ERR_INVALID);
}

int64_t ahmc_glm_source(int32_t family, int32_t D, int32_t n, char* buf, int64_t len) {
    const std::string s = glm_group_source(family, D, n);
    if (buf && len > 0) snprintf(buf, (size_t)len, "%s", s.c_str());
    return (int64_t)s.size();
}

int ahmc_model_create_glm(ahmc_ctx* ctx, int32_t family, int32_t D, int32_t n, const double* X, const double* y,
                          const double* prior_prec, double c0, ahmc_model** out) {
    if (!ctx || !out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/out");
    *out = nullptr;
    if (family != AHMC_GLM_BERNOULLI_LOGIT && family != AHMC_GLM_POISSON_LOG)
        return fail(ctx, AHMC_ERR_INVALID, "unknown GLM family %d", family);
    if (n < 1 || D < 1 || D > 512) return fail(ctx, AHMC_ERR_INVALID, "a GLM target needs n >= 1 rows and D in 1..512 (got n=%d, D=%d)", n, D);
    if (!X || !y) return fail(ctx, AHMC_ERR_INVALID, "X / y is NULL");
    for (size_t i = 0; i < (size_t)n * D; ++i)
        if (!std::isfinite(X[i])) return fail(ctx, AHMC_ERR_INVALID, "X[%zu, %zu] is not finite", i / D, i % D);
    for (int d = 0; prior_prec && d < D; ++d)
        if (!std::isfinite(prior_prec[d]) || prior_prec[d] < 0.0)
            return fail(ctx, AHMC_ERR_INVALID, "prior_prec[%d] = %g: precisions are finite and >= 0", d, prior_prec[d]);
    double lgam = 0.0;
    for (int i = 0; i < n; ++i) {
        if (!std::isfinite(y[i])) return fail(ctx, AHMC_ERR_INVALID, "y[%d] is not finite", i);
        if (family == AHMC_GLM_BERNOULLI_LOGIT && y[i] != 0.0 && y[i] != 1.0)
            return fail(ctx, AHMC_ERR_INVALID, "y[%d] = %g: a Bernoulli response is 0 or 1", i, y[i]);
        if (family == AHMC_GLM_POISSON_LOG) {
            if (y[i] < 0.0 || y[i] != std::floor(y[i]))
                return fail(ctx, AHMC_ERR_INVALID, "y[%d] = %g: a Poisson response is a non-negative integer", i, y[i]);
            lgam += std::lgamma(y[i] + 1.0);
        }
    }
    DeviceGuard g(ctx->device);
    ahmc_model* m = new (std::nothrow) ahmc_model();
    if (!m) return fail(ctx, AHMC_ERR_NOMEM, "out of host memory");
    m->kind = AHMC_MODEL_USER;
    m->D = D;
    m->c0 = c0 - lgam;
    m->glm_family = family;
    m->glm_n = n;
    char why[256];
    // without NVRTC the model still exists: calls that need the run-time compiled kernels fail at first use
    m->rtc = user_module_create(glm_group_source(family, D, n).c_str(), why, sizeof why);
    std::vector<double> params((size_t)D + (size_t)n * D + n, 0.0);
    if (prior_prec) memcpy(params.data(), prior_prec, sizeof(double) * D);
    memcpy(params.data() + D, X, sizeof(double) * (size_t)n * D);
    memcpy(params.data() + D + (size_t)n * D, y, sizeof(double) * n);
    const int lds = glm_lds(D);
    std::vector<double> Xp(glm_padded_doubles(D, n), 0.0);
    for (int i = 0; i < n; ++i) memcpy(Xp.data() + (size_t)i * lds, X + (size_t)i * D, sizeof(double) * D);
    if (cudaMalloc((void**)&m->d_p0, params.size() * 8) != cudaSuccess || cudaMalloc((void**)&m->d_glm_X, Xp.size() * 8) != cudaSuccess) {
        ahmc_model_destroy(ctx, m);
        return fail(ctx, AHMC_ERR_NOMEM, "cudaMalloc for the GLM data failed");
    }
    cudaError_t e = cudaMemcpy(m->d_p0, params.data(), params.size() * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(m->d_glm_X, Xp.data(), Xp.size() * 8, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        ahmc_model_destroy(ctx, m);
        return fail(ctx, AHMC_ERR_CUDA, "copying the GLM data failed: %s", cudaGetErrorString(e));
    }
    *out = m;
    return AHMC_OK;
}

int ahmc_model_destroy(ahmc_ctx* ctx, ahmc_model* m) {
    if (!m) return AHMC_OK;
    if (ctx) {
        DeviceGuard g(ctx->device);
        cudaFree(m->d_p0);
        cudaFree(m->d_p1);
        cudaFree(m->d_p1_pad);
        cudaFree(m->d_p1_coop);
        cudaFree(m->d_glm_X);
        if (m->rtc) {
            cudaStreamSynchronize(ctx->stream);
            user_module_destroy(m->rtc);
        }
    }
    delete m;
    return AHMC_OK;
}

// ---------------------------------------------------------------------------------------------- phasepoint
int ahmc_phasepoint_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                        const ahmc_phasepoint* z, uint32_t flags) {
    if (!ctx || !model || !metric) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/model/metric");
    int rc = check_common(ctx, model, metric, D, N, true);
    if (rc) return rc;
    if ((rc = check_pp(ctx, z, D, "z", true, N))) return rc;
    if (N == 0) return AHMC_OK;
    DeviceGuard g(ctx->device);
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    PhasepointArgs a{};
    a.model = model_dev(model);
    a.D = D;
    a.N = N;
    a.ld = z->ld;
    rc = st.stage([&](Stager& s) {
        stage_metric(s, metric, D, N, &a.metric);
        s.in2d((const double*)z->theta, D, z->ld, N, &a.th);
        s.in2d((const double*)z->r, D, z->ld, N, &a.r);
        s.out(z->lp_value, (size_t)N, &a.lp);
        s.out2d(z->lp_gradient, D, z->ld, N, &a.g);
        s.out(z->lk_value, (size_t)N, &a.lk);
        s.out2d(z->lk_gradient, D, z->ld, N, &a.dr);
    });
    if (rc) return rc;
    int nl = 0;
    if (model->kind == AHMC_MODEL_CALLBACK) {  // user closure, then the metric half of phasepoint
        SplitWork w;
        if ((rc = split_workspace(ctx, D, N, z->ld, false, &w))) return rc;
        if ((rc = call_user(ctx, model, a.th, w.cb_lp, w.cb_grad, D, N, z->ld))) return rc;
        SplitArgs sa{};
        sa.metric = a.metric; sa.D = D; sa.N = N; sa.fwd = 1; sa.mul = 1.0; sa.no_kick = 1;
        sa.r = const_cast<double*>(a.r); sa.g = a.g; sa.lp = a.lp; sa.lk = a.lk; sa.dr = a.dr;
        sa.cb_lp = w.cb_lp; sa.cb_grad = w.cb_grad; sa.ld = z->ld;
        CU(launch_kick_energy(sa, ctx->stream, &nl));
    } else if (glm_tile_eligible(model, a.metric, flags)) {  // one pass of the tile kernel over the input point
        GlmArgs ga = glm_args(model, a.metric, N);
        ga.fwd = 1; ga.th_in = a.th; ga.r_in = a.r; ga.ld_in = ga.ld_out = z->ld;
        ga.g_out = a.g; ga.dr_out = a.dr; ga.lp_out = a.lp; ga.lk_out = a.lk;
        CU(launch_glm_traj(ga, ctx->stream, &nl));
    } else {
        CU(launch_phasepoint(a, ctx->stream, &nl));
    }
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

// ---------------------------------------------------------------------------------------------- leapfrog
static int copy_pp_device(ahmc_ctx* ctx, int32_t D, int64_t N, const ahmc_phasepoint* a, const ahmc_phasepoint* b,
                          cudaMemcpyKind kind) {
    auto cp2 = [&](double* dst, const double* src) -> cudaError_t {
        if (!dst || !src || dst == src) return cudaSuccess;
        return cudaMemcpy2DAsync(dst, (size_t)b->ld * sizeof(double), src, (size_t)a->ld * sizeof(double),
                                 (size_t)D * sizeof(double), (size_t)N, kind, ctx->stream);
    };
    auto cp1 = [&](double* dst, const double* src) -> cudaError_t {
        if (!dst || !src || dst == src) return cudaSuccess;
        return cudaMemcpyAsync(dst, src, (size_t)N * sizeof(double), kind, ctx->stream);
    };
    CU(cp2(b->theta, a->theta));
    CU(cp2(b->r, a->r));
    CU(cp2(b->lp_gradient, a->lp_gradient));
    CU(cp2(b->lk_gradient, a->lk_gradient));
    CU(cp1(b->lp_value, a->lp_value));
    CU(cp1(b->lk_value, a->lk_value));
    return AHMC_OK;
}

// device alias of a page-locked, device-mapped host pointer (cudaHostAlloc / cudaHostRegister memory under unified
// addressing), or nullptr for pageable memory
static void* pinned_alias(const void* p) {
    if (!p) return nullptr;
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    if (at.type != cudaMemoryTypeHost || !at.devicePointer) return nullptr;
    return at.devicePointer;
}

static int pipe_resources(ahmc_ctx* ctx) {
    if (ctx->pipe[0]) return AHMC_OK;
    for (cudaStream_t& s : ctx->pipe) CU(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&ctx->ev_a, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&ctx->ev_down, cudaEventDisableTiming));
    for (int i = 0; i < kMaxPipeChunks; ++i) {
        CU(cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&ctx->ev_k[i], cudaEventDisableTiming));
    }
    return AHMC_OK;
}

// HOST_BUFFERS fast lane.  The chain axis is cut into chunks (chains are independent, so a chunk is a complete
// sub-problem) that flow upload -> kernel -> download through separate streams linked chunk by chunk with events, so
// the upload of chunk i+1 overlaps the kernel and the download of chunk i (PCIe is full duplex): the call costs about
// max(H2D, D2H) + one chunk instead of their sum.  Same kernels, bit-identical results to the one-shot path.
//   upload   : copy engines on one stream, or -- page-locked inputs only -- none at all: the kernel loads from host
//              memory directly, in one chunk;
//   download : copy engines on a second stream, or -- page-locked outputs only -- none: the kernel's stores go straight
//              to host memory as posted PCIe writes.
// Each side is direct exactly when all of its buffers are page-locked.  A copy-engine upload takes 2 chunks from 1024
// chains on (1 below).  When every buffer is page-locked and N >= 1024 the transport is measured instead (kPipeCands).
static int leapfrog_host_pipelined(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D,
                                   int64_t N, double eps, const double* eps_chain, int32_t n_steps,
                                   double temper_alpha, const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out,
                                   uint32_t* status, int32_t* steps_done, uint32_t flags) {
    const auto t_enter = std::chrono::steady_clock::now();
    auto since = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enter).count(); };
    int rc = pipe_resources(ctx);
    if (rc) return rc;
    const bool per_chain_minv = metric->kind == AHMC_METRIC_DIAG && metric->chain_stride != 0;

    // which buffers can the device address directly?
    bool in_pinned = true, out_pinned = true;
    auto alias = [](const void* p, bool& all) -> void* {
        if (!p) return nullptr;
        void* d = pinned_alias(p);
        if (!d) all = false;
        return d;
    };
    const double* a_th = (const double*)alias(z_in->theta, in_pinned);
    const double* a_r = (const double*)alias(z_in->r, in_pinned);
    const double* a_g = (const double*)alias(z_in->lp_gradient, in_pinned);
    const double* a_eps = (const double*)alias(eps_chain, in_pinned);
    const double* a_minv = per_chain_minv ? (const double*)alias(metric->Minv, in_pinned) : nullptr;
    double* b_th = (double*)alias(z_out->theta, out_pinned);
    double* b_r = (double*)alias(z_out->r, out_pinned);
    double* b_g = (double*)alias(z_out->lp_gradient, out_pinned);
    double* b_dr = (double*)alias(z_out->lk_gradient, out_pinned);
    double* b_lp = (double*)alias(z_out->lp_value, out_pinned);
    double* b_lk = (double*)alias(z_out->lk_value, out_pinned);
    uint32_t* b_st = (uint32_t*)alias(status, out_pinned);
    int32_t* b_sd = (int32_t*)alias(steps_done, out_pinned);

    const bool has_g = z_in->lp_gradient != nullptr;
    PipeTransport tp{in_pinned, out_pinned, in_pinned ? 1 : N >= 1024 ? 2 : 1};
    // ---- transport choice.  Page-locked buffers can be moved in several ways whose ranking depends on the HOST
    // (SM-issued reads of system memory are at the mercy of the platform's read-completion latency, copy engines are
    // not), so the first calls of a given shape try each candidate in turn -- results are bit-identical in every mode,
    // nothing extra is executed -- and the fastest is kept for the life of the context.
    constexpr int kRounds = 3;  // round 0 warms every candidate up (arena growth, first-touch), rounds 1.. are timed
    ahmc_ctx::PipeTune* tune = nullptr;
    int trial = -1;
    if (in_pinned && out_pinned && N >= 1024) {
        const int key = (has_g ? 1 : 0) | (z_out->lk_gradient ? 2 : 0) | (eps_chain ? 4 : 0) | (per_chain_minv ? 8 : 0);
        for (auto& t : ctx->tune)
            if (t.N == N && t.D == D && t.key == key) tune = &t;
        if (!tune) {
            ahmc_ctx::PipeTune t{};
            t.N = N; t.D = D; t.key = key; t.calls = 0; t.chosen = -1;
            for (double& b : t.best_ms) b = 1e30;
            ctx->tune.push_back(t);
            tune = &ctx->tune.back();
        }
        int c = tune->chosen;
        if (c < 0) {
            trial = tune->calls % kPipeNCand;
            c = trial;
        }
        tp = kPipeCands[c];
    }
    int64_t chunk = (N + tp.chunks - 1) / tp.chunks;
    chunk = (chunk + 3) & ~(int64_t)3;

    // device staging for whatever is not addressed directly
    const int64_t ldi = z_in->ld, ldo = z_out->ld;
    const size_t nMinv = metric_minv_count(metric, D, N);
    const bool stage_in = !tp.up_direct, stage_out = !tp.down_direct;
    // a launch that reads or writes host memory directly is capped at one resident CTA per SM (see PipeTransport)
    const int occ_cap = tp.up_direct || tp.down_direct ? 1 : 0;
    const bool hasU = metric->kind == AHMC_METRIC_DENSE && metric->cholU;
    double *dMinv, *dU, *dEps, *dTh, *dR, *dG, *oTh, *oR, *oG, *oDr, *oLp, *oLk;
    uint32_t* oSt;
    int32_t* oSd;
    auto layout = [&](Carver& c) {
        dMinv = c.take<double>(nMinv, nMinv && !(per_chain_minv && !stage_in));
        dU = c.take<double>((size_t)D * D, hasU);
        dEps = c.take<double>((size_t)N, stage_in);
        dTh = c.take<double>((size_t)ldi * N, stage_in);
        dR = c.take<double>((size_t)ldi * N, stage_in);
        dG = c.take<double>((size_t)ldi * N, stage_in && has_g);
        oTh = c.take<double>((size_t)ldo * N, stage_out);
        oR = c.take<double>((size_t)ldo * N, stage_out);
        oG = c.take<double>((size_t)ldo * N, stage_out);
        oDr = c.take<double>((size_t)ldo * N, stage_out);
        oLp = c.take<double>((size_t)N, stage_out);
        oLk = c.take<double>((size_t)N, stage_out);
        oSt = c.take<uint32_t>((size_t)N, stage_out);
        oSd = c.take<int32_t>((size_t)N, stage_out);
    };
    Carver size;
    layout(size);
    if ((rc = ensure_arena(ctx, size.off))) return rc;
    Carver arena{(char*)ctx->arena.p};
    layout(arena);

    cudaStream_t s_cmp = ctx->stream, s_up = ctx->pipe[0], s_down = ctx->pipe[1];

    // everything is ordered after earlier work on the context stream; shared parameters (re-read by every chain, so
    // always staged) go first on the compute stream itself
    CU(cudaEventRecord(ctx->ev_a, s_cmp));
    if (stage_in) CU(cudaStreamWaitEvent(s_up, ctx->ev_a, 0));
    if (nMinv && !per_chain_minv) CU(cudaMemcpyAsync(dMinv, metric->Minv, nMinv * 8, cudaMemcpyHostToDevice, s_cmp));
    if (hasU) CU(cudaMemcpyAsync(dU, metric->cholU, (size_t)D * D * 8, cudaMemcpyHostToDevice, s_cmp));

    const int n_abs = n_steps < 0 ? -n_steps : n_steps;
    int nl = 0, k = 0;
    for (int64_t c0 = 0; c0 < N; c0 += chunk, ++k) {
        const int64_t n = (c0 + chunk <= N) ? chunk : N - c0;
        if (stage_in) {
            CU(copy_rows(dTh + ldi * c0, z_in->theta + ldi * c0, (size_t)D * 8, (size_t)ldi * 8, (size_t)n, cudaMemcpyHostToDevice, s_up));
            if (eps_chain) CU(cudaMemcpyAsync(dEps + c0, eps_chain + c0, (size_t)n * 8, cudaMemcpyHostToDevice, s_up));
            CU(copy_rows(dR + ldi * c0, z_in->r + ldi * c0, (size_t)D * 8, (size_t)ldi * 8, (size_t)n, cudaMemcpyHostToDevice, s_up));
            if (per_chain_minv)
                CU(cudaMemcpyAsync(dMinv + metric->chain_stride * c0, metric->Minv + metric->chain_stride * c0,
                                   (size_t)metric->chain_stride * n * 8, cudaMemcpyHostToDevice, s_up));
            if (has_g)
                CU(copy_rows(dG + ldi * c0, z_in->lp_gradient + ldi * c0, (size_t)D * 8, (size_t)ldi * 8, (size_t)n, cudaMemcpyHostToDevice, s_up));
            CU(cudaEventRecord(ctx->ev_in[k], s_up));
            CU(cudaStreamWaitEvent(s_cmp, ctx->ev_in[k], 0));
        }
        LeapfrogArgs a{};
        a.model = model_dev(model);
        const double* minv_k = !nMinv ? nullptr
                               : !per_chain_minv ? dMinv
                               : stage_in ? dMinv + metric->chain_stride * c0 : a_minv + metric->chain_stride * c0;
        a.metric = MetricDev{metric->kind, minv_k, per_chain_minv ? metric->chain_stride : 0, hasU ? dU : nullptr};
        a.D = D;
        a.N = n;
        a.eps = eps;
        a.eps_chain = !eps_chain ? nullptr : stage_in ? dEps + c0 : a_eps + c0;
        a.n_steps = n_abs;
        a.fwd = n_steps > 0;
        a.temper_alpha = temper_alpha;
        a.th_in = (stage_in ? dTh : a_th) + ldi * c0;
        a.r_in = (stage_in ? dR : a_r) + ldi * c0;
        a.g_in = !has_g ? nullptr : (stage_in ? dG : a_g) + ldi * c0;
        a.ld_in = ldi;
        a.th_out = (stage_out ? oTh : b_th) + ldo * c0;
        a.r_out = (stage_out ? oR : b_r) + ldo * c0;
        a.g_out = (stage_out ? oG : b_g) + ldo * c0;
        a.dr_out = !z_out->lk_gradient ? nullptr : (stage_out ? oDr : b_dr) + ldo * c0;
        a.lp_out = (stage_out ? oLp : b_lp) + c0;
        a.lk_out = (stage_out ? oLk : b_lk) + c0;
        a.ld_out = ldo;
        a.status = !status ? nullptr : (stage_out ? oSt : b_st) + c0;
        a.steps_done = !steps_done ? nullptr : (stage_out ? oSd : b_sd) + c0;
        a.flags = flags;
        a.resident_blocks_per_sm = occ_cap;
        CU(launch_leapfrog(a, s_cmp, &nl));
        if (stage_out) {
            CU(cudaEventRecord(ctx->ev_k[k], s_cmp));
            CU(cudaStreamWaitEvent(s_down, ctx->ev_k[k], 0));
            const size_t w = (size_t)D * 8, pitch = (size_t)ldo * 8;  // rows d < D only: the caller's padding stays
            CU(copy_rows(z_out->theta + ldo * c0, a.th_out, w, pitch, (size_t)n, cudaMemcpyDeviceToHost, s_down));
            CU(copy_rows(z_out->r + ldo * c0, a.r_out, w, pitch, (size_t)n, cudaMemcpyDeviceToHost, s_down));
            CU(copy_rows(z_out->lp_gradient + ldo * c0, a.g_out, w, pitch, (size_t)n, cudaMemcpyDeviceToHost, s_down));
            if (a.dr_out) CU(copy_rows(z_out->lk_gradient + ldo * c0, a.dr_out, w, pitch, (size_t)n, cudaMemcpyDeviceToHost, s_down));
        }
    }
    ctx->launches += nl;
    if (stage_out) {
        // the per-chain scalars of all chunks go back in one copy each (stream order puts them after the last kernel)
        CU(cudaMemcpyAsync(z_out->lp_value, oLp, (size_t)N * 8, cudaMemcpyDeviceToHost, s_down));
        CU(cudaMemcpyAsync(z_out->lk_value, oLk, (size_t)N * 8, cudaMemcpyDeviceToHost, s_down));
        if (status) CU(cudaMemcpyAsync(status, oSt, (size_t)N * 4, cudaMemcpyDeviceToHost, s_down));
        if (steps_done) CU(cudaMemcpyAsync(steps_done, oSd, (size_t)N * 4, cudaMemcpyDeviceToHost, s_down));
        CU(cudaEventRecord(ctx->ev_down, s_down));
        CU(cudaStreamWaitEvent(s_cmp, ctx->ev_down, 0));
    }
    // host buffers are valid once everything joined into the context stream has retired
    CU(cudaStreamSynchronize(s_cmp));
    {
        char buf[96];
        snprintf(buf, sizeof buf, "up=%s down=%s chunks=%d%s%s", tp.up_direct ? "direct" : "ce1", tp.down_direct ? "direct" : "ce",
                 k, occ_cap ? " occ=1" : "", tune ? (tune->chosen >= 0 ? " (autotuned)" : " (autotune trial)") : "");
        ctx->transport = buf;
    }
    if (tune && trial >= 0) {
        const double ms = since();
        if (tune->calls >= kPipeNCand && ms < tune->best_ms[trial]) tune->best_ms[trial] = ms;
        if (++tune->calls >= kPipeNCand * kRounds) {
            int best = 0;
            for (int c = 1; c < kPipeNCand; ++c)
                if (tune->best_ms[c] < tune->best_ms[best]) best = c;
            tune->chosen = best;
        }
    }
    return AHMC_OK;
}

int ahmc_leapfrog_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                      double eps, const double* eps_chain, int32_t n_steps, double temper_alpha,
                      const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out, uint32_t* status,
                      int32_t* steps_done, uint32_t flags) {
    if (!ctx || !model || !metric) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/model/metric");
    int rc = check_common(ctx, model, metric, D, N, true);
    if (!rc && D > 512 && temper_alpha > 0.0) rc = fail(ctx, AHMC_ERR_UNSUPPORTED, "TemperedLeapfrog at D > 512 is not built");
    if (rc) return rc;
    // z_in: only theta and r are required.  The cached energies are not read, and a NULL z_in->lp_gradient means "not
    // cached": built-in targets recompute dH/dtheta at the start point on the device (bit-identical to the value
    // phasepoint / a previous step produced), which saves a third of the upload of a host-buffer call.
    if ((rc = check_pp(ctx, z_in, D, "z_in", false, N))) return rc;
    if ((rc = check_pp(ctx, z_out, D, "z_out", true, N))) return rc;
    if (N == 0) return AHMC_OK;
    if (!z_in->lp_gradient && model->kind == AHMC_MODEL_CALLBACK)
        return fail(ctx, AHMC_ERR_INVALID, "z_in.lp_gradient is NULL: a callback target needs the cached gradient (call ahmc_phasepoint_f64 first)");
    DeviceGuard g(ctx->device);
    const bool host = flags & AHMC_FLAG_HOST_BUFFERS;
    const int n_abs = n_steps < 0 ? -n_steps : n_steps;
    if (n_abs == 0 && !z_in->lp_gradient)
        return fail(ctx, AHMC_ERR_INVALID, "n_steps == 0 returns z unchanged and needs z_in.lp_gradient");
    if (n_abs == 0) {  // the loop body never runs: z is returned unchanged (integrator.jl:233)
        rc = copy_pp_device(ctx, D, N, z_in, z_out, host ? cudaMemcpyHostToHost : cudaMemcpyDeviceToDevice);
        if (rc) return rc;
        CU(cudaStreamSynchronize(ctx->stream));
        if (host) {
            if (status) memset(status, 0, sizeof(uint32_t) * (size_t)N);
            if (steps_done) memset(steps_done, 0, sizeof(int32_t) * (size_t)N);
        } else {
            if (status) CU(cudaMemsetAsync(status, 0, sizeof(uint32_t) * (size_t)N, ctx->stream));
            if (steps_done) CU(cudaMemsetAsync(steps_done, 0, sizeof(int32_t) * (size_t)N, ctx->stream));
            if (!(flags & AHMC_FLAG_ASYNC)) CU(cudaStreamSynchronize(ctx->stream));
        }
        return AHMC_OK;
    }
    // dense targets / metrics go through the staged lane below, which can pick the tiled kernel
    const bool host_fast = host && !(flags & AHMC_FLAG_COMPAT_BREAK_ALL) && model->kind != AHMC_MODEL_CALLBACK &&
                           model->kind != AHMC_MODEL_DENSE_GAUSS && metric->kind != AHMC_METRIC_DENSE;
    if (host_fast && N >= 256)
        return leapfrog_host_pipelined(ctx, model, metric, D, N, eps, eps_chain, n_steps, temper_alpha, z_in, z_out,
                                       status, steps_done, flags);
    Stager st(ctx, host);
    LeapfrogArgs a{};
    a.model = model_dev(model);
    a.D = D;
    a.N = N;
    a.eps = eps;
    a.n_steps = n_abs;
    a.fwd = n_steps > 0;
    a.temper_alpha = temper_alpha;
    a.lp_in = nullptr;
    a.lk_in = nullptr;
    rc = st.stage([&](Stager& s) {
        stage_metric(s, metric, D, N, &a.metric);
        s.in(eps_chain, (size_t)N, &a.eps_chain);
        stage_pp_in(s, z_in, D, N, a);
        stage_pp_out(s, z_out, D, N, a, &a.dr_out);
        s.out(status, (size_t)N, &a.status);
        s.out(steps_done, (size_t)N, &a.steps_done);
    });
    if (rc) return rc;
    a.flags = flags;
    const bool compat = flags & AHMC_FLAG_COMPAT_BREAK_ALL;
    a.min_break = nullptr;
    a.only_mask = nullptr;
    const Engine e = trajectory_engine(model, a.metric, flags, temper_alpha, a.g_in != nullptr);
    if (e != Engine::Fused) {
        SplitWork w{};
        if (e == Engine::Split && (rc = split_workspace(ctx, D, N, z_out->ld, false, &w))) return rc;
        int nl = 0;
        rc = run_trajectory(ctx, model, e, a, w, compat, &nl);
        ctx->launches += nl;
        if (rc) return rc;
        return finish_call(ctx, st, flags);
    }
    if (compat) {
        const int big = 0x7fffffff;
        CU(cudaMemcpyAsync(ctx->d_min_break, &big, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        a.min_break = ctx->d_min_break;
    }
    int nl = 0;
    CU(launch_leapfrog(a, ctx->stream, &nl));
    if (compat) {
        // reference quirk Q1: `isfinite(z)` is all(...) over every chain, so the first non-finite step
        // stops ALL chains.  Re-run everyone for exactly that many steps (inputs are untouched unless
        // the caller aliased z_out = z_in, which COMPAT mode therefore forbids).
        int mb = 0;
        CU(cudaMemcpyAsync(&mb, ctx->d_min_break, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        if (mb < n_abs) {
            if (!host && z_in->theta == z_out->theta)
                return fail(ctx, AHMC_ERR_INVALID, "COMPAT_BREAK_ALL cannot re-run an in-place call (z_out aliases z_in)");
            a.n_steps = mb;
            a.min_break = nullptr;
            a.flags |= AHMC_FLAG_EXACT_CHECKS;
            CU(launch_leapfrog(a, ctx->stream, &nl));
        }
    }
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

// ---------------------------------------------------------------------------------------------- rand_momentum
int ahmc_rand_momentum_f64(ahmc_ctx* ctx, const ahmc_metric* metric, int32_t D, int64_t N, const ahmc_rng* rng,
                           double* r, int64_t ld, uint32_t flags) {
    if (!ctx || !metric || !rng || !r) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/metric/rng/r");
    int rc = check_common(ctx, nullptr, metric, D, N, true);
    if (!rc && !rng->normal_tape) rc = check_philox_d(ctx, D);
    if (!rc && !rng->normal_tape) rc = check_philox_offset(ctx, rng->offset, 1);
    if (rc) return rc;
    if (ld < D) return fail(ctx, AHMC_ERR_INVALID, "ld < D");
    if (metric->kind == AHMC_METRIC_DENSE && !metric->cholU)
        return fail(ctx, AHMC_ERR_INVALID, "Dense metric needs cholU for rand_momentum (metric.jl:311-320)");
    if (N == 0) return AHMC_OK;
    DeviceGuard g(ctx->device);
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    MomentumArgs a{};
    a.D = D;
    a.N = N;
    a.seed = rng->seed;
    a.offset = rng->offset;
    a.ld = ld;
    rc = st.stage([&](Stager& s) {
        stage_metric(s, metric, D, N, &a.metric);
        s.in(rng->normal_tape, (size_t)D * N, &a.normal_tape);
        s.out2d(r, D, ld, N, &a.r);
    });
    if (rc) return rc;
    int nl = 0;
    CU(launch_rand_momentum(a, ctx->stream, &nl));
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

// ---------------------------------------------------------------------------------------------- transitions
// the statistics a sampler writes: max_hamiltonian_energy_error NUTS only (`max_dH`), tree_depth NUTS and the multinomial
// draw's offset (`depth`).  A field it does not write is not staged, so a host-buffer call leaves the caller's array as
// it was, as a device-pointer call does
static void stage_stats(Stager& st, const ahmc_stats* s, int64_t N, StatsDev* d, bool max_dH, bool depth) {
    memset(d, 0, sizeof *d);
    if (!s) return;
    st.out(s->n_steps, (size_t)N, &d->n_steps);
    st.out(s->is_accept, (size_t)N, &d->is_accept);
    st.out(s->acceptance_rate, (size_t)N, &d->acceptance_rate);
    st.out(s->log_density, (size_t)N, &d->log_density);
    st.out(s->hamiltonian_energy, (size_t)N, &d->hamiltonian_energy);
    st.out(s->hamiltonian_energy_error, (size_t)N, &d->hamiltonian_energy_error);
    if (max_dH) st.out(s->max_hamiltonian_energy_error, (size_t)N, &d->max_hamiltonian_energy_error);
    if (depth) st.out(s->tree_depth, (size_t)N, &d->tree_depth);
    st.out(s->numerical_error, (size_t)N, &d->numerical_error);
}

static void stage_rng(Stager& st, const ahmc_rng* r, int32_t D, int64_t N, bool nuts, RngDev* d) {
    d->seed = r->seed;
    d->offset = r->offset;
    d->partial_alpha = r->partial_refresh_alpha;
    d->temper_alpha = r->temper_alpha > 0.0 ? r->temper_alpha : 0.0;
    d->exp_stride = nuts ? r->exp_stride : 1;
    d->dir_stride = r->dir_stride;
    st.in(r->normal_tape, (size_t)D * N, &d->normal_tape);
    st.in(r->exp_tape, (size_t)(nuts ? r->exp_stride : 1) * N, &d->exp_tape);
    st.in(nuts ? r->dir_tape : (const uint8_t*)nullptr, (size_t)r->dir_stride * N, &d->dir_tape);
}

// the momentum refresh (partial_refresh_alpha) and integrator (temper_alpha) a transition's rng asks for
static int check_refresh_rng(ahmc_ctx* ctx, const ahmc_rng* rng) {
    if (!(rng->partial_refresh_alpha > -1.0 && rng->partial_refresh_alpha < 1.0))
        return fail(ctx, AHMC_ERR_INVALID, "partial_refresh_alpha must be in (-1, 1)");
    if (!(rng->temper_alpha >= 0.0) || std::isinf(rng->temper_alpha))
        return fail(ctx, AHMC_ERR_INVALID, "temper_alpha must be 0 (plain Leapfrog) or a finite alpha > 0 (TemperedLeapfrog)");
    return AHMC_OK;
}
// what every transition needs of its metric and output phase point
static int check_transition_io(ahmc_ctx* ctx, const ahmc_metric* metric, const ahmc_phasepoint* z_out, uint32_t flags) {
    if (metric->kind == AHMC_METRIC_DENSE && !metric->cholU && !(flags & AHMC_FLAG_NO_REFRESH))
        return fail(ctx, AHMC_ERR_INVALID, "Dense metric needs cholU for the momentum refresh (metric.jl:311-320)");
    if (z_out->lk_gradient)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "transition entry points do not emit lk_gradient; call ahmc_phasepoint_f64 if needed");
    return AHMC_OK;
}

// ---- in-launch adaptation (ahmc_nuts_adapt_sample_f64, ahmc_hmc_adapt_sample_f64): the cfg checks after the metric /
// sampler family checks of each entry point, the staging of the adaptors' buffers, and the per-chain workspace
// The metric / estimator pairs an adaptive launch accepts, checked before everything else of the cfg: the diagonal
// estimators adapt a Diag metric; a Dense metric (shared or per chain, as the starting point) adapts its step size only or
// runs WelfordCov, on built-in and run-time compiled targets alike (GLM targets adapt in their general form).
static int check_adapt_metric(ahmc_ctx* ctx, const ahmc_adapt_cfg* cfg, const ahmc_metric* metric) {
    if (cfg->adapt_metric == AHMC_ADAPT_WELFORD_COV && metric->kind != AHMC_METRIC_DENSE)
        return fail(ctx, AHMC_ERR_INVALID, "cfg.adapt_metric = AHMC_ADAPT_WELFORD_COV adapts a dense M^-1: it needs the Dense metric");
    if (metric->kind == AHMC_METRIC_DENSE) {
        if (cfg->adapt_metric != AHMC_ADAPT_STEPSIZE && cfg->adapt_metric != AHMC_ADAPT_WELFORD_COV)
            return fail(ctx, AHMC_ERR_UNSUPPORTED, "in-launch adaptation of a Dense metric: AHMC_ADAPT_STEPSIZE or AHMC_ADAPT_WELFORD_COV "
                                                   "(WelfordVar / NutpieVar estimate a diagonal M^-1)");
        // the launch copies the starting factor into the chain's cholU_chain row (and reads the chain's row for every
        // momentum refresh), so it is required even with AHMC_FLAG_NO_REFRESH
        if (!metric->cholU)
            return fail(ctx, AHMC_ERR_INVALID, "in-launch adaptation with a Dense metric needs its cholU (metric.jl:104-109)");
        return AHMC_OK;
    }
    if (metric->kind != AHMC_METRIC_DIAG)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "in-launch adaptation needs the Diag metric (per-chain diagonal M^-1) or the Dense metric");
    return AHMC_OK;
}
static int check_adapt_cfg(ahmc_ctx* ctx, const ahmc_adapt_cfg* cfg, const ahmc_rng* rng, int32_t n_transitions) {
    if (rng->normal_tape || rng->exp_tape || rng->dir_tape)
        return fail(ctx, AHMC_ERR_INVALID, "in-launch adaptation draws from the Philox streams (no tapes)");
    if (cfg->n_adapts < 0 || cfg->n_adapts > n_transitions)
        return fail(ctx, AHMC_ERR_INVALID, "need 0 <= n_adapts <= n_transitions");
    if (!cfg->eps_chain) return fail(ctx, AHMC_ERR_INVALID, "cfg.eps_chain (N, in/out) is required");
    if (cfg->adapt_metric < AHMC_ADAPT_STEPSIZE || cfg->adapt_metric > AHMC_ADAPT_WELFORD_COV)
        return fail(ctx, AHMC_ERR_INVALID, "cfg.adapt_metric must be AHMC_ADAPT_STEPSIZE (0), AHMC_ADAPT_WELFORD (1), AHMC_ADAPT_NUTPIE (2) "
                                           "or AHMC_ADAPT_WELFORD_COV (3)");
    if (cfg->adapt_metric && !cfg->Minv_chain)
        return fail(ctx, AHMC_ERR_INVALID, "cfg.Minv_chain (N x D, out; N x D x D with WelfordCov) is required with adapt_metric");
    if (cfg->adapt_metric == AHMC_ADAPT_WELFORD_COV && !cfg->cholU_chain)
        return fail(ctx, AHMC_ERR_INVALID, "cfg.cholU_chain (N x D x D, out) is required with AHMC_ADAPT_WELFORD_COV");
    if (cfg->init_buffer < 0 || cfg->term_buffer < 0 || cfg->window_size < 1)
        return fail(ctx, AHMC_ERR_INVALID, "need init_buffer >= 0, term_buffer >= 0, window_size >= 1");
    if (!(cfg->gamma > 0.0) || !(cfg->t0 >= 0.0) || !(cfg->delta > 0.0 && cfg->delta < 1.0))
        return fail(ctx, AHMC_ERR_INVALID, "need gamma > 0, t0 >= 0, 0 < delta < 1");
    return AHMC_OK;
}
// in-launch adaptation: the metric / estimator pair, then `refusal` (why this sampler configuration cannot adapt inside
// its launch, or nullptr), then the cfg
static int check_adapt(ahmc_ctx* ctx, const ahmc_metric* metric, const ahmc_adapt_cfg* cfg,
                       const ahmc_rng* rng, int32_t n_transitions, const char* refusal) {
    int rc = check_adapt_metric(ctx, cfg, metric);
    if (rc) return rc;
    if (refusal) return fail(ctx, AHMC_ERR_UNSUPPORTED, "%s", refusal);
    return check_adapt_cfg(ctx, cfg, rng, n_transitions);
}
// fills `ad` with the schedule and constants of the adaptors
static int adapt_schedule(ahmc_ctx* ctx, const ahmc_adapt_cfg* cfg, AdaptDev* ad) {
    ad->enabled = 1;
    ad->n_adapts = cfg->n_adapts;
    ad->delta = cfg->delta;
    ad->gamma = cfg->gamma;
    ad->t0 = cfg->t0;
    ad->kappa = cfg->kappa;
    ad->adapt_metric = cfg->adapt_metric;
    ad->n_min = cfg->n_min > 0 ? cfg->n_min : 10;
    if (!stan_window_schedule(*ad, cfg->init_buffer, cfg->term_buffer, cfg->window_size, cfg->n_adapts))
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "the window schedule (stan_adaptor.jl:13-50) needs more than %d splits",
                    (int)(sizeof(ad->splits) / sizeof(ad->splits[0])));
    return AHMC_OK;
}
// stages the adaptors' eps / M^-1 / trace buffers into `ad`; *eps_chain = the per-chain step sizes the kernel reads
static void stage_adapt(Stager& st, const ahmc_metric* metric, const ahmc_adapt_cfg* cfg, int32_t D, int64_t N,
                        int32_t n_transitions, AdaptDev* ad, const double** eps_chain) {
    st.inout(cfg->eps_chain, (size_t)N, &ad->eps);
    *eps_chain = ad->eps;
    ad->minv = ad->cholU = nullptr;
    if (metric->kind == AHMC_METRIC_DENSE) {  // the chain's M^-1 / factor rows: both or neither (step size only)
        if (cfg->Minv_chain && cfg->cholU_chain) {
            st.out(cfg->Minv_chain, (size_t)N * D * D, &ad->minv);
            st.out(cfg->cholU_chain, (size_t)N * D * D, &ad->cholU);
        }
    } else {
        st.out(cfg->Minv_chain, (size_t)N * D, &ad->minv);
    }
    st.out(cfg->eps_trace, (size_t)N * n_transitions, &ad->eps_trace);
}
// the context's per-chain workspace (NUTS trees, in-launch adaptors' estimators, D > 512 start points): at least `need` bytes
static int chain_workspace(ahmc_ctx* ctx, size_t need, double** out) {
    int rc = ensure(ctx, ctx->chain_ws, need, "the NUTS workspace");
    *out = (double*)ctx->chain_ws.p;
    return rc;
}
// adapt_summary's workspace (K5): [completion counter (as 2 doubles)] [block partials], for `blocks` blocks.  The counter
// starts at zero and the kernel leaves it at zero, so it is cleared only when the buffer is new.
static int summary_workspace(ahmc_ctx* ctx, int32_t D, int blocks, unsigned** counter, double** partial) {
    const size_t need = ((size_t)blocks * (D + 1) + 2) * sizeof(double);
    const bool grows = need > ctx->summary_ws.bytes;
    int rc = ensure(ctx, ctx->summary_ws, need, "the adaptor workspace");
    if (rc) return rc;
    if (grows) CU(cudaMemsetAsync(ctx->summary_ws.p, 0, need, ctx->stream));
    *counter = (unsigned*)ctx->summary_ws.p;
    *partial = (double*)ctx->summary_ws.p + 2;
    return AHMC_OK;
}

static int hmc_impl(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                    double eps, const double* eps_chain, int32_t n_steps, int32_t n_transitions, const ahmc_rng* rng,
                    const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out, double* draws, const ahmc_stats* stats,
                    uint32_t flags, const ahmc_adapt_cfg* cfg = nullptr) {
    if (!ctx || !model || !metric || !rng) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/model/metric/rng");
    if (n_transitions < 1) return fail(ctx, AHMC_ERR_INVALID, "n_transitions must be >= 1");
    int rc;
    if (cfg &&
        (rc = check_adapt(ctx, metric, cfg, rng, n_transitions,
                          model->kind == AHMC_MODEL_CALLBACK
                              ? "in-launch adaptation needs a device-resident target: callback (split-step) models cannot run inside one launch; express the target as CUDA source (ahmc_model_create_user)"
                              : nullptr)))
        return rc;
    if (n_transitions > 1 && (rng->normal_tape || rng->exp_tape))
        return fail(ctx, AHMC_ERR_INVALID, "random tapes describe ONE transition; multi-transition sampling uses the Philox streams");
    if (n_transitions > 1 && model->kind == AHMC_MODEL_CALLBACK)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "multi-transition sampling needs a device-resident target");
    if (rng->partial_refresh_alpha != 0.0 && model->kind == AHMC_MODEL_CALLBACK)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "partial momentum refreshment is not wired into the split-step path");
    if ((rc = check_refresh_rng(ctx, rng))) return rc;
    rc = check_common(ctx, model, metric, D, N, true);
    if (!rc && D > 512 && rng->temper_alpha > 0.0) rc = fail(ctx, AHMC_ERR_UNSUPPORTED, "TemperedLeapfrog at D > 512 is not built");
    if (!rc && D > 512 && !(flags & AHMC_FLAG_NO_REFRESH) && !rng->normal_tape) rc = check_philox_d(ctx, D);
    if (!rc && (!rng->exp_tape || (!(flags & AHMC_FLAG_NO_REFRESH) && !rng->normal_tape)))
        rc = check_philox_offset(ctx, rng->offset, n_transitions);
    if (rc) return rc;
    if ((rc = check_pp(ctx, z_in, D, "z_in", true, N))) return rc;
    if ((rc = check_pp(ctx, z_out, D, "z_out", true, N))) return rc;
    if (n_steps < 1) return fail(ctx, AHMC_ERR_INVALID, "n_steps must be >= 1 (nsteps(tau) = max(1, ...), trajectory.jl:240-243)");
    if (flags & AHMC_FLAG_COMPAT_BREAK_ALL)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "COMPAT_BREAK_ALL is only available on ahmc_leapfrog_f64");
    if ((rc = check_transition_io(ctx, metric, z_out, flags))) return rc;
    if (N == 0) return AHMC_OK;
    HmcArgs h{};
    if (cfg && (rc = adapt_schedule(ctx, cfg, &h.ad))) return rc;
    DeviceGuard g(ctx->device);
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    LeapfrogArgs& a = h.lf;
    a.model = model_dev(model);
    a.D = D;
    a.N = N;
    a.eps = eps;
    a.n_steps = n_steps;
    a.fwd = 1;
    a.temper_alpha = 0.0;
    a.dr_out = nullptr;
    a.flags = flags;
    h.n_transitions = n_transitions;
    h.refresh = (flags & AHMC_FLAG_NO_REFRESH) ? 0 : 1;
    rc = st.stage([&](Stager& s) {
        stage_metric(s, metric, D, N, &a.metric);
        if (cfg) stage_adapt(s, metric, cfg, D, N, n_transitions, &h.ad, &a.eps_chain);
        else s.in(eps_chain, (size_t)N, &a.eps_chain);
        stage_pp_in(s, z_in, D, N, a, &a.lp_in);
        stage_pp_out(s, z_out, D, N, a);
        stage_rng(s, rng, D, N, false, &h.rng);
        stage_stats(s, stats, N * n_transitions, &h.st, false, false);
        s.out(draws, (size_t)D * N * n_transitions, &h.draws);
    });
    if (rc) return rc;
    int nl = 0;
    Engine e = trajectory_engine(model, a.metric, flags, h.rng.temper_alpha, true);
    // K4 and K6 run a transition in stages (sequenced_transitions), whose momentum refresh is a full one; in-launch
    // adaptation is built into hmc_kernel only
    if ((e == Engine::Dense || e == Engine::Glm) && (cfg || h.rng.partial_alpha != 0.0)) e = Engine::Fused;
    // K4 serves one transition into a separate z_out, without draws.  Sampling launches (several transitions, draws, or
    // z_out = z_in to chain calls in place) stay on hmc_kernel, so that a run's draws do not depend on how it is split
    // into launches: K4's DMMA products round differently from hmc_kernel's
    if (e == Engine::Dense && (n_transitions > 1 || a.th_out == a.th_in || draws)) e = Engine::Fused;
    if (e != Engine::Fused) {
        rc = sequenced_transitions(ctx, model, e, h, &nl);
        if (rc) return rc;
        ctx->launches += nl;
        return finish_call(ctx, st, flags);
    }
    if (cfg || D > 512) {  // the adaptors' estimator state: chain_adapt_doubles per chain; at D > 512 also the
                           // transition's start point, kBigHmcVectors D-vectors per chain ahead of it (ahmc_bigd_hmc.cu)
        h.scratch_stride = (long long)(D > 512 ? kBigHmcVectors : 0) * D + (cfg ? chain_adapt_doubles(cfg->adapt_metric, D) : 0);
        if ((rc = chain_workspace(ctx, (size_t)h.scratch_stride * (size_t)N * sizeof(double), &h.scratch))) return rc;
    }
    CU(launch_hmc(h, ctx->stream, &nl));
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

static int nuts_impl(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                     double eps, const double* eps_chain, int32_t max_depth, double delta_max, int32_t n_transitions,
                     const ahmc_rng* rng, const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out, double* draws,
                     const ahmc_stats* stats, uint32_t flags, const ahmc_adapt_cfg* cfg = nullptr) {
    if (!ctx || !model || !metric || !rng) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/model/metric/rng");
    if (n_transitions < 1) return fail(ctx, AHMC_ERR_INVALID, "n_transitions must be >= 1");
    int rc;
    if (cfg && (rc = check_adapt(ctx, metric, cfg, rng, n_transitions,
                                 (flags & (AHMC_FLAG_NUTS_SLICE_TS | AHMC_FLAG_NUTS_CLASSIC | AHMC_FLAG_NUTS_STRICT))
                                     ? "in-launch adaptation is built for MultinomialTS + GeneralisedNoUTurn"
                                     : nullptr)))
        return rc;
    if (n_transitions > 1 && (rng->normal_tape || rng->exp_tape || rng->dir_tape))
        return fail(ctx, AHMC_ERR_INVALID, "random tapes describe ONE transition; multi-transition sampling uses the Philox streams");
    if ((rc = check_refresh_rng(ctx, rng))) return rc;
    // (every NUTS launch: a tree that outgrows its exponential or direction tape continues on the Philox streams)
    if ((rc = check_philox_offset(ctx, rng->offset, n_transitions))) return rc;
    if ((rc = check_common(ctx, model, metric, D, N))) return rc;
    if ((rc = check_pp(ctx, z_in, D, "z_in", true, N))) return rc;
    if ((rc = check_pp(ctx, z_out, D, "z_out", true, N))) return rc;
    if (max_depth < 0 || max_depth > 20) return fail(ctx, AHMC_ERR_INVALID, "max_depth must be in 0..20");
    if (cfg && max_depth == 0)  // no leaf is ever built: acceptance_rate = 0/0 (as in the reference) would poison dual averaging
        return fail(ctx, AHMC_ERR_INVALID, "in-launch adaptation needs max_depth >= 1");
    if ((flags & AHMC_FLAG_NUTS_CLASSIC) && (flags & AHMC_FLAG_NUTS_STRICT))
        return fail(ctx, AHMC_ERR_INVALID, "AHMC_FLAG_NUTS_CLASSIC and AHMC_FLAG_NUTS_STRICT are mutually exclusive");
    if (model->kind == AHMC_MODEL_CALLBACK)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "NUTS needs a device-resident target: callback (split-step) models are supported by ahmc_leapfrog_f64 / ahmc_hmc_transition_f64 / ahmc_phasepoint_f64 only; express the target as CUDA source (ahmc_model_create_user) to run NUTS on it");
    if (model->kind == AHMC_MODEL_USER && (flags & (AHMC_FLAG_NUTS_SLICE_TS | AHMC_FLAG_NUTS_CLASSIC | AHMC_FLAG_NUTS_STRICT)))
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "run-time compiled targets: MultinomialTS + GeneralisedNoUTurn only");
    if ((rc = check_transition_io(ctx, metric, z_out, flags))) return rc;
    if (rng->exp_tape && rng->exp_stride < 1) return fail(ctx, AHMC_ERR_INVALID, "exp_tape needs exp_stride >= 1");
    if (rng->dir_tape && rng->dir_stride < max_depth) return fail(ctx, AHMC_ERR_INVALID, "dir_tape needs dir_stride >= max_depth");
    if (N == 0) return AHMC_OK;
    NutsArgs a{};
    if (cfg && (rc = adapt_schedule(ctx, cfg, &a.ad))) return rc;
    DeviceGuard g(ctx->device);
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    a.model = model_dev(model);
    a.D = D;
    a.N = N;
    a.eps = eps;
    a.max_depth = max_depth;
    a.delta_max = delta_max;
    a.sampler = (flags & AHMC_FLAG_NUTS_SLICE_TS) ? 1 : 0;
    a.criterion = (flags & AHMC_FLAG_NUTS_STRICT) ? 2 : (flags & AHMC_FLAG_NUTS_CLASSIC) ? 1 : 0;
    a.refresh = (flags & AHMC_FLAG_NO_REFRESH) ? 0 : 1;
    a.dr_out = nullptr;
    a.n_transitions = n_transitions;
    rc = st.stage([&](Stager& s) {
        stage_metric(s, metric, D, N, &a.metric);
        if (cfg) stage_adapt(s, metric, cfg, D, N, n_transitions, &a.ad, &a.eps_chain);
        else s.in(eps_chain, (size_t)N, &a.eps_chain);
        stage_pp_in(s, z_in, D, N, a, &a.lp_in);
        stage_pp_out(s, z_out, D, N, a);
        stage_rng(s, rng, D, N, true, &a.rng);
        stage_stats(s, stats, N * n_transitions, &a.st, true, true);
        s.out(draws, (size_t)D * N * n_transitions, &a.draws);
    });
    if (rc) return rc;
    if (a.metric.kind == AHMC_METRIC_DENSE && a.metric.chain_stride == 0 && !cfg && D > 16 && D <= 512) {
        // the cooperative form streams Minv / cholU in chunks of columns: hand it copies whose columns are padded to the
        // shared-memory leading dimension, so that a chunk is one bulk copy (two small kernels per call, on the stream).
        // (A per-chain Dense metric, and the Dense adaptive form, run warp per chain: no shared matrix to pad.)
        const size_t per = coop_padded_doubles(D);
        if ((rc = ensure(ctx, ctx->coop_ws, 2 * per * sizeof(double), "the column-padded metric"))) return rc;
        double* coop = (double*)ctx->coop_ws.p;
        CU(launch_pad_columns(a.metric.Minv, D, coop, ctx->stream));
        a.metric.Minv_coop = coop;
        int n_prep = 1;
        if (a.metric.cholU) {
            CU(launch_pad_columns(a.metric.cholU, D, coop + per, ctx->stream));
            a.metric.cholU_coop = coop + per;
            ++n_prep;
        }
        ctx->launches += n_prep;
    }
    // per-chain tree workspace
    a.scratch_stride = nuts_scratch_doubles_per_chain(D, max_depth, cfg ? chain_adapt_doubles(cfg->adapt_metric, D) : 0);
    if ((rc = chain_workspace(ctx, (size_t)a.scratch_stride * (size_t)N * sizeof(double), &a.scratch))) return rc;
    int nl = 0;
    CU(launch_nuts(a, ctx->stream, &nl));
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

int ahmc_leapfrog_trajectory_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D,
                                 int64_t N, double eps, const double* eps_chain, int32_t n_steps, double temper_alpha,
                                 const ahmc_phasepoint* z_in, const ahmc_phasepoint* traj, int64_t step_stride,
                                 int32_t* steps_done, uint32_t flags) {
    if (!ctx || !model || !metric) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/model/metric");
    int rc = check_common(ctx, model, metric, D, N);
    if (rc) return rc;
    if ((rc = check_pp(ctx, z_in, D, "z_in", true, N))) return rc;
    const int n_abs = n_steps < 0 ? -n_steps : n_steps;
    if (n_abs == 0 || N == 0) return AHMC_OK;  // res = Vector{P}(undef, 0)
    if ((rc = check_pp(ctx, traj, D, "traj", true, N))) return rc;
    if (step_stride < traj->ld * N) return fail(ctx, AHMC_ERR_INVALID, "step_stride must be >= ld*N");
    if (model->kind == AHMC_MODEL_CALLBACK || model->kind == AHMC_MODEL_USER)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "full_trajectory: built-in targets only (callback / run-time compiled targets: loop over ahmc_leapfrog_f64)");
    DeviceGuard g(ctx->device);
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    TrajArgs a{};
    a.model = model_dev(model);
    a.D = D; a.N = N; a.eps = eps;
    a.n_steps = n_abs; a.fwd = n_steps > 0; a.temper_alpha = temper_alpha;
    a.step_stride = step_stride;
    rc = st.stage([&](Stager& s) {
        stage_metric(s, metric, D, N, &a.metric);
        s.in(eps_chain, (size_t)N, &a.eps_chain);
        stage_pp_in(s, z_in, D, N, a);
        stage_pp_out(s, traj, D, N, a, &a.dr_out, n_abs, step_stride);
        s.out(steps_done, (size_t)N, &a.steps_done);
    });
    if (rc) return rc;
    int nl = 0;
    CU(launch_trajectory(a, ctx->stream, &nl));
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

int ahmc_hmc_multinomial_transition_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D,
                                        int64_t N, double eps, const double* eps_chain, int32_t n_steps,
                                        int32_t n_steps_fwd, const ahmc_rng* rng, const ahmc_phasepoint* z_in,
                                        const ahmc_phasepoint* z_out, const ahmc_stats* stats, uint32_t flags) {
    if (!ctx || !model || !metric || !rng) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/model/metric/rng");
    int rc = check_common(ctx, model, metric, D, N);
    if (rc) return rc;
    if ((rc = check_pp(ctx, z_in, D, "z_in", true, N))) return rc;
    if ((rc = check_pp(ctx, z_out, D, "z_out", true, N))) return rc;
    if (n_steps < 1 || n_steps_fwd < 0 || n_steps_fwd > n_steps)
        return fail(ctx, AHMC_ERR_INVALID, "need n_steps >= 1 and 0 <= n_steps_fwd <= n_steps (rand(0:n_steps), trajectory.jl:373)");
    if (model->kind == AHMC_MODEL_CALLBACK || model->kind == AHMC_MODEL_USER)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "MultinomialTS static transitions: built-in targets only");
    if ((rc = check_transition_io(ctx, metric, z_out, flags))) return rc;
    if ((rc = check_refresh_rng(ctx, rng))) return rc;
    if ((!rng->exp_tape || (!(flags & AHMC_FLAG_NO_REFRESH) && !rng->normal_tape)) && (rc = check_philox_offset(ctx, rng->offset, 1)))
        return rc;
    if (N == 0) return AHMC_OK;
    DeviceGuard g(ctx->device);
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    MultinomialArgs a{};
    a.model = model_dev(model);
    a.D = D; a.N = N; a.eps = eps;
    a.n_steps = n_steps; a.n_fwd = n_steps_fwd;
    a.refresh = (flags & AHMC_FLAG_NO_REFRESH) ? 0 : 1;
    rc = st.stage([&](Stager& s) {
        stage_metric(s, metric, D, N, &a.metric);
        s.in(eps_chain, (size_t)N, &a.eps_chain);
        stage_pp_in(s, z_in, D, N, a, &a.lp_in);
        stage_pp_out(s, z_out, D, N, a);
        stage_rng(s, rng, D, N, false, &a.rng);
        stage_stats(s, stats, N, &a.st, false, true);
    });
    if (rc) return rc;
    if ((rc = ensure(ctx, ctx->energy_ws, (size_t)(n_steps + 1) * (size_t)N * sizeof(double), "the multinomial energy tape")))
        return rc;
    a.energies = (double*)ctx->energy_ws.p;
    int nl = 0;
    CU(launch_multinomial(a, ctx->stream, &nl));
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

int ahmc_hmc_transition_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                            double eps, const double* eps_chain, int32_t n_steps, const ahmc_rng* rng,
                            const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out, const ahmc_stats* stats,
                            uint32_t flags) {
    return hmc_impl(ctx, model, metric, D, N, eps, eps_chain, n_steps, 1, rng, z_in, z_out, nullptr, stats, flags);
}

int ahmc_nuts_transition_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                             double eps, const double* eps_chain, int32_t max_depth, double delta_max,
                             const ahmc_rng* rng, const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out,
                             const ahmc_stats* stats, uint32_t flags) {
    return nuts_impl(ctx, model, metric, D, N, eps, eps_chain, max_depth, delta_max, 1, rng, z_in, z_out, nullptr, stats,
                     flags);
}

int ahmc_hmc_sample_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                        double eps, const double* eps_chain, int32_t n_steps, int32_t n_transitions, const ahmc_rng* rng,
                        const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out, double* draws,
                        const ahmc_stats* stats, uint32_t flags) {
    return hmc_impl(ctx, model, metric, D, N, eps, eps_chain, n_steps, n_transitions, rng, z_in, z_out, draws, stats, flags);
}

int ahmc_nuts_sample_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                         double eps, const double* eps_chain, int32_t max_depth, double delta_max, int32_t n_transitions,
                         const ahmc_rng* rng, const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out, double* draws,
                         const ahmc_stats* stats, uint32_t flags) {
    return nuts_impl(ctx, model, metric, D, N, eps, eps_chain, max_depth, delta_max, n_transitions, rng, z_in, z_out,
                     draws, stats, flags);
}

int ahmc_nuts_adapt_sample_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                               int32_t max_depth, double delta_max, int32_t n_transitions, const ahmc_adapt_cfg* cfg,
                               const ahmc_rng* rng, const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out,
                               double* draws, const ahmc_stats* stats, uint32_t flags) {
    if (!cfg) return fail(ctx, AHMC_ERR_INVALID, "NULL cfg");
    return nuts_impl(ctx, model, metric, D, N, 0.0, nullptr, max_depth, delta_max, n_transitions, rng, z_in, z_out, draws,
                     stats, flags, cfg);
}

int ahmc_hmc_adapt_sample_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                              int32_t n_steps, int32_t n_transitions, const ahmc_adapt_cfg* cfg, const ahmc_rng* rng,
                              const ahmc_phasepoint* z_in, const ahmc_phasepoint* z_out, double* draws,
                              const ahmc_stats* stats, uint32_t flags) {
    if (!cfg) return fail(ctx, AHMC_ERR_INVALID, "NULL cfg");
    return hmc_impl(ctx, model, metric, D, N, 0.0, nullptr, n_steps, n_transitions, rng, z_in, z_out, draws, stats, flags, cfg);
}

// ---------------------------------------------------------------------------------------------- adaptor stats
int ahmc_adapt_summary_f64(ahmc_ctx* ctx, int32_t D, int64_t N, const double* theta, int64_t ld,
                           const double* acceptance_rate, double* out, uint32_t flags) {
    if (!ctx || !theta || !out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/theta/out");
    if (D < 1 || N < 1 || ld < D) return fail(ctx, AHMC_ERR_INVALID, "need D >= 1, N >= 1, ld >= D");
    DeviceGuard g(ctx->device);
    const int blocks = (int)(N < ctx->sm_count ? N : ctx->sm_count);
    unsigned* counter;
    double* partial;
    int rc = summary_workspace(ctx, D, blocks, &counter, &partial);
    if (rc) return rc;
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    const double *d_theta, *d_alpha;
    double* d_out;
    rc = st.stage([&](Stager& s) {
        s.in2d(theta, D, ld, N, &d_theta);
        s.in(acceptance_rate, (size_t)N, &d_alpha);
        s.out(out, (size_t)(2 + 2 * D), &d_out);
    });
    if (rc) return rc;
    int nl = 0;
    CU(launch_adapt_summary(D, N, d_theta, ld, d_alpha, d_out, partial, counter, blocks, ctx->stream, &nl));
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

int ahmc_adapt_cov_f64(ahmc_ctx* ctx, int32_t D, int64_t N, const double* theta, int64_t ld, const double* mean,
                       double* out, uint32_t flags) {
    if (!ctx || !theta || !mean || !out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/theta/mean/out");
    if (D < 1 || N < 1 || ld < D) return fail(ctx, AHMC_ERR_INVALID, "need D >= 1, N >= 1, ld >= D");
    DeviceGuard g(ctx->device);
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    const double *d_theta, *d_mean;
    double* d_out;
    int rc = st.stage([&](Stager& s) {
        s.in2d(theta, D, ld, N, &d_theta);
        s.in(mean, (size_t)D, &d_mean);
        s.out(out, (size_t)D * D, &d_out);
    });
    if (rc) return rc;
    int nl = 0;
    CU(launch_adapt_cov(D, N, d_theta, ld, d_mean, d_out, ctx->stream, &nl));
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

int ahmc_find_good_stepsize_f64(ahmc_ctx* ctx, const ahmc_model* model, const ahmc_metric* metric, int32_t D, int64_t N,
                                const ahmc_phasepoint* z, const ahmc_rng* rng, double initial_step_size, int32_t max_n_iters,
                                double* eps_out, double* r_out, uint32_t flags) {
    if (!ctx || !model || !metric || !rng || !eps_out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/model/metric/rng/eps_out");
    int rc = check_common(ctx, model, metric, D, N, true);
    if (!rc && D > 512 && !rng->normal_tape) rc = check_philox_d(ctx, D);
    if (!rc && !rng->normal_tape) rc = check_philox_offset(ctx, rng->offset, 1);
    if (rc) return rc;
    if (!z || (N > 0 && (!z->theta || !z->lp_value || !z->lp_gradient)))
        return fail(ctx, AHMC_ERR_INVALID, "z.theta / lp_value / lp_gradient is NULL (call ahmc_phasepoint_f64 first)");
    if (N > 0 && z->ld < D) return fail(ctx, AHMC_ERR_INVALID, "z.ld < D");
    if (!(initial_step_size > 0.0) || max_n_iters < 0) return fail(ctx, AHMC_ERR_INVALID, "need initial_step_size > 0, max_n_iters >= 0");
    if (model->kind == AHMC_MODEL_CALLBACK)
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "find_good_stepsize in one launch needs the gradient inside the kernel (built-in targets)");
    if (N == 0) return AHMC_OK;
    DeviceGuard g(ctx->device);
    Stager st(ctx, flags & AHMC_FLAG_HOST_BUFFERS);
    FindEpsArgs a{};
    a.model = model_dev(model);
    a.D = D;
    a.N = N;
    a.ld = z->ld;
    a.seed = rng->seed;
    a.offset = rng->offset;
    a.eps0 = initial_step_size;
    a.max_iters = max_n_iters;
    rc = st.stage([&](Stager& s) {
        stage_metric(s, metric, D, N, &a.metric);
        s.in2d((const double*)z->theta, D, z->ld, N, &a.th);
        s.in2d((const double*)z->lp_gradient, D, z->ld, N, &a.g);
        s.in((const double*)z->lp_value, (size_t)N, &a.lp);
        s.in(rng->normal_tape, (size_t)D * N, &a.normal_tape);
        s.out(eps_out, (size_t)N, &a.eps_out);
        s.out2d(r_out, D, z->ld, N, &a.r_out);
    });
    if (rc) return rc;
    if (D > 512 && (rc = chain_workspace(ctx, (size_t)kBigFindEpsVectors * D * (size_t)N * sizeof(double), &a.scratch))) return rc;
    int nl = 0;
    CU(launch_find_eps(a, ctx->stream, &nl));
    ctx->launches += nl;
    return finish_call(ctx, st, flags);
}

// ------------------------------------------------------------------------------------------ comm + pooled adaptor
struct ahmc_comm {
    void* nccl = nullptr;
    int nranks = 1, rank = 0;
    bool owned = false;
};
struct ahmc_pooled {
    int D = 0;
    int64_t N = 0;
    void* dev = nullptr;  // one allocation: state | eps_chain | minv | w_mu | w_M2 | record | merged
    void* state = nullptr;
    double *eps_chain = nullptr, *minv = nullptr, *w_mu = nullptr, *w_M2 = nullptr, *record = nullptr, *merged = nullptr;
    DevBuf gathered;  // every rank's record (more than one rank)
};

int ahmc_comm_unique_id(ahmc_ctx* ctx, void* id128_out) {
    if (!ctx || !id128_out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/id");
    if (const char* why = nccl_bind()) return fail(ctx, AHMC_ERR_UNSUPPORTED, "NCCL unavailable: %s", why);
    int rc = nccl_unique_id(id128_out);
    if (rc) return fail(ctx, AHMC_ERR_CUDA, "ncclGetUniqueId: %s", nccl_err(rc));
    return AHMC_OK;
}
int ahmc_comm_create(ahmc_ctx* ctx, const void* id128, int32_t nranks, int32_t rank, ahmc_comm** out) {
    if (!ctx || !id128 || !out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/id/out");
    if (nranks < 1 || rank < 0 || rank >= nranks) return fail(ctx, AHMC_ERR_INVALID, "need 0 <= rank < nranks");
    if (const char* why = nccl_bind()) return fail(ctx, AHMC_ERR_UNSUPPORTED, "NCCL unavailable: %s", why);
    DeviceGuard g(ctx->device);
    void* c = nullptr;
    int rc = nccl_comm_init(&c, nranks, id128, rank);
    if (rc) return fail(ctx, AHMC_ERR_CUDA, "ncclCommInitRank: %s", nccl_err(rc));
    ahmc_comm* m = new (std::nothrow) ahmc_comm;
    if (!m) return fail(ctx, AHMC_ERR_NOMEM, "out of host memory");
    m->nccl = c; m->nranks = nranks; m->rank = rank; m->owned = true;
    *out = m;
    return AHMC_OK;
}
int ahmc_comm_from_nccl(ahmc_ctx* ctx, void* nccl_comm, int32_t nranks, int32_t rank, ahmc_comm** out) {
    if (!ctx || !nccl_comm || !out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/comm/out");
    if (nranks < 1 || rank < 0 || rank >= nranks) return fail(ctx, AHMC_ERR_INVALID, "need 0 <= rank < nranks");
    if (const char* why = nccl_bind()) return fail(ctx, AHMC_ERR_UNSUPPORTED, "NCCL unavailable: %s", why);
    ahmc_comm* m = new (std::nothrow) ahmc_comm;
    if (!m) return fail(ctx, AHMC_ERR_NOMEM, "out of host memory");
    m->nccl = nccl_comm; m->nranks = nranks; m->rank = rank; m->owned = false;
    *out = m;
    return AHMC_OK;
}
int ahmc_comm_destroy(ahmc_ctx* ctx, ahmc_comm* comm) {
    if (!ctx) return AHMC_ERR_INVALID;
    if (!comm) return AHMC_OK;
    DeviceGuard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (comm->owned && comm->nccl) nccl_comm_destroy(comm->nccl);
    delete comm;
    return AHMC_OK;
}

int ahmc_adapt_allgather_f64(ahmc_ctx* ctx, ahmc_comm* comm, const double* record, int64_t n, double* out, uint32_t flags) {
    if (!ctx || !record || !out || n < 1) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/record/out or n < 1");
    if (flags & AHMC_FLAG_HOST_BUFFERS) return fail(ctx, AHMC_ERR_UNSUPPORTED, "the exchange takes device pointers");
    DeviceGuard g(ctx->device);
    if (!comm || comm->nranks == 1) {
        if (out != record) CU(cudaMemcpyAsync(out, record, (size_t)n * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    } else {
        int rc = nccl_allgather_f64(record, out, (size_t)n, comm->nccl, ctx->stream);
        if (rc) return fail(ctx, AHMC_ERR_CUDA, "ncclAllGather: %s", nccl_err(rc));
    }
    if (!(flags & AHMC_FLAG_ASYNC)) CU(cudaStreamSynchronize(ctx->stream));
    return AHMC_OK;
}

int ahmc_pooled_create(ahmc_ctx* ctx, int32_t D, int64_t N, const ahmc_pooled_cfg* cfg, const double* Minv0, ahmc_pooled** out) {
    if (!ctx || !cfg || !out) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/cfg/out");
    if (D < 1 || N < 1) return fail(ctx, AHMC_ERR_INVALID, "need D >= 1, N >= 1");
    if (cfg->n_adapts < 0 || !(cfg->eps0 > 0.0)) return fail(ctx, AHMC_ERR_INVALID, "need n_adapts >= 0 and eps0 > 0");
    AdaptDev sched{};
    if (!stan_window_schedule(sched, cfg->init_buffer, cfg->term_buffer, cfg->window_size, cfg->n_adapts))
        return fail(ctx, AHMC_ERR_UNSUPPORTED, "the window schedule has more than 12 window ends");
    DeviceGuard g(ctx->device);
    ahmc_pooled* a = new (std::nothrow) ahmc_pooled;
    if (!a) return fail(ctx, AHMC_ERR_NOMEM, "out of host memory");
    a->D = D;
    a->N = N;
    const size_t rec = (size_t)(2 + 2 * D) * 8;
    auto layout = [&](Carver& c) {
        a->state = c.take<char>(pooled_state_bytes());
        a->eps_chain = c.take<double>((size_t)N);
        a->minv = c.take<double>((size_t)D);
        a->w_mu = c.take<double>((size_t)D);
        a->w_M2 = c.take<double>((size_t)D);
        a->record = c.take<double>((size_t)(2 + 2 * D));
        a->merged = c.take<double>((size_t)(2 + 2 * D));
    };
    Carver size;
    layout(size);
    if (cudaMalloc(&a->dev, size.off) != cudaSuccess) {
        delete a;
        return fail(ctx, AHMC_ERR_NOMEM, "cudaMalloc(%zu) for the pooled adaptor failed", size.off);
    }
    Carver c{(char*)a->dev};
    layout(c);
    std::vector<char> img(pooled_state_bytes());
    pooled_state_init(img.data(), cfg->eps0, sched, cfg->delta, cfg->gamma, cfg->t0, cfg->kappa, cfg->n_adapts,
                      cfg->adapt_metric, cfg->n_min);
    CU(cudaMemcpyAsync(a->state, img.data(), img.size(), cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemsetAsync(a->w_mu, 0, (size_t)D * 8, ctx->stream));
    CU(cudaMemsetAsync(a->w_M2, 0, (size_t)D * 8, ctx->stream));
    CU(cudaMemsetAsync(a->merged, 0, rec, ctx->stream));
    if (Minv0) CU(cudaMemcpyAsync(a->minv, Minv0, (size_t)D * 8, cudaMemcpyHostToDevice, ctx->stream));
    else CU(launch_fill(a->minv, D, 1.0, ctx->stream));
    CU(launch_fill(a->eps_chain, N, cfg->eps0, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));  // img / Minv0 are host memory of this frame
    *out = a;
    return AHMC_OK;
}
int ahmc_pooled_destroy(ahmc_ctx* ctx, ahmc_pooled* a) {
    if (!ctx) return AHMC_ERR_INVALID;
    if (!a) return AHMC_OK;
    DeviceGuard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaFree(a->dev);
    cudaFree(a->gathered.p);
    delete a;
    return AHMC_OK;
}
double* ahmc_pooled_eps(ahmc_pooled* a) { return a ? a->eps_chain : nullptr; }
double* ahmc_pooled_minv(ahmc_pooled* a) { return a ? a->minv : nullptr; }

int ahmc_adapt_exchange_f64(ahmc_ctx* ctx, ahmc_comm* comm, ahmc_pooled* a, int32_t D, int64_t N, const double* theta,
                            int64_t ld, const double* acceptance_rate, double* eps_trace, uint32_t flags) {
    if (!ctx || !a || !theta || !acceptance_rate) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/adaptor/theta/acceptance_rate");
    if (flags & AHMC_FLAG_HOST_BUFFERS) return fail(ctx, AHMC_ERR_UNSUPPORTED, "the exchange takes device pointers");
    if (D != a->D || N != a->N || ld < D) return fail(ctx, AHMC_ERR_INVALID, "D / N differ from the adaptor's, or ld < D");
    DeviceGuard g(ctx->device);
    const int R = comm ? comm->nranks : 1;
    const size_t rec = (size_t)(2 + 2 * D);
    int rc;
    if (R > 1 && (rc = ensure(ctx, a->gathered, rec * 8 * (size_t)R, "the gathered records"))) return rc;
    // K5: this rank's record
    const int blocks = (int)(N < ctx->sm_count ? N : ctx->sm_count);
    unsigned* counter;
    double* partial;
    if ((rc = summary_workspace(ctx, D, blocks, &counter, &partial))) return rc;
    int nl = 0;
    CU(launch_adapt_summary(D, N, theta, ld, acceptance_rate, a->record, partial, counter, blocks, ctx->stream, &nl));
    const double* gathered = a->record;
    if (R > 1) {
        if ((rc = nccl_allgather_f64(a->record, (double*)a->gathered.p, rec, comm->nccl, ctx->stream)))
            return fail(ctx, AHMC_ERR_CUDA, "ncclAllGather: %s", nccl_err(rc));
        gathered = (double*)a->gathered.p;
    }
    CU(launch_pooled_update(a->state, gathered, R, D, a->w_mu, a->w_M2, a->minv, a->eps_chain, N, eps_trace, a->merged,
                            ctx->stream, &nl));
    ctx->launches += nl;
    if (!(flags & AHMC_FLAG_ASYNC)) CU(cudaStreamSynchronize(ctx->stream));
    return AHMC_OK;
}

int ahmc_pooled_state(ahmc_ctx* ctx, ahmc_pooled* a, double* eps, double* Minv, int32_t* iteration, double* merged_record) {
    if (!ctx || !a) return fail(ctx, AHMC_ERR_INVALID, "NULL ctx/adaptor");
    DeviceGuard g(ctx->device);
    std::vector<char> img(pooled_state_bytes());
    CU(cudaMemcpyAsync(img.data(), a->state, img.size(), cudaMemcpyDeviceToHost, ctx->stream));
    if (Minv) CU(cudaMemcpyAsync(Minv, a->minv, (size_t)a->D * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (merged_record) CU(cudaMemcpyAsync(merged_record, a->merged, (size_t)(2 + 2 * a->D) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    int it = 0;
    pooled_state_read(img.data(), eps, &it, nullptr, nullptr);
    if (iteration) *iteration = it;
    return AHMC_OK;
}

}  // extern "C"
