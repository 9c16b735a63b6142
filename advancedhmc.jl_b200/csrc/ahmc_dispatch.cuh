// ahmc_dispatch.cuh -- host-side launch dispatch: run-time layout (G, E), model kind and metric form -> the compile-time
// template arguments of a kernel, and the launch itself.  Every launcher of the register-resident and D > 512 kernels goes
// through these tables, so which kernels exist and which run-time kinds reach them is stated once.
// Host only: not part of what NVRTC compiles for user targets, nor of the CPU SIMT emulation.
#pragma once
#include <type_traits>

#include "ahmc_kernels.cuh"

namespace ahmc {

template <int V>
using IC = std::integral_constant<int, V>;
template <int... V>
struct Kinds {};

// the built-in targets and the metric forms a launch instantiates (metric_form: kMetricDenseChain for a per-chain Dense metric)
using AllModels = Kinds<AHMC_MODEL_STD_NORMAL, AHMC_MODEL_DIAG_GAUSS, AHMC_MODEL_DENSE_GAUSS, AHMC_MODEL_FUNNEL>;
using AllMetrics = Kinds<AHMC_METRIC_UNIT, AHMC_METRIC_DIAG, AHMC_METRIC_DENSE, kMetricDenseChain>;
// D > 512 (bigd_supported): the streaming kernels exist for these only
using BigModels = Kinds<AHMC_MODEL_STD_NORMAL, AHMC_MODEL_DIAG_GAUSS, AHMC_MODEL_FUNNEL>;
using BigMetrics = Kinds<AHMC_METRIC_UNIT, AHMC_METRIC_DIAG>;

// f(IC<k>{}) for the kind k of the list equal to `kind`; `none` if the list does not hold it
template <int... V, class F>
cudaError_t with_kind(Kinds<V...>, int kind, F&& f, cudaError_t none = cudaErrorInvalidValue) {
    cudaError_t r = none;
    (void)((kind == V && (r = f(IC<V>{}), true)) || ...);
    return r;
}

// f(IC<G>{}, IC<E>{}) for the register-resident layouts pick_layout (ahmc_leapfrog.cu) returns, and only those
template <class F>
cudaError_t with_layout(int G, int E, F&& f) {
    if (G == 4 && E == 1) return f(IC<4>{}, IC<1>{});
    if (G == 8 && E == 1) return f(IC<8>{}, IC<1>{});
    if (G == 16 && E == 1) return f(IC<16>{}, IC<1>{});
    if (G == 32 && E == 1) return f(IC<32>{}, IC<1>{});
    if (G == 32 && E == 2) return f(IC<32>{}, IC<2>{});
    if (G == 32 && E == 4) return f(IC<32>{}, IC<4>{});
    if (G == 32 && E == 8) return f(IC<32>{}, IC<8>{});
    if (G == 32 && E == 16) return f(IC<32>{}, IC<16>{});
    return cudaErrorInvalidValue;
}

// f(MODEL, METRIC) as integral constants for (model, metric) in the caller's lists; `none` for any other pair
template <class Models, class Metrics, class F>
cudaError_t with_model_metric(Models models, Metrics metrics, int model, int metric, F&& f, cudaError_t none = cudaErrorInvalidValue) {
    return with_kind(models, model, [&](auto M) { return with_kind(metrics, metric, [&](auto K) { return f(M, K); }, none); }, none);
}
// f(MODEL, METRIC, G, E): (model, metric) from the caller's lists, (G, E) from the layout table
template <class Models, class Metrics, class F>
cudaError_t with_model_metric_layout(Models models, Metrics metrics, int model, int metric, int G, int E, F&& f) {
    return with_model_metric(models, metrics, model, metric, [&](auto M, auto K) {
        return with_layout(G, E, [&](auto g, auto e) { return f(M, K, g, e); });
    });
}

// launch with `smem` bytes of dynamic shared memory; beyond 48 KB the kernel has to opt in first
template <class Args>
cudaError_t launch_kernel(void (*kernel)(Args), long long blocks, int threads, size_t smem, cudaStream_t st, const Args& a) {
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    kernel<<<(unsigned)blocks, threads, smem, st>>>(a);
    return cudaGetLastError();
}
// one group of G lanes per chain, kBlockThreads per CTA
template <class Args>
cudaError_t launch_warps(void (*kernel)(Args), long long N, int G, size_t smem, cudaStream_t st, const Args& a) {
    const int chains_per_block = kBlockThreads / G;
    return launch_kernel(kernel, (N + chains_per_block - 1) / chains_per_block, kBlockThreads, smem, st, a);
}

}  // namespace ahmc
