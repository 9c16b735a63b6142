// ahmc_nuts.cu -- K3 entry: workspace size, family dispatch, and the default family
// (MultinomialTS + GeneralisedNoUTurn, what `NUTS(delta)` builds).  Kernel: ahmc_nuts_kernel.cuh.
#include "ahmc_nuts_kernel.cuh"

namespace ahmc {

long long nuts_scratch_doubles_per_chain(int D, int max_depth, long long adapt_doubles) {
    return nuts_level_doubles(D, max_depth) + adapt_doubles;
}

// A (D x D, column-major) -> columns of leading dimension coop_lds(D), rows >= D zero: what the cooperative products stream
__global__ void pad_columns_kernel(const double* __restrict__ A, int D, int lds, double* __restrict__ out) {
    const long long n = (long long)D * lds;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i / lds), r = (int)(i - (long long)k * lds);
        out[i] = r < D ? A[(long long)k * D + r] : 0.0;
    }
}
size_t coop_padded_doubles(int D) { return (size_t)D * coop_lds(D); }
cudaError_t launch_pad_columns(const double* A, int D, double* out, cudaStream_t st) {
    pad_columns_kernel<<<64, 256, 0, st>>>(A, D, coop_lds(D), out);
    return cudaGetLastError();
}

cudaError_t launch_nuts_variants(const NutsArgs& a, cudaStream_t st);  // ahmc_nuts_var.cu
cudaError_t launch_nuts_adaptive(const NutsArgs& a, cudaStream_t st);  // ahmc_nuts_adapt.cu
cudaError_t launch_nuts_nutpie(const NutsArgs& a, cudaStream_t st);    // ahmc_nuts_nutpie.cu
cudaError_t launch_nuts_cov(const NutsArgs& a, cudaStream_t st);       // ahmc_nuts_cov.cu

cudaError_t launch_nuts(const NutsArgs& a, cudaStream_t st, int* n_launches) {
    if (n_launches) *n_launches += 1;
    // (adaptive: the metric kind and estimator form of the instantiation, decided once for both kinds of target)
    const AdaptKernel ak = a.ad.enabled ? adapt_kernel(a.ad, a.metric) : AdaptKernel{metric_form(a.metric), 0};
    if (a.model.kind == AHMC_MODEL_USER) {  // run-time compiled kernel of a user target (default / adaptive family, ahmc_user.cu)
        int G, E;
        if (!pick_layout(a.D, &G, &E) || a.sampler != 0 || a.criterion != 0) return cudaErrorInvalidValue;
        if (a.ad.enabled && a.metric.kind != AHMC_METRIC_DIAG && a.metric.kind != AHMC_METRIC_DENSE) return cudaErrorInvalidValue;
        const int cpb = kBlockThreads / G;
        const int maxd = a.max_depth > 0 ? a.max_depth : 1;
        const size_t sm = smem_bytes(AHMC_MODEL_USER, ak.metric_kind, a.D, G) + (size_t)cpb * maxd * kLevelScalars * sizeof(double);
        return user_launch((UserModule*)a.model.user, a.ad.enabled ? UK_NUTS_ADAPT : UK_NUTS, ak.metric_kind, G, E, &a,
                           (unsigned)((a.N + cpb - 1) / cpb), sm, st, ak.form);
    }
    if (a.ad.enabled) {
        switch (ak.form) {
            case AHMC_ADAPT_WELFORD_COV: return launch_nuts_cov(a, st);
            case AHMC_ADAPT_NUTPIE: return launch_nuts_nutpie(a, st);
            default: return launch_nuts_adaptive(a, st);
        }
    }
    if (a.sampler != 0 || a.criterion != 0) return launch_nuts_variants(a, st);
    return nuts_dispatch<false, false, false>(a, st);
}

}  // namespace ahmc
