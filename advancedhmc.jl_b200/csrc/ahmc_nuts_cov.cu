// ahmc_nuts_cov.cu -- K3, adaptive family for the Dense metric: every chain runs its own NesterovDualAveraging and, with
// AHMC_ADAPT_WELFORD_COV, a windowed WelfordCov (massmatrix.jl:284-340) whose estimate is factorised at each window end
// (ahmc_chain_adapt.cuh).  The chain's trajectories read its own M^-1 and factor, so the warp-per-chain form runs (never
// the cooperative one, whose warps share one matrix).  A translation unit of its own, like the other estimator forms.
#include "ahmc_nuts_kernel.cuh"

namespace ahmc {

cudaError_t launch_nuts_cov(const NutsArgs& a, cudaStream_t st) {
    if (a.sampler != 0 || a.criterion != 0) return cudaErrorInvalidValue;
    return nuts_dispatch<false, AHMC_ADAPT_WELFORD_COV, true>(a, st);
}

}  // namespace ahmc
