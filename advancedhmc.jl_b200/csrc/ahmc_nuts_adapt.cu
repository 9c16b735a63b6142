// ahmc_nuts_adapt.cu -- K3, adaptive family: every chain runs its own NesterovDualAveraging and windowed WelfordVar
// (the reference's vectorised adaptors: src/adaptation/stepsize.jl:178-210, massmatrix.jl:141-157,
// stan_adaptor.jl:137-159) INSIDE the persistent launch, so a whole warm-up + sampling run is one kernel and no chain
// waits for another chain's tree.  Diag metric (per-chain M^-1), MultinomialTS + GeneralisedNoUTurn.  The NutpieVar
// form is compiled in ahmc_nuts_nutpie.cu.
#include "ahmc_nuts_kernel.cuh"

namespace ahmc {

cudaError_t launch_nuts_adaptive(const NutsArgs& a, cudaStream_t st) {
    if (a.sampler != 0 || a.criterion != 0) return cudaErrorInvalidValue;
    return nuts_dispatch<false, AHMC_ADAPT_WELFORD, true>(a, st);
}

}  // namespace ahmc
