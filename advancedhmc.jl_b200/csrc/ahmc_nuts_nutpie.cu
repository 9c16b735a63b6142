// ahmc_nuts_nutpie.cu -- K3, adaptive family with NutpieVar as each chain's metric estimator (massmatrix.jl:172-250):
// the form of ahmc_nuts_adapt.cu whose adaptor pushes positions and gradients (ahmc_chain_adapt.cuh).  A translation unit
// of its own so that the two adaptive forms compile in parallel.
#include "ahmc_nuts_kernel.cuh"

namespace ahmc {

cudaError_t launch_nuts_nutpie(const NutsArgs& a, cudaStream_t st) {
    if (a.sampler != 0 || a.criterion != 0) return cudaErrorInvalidValue;
    return nuts_dispatch<false, AHMC_ADAPT_NUTPIE, true>(a, st);
}

}  // namespace ahmc
