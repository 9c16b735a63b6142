// ahmc_glm.cuh -- K6 (ahmc_glm.cu): argument block, tile shape and launch declarations of the tiled trajectory kernel
// for generalised linear model targets (AHMC_GLM_BERNOULLI_LOGIT / AHMC_GLM_POISSON_LOG with a Gaussian prior).
#pragma once
#include <string>

#include "ahmc_kernels.cuh"

namespace ahmc {

// rows of the padded design matrix: n rounded up to the largest chunk, so every chunk size divides it
constexpr int kGlmMaxChunk = 64;
__host__ __device__ constexpr int glm_lds(int D) { return ((D + 7) / 8) * 8 + 4; }  // leading dimension of a stored row
inline size_t glm_padded_doubles(int D, int n) {
    return (size_t)((n + kGlmMaxChunk - 1) / kGlmMaxChunk) * kGlmMaxChunk * (size_t)glm_lds(D);
}

struct GlmArgs {
    int family;  // AHMC_GLM_*
    int D, n;
    int nc, stages;       // rows per chunk (8, 16, 32 or 64) and pipeline stages (2 or 3): glm_tile_shape
    long long N;
    const double* Xp;     // padded design matrix: row i at i * glm_lds(D), columns >= D and rows >= n zero
    const double* y;      // n
    const double* prec;   // D prior precisions
    double c0;
    const double* Minv;   // Diag metric: D (chain_stride 0) or chain c's at chain_stride * c; nullptr: Unit
    long long chain_stride;
    double eps;
    const double* eps_chain;
    int n_steps, fwd;     // n_steps == 0: phasepoint (energies, gradient and dH/dr of the input point)
    const double *th_in, *r_in, *g_in;  // g_in nullable: one pass at the start point
    long long ld_in;
    double *th_out, *r_out, *g_out, *dr_out, *lp_out, *lk_out;  // th_out / r_out / dr_out nullable
    long long ld_out;
    uint32_t* status;     // nullable
    int32_t* steps_done;  // nullable
};

// the tile a (D, n) runs on: RB row blocks of 8 coordinates per warp, CB column blocks of 8 chains, chunk rows, stages and
// the dynamic shared memory.  false: no tile (D > 256, or the stages do not fit) -- the caller takes the general form.
bool glm_tile_shape(int D, int n, int* RB, int* CB, int* nc, int* stages, size_t* smem);
// CUDA source of the target in the group form of run-time compiled targets (params = [prior_prec | X | y])
std::string glm_group_source(int family, int D, int n);
#ifndef AHMC_SIMT_EMULATION
cudaError_t launch_glm_traj(const GlmArgs& a, cudaStream_t st, int* n_launches);
#endif

}  // namespace ahmc
