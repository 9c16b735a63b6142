// glm_emu.cpp -- K6, the chain-tile trajectory kernel for GLM targets (advancedhmc.jl_b200/csrc/ahmc_glm.cu:
// `glm_traj_kernel`, unmodified) under the CPU SIMT emulator.  The kernel's PTX wrappers (mbarrier, bulk copy, DMMA) are
// restated in simt_emu.cpp with the same contracts.  TEST INFRASTRUCTURE ONLY (tests/test_glm_cpu.py).
#define AHMC_SIMT_EMULATION 1
#define __shared__ static
#include <cstring>
#include <vector>

#include "ahmc_glm.cu"

void emu_launch(void (*kernel)(const void*), const void* args, int blocks, int threads);

namespace ahmc {
unsigned char* emu_dynamic_smem = nullptr;
}
using namespace ahmc;

template <int RB, int CB, int FAM>
static void glm_thunk(const void* p) { glm_traj_kernel<RB, CB, FAM>(*static_cast<const GlmArgs*>(p)); }

struct EmuGlm {
    int32_t family, D, n;
    int64_t N;
    const double *X, *y, *prec;  // X: n x D row-major
    double c0;
    const double* Minv;
    int64_t chain_stride;
    double eps;
    const double* eps_chain;
    int32_t n_steps, fwd;
    const double *th_in, *r_in, *g_in;
    double *th_out, *r_out, *g_out, *dr_out, *lp_out, *lk_out;
    uint32_t* status;
    int32_t* steps_done;
    int32_t nc_out, stages_out;
};

extern "C" int emu_glm(EmuGlm* e) {
    GlmArgs a{};
    int RB, CB;
    size_t sm;
    if (!glm_tile_shape(e->D, e->n, &RB, &CB, &a.nc, &a.stages, &sm)) return -1;
    e->nc_out = a.nc;
    e->stages_out = a.stages;
    const int lds = glm_lds(e->D);
    std::vector<double> Xp(glm_padded_doubles(e->D, e->n), 0.0);
    for (int i = 0; i < e->n; ++i) std::memcpy(Xp.data() + (size_t)i * lds, e->X + (size_t)i * e->D, sizeof(double) * e->D);
    a.family = e->family; a.D = e->D; a.n = e->n; a.N = e->N; a.Xp = Xp.data(); a.y = e->y; a.prec = e->prec; a.c0 = e->c0;
    a.Minv = e->Minv; a.chain_stride = e->chain_stride; a.eps = e->eps; a.eps_chain = e->eps_chain;
    a.n_steps = e->n_steps; a.fwd = e->fwd; a.th_in = e->th_in; a.r_in = e->r_in; a.g_in = e->g_in; a.ld_in = e->D;
    a.th_out = e->th_out; a.r_out = e->r_out; a.g_out = e->g_out; a.dr_out = e->dr_out; a.lp_out = e->lp_out; a.lk_out = e->lk_out;
    a.ld_out = e->D; a.status = e->status; a.steps_done = e->steps_done;
    void (*fn)(const void*) = nullptr;
    const bool logit = e->family == AHMC_GLM_BERNOULLI_LOGIT;
    if (CB != 2) return -2;
    if (RB == 1) fn = logit ? glm_thunk<1, 2, 0> : glm_thunk<1, 2, 1>;
    else if (RB == 2) fn = logit ? glm_thunk<2, 2, 0> : glm_thunk<2, 2, 1>;
    else if (RB == 3) fn = logit ? glm_thunk<3, 2, 0> : glm_thunk<3, 2, 1>;
    else fn = logit ? glm_thunk<4, 2, 0> : glm_thunk<4, 2, 1>;
    std::vector<double> smem(sm / sizeof(double) + 2, 0.0);
    emu_dynamic_smem = reinterpret_cast<unsigned char*>(smem.data());
    emu_launch(fn, &a, (int)((e->N + 8 * CB - 1) / (8 * CB)), kGlmThreads);
    emu_dynamic_smem = nullptr;
    return 0;
}
