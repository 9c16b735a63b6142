// glm_emu.cpp -- K6, the chain-tile trajectory kernel for GLM targets (advancedhmc.jl_b200/csrc/ahmc_glm.cu:
// `glm_traj_kernel`, unmodified) under the CPU SIMT emulator.  The kernel's PTX wrappers (mbarrier, bulk copy, DMMA) are
// restated in simt_emu.cpp with the same contracts.  TEST INFRASTRUCTURE ONLY (tests/test_glm_cpu.py).
#define AHMC_SIMT_EMULATION 1
#define __shared__ static
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <vector>

#include "ahmc_glm.cu"
#include "emu_smem.h"
#include "emu_harness.h"

namespace ahmc {
unsigned char* emu_dynamic_smem = nullptr;
}
EMU_DEFINE_SMEM_ARENA();
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
    int64_t ld_in, ld_out;  // leading dimensions of the D x N inputs / outputs (0: D)
};
EMU_EXPORT_SIZEOF(EmuGlm);

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
    a.n_steps = e->n_steps; a.fwd = e->fwd; a.th_in = e->th_in; a.r_in = e->r_in; a.g_in = e->g_in; a.ld_in = e->ld_in ? e->ld_in : e->D;
    a.th_out = e->th_out; a.r_out = e->r_out; a.g_out = e->g_out; a.dr_out = e->dr_out; a.lp_out = e->lp_out; a.lk_out = e->lk_out;
    a.ld_out = e->ld_out ? e->ld_out : e->D; a.status = e->status; a.steps_done = e->steps_done;
    void (*fn)(const void*) = nullptr;
    const bool logit = e->family == AHMC_GLM_BERNOULLI_LOGIT;
    if (CB != 2) return -2;
    if (RB == 1) fn = logit ? glm_thunk<1, 2, 0> : glm_thunk<1, 2, 1>;
    else if (RB == 2) fn = logit ? glm_thunk<2, 2, 0> : glm_thunk<2, 2, 1>;
    else if (RB == 3) fn = logit ? glm_thunk<3, 2, 0> : glm_thunk<3, 2, 1>;
    else fn = logit ? glm_thunk<4, 2, 0> : glm_thunk<4, 2, 1>;
    emu_dynamic_smem = emu_smem_base();
    emu_smem_begin(emu_dynamic_smem, sm, 0, "glm_traj_kernel");
    emu_launch(fn, &a, (int)((e->N + 8 * CB - 1) / (8 * CB)), kGlmThreads);
    emu_smem_end();
    emu_dynamic_smem = nullptr;
    return 0;
}

#ifdef RACE_GLM
// K6: a 9-coordinate Bernoulli-logit target with 70 rows (two chunks, a partial last one), a ragged second tile
int main() {
    const int D = 9, n = 70, N = 17, steps = 2;
    std::vector<double> X((size_t)n * D), y(n), prec(D, 1.0), th((size_t)N * D), r((size_t)N * D), o((size_t)6 * N * D), lp(N), lk(N);
    std::vector<uint32_t> status(N);
    std::vector<int32_t> done(N);
    srand(3);
    auto u = [] { return rand() / (double)RAND_MAX - 0.5; };
    for (auto& x : X) x = u();
    for (auto& v : y) v = u() > 0.0 ? 1.0 : 0.0;
    for (auto& v : th) v = 0.3 * u();
    for (auto& v : r) v = u();
    EmuGlm e{};
    e.family = AHMC_GLM_BERNOULLI_LOGIT; e.D = D; e.n = n; e.N = N; e.X = X.data(); e.y = y.data(); e.prec = prec.data();
    e.eps = 0.05; e.n_steps = steps; e.fwd = 1; e.th_in = th.data(); e.r_in = r.data();
    double* p = o.data();
    e.th_out = p; e.r_out = p + N * D; e.g_out = p + 2 * N * D; e.dr_out = p + 3 * N * D; e.lp_out = lp.data(); e.lk_out = lk.data();
    e.status = status.data(); e.steps_done = done.data();
    const int rc = emu_glm(&e);
    int bad = rc != 0;
    for (int c = 0; c < N; ++c) bad |= status[c] != 0 || done[c] != steps || !std::isfinite(lp[c]);
    std::printf("glm D %d n %d N %d: rc %d\n", D, n, N, bad);
    return bad;
}
#endif
