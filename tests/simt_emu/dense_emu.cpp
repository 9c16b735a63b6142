// dense_emu.cpp -- K4, the tile-per-CTA trajectory kernel for GEMM-shaped operators (advancedhmc.jl_b200/csrc/
// ahmc_dense.cu: `dense_traj_kernel`, `pad_norm_kernel`, `vec_norm_kernel`, unmodified) under the CPU SIMT emulator.
// The kernel's PTX wrappers (mbarrier, bulk copy, DMMA) are restated in simt_emu.cpp with the same contracts.
// TEST INFRASTRUCTURE ONLY (tests/test_simt_emulation.py).
#define AHMC_SIMT_EMULATION 1
#define __shared__ static  // static shared variables; blocks run one at a time
#include <cstdlib>
#include <cstdio>
#include <atomic>
#include <thread>
#include <vector>

#include "ahmc_dense.cu"
#include "emu_smem.h"
#include "emu_harness.h"

namespace ahmc {
unsigned char* emu_dynamic_smem = nullptr;
// (the mbarrier / bulk-copy / DMMA contracts live in simt_emu.cpp: the cooperative NUTS products use them too)
}  // namespace ahmc
EMU_DEFINE_SMEM_ARENA();
using namespace ahmc;

template <int RB, int CB, int MINB>
static void dense_thunk(const void* p) { dense_traj_kernel<RB, CB, MINB>(*static_cast<const DenseArgs*>(p)); }
struct PadArgs {
    const double* A;
    int D, Dp;
    double* Ap;
    double* norm;
};
static void pad_thunk(const void* p) {
    const PadArgs& a = *static_cast<const PadArgs*>(p);
    pad_norm_kernel(a.A, a.D, a.Dp, a.Ap, a.norm);
}
static void vec_thunk(const void* p) {
    const PadArgs& a = *static_cast<const PadArgs*>(p);
    vec_norm_kernel(a.A, a.D, a.norm);
}

struct EmuDense {
    int32_t D;
    int64_t N;
    const double *P, *w, *mu;  // P: D x D column-major precision or null; w: 1/s^2 or null
    double c0;
    const double *Minv, *Mdiag;  // Minv: D x D column-major or null
    double eps;
    const double* eps_chain;
    int32_t n_steps, fwd;
    const double *th_in, *r_in, *g_in;
    double *th_out, *r_out, *g_out, *dr_out, *lp_out, *lk_out;
    uint32_t* status;
    int32_t* steps_done;
    uint8_t* need_exact;
    int32_t wide_tile;  // RB == 2 only: 1 -> the <2,4> (32-chain) form instead of the default <2,2,2>
    double norms_out[2];
    int64_t ld_in, ld_out;  // leading dimensions of the D x N inputs / outputs (0: D)
};
EMU_EXPORT_SIZEOF(EmuDense);

extern "C" int emu_dense_stages() { return kStages; }
extern "C" int emu_dense(EmuDense* q) {
    // (mbarrier table: reset per block by emu_launch)
    int Dp, RB, CB_shape;
    if (!dense_tile_shape(q->D, &Dp, &RB, &CB_shape)) return -1;
    std::vector<double> Pp, Mp;
    double norms[2] = {0.0, 0.0};
    PadArgs pa{};
    if (q->Minv) {
        Mp.assign(dense_mat_doubles(Dp), -1.0);
        pa = PadArgs{q->Minv, q->D, Dp, Mp.data(), &norms[0]};
        emu_launch(pad_thunk, &pa, 1, 256);
    } else {
        pa = PadArgs{q->Mdiag, q->D, Dp, nullptr, &norms[0]};
        emu_launch(vec_thunk, &pa, 1, 32);
    }
    if (q->P) {
        Pp.assign(dense_mat_doubles(Dp), -1.0);
        pa = PadArgs{q->P, q->D, Dp, Pp.data(), &norms[1]};
        emu_launch(pad_thunk, &pa, 1, 256);
    } else {
        pa = PadArgs{q->w, q->D, Dp, nullptr, &norms[1]};
        emu_launch(vec_thunk, &pa, 1, 32);
    }
    q->norms_out[0] = norms[0];
    q->norms_out[1] = norms[1];
    DenseArgs a{};
    a.D = q->D; a.Dp = Dp; a.N = q->N; a.P = q->P ? Pp.data() : nullptr; a.w = q->w; a.mu = q->mu; a.c0 = q->c0;
    a.Minv = q->Minv ? Mp.data() : nullptr; a.Mdiag = q->Mdiag; a.norms = norms; a.eps = q->eps; a.eps_chain = q->eps_chain;
    a.n_steps = q->n_steps; a.fwd = q->fwd; a.th_in = q->th_in; a.r_in = q->r_in; a.g_in = q->g_in; a.ld_in = q->ld_in ? q->ld_in : q->D;
    a.th_out = q->th_out; a.r_out = q->r_out; a.g_out = q->g_out; a.dr_out = q->dr_out; a.lp_out = q->lp_out; a.lk_out = q->lk_out;
    a.ld_out = q->ld_out ? q->ld_out : q->D; a.status = q->status; a.steps_done = q->steps_done; a.need_exact = q->need_exact;
    void (*fn)(const void*) = nullptr;
    int CB = 0;  // the instantiation's, as launch_dense_traj picks it (RB == 2 may ask for the 32-chain form instead)
    if (RB == 1) fn = dense_thunk<1, 4, 1>, CB = 4;
    else if (RB == 2 && q->wide_tile) fn = dense_thunk<2, 4, 1>, CB = 4;
    else if (RB == 2) fn = dense_thunk<2, 2, 2>, CB = 2;
    else if (RB == 3) fn = dense_thunk<3, 2, 1>, CB = 2;
    else if (RB == 4) fn = dense_thunk<4, 2, 1>, CB = 2;
    else if (RB == 5) fn = dense_thunk<5, 1, 1>, CB = 1;
    else if (RB == 6) fn = dense_thunk<6, 1, 1>, CB = 1;
    else if (RB == 7) fn = dense_thunk<7, 1, 1>, CB = 1;
    else if (RB == 8) fn = dense_thunk<8, 1, 1>, CB = 1;
    else return -2;
    const int CT = 8 * CB;
    emu_dynamic_smem = emu_smem_base();
    emu_smem_begin(emu_dynamic_smem, dense_smem_bytes(Dp, CB), 2 * sizeof(int) /* s_flag, s_k */, "dense_traj_kernel");
    emu_launch(fn, &a, (int)((q->N + CT - 1) / CT), kDenseThreads);
    emu_smem_end();
    emu_dynamic_smem = nullptr;
    return 0;
}

#ifdef RACE_DENSE
static int run(int D, int N, bool denseP, bool denseM, int n, int wide) {
    std::vector<double> P((size_t)D * D, 0.0), M((size_t)D * D, 0.0), w(D), md(D), mu(D, 0.1), th((size_t)N * D), r((size_t)N * D),
        g((size_t)N * D), o((size_t)4 * N * D), lp(N), lk(N);
    srand(3 + D);
    auto u = [] { return rand() / (double)RAND_MAX; };
    for (int i = 0; i < D; ++i) {
        P[(size_t)i * D + i] = 1.0 + 0.01 * i;
        M[(size_t)i * D + i] = 0.5 + 0.002 * i;
        if (i) P[(size_t)i * D + i - 1] = P[(size_t)(i - 1) * D + i] = 0.1, M[(size_t)i * D + i - 1] = M[(size_t)(i - 1) * D + i] = 0.05;
        w[i] = 0.8 + 0.4 * u();
        md[i] = 0.7 + 0.5 * u();
    }
    for (auto* v : {&th, &r, &g})
        for (auto& x : *v) x = u() - 0.5;
    std::vector<uint32_t> st(N);
    std::vector<int32_t> done(N);
    std::vector<uint8_t> need(N);
    EmuDense q{};
    q.D = D; q.N = N; q.P = denseP ? P.data() : nullptr; q.w = denseP ? nullptr : w.data(); q.mu = mu.data();
    q.Minv = denseM ? M.data() : nullptr; q.Mdiag = denseM ? nullptr : md.data(); q.eps = 0.1; q.n_steps = n; q.fwd = 1;
    q.th_in = th.data(); q.r_in = r.data(); q.g_in = g.data();
    q.th_out = o.data(); q.r_out = o.data() + (size_t)N * D; q.g_out = o.data() + (size_t)2 * N * D; q.dr_out = o.data() + (size_t)3 * N * D;
    q.lp_out = lp.data(); q.lk_out = lk.data(); q.status = st.data(); q.steps_done = done.data(); q.need_exact = need.data();
    q.wide_tile = wide;
    const int rc = emu_dense(&q);
    std::printf("dense D %d N %d P %d M %d: rc %d lp0 %.6f need0 %d\n", D, N, (int)denseP, (int)denseM, rc, lp[0], (int)need[0]);
    return rc != 0 || need[0] != 0;
}

int main() {
    int bad = 0;
    bad |= run(40, 37, true, true, 4, 0);    // <1,4>: two products per step, ragged second tile
    bad |= run(100, 20, true, false, 3, 0);  // <2,2,2>
    bad |= run(70, 33, false, true, 3, 1);   // <2,4>
    bad |= run(130, 9, true, true, 2, 0);    // <3,2>: 12 chunks per product
    return bad;
}
#endif
