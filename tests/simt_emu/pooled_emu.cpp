// pooled_emu.cpp -- the device-side pooled adaptor (advancedhmc.jl_b200/csrc/ahmc_pooled.cu `pooled_update_kernel`, unmodified)
// under the CPU SIMT emulator: the rank-ordered merge of R per-rank records, dual averaging, WelfordVar and the Stan window
// logic -- the multi-rank arithmetic of the exchange, checkable without a GPU or NCCL.  TEST INFRASTRUCTURE ONLY.
#define AHMC_SIMT_EMULATION 1
#define __shared__ static  // static shared variables only; one block
#include <cstdlib>
#include <vector>

#include "ahmc_pooled.cu"
#include "emu_harness.h"

using namespace ahmc;

struct UpdArgs {
    PooledState* st;
    const double* gathered;
    int R, D;
    double *w_mu, *w_M2, *Minv, *eps_chain;
    long long N;
    double *trace, *merged;
};
static void upd_thunk(const void* p) {
    const UpdArgs& a = *static_cast<const UpdArgs*>(p);
    pooled_update_kernel(a.st, a.gathered, a.R, a.D, a.w_mu, a.w_M2, a.Minv, a.eps_chain, a.N, a.trace, a.merged);
}

struct PooledHandle {
    std::vector<char> state;
    std::vector<double> w_mu, w_M2, Minv, eps_chain, merged;
    int D;
    long long N;
};

extern "C" void* emu_pooled_create(int D, long long N, int n_adapts, int init_buffer, int term_buffer, int window_size, double eps0,
                                   double delta, int adapt_metric, int n_min) {
    AdaptDev sched{};
    if (!stan_window_schedule(sched, init_buffer, term_buffer, window_size, n_adapts)) return nullptr;
    PooledHandle* e = new PooledHandle;
    e->D = D;
    e->N = N;
    e->state.resize(pooled_state_bytes());
    pooled_state_init(e->state.data(), eps0, sched, delta, 0.05, 10.0, 0.75, n_adapts, adapt_metric, n_min);
    e->w_mu.assign(D, 0.0);
    e->w_M2.assign(D, 0.0);
    e->Minv.assign(D, 1.0);
    e->eps_chain.assign(N, eps0);
    e->merged.assign(2 + 2 * D, 0.0);
    return e;
}
// one exchange: `gathered` = R records of (2 + 2D) doubles in rank order
extern "C" int emu_pooled_update(void* h, const double* gathered, int R, double* eps_out, double* minv_out, double* merged_out) {
    PooledHandle* e = static_cast<PooledHandle*>(h);
    UpdArgs a{reinterpret_cast<PooledState*>(e->state.data()), gathered, R, e->D, e->w_mu.data(), e->w_M2.data(), e->Minv.data(),
              e->eps_chain.data(), e->N, nullptr, e->merged.data()};
    emu_launch(upd_thunk, &a, 1, 256);
    int it = 0;
    pooled_state_read(e->state.data(), eps_out, &it, nullptr, nullptr);
    for (int d = 0; d < e->D; ++d) minv_out[d] = e->Minv[d];
    for (int k = 0; k < 2 + 2 * e->D; ++k) merged_out[k] = e->merged[k];
    for (long long c = 0; c < e->N; ++c)
        if (e->eps_chain[c] != *eps_out) return -1;
    return it;
}
extern "C" void emu_pooled_destroy(void* h) { delete static_cast<PooledHandle*>(h); }
