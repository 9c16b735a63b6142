// simt_emu.cpp -- a minimal CPU emulator of CUDA's warp-synchronous execution model, enough to run the product's NUTS
// kernel SOURCE (advancedhmc.jl_b200/csrc/ahmc_nuts_kernel.cuh, unmodified) on the host: every CUDA thread of a block is
// a host thread; the 32 threads of a warp meet at a barrier in every shuffle / vote / __syncwarp, which is exactly the
// convergence the kernel's warp-uniform control flow guarantees on the device.  Blocks run one after another.
// TEST INFRASTRUCTURE ONLY (tests/test_simt_emulation.py): it lets kernel changes be checked against the oracle without
// a GPU; it says nothing about performance.
#include <pthread.h>

#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "cuda_runtime.h"
#include "emu_smem.h"

thread_local EmuUint3 threadIdx = {0, 0, 0}, blockIdx = {0, 0, 0};
EmuUint3 blockDim = {1, 1, 1}, gridDim = {1, 1, 1};

namespace {
struct Warp {
    pthread_barrier_t bar;
    uint64_t slot[32];
    double slot_b[32];
    unsigned pred[32];
};
thread_local Warp* tls_warp = nullptr;
thread_local int tls_lane = 0;
thread_local pthread_barrier_t* tls_block_bar = nullptr;
}  // namespace

void __syncthreads() { pthread_barrier_wait(tls_block_bar); }
static std::atomic<int> g_block_or{0};  // blocks run one at a time
int __syncthreads_or(int pred) {
    if (pred) g_block_or.store(1);
    pthread_barrier_wait(tls_block_bar);
    const int r = g_block_or.load();
    pthread_barrier_wait(tls_block_bar);
    if (threadIdx.x == 0) g_block_or.store(0);
    pthread_barrier_wait(tls_block_bar);
    return r;
}
unsigned atomicAdd(unsigned* addr, unsigned v) { return std::atomic_ref<unsigned>(*addr).fetch_add(v); }

int emu_lane() { return tls_lane; }
void emu_syncwarp() { pthread_barrier_wait(&tls_warp->bar); }
unsigned emu_ballot(bool p) {
    Warp* w = tls_warp;
    w->pred[tls_lane] = p ? 1u : 0u;
    pthread_barrier_wait(&w->bar);
    unsigned m = 0;
    for (int i = 0; i < 32; ++i) m |= w->pred[i] << i;
    pthread_barrier_wait(&w->bar);
    return m;
}
uint64_t emu_shfl(uint64_t bits, int src_lane) {
    Warp* w = tls_warp;
    w->slot[tls_lane] = bits;
    pthread_barrier_wait(&w->bar);
    const uint64_t out = w->slot[src_lane & 31];
    pthread_barrier_wait(&w->bar);
    return out;
}
unsigned emu_reduce_max(unsigned mask, unsigned v) {
    Warp* w = tls_warp;
    w->slot[tls_lane] = v;
    pthread_barrier_wait(&w->bar);
    unsigned m = 0;
    for (int i = 0; i < 32; ++i)
        if ((mask >> i) & 1u) m = w->slot[i] > m ? (unsigned)w->slot[i] : m;
    pthread_barrier_wait(&w->bar);
    return m;
}
int atomicOr(int* addr, int v) { return std::atomic_ref<int>(*addr).fetch_or(v); }
void emu_gather2(double a, double b, double* a32, double* b32) {
    Warp* w = tls_warp;
    std::memcpy(&w->slot[tls_lane], &a, 8);
    w->slot_b[tls_lane] = b;
    pthread_barrier_wait(&w->bar);
    std::memcpy(a32, w->slot, 32 * 8);
    std::memcpy(b32, w->slot_b, 32 * 8);
    pthread_barrier_wait(&w->bar);
}
int atomicMin(int* addr, int v) {
    std::atomic_ref<int> a(*addr);
    int old = a.load();
    while (old > v && !a.compare_exchange_weak(old, v)) {
    }
    return old;
}

namespace ahmc {
void emu_reset_barriers();             // (below) forget the previous block's mbarriers
void emu_check_barriers_at_exit(int);  // (below) no bulk copy may still be in flight when a block exits
}

// ---- the launch's dynamic shared memory (emu_smem.h): exact size, poisoned before every block, guarded on both sides
namespace {
unsigned char* g_smem = nullptr;  // [g_smem, g_smem + g_smem_bytes): the launch's dynamic shared memory
size_t g_smem_bytes = 0;
const char* g_smem_kernel = "";
int g_poison = EMU_POISON_NAN;
constexpr uint64_t kPoisonNan = 0x7ff8badc0ffee5a5ull;  // a quiet NaN whose payload is easy to recognise in a dump
uint64_t poison_word(size_t i) {
    if (g_poison == EMU_POISON_HUGE) {
        const double v = (i & 1) ? -1e300 : 1e300;
        uint64_t b;
        std::memcpy(&b, &v, 8);
        return b;
    }
    return kPoisonNan;
}
void poison_fill() {
    unsigned char* lo = g_smem - kEmuSmemGuard;
    const size_t words = (2 * kEmuSmemGuard + g_smem_bytes + 7) / 8;
    for (size_t i = 0; i < words; ++i) {
        const uint64_t w = poison_word(i);
        std::memcpy(lo + 8 * i, &w, 8);
    }
}
void guard_check(int block) {
    unsigned char* lo = g_smem - kEmuSmemGuard;
    const size_t end = 2 * kEmuSmemGuard + g_smem_bytes;
    for (size_t off = 0; off < end; ++off) {
        if (off == kEmuSmemGuard) off = kEmuSmemGuard + g_smem_bytes;  // (the launch's own bytes may hold anything)
        if (off >= end) break;
        const uint64_t w = poison_word(off / 8);
        if (lo[off] != reinterpret_cast<const unsigned char*>(&w)[off % 8]) {
            const long long rel = (long long)off - (long long)kEmuSmemGuard;
            std::fprintf(stderr, "[simt_emu] %s block %d wrote shared memory outside its %zu-byte launch: byte offset %lld\n", g_smem_kernel,
                         block, g_smem_bytes, rel);
            std::abort();
        }
    }
}
}  // namespace
void emu_smem_begin(unsigned char* base, size_t bytes, size_t static_bytes, const char* kernel) {
    if (bytes + static_bytes > kEmuSmemLimit) {
        std::fprintf(stderr, "[simt_emu] %s asks for %zu bytes of dynamic + %zu of static shared memory: more than the %zu a block may have\n",
                     kernel, bytes, static_bytes, kEmuSmemLimit);
        std::abort();
    }
    if ((reinterpret_cast<uintptr_t>(base) & 127u) != 0) {
        std::fprintf(stderr, "[simt_emu] %s: the dynamic shared memory must start 128-byte aligned\n", kernel);
        std::abort();
    }
    g_smem = base;
    g_smem_bytes = bytes;
    g_smem_kernel = kernel;
}
void emu_smem_end() {
    g_smem = nullptr;
    g_smem_bytes = 0;
    g_smem_kernel = "";
}
extern "C" void emu_set_poison(int mode) { g_poison = mode; }
extern "C" int emu_get_poison() { return g_poison; }
bool emu_in_smem(const void* p, size_t bytes) {
    const unsigned char* c = static_cast<const unsigned char*>(p);
    return g_smem && c >= g_smem && bytes <= g_smem_bytes && (size_t)(c - g_smem) <= g_smem_bytes - bytes;
}
const char* emu_smem_kernel() { return g_smem_kernel; }

// run `kernel(args)` for a 1-D grid of `blocks` blocks of `threads` threads (threads % 32 == 0)
void emu_launch(void (*kernel)(const void*), const void* args, int blocks, int threads) {
    blockDim = {(unsigned)threads, 1, 1};
    gridDim = {(unsigned)blocks, 1, 1};
    const int nwarps = threads / 32;
    for (int b = 0; b < blocks; ++b) {
        ahmc::emu_reset_barriers();
        if (g_smem) poison_fill();
        std::vector<Warp> warps(nwarps);
        for (auto& w : warps) pthread_barrier_init(&w.bar, nullptr, 32);
        pthread_barrier_t block_bar;
        pthread_barrier_init(&block_bar, nullptr, threads);
        std::vector<std::thread> ts;
        ts.reserve(threads);
        for (int t = 0; t < threads; ++t)
            ts.emplace_back([&, t, b] {
                threadIdx = {(unsigned)t, 0, 0};
                blockIdx = {(unsigned)b, 0, 0};
                tls_warp = &warps[t / 32];
                tls_lane = t % 32;
                tls_block_bar = &block_bar;
                kernel(args);
            });
        for (auto& th : ts) th.join();
        for (auto& w : warps) pthread_barrier_destroy(&w.bar);
        pthread_barrier_destroy(&block_bar);
        ahmc::emu_check_barriers_at_exit(b);
        if (g_smem) guard_check(b);
    }
}

// ---- mbarrier / bulk copy / fp64 MMA contracts of the kernels' PTX wrappers (ahmc_device.cuh) --------------------------
//   * an mbarrier is (completed phases, pending arrivals, pending transaction bytes); `mbar_wait(parity)` returns once
//     the phase of that parity has completed; `mbar_init` on an invalidated barrier re-arms it;
//   * `bulk_g2s` copies synchronously and completes its bytes on the barrier;
//   * `dmma` is `mma.sync.aligned.m8n8k4.row.col.f64`: lane l holds A[l/4][l%4], B[l%4][l/4] and C[l/4][2(l%4)+{0,1}].
// Every use is checked against the PTX ISA's rules, and a violation aborts naming the rule (the device would fault, hang
// or corrupt shared memory instead):
//   * a barrier is 8-byte aligned, inside the launch's dynamic shared memory, initialised with a count in 1 .. 2^20-1,
//     and not initialised again before it is invalidated; arrive / expect_tx / wait / complete_tx need a live barrier;
//   * an arrival needs a pending arrival (the phase cannot complete twice), pending tx bytes stay within 2^20-1,
//     and a barrier is invalidated only between phases (no arrivals and no bytes pending);
//   * a bulk copy has a 16-byte aligned source and destination, a size that is a positive multiple of 16, and lands
//     inside the launch's dynamic shared memory; no copy is in flight when the block exits.
namespace ahmc {
// An mbarrier lives in the kernel's shared memory as one 64-bit word; here: bits 0..11 completed phases, 12..31 pending
// arrivals of the current phase, 32..63 pending transaction bytes (biased by 2^31: complete_tx may precede expect_tx).
// The expected arrival count and the state of each barrier are kept beside it (indexed by its address).
namespace {
constexpr uint64_t kTxBias = 1ull << 31;
constexpr int64_t kTxMax = (1 << 20) - 1;
constexpr uint32_t kCountMax = (1u << 20) - 1;
struct BarInfo {
    uint64_t* bar;
    std::atomic<uint32_t> count;
    std::atomic<int> live;  // initialised and not invalidated since
};
BarInfo bar_info[16];
std::atomic<int> n_bar_info{0};
[[noreturn]] void violation(const char* what, const void* bar) {
    std::fprintf(stderr, "[simt_emu] %s: %s (thread %u block %u barrier %p)\n", emu_smem_kernel(), what, threadIdx.x, blockIdx.x, bar);
    std::abort();
}
BarInfo* find_bar(const uint64_t* bar) {
    for (int i = 0; i < n_bar_info.load(); ++i)
        if (bar_info[i].bar == bar) return &bar_info[i];
    return nullptr;
}
void check_placement(const uint64_t* bar) {
    if ((reinterpret_cast<uintptr_t>(bar) & 7u) != 0) violation("mbarrier not 8-byte aligned", bar);
    if (!emu_in_smem(bar, 8)) violation("mbarrier outside the launch's dynamic shared memory", bar);
}
BarInfo& live_bar(uint64_t* bar, const char* op) {
    check_placement(bar);
    BarInfo* i = find_bar(bar);
    if (!i || !i->live.load()) {
        static thread_local char msg[96];
        std::snprintf(msg, sizeof msg, "%s on an mbarrier that is not initialised (or was invalidated)", op);
        violation(msg, bar);
    }
    return *i;
}
// apply (arrivals, +/- bytes) atomically; complete the phase when both reach zero
void bar_update(uint64_t* bar, uint32_t arrivals, int64_t tx, const char* op) {
    BarInfo& info = live_bar(bar, op);
    std::atomic_ref<uint64_t> b(*bar);
    uint64_t old = b.load(), neu;
    do {
        uint64_t phases = old & 0xfffu, pend = (old >> 12) & 0xfffffu;
        int64_t bytes = (int64_t)(old >> 32) - (int64_t)kTxBias + tx;
        if (arrivals > pend) violation("arrival on an mbarrier with no arrivals pending in its phase", bar);
        if (bytes > kTxMax || bytes < -kTxMax) violation("more than 2^20-1 transaction bytes pending on an mbarrier", bar);
        pend -= arrivals;
        if (pend == 0 && bytes == 0) {
            phases = (phases + 1) & 0xfffu;
            pend = info.count.load();
        }
        neu = phases | (pend << 12) | ((uint64_t)(bytes + (int64_t)kTxBias) << 32);
    } while (!b.compare_exchange_weak(old, neu));
}
}  // namespace
void emu_reset_barriers() {
    for (int i = 0; i < 16; ++i) bar_info[i].live.store(0);
    n_bar_info.store(0);
}
void emu_check_barriers_at_exit(int block) {
    for (int i = 0; i < n_bar_info.load(); ++i) {
        if (!bar_info[i].live.load()) continue;
        const uint64_t v = std::atomic_ref<uint64_t>(*bar_info[i].bar).load();
        if ((int64_t)(v >> 32) - (int64_t)kTxBias != 0) {
            std::fprintf(stderr, "[simt_emu] %s block %d exits with bulk-copy bytes pending on mbarrier %p\n", emu_smem_kernel(), block,
                         (void*)bar_info[i].bar);
            std::abort();
        }
    }
}
void mbar_init(uint64_t* bar, int count) {  // thread 0 only, before the block barrier
    check_placement(bar);
    if (count < 1 || (uint32_t)count > kCountMax) violation("mbarrier initialised with a count outside 1 .. 2^20-1", bar);
    BarInfo* i = find_bar(bar);
    if (i && i->live.load()) violation("mbarrier initialised again without being invalidated first", bar);
    if (!i) {
        const int k = n_bar_info.load();
        if (k == 16) violation("more than 16 mbarriers in one block", bar);
        i = &bar_info[k];
        i->bar = bar;
        n_bar_info.store(k + 1);
    }
    i->count.store((uint32_t)count);
    std::atomic_ref<uint64_t>(*bar).store(((uint64_t)count << 12) | (kTxBias << 32));
    i->live.store(1);
}
void mbar_fence_init() {}
void mbar_inval(uint64_t* bar) {
    BarInfo& i = live_bar(bar, "mbarrier.inval");
    const uint64_t v = std::atomic_ref<uint64_t>(*bar).load();
    if (((v >> 12) & 0xfffffu) != i.count.load() || (int64_t)(v >> 32) != (int64_t)kTxBias)
        violation("mbarrier invalidated with arrivals or transaction bytes still pending", bar);
    i.live.store(0);
}
void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { bar_update(bar, 1, (int64_t)bytes, "mbarrier.arrive.expect_tx"); }
void mbar_arrive(uint64_t* bar) { bar_update(bar, 1, 0, "mbarrier.arrive"); }
void mbar_wait(uint64_t* bar, uint32_t parity) {
    live_bar(bar, "mbarrier.try_wait");
    // spin briefly, then sleep: a block is 256 host threads on a handful of cores, and waiters must not starve the workers
    for (int spins = 0; (uint32_t)(std::atomic_ref<uint64_t>(*bar).load() & 1u) == parity; ++spins) {
        if (spins < 16) std::this_thread::yield();
        else std::this_thread::sleep_for(std::chrono::microseconds(50));
        if (spins == 400000) {  // ~20 s: a protocol error in the kernel under test -- say where instead of hanging the suite
            const uint64_t v = std::atomic_ref<uint64_t>(*bar).load();
            std::fprintf(stderr, "[simt_emu] mbar_wait stuck: thread %u block %u barrier %p parity %u state phases=%llu pending=%llu tx=%lld\n",
                         threadIdx.x, blockIdx.x, (void*)bar, parity, (unsigned long long)(v & 0xfffu),
                         (unsigned long long)((v >> 12) & 0xfffffu), (long long)(v >> 32) - (long long)kTxBias);
            std::abort();
        }
    }
}
void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    if ((reinterpret_cast<uintptr_t>(src) & 15u) != 0) violation("cp.async.bulk source not 16-byte aligned", bar);
    if ((reinterpret_cast<uintptr_t>(dst) & 15u) != 0) violation("cp.async.bulk destination not 16-byte aligned", bar);
    if (bytes == 0 || (bytes & 15u) != 0) violation("cp.async.bulk size not a positive multiple of 16", bar);
    if (!emu_in_smem(dst, bytes)) violation("cp.async.bulk destination outside the launch's dynamic shared memory", bar);
    live_bar(bar, "cp.async.bulk complete_tx");
    std::memcpy(dst, src, bytes);
    bar_update(bar, 0, -(int64_t)bytes, "cp.async.bulk complete_tx");
}
void dmma(double& d0, double& d1, double a, double b) {
    double A[32], B[32];
    emu_gather2(a, b, A, B);
    const int lane = emu_lane(), row = lane >> 2, c0 = 2 * (lane & 3);
    for (int k = 0; k < 4; ++k) {
        d0 = fma(A[row * 4 + k], B[c0 * 4 + k], d0);
        d1 = fma(A[row * 4 + k], B[(c0 + 1) * 4 + k], d1);
    }
}
}  // namespace ahmc
