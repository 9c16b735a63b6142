// ahmc_device.cuh -- device-side building blocks shared by every kernel of libahmc_b200 (sm_90a).
//
// Work decomposition ("group-distributed vectors"): one chain is owned by a GROUP of G consecutive
// lanes of a warp (G in {4,8,16,32}); lane l of the group holds E coordinates d = l + G*e, e < E, so a
// chain's D <= G*E doubles live in registers for the whole trajectory and every global access of the
// group is a run of G consecutive doubles (Julia column-major D x N: a chain is contiguous).  Per-chain
// scalars (log pi, kinetic energy, U-turn dots) are xor-butterfly shuffles inside the group, so all
// lanes of a group hold bit-identical sums.  No shared memory, no block barrier on the Unit/Diag path.
//
// Reference semantics implemented here (citations relative to the AdvancedHMC.jl checkout):
//   dH/dtheta = (lp, -grad lp)        src/hamiltonian.jl:45-48
//   dH/dr, neg_energy                 src/hamiltonian.jl:50-68, 155-184
//   PhasePoint -Inf mapping, isfinite src/hamiltonian.jl:95-104, 141-142
//   one leapfrog step                 src/integrator.jl:233-247  (+ temper :198-209)
#pragma once
#if defined(__CUDACC_RTC__)
// run-time compilation of the user-model kernels (ahmc_user.cu): no host headers are available to NVRTC
typedef unsigned char uint8_t;
typedef int int32_t;
typedef unsigned int uint32_t;
typedef long long int64_t;
typedef unsigned long long uint64_t;
#define CUDART_INF __longlong_as_double(0x7ff0000000000000LL)
#define CUDART_NAN __longlong_as_double(0xfff8000000000000LL)
#else
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>
#endif

#include "../../include/ahmc_b200.h"

#if defined(AHMC_NVRTC_USER_MODEL)
// The user's target (AHMC_MODEL_USER, ahmc_model_create_user): CUDA source handed over at run time defines ONE of
//   __device__ double ahmc_user_logp_grad(const double* theta, double* grad, int D, const double* params);
//       log pi(theta) of one chain; writes the PLUS gradient into grad[0..D).  theta / grad are D-vectors in shared memory;
//       one lane of the chain's group runs it.
//   __device__ double ahmc_user_coord(int d, double theta_d, const double* params, double* grad_d);      (and #define AHMC_USER_COORDWISE)
//       for targets that are a sum over coordinates: the term of coordinate d and its derivative; every lane evaluates
//       its own coordinates and the terms are summed by warp shuffles (as fast as the built-in diagonal targets).
//   __device__ double ahmc_user_logp_grad_group(const double* theta, double* grad, int D, const double* params,
//                                               ahmc_group g);                                      (and #define AHMC_USER_GROUPWISE)
//       the general target evaluated by ALL G lanes of the chain's group together (g.lane in 0..G-1, g.size = G).  theta
//       (read-only) and grad are the group's two shared-memory D-vectors; each grad[d] (PLUS gradient) is written by
//       exactly one lane, whichever the user picks.  Returns the calling lane's share of log pi: the library sums the G
//       shares in a fixed order (Grp::sum) and adds c0.  The library syncs the group before the call (theta staged) and
//       after it (before the lanes read grad).  Inside, the group may use ahmc_group_sum / _bcast / _sync (defined at the
//       end of this file).
#if defined(AHMC_USER_COORDWISE) && defined(AHMC_USER_GROUPWISE)
#error "the user target defines both AHMC_USER_COORDWISE and AHMC_USER_GROUPWISE: select one contract"
#endif
struct ahmc_group {
    int lane;  // 0 .. size-1: this lane's index in the chain's group
    int size;  // G in {4, 8, 16, 32}
};
__device__ double ahmc_user_logp_grad(const double* theta, double* grad, int D, const double* params);
__device__ double ahmc_user_coord(int d, double theta_d, const double* params, double* grad_d);
__device__ double ahmc_user_logp_grad_group(const double* theta, double* grad, int D, const double* params, ahmc_group g);
#endif

namespace ahmc {

constexpr unsigned FULL = 0xffffffffu;

struct ModelDev {
    int kind;
    int D;
    const double* p0;  // DIAG_GAUSS: mean; DENSE_GAUSS: mean; USER: the user's parameter array
    const double* p1;  // DIAG_GAUSS: w = 1/s^2 ; DENSE_GAUSS: precision D x D (column-major)
    double c0;
    const void* user;  // USER: host-side handle of the run-time compiled kernels (never dereferenced on the device)
    const double* p1_coop;  // DENSE_GAUSS, nullable: the precision with padded columns (leading dimension coop_lds(D), zero
                            // filled) -- the cooperative products then fetch a whole chunk of columns with ONE bulk copy
};

// doubles of per-group shared-memory slab a kernel family needs: dense operators stage one D-vector, a user target a
// second one for the gradient
template <int MODEL>
__host__ __device__ constexpr int slab_vectors() { return MODEL == AHMC_MODEL_USER ? 2 : 1; }

// The template metric kind of a per-chain Dense metric (chain_stride >= D*D: chain c's M^-1 and factor at chain_stride*c),
// internal to the kernels -- the C ABI's kind stays AHMC_METRIC_DENSE.  Its kernels are instantiations of their own, so the
// shared-matrix Dense kernels are compiled exactly as before: only these index the matrices by the chain, and they read
// them with coherent loads, because the in-launch WelfordCov warm-up writes a chain's rows during the launch.
constexpr int kMetricDenseChain = 3;
__host__ __device__ constexpr bool is_dense_metric(int kind) { return kind == AHMC_METRIC_DENSE || kind == kMetricDenseChain; }

struct MetricDev {
    int kind;
    const double* Minv;
    long long chain_stride;
    const double* cholU;
    const double* Minv_coop;   // Dense, nullable: Minv / cholU with padded columns (see ModelDev::p1_coop)
    const double* cholU_coop;
};
// the template metric kind a launch instantiates for this metric: kMetricDenseChain for a per-chain Dense metric
__host__ __device__ inline int metric_form(const MetricDev& m) {
    return m.kind == AHMC_METRIC_DENSE && m.chain_stride != 0 ? kMetricDenseChain : m.kind;
}

// ------------------------------------------------------------------------------------------------
// group collectives
// ------------------------------------------------------------------------------------------------
template <int G>
struct Grp {
    static __device__ __forceinline__ double sum(double v) {
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
        return v;
    }
    static __device__ __forceinline__ double max(double v) {
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(FULL, v, o));
        return v;
    }
    // value held by lane `src` (0..G-1) of my group
    static __device__ __forceinline__ double bcast(double v, int src) { return __shfl_sync(FULL, v, src, G); }
    static __device__ __forceinline__ unsigned gmask() {
        if (G == 32) return FULL;
        unsigned lane = threadIdx.x & 31u;
        return ((1u << G) - 1u) << (lane & ~(unsigned)(G - 1));
    }
    static __device__ __forceinline__ bool all(bool p) {
        unsigned b = __ballot_sync(FULL, p);
        unsigned m = gmask();
        return (b & m) == m;
    }
    static __device__ __forceinline__ bool any(bool p) {
        unsigned b = __ballot_sync(FULL, p);
        return (b & gmask()) != 0u;
    }
};

__device__ __forceinline__ bool finite_d(double x) { return (__double2hiint(x) & 0x7ff00000) != 0x7ff00000; }
// exponent field of x >= biased exponent `ebits` (pre-shifted by 20); NaN/Inf always "big"
__device__ __forceinline__ bool big_d(double x, int ebits) { return (__double2hiint(x) & 0x7ff00000) >= ebits; }
__device__ __forceinline__ double map_nonfinite(double v) { return finite_d(v) ? v : -CUDART_INF; }
constexpr int expo_bits(int e) { return (1023 + e) << 20; }

// ------------------------------------------------------------------------------------------------
// group-distributed vector I/O:  element e of lane l  <->  d = l + G*e
// ------------------------------------------------------------------------------------------------
template <int G, int E>
__device__ __forceinline__ void vload(double (&x)[E], const double* __restrict__ base, int l, int D) {
#pragma unroll
    for (int e = 0; e < E; ++e) {
        int d = l + G * e;
        x[e] = (d < D) ? __ldg(base + d) : 0.0;
    }
}
template <int G, int E>
__device__ __forceinline__ void vload_nc(double (&x)[E], const double* base, int l, int D) {
#pragma unroll
    for (int e = 0; e < E; ++e) {
        int d = l + G * e;
        x[e] = (d < D) ? base[d] : 0.0;
    }
}
template <int G, int E>
__device__ __forceinline__ void vstore(double* base, const double (&x)[E], int l, int D) {
#pragma unroll
    for (int e = 0; e < E; ++e) {
        int d = l + G * e;
        if (d < D) base[d] = x[e];
    }
}

// ------------------------------------------------------------------------------------------------
// lane-contiguous vector I/O (K1 fast path, G = 32): lane l owns V = min(E, 4) CONSECUTIVE doubles of every
// 32*V-wide block, element e  <->  d = 32*V*(e / V) + V*l + (e % V).  A lane moves its V doubles with 128-bit
// accesses instead of V scalar ones (sm_90 has no wider per-thread load or store: V = 4 is two of them, at d0 and
// d0 + 2).  Used for FULL tiles only (D == 32*E, 8*V-byte aligned rows; the host checks): no bounds predicate, no
// zero fill.
// ------------------------------------------------------------------------------------------------
template <int E>
struct Contig {
    static constexpr int V = E >= 4 ? 4 : E;
    static __device__ __forceinline__ int dim(int l, int e) { return 32 * V * (e / V) + V * l + (e % V); }
};
template <int E>
__device__ __forceinline__ void cload(double (&x)[E], const double* base, int l, int D) {
    constexpr int V = Contig<E>::V;
#pragma unroll
    for (int b = 0; b < E / V; ++b) {
        const int d0 = 32 * V * b + V * l;
        if constexpr (V == 4) {
            const double2 v0 = *reinterpret_cast<const double2*>(base + d0);
            const double2 v1 = *reinterpret_cast<const double2*>(base + d0 + 2);
            x[4 * b] = v0.x; x[4 * b + 1] = v0.y; x[4 * b + 2] = v1.x; x[4 * b + 3] = v1.y;
        } else if constexpr (V == 2) {
            double2 v = *reinterpret_cast<const double2*>(base + d0);
            x[2 * b] = v.x; x[2 * b + 1] = v.y;
        } else {
            x[b] = base[d0];
        }
    }
}
template <int E>
__device__ __forceinline__ void cstore(double* base, const double (&x)[E], int l, int D) {
    constexpr int V = Contig<E>::V;
#pragma unroll
    for (int b = 0; b < E / V; ++b) {
        const int d0 = 32 * V * b + V * l;
        if constexpr (V == 4) {
            *reinterpret_cast<double2*>(base + d0) = make_double2(x[4 * b], x[4 * b + 1]);
            *reinterpret_cast<double2*>(base + d0 + 2) = make_double2(x[4 * b + 2], x[4 * b + 3]);
        } else if constexpr (V == 2) {
            *reinterpret_cast<double2*>(base + d0) = make_double2(x[2 * b], x[2 * b + 1]);
        } else {
            base[d0] = x[b];
        }
    }
}
// vector load in the layout a trajectory functor asks for (coefficients follow the state's layout)
template <bool CONTIG, int G, int E>
__device__ __forceinline__ void lload(double (&x)[E], const double* base, int l, int D) {
    if constexpr (CONTIG) cload<E>(x, base, l, D);
    else vload<G, E>(x, base, l, D);
}
template <bool CONTIG, int G, int E>
__device__ __forceinline__ bool lin(int l, int e, int D) { return CONTIG ? true : (l + G * e) < D; }

// max over the group of a 32-bit unsigned (one REDUX for a full warp)
template <int G>
__device__ __forceinline__ unsigned grp_umax(unsigned v) {
    if constexpr (G == 32) {
        return __reduce_max_sync(FULL, v);
    } else {
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) {
            const unsigned w = __shfl_xor_sync(FULL, v, o);
            v = w > v ? w : v;
        }
        return v;
    }
}

// y = A x for a D x D column-major matrix in global memory, x/y group-distributed.
// xs: this group's private slab of >= D doubles in shared memory.  (Dense metric / dense Gaussian
// target; the register-tiled CTA kernel for these shapes is a separate code path.)
template <int G, int E>
__device__ __forceinline__ void matvec(const double* __restrict__ A, int D, const double (&x)[E], double (&y)[E],
                                       double* xs, int l) {
    __syncwarp();
#pragma unroll
    for (int e = 0; e < E; ++e) {
        int d = l + G * e;
        if (d < D) xs[d] = x[e];
        y[e] = 0.0;
    }
    __syncwarp();
    for (int k = 0; k < D; ++k) {
        double xk = xs[k];
        const double* col = A + (long long)D * k;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            int d = l + G * e;
            if (d < D) y[e] = fma(__ldg(col + d), xk, y[e]);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// mbarrier / bulk-copy / fp64-MMA wrappers (K4's tile product, ahmc_dense.cu, and the cooperative products below).
// Under the CPU SIMT emulation the harness provides them with the same contracts (tests/simt_emu/simt_emu.cpp): an
// mbarrier is (completed phases, pending arrivals, pending transaction bytes), `mbar_wait(parity)` returns once the phase
// of that parity has completed, `bulk_g2s` copies synchronously and completes its bytes on the barrier, `dmma` is
// mma.sync.aligned.m8n8k4.row.col.f64 (wgmma has no f64 kind): lane l holds A[l/4][l%4], B[l%4][l/4], C[l/4][2(l%4)+{0,1}].
// ------------------------------------------------------------------------------------------------
#ifdef AHMC_SIMT_EMULATION
void mbar_init(uint64_t* bar, int count);
void mbar_inval(uint64_t* bar);
void mbar_fence_init();
void mbar_expect_tx(uint64_t* bar, uint32_t bytes);
void mbar_arrive(uint64_t* bar);
void mbar_wait(uint64_t* bar, uint32_t parity);
void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar);
void dmma(double& d0, double& d1, double a, double b);
#else
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_inval(uint64_t* bar) { asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}
#endif  // AHMC_SIMT_EMULATION

// ------------------------------------------------------------------------------------------------
// CTA-cooperative dense products for kernels that own ONE chain per warp (G = 32) and whose warps can rendezvous (the
// NUTS form for dense operators): all kCoopWarps warps of the block call at the same point, each with its own chain's
// vector.  The matrix is streamed from L2 into shared memory ONCE per block, coop_kc<E>() columns per stage, by bulk copies
// (cp.async.bulk, one per column, issued by warp 0, completion on the stage's "full" mbarrier); a stage is handed back
// through its "empty" mbarrier (one arrival per warp), which only the issuing warp waits on -- no block barrier inside the
// product.  Y[D x 8] = A X[D x 8] runs on the fp64 tensor pipe: a warp owns 16-row blocks q = w, w + 8, ... ; lane
// (fr = l/4, fk = l%4) reads rows 16q + 2fr + {0,1} of column fk as ONE 128-bit shared load = the A fragments of two
// m8n8k4 tiles (tile j holds rows 16q + 2fr' + j, fr' = 0..7: which rows form a tile is free, C's rows follow), and the B
// fragment (the 8 chains' x at 4 consecutive k) as one 64-bit load: 3 shared loads per 4 DMMAs at D = 256.
// Shared-memory layout (doubles, from `base`): X slab [D][8] (transposed: the 8 chains' x[k] adjacent) | Y slab [8][D] |
// coop_stages(D) stages [coop_kc<E>()][lds] (lds = D rounded up to 16, + 4: the 16-row fragment blocks of a ragged D stay inside
// their column -- rows beyond D are read, never used -- column starts are 16-byte aligned and the 128-bit fragment loads of
// 4 columns fall into distinct banks) | 16 doubles of slack | 2 coop_stages(D) mbarriers.  Idle warps still take part.
// ------------------------------------------------------------------------------------------------
// matrix columns per stage = per bulk copy and per pair of barrier operations, by the kernel's layout (E coordinates per
// lane, D <= 32 E).  Beyond D = 256 the stages must shrink to fit the 227 KB of shared memory a block may have.
template <int E>
__host__ __device__ constexpr int coop_kc() { return E <= 8 ? 24 : 16; }
// stages of the L2 -> shared-memory pipeline (stages - 1 chunks in flight): the kernels that use it run one block per SM,
// so shared memory is there to spend on depth while a stage is D x 8 doubles
__host__ __device__ constexpr int coop_stages(int D) { return D <= 256 ? 3 : 2; }
constexpr int kCoopWarps = 8;    // warps (= chains) per block of the kernels that use it
constexpr int kCoopThreads = 32 * kCoopWarps;
__host__ __device__ constexpr int coop_lds(int D) { return ((D + 15) & ~15) + 4; }
__host__ __device__ constexpr int coop_stage_doubles(int D, int KC) { return KC * coop_lds(D); }
__host__ __device__ constexpr int coop_smem_doubles(int D, int KC) { return 2 * kCoopWarps * D + coop_stages(D) * coop_stage_doubles(D, KC) + 16 + 2 * coop_stages(D); }

// `ncols` columns (src + k*D, `rows` leading entries each) -> stage columns of leading dimension coop_lds(D); completes on
// `full`.  Called by ALL lanes of warp 0, converged.  bulk: 16-byte aligned source columns and an even number of rows.
// `padded` (nullable): the same columns in a copy of the matrix whose leading dimension already is coop_lds(D) -- the chunk
// is then ONE contiguous bulk copy instead of one per column (a bulk copy costs the copy engine of the SM a fixed time
// that 2 KB does not amortise).
__device__ __forceinline__ void coop_issue(double* stage, const double* __restrict__ src, const double* __restrict__ padded, int ncols,
                                           int rows, int D, bool bulk, uint64_t* full) {
    const int lane = threadIdx.x & 31;
    const int lds = coop_lds(D);
    if (padded) {
        if (lane == 0) {
            const uint32_t bytes = (uint32_t)(ncols * lds * 8);
            mbar_expect_tx(full, bytes);
            bulk_g2s(stage, padded, bytes, full);
        }
        return;
    }
    if (bulk) {
        if (lane == 0) mbar_expect_tx(full, (uint32_t)(ncols * rows * 8));
        if (lane < ncols) bulk_g2s(stage + lane * lds, src + (long long)lane * D, (uint32_t)(rows * 8), full);
    } else {
        for (int k = 0; k < ncols; ++k)
            for (int d = lane; d < rows; d += 32) stage[k * lds + d] = __ldg(src + (long long)k * D + d);
        __syncwarp();
        if (lane == 0) mbar_arrive(full);
    }
}
// (re)arm the pipeline's barriers for one cooperative call; thread 0, before the call's first block barrier.  The kernel
// initialises them once (coop_begin) so that every later call can invalidate and re-initialise: phases start at 0 per call.
__device__ __forceinline__ uint64_t* coop_bars(double* base, int D, int KC) {
    return reinterpret_cast<uint64_t*>(base + 2 * kCoopWarps * D + coop_stages(D) * coop_stage_doubles(D, KC) + 16);
}
__device__ __forceinline__ void coop_arm(uint64_t* bars, int S, bool first) {
    for (int s = 0; s < S; ++s) {
        if (!first) {
            mbar_inval(&bars[s]);
            mbar_inval(&bars[S + s]);
        }
        mbar_init(&bars[s], 1);               // full: the issuing lane's arrival (+ the copied bytes)
        mbar_init(&bars[S + s], kCoopWarps);  // empty: one arrival per warp
    }
    mbar_fence_init();
}
// once per kernel, by every thread of the block, before the first cooperative call
template <int E>
__device__ __forceinline__ void coop_begin(double* base, int D) {
    if (threadIdx.x == 0) coop_arm(coop_bars(base, D, coop_kc<E>()), coop_stages(D), true);
    __syncthreads();
}

template <int E>
__device__ __forceinline__ void matvec_coop(const double* __restrict__ A, const double* __restrict__ Ap, int D, const double (&x)[E],
                                            double (&y)[E], double* base, int l) {
    constexpr int nw = kCoopWarps, KC = coop_kc<E>();
    const int S = coop_stages(D);
    static_assert(nw == 8, "the DMMA tile has 8 columns: one per chain of the block");
    const int w = threadIdx.x >> 5;
    double* Xs = base;                 // [D][nw]
    double* Ys = base + nw * D;        // [nw][D]
    double* As = base + 2 * nw * D;    // S x [KC][lds]
    uint64_t* bars = coop_bars(base, D, KC);
    const int lds = coop_lds(D), stage_doubles = coop_stage_doubles(D, KC);
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int d = l + 32 * e;
        if (d < D) Xs[d * nw + w] = x[e];
    }
    if (threadIdx.x == 0) coop_arm(bars, S, false);
    __syncthreads();  // X slab and barriers visible; every warp has left the previous cooperative call
    const int nchunks = (D + KC - 1) / KC;
    const bool bulk = ((D & 1) == 0) && ((reinterpret_cast<unsigned long long>(A) & 15ull) == 0);
    auto chunk_cols = [&](int c) { return (D - c * KC < KC) ? D - c * KC : KC; };
    if (w == 0)
        for (int c = 0; c < S && c < nchunks; ++c)
            coop_issue(As + c * stage_doubles, A + (long long)D * c * KC, Ap ? Ap + (long long)lds * c * KC : nullptr, chunk_cols(c), D, D,
                       bulk, &bars[c]);
    constexpr int PBW = (E + 3) / 4;  // 16-row blocks per warp: ceil(D / 16) <= 2 E blocks over 8 warps
    double acc[PBW][2][2];            // [block][row 2fr + j][chain 2fk + jj]
#pragma unroll
    for (int p = 0; p < PBW; ++p) acc[p][0][0] = acc[p][0][1] = acc[p][1][0] = acc[p][1][1] = 0.0;
    const int fk = l & 3, fr = l >> 2;
    int stage = 0, pstage = 0;
    uint32_t par = 0, ppar = 0;
    for (int c = 0; c < nchunks; ++c) {
        mbar_wait(&bars[stage], par);  // chunk c has landed
        const double* as = As + stage * stage_doubles + 2 * fr;
        const int kc = chunk_cols(c);
        const double* xk = Xs + (c * KC) * nw + fr;
        if (kc == KC) {
#pragma unroll
            for (int ks = 0; ks < KC / 4; ++ks) {
                const int kl = 4 * ks + fk;
                const double b = xk[kl * nw];  // B[k][chain = fr]
#pragma unroll
                for (int p = 0; p < PBW; ++p) {
                    const int q = w + nw * p;
                    if (D >= 16 * nw * PBW || 16 * q < D) {  // (rows >= D of a ragged block: read, accumulated, never stored)
                        const double2 a2 = *reinterpret_cast<const double2*>(as + kl * lds + 16 * q);
                        dmma(acc[p][0][0], acc[p][0][1], a2.x, b);
                        dmma(acc[p][1][0], acc[p][1][1], a2.y, b);
                    }
                }
            }
        } else {  // the ragged last chunk: columns >= D contribute exact zeros
#pragma unroll
            for (int ks = 0; ks < KC / 4; ++ks) {
                const int kl = 4 * ks + fk;
                const bool kin = kl < kc;
                const double b = kin ? xk[kl * nw] : 0.0;
#pragma unroll
                for (int p = 0; p < PBW; ++p) {
                    const int q = w + nw * p;
                    if (16 * q < D) {
                        double2 a2 = make_double2(0.0, 0.0);
                        if (kin) a2 = *reinterpret_cast<const double2*>(as + kl * lds + 16 * q);
                        dmma(acc[p][0][0], acc[p][0][1], a2.x, b);
                        dmma(acc[p][1][0], acc[p][1][1], a2.y, b);
                    }
                }
            }
        }
        __syncwarp();
        if (l == 0) mbar_arrive(&bars[S + stage]);  // this warp is done with the stage
        // warp 0 refills the stage of the PREVIOUS chunk (its last readers are at most one chunk behind) with chunk c-1+S
        if (w == 0 && c >= 1 && c - 1 + S < nchunks) {
            mbar_wait(&bars[S + pstage], ppar);
            const int cn = c - 1 + S;
            coop_issue(As + pstage * stage_doubles, A + (long long)D * cn * KC, Ap ? Ap + (long long)lds * cn * KC : nullptr,
                       chunk_cols(cn), D, D, bulk, &bars[pstage]);
        }
        pstage = stage;
        ppar = par;
        if (++stage == S) {
            stage = 0;
            par ^= 1u;
        }
    }
#pragma unroll
    for (int p = 0; p < PBW; ++p) {
        const int row = 16 * (w + nw * p) + 2 * fr;
#pragma unroll
        for (int j = 0; j < 2; ++j)
            if (row + j < D) {
                Ys[(2 * fk) * D + row + j] = acc[p][j][0];
                Ys[(2 * fk + 1) * D + row + j] = acc[p][j][1];
            }
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int d = l + 32 * e;
        y[e] = (d < D) ? Ys[w * D + d] : 0.0;
    }
}

// matvec for a chain's own matrix (kMetricDenseChain), which the same launch may write: coherent loads, no read-only path
template <int G, int E>
__device__ __forceinline__ void matvec_coherent(const double* A, int D, const double (&x)[E], double (&y)[E], double* xs, int l) {
    __syncwarp();
#pragma unroll
    for (int e = 0; e < E; ++e) {
        int d = l + G * e;
        if (d < D) xs[d] = x[e];
        y[e] = 0.0;
    }
    __syncwarp();
    for (int k = 0; k < D; ++k) {
        double xk = xs[k];
        const double* col = A + (long long)D * k;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            int d = l + G * e;
            if (d < D) y[e] = fma(col[d], xk, y[e]);
        }
    }
}

// solve U x = z (U upper triangular, column-major) for a group-distributed vector; result in x.
// Back substitution, one pivot per iteration (metric.jl:311-320 `ldiv!(cholMinv, r)`).
template <int G, int E>
__device__ __forceinline__ void upper_solve(const double* __restrict__ U, int D, double (&x)[E], int l) {
    for (int i = D - 1; i >= 0; --i) {
        int le = i % G, ee = i / G;
        double xi = 0.0;
#pragma unroll
        for (int e = 0; e < E; ++e)
            if (e == ee) xi = x[e];
        xi = Grp<G>::bcast(xi, le) / __ldg(U + i + (long long)D * i);
        const double* col = U + (long long)D * i;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            int d = l + G * e;
            if (d == i)
                x[e] = xi;
            else if (d < i)
                x[e] = fma(-__ldg(col + d), xi, x[e]);
        }
    }
}

// upper_solve for a chain's own factor (kMetricDenseChain): coherent loads, as matvec_coherent
template <int G, int E>
__device__ __forceinline__ void upper_solve_coherent(const double* U, int D, double (&x)[E], int l) {
    for (int i = D - 1; i >= 0; --i) {
        int le = i % G, ee = i / G;
        double xi = 0.0;
#pragma unroll
        for (int e = 0; e < E; ++e)
            if (e == ee) xi = x[e];
        xi = Grp<G>::bcast(xi, le) / U[i + (long long)D * i];
        const double* col = U + (long long)D * i;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            int d = l + G * e;
            if (d == i)
                x[e] = xi;
            else if (d < i)
                x[e] = fma(-col[d], xi, x[e]);
        }
    }
}

// CTA-cooperative back substitution U X = Z for the block's 8 chains (see matvec_coop): blocked by 8 columns, last block
// first.  Per block: (1) every warp solves ITS chain's 8 x 8 diagonal system from the staged columns (lanes 0..7 hold the
// block's entries; 8 dependent steps of multiply-by-1/U_ii, shuffle, FMA); (2) after a block barrier the rows above the
// block are updated for ALL chains at once on the fp64 tensor pipe, Z[rows][8] -= U[rows, block] X[block][8], the 16-row
// blocks dealt round-robin to the warps as in matvec_coop.  The warp-private form above costs a serial chain of D pivots
// each waiting on L2 (~600 cycles x D per transition at D = 256, more than the whole tree of a short NUTS transition);
// the first cooperative version (pivot by pivot from shared memory) still spent 170 instructions per pivot per warp.
// x / U_ii is computed as x * (1 / U_ii): one rounding more than the reference's `ldiv!` (metric.jl:311-320).
// Only the upper triangle of U is ever used (what lies below may be anything, like the parent of Julia's `.U`).
template <int E>
__device__ __forceinline__ void upper_solve_coop(const double* __restrict__ U, const double* __restrict__ Up, int D, double (&x)[E],
                                                 double* base, int l) {
    constexpr int nw = kCoopWarps, KC = coop_kc<E>();
    const int S = coop_stages(D);
    const int w = threadIdx.x >> 5;
    double* Xs = base;               // [D][nw]: right-hand sides in, solutions out
    double* As = base + 2 * nw * D;  // S x [KC][lds]
    uint64_t* bars = coop_bars(base, D, KC);
    const int lds = coop_lds(D), stage_doubles = coop_stage_doubles(D, KC);
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int d = l + 32 * e;
        if (d < D) Xs[d * nw + w] = x[e];
    }
    if (threadIdx.x == 0) coop_arm(bars, S, false);
    __syncthreads();
    const int nb = (D + KC - 1) / KC;
    const bool bulk = ((D & 1) == 0) && ((reinterpret_cast<unsigned long long>(U) & 15ull) == 0);
    auto blk_cols = [&](int b) { return (D - b * KC < KC) ? D - b * KC : KC; };
    auto blk_rows = [&](int b) { return (b * KC + KC < D) ? b * KC + KC : D; };  // rows 0 .. end of the diagonal block
    // step j handles block b = nb - 1 - j
    if (w == 0)
        for (int j = 0; j < S && j < nb; ++j) {
            const int b = nb - 1 - j;
            coop_issue(As + j * stage_doubles, U + (long long)D * b * KC, Up ? Up + (long long)lds * b * KC : nullptr, blk_cols(b),
                       blk_rows(b), D, bulk, &bars[j]);
        }
    const int fk = l & 3, fr = l >> 2;
    int stage = 0;
    uint32_t par = 0;
    for (int j = 0; j < nb; ++j) {
        const int b = nb - 1 - j, k0 = b * KC, kc = blk_cols(b);
        mbar_wait(&bars[stage], par);
        const double* us = As + stage * stage_doubles;
        {   // (1) diagonal block, chain w: lane i < kc holds entry k0 + i
            const bool in = l < kc;
            double z = in ? Xs[(k0 + l) * nw + w] : 0.0;
            const double inv = in ? 1.0 / us[l * lds + k0 + l] : 0.0;
#pragma unroll
            for (int i = KC - 1; i >= 0; --i) {
                if (i < kc) {  // (uniform)
                    const double xi = __shfl_sync(FULL, z * inv, i);  // x_i = z_i / U_ii, final once every j > i is eliminated
                    if (l == i) z = xi;
                    else if (l < i) z = fma(-us[i * lds + k0 + l], xi, z);
                }
            }
            if (in) Xs[(k0 + l) * nw + w] = z;
        }
        __syncthreads();  // the block's solutions of all 8 chains are in the slab
        {   // (2) rows [0, k0) -= U[rows, block] * X[block]
            const int npb = (k0 + 15) >> 4;
            for (int q = w; q < npb; q += nw) {
                const int row = 16 * q + 2 * fr;
                double2 c0 = *reinterpret_cast<const double2*>(Xs + row * nw + 2 * fk);        // row,     chains 2fk, 2fk+1
                double2 c1 = *reinterpret_cast<const double2*>(Xs + (row + 1) * nw + 2 * fk);  // row + 1  (rows >= k0: read, never stored)
#pragma unroll
                for (int ks = 0; ks < KC / 4; ++ks) {
                    const int kl = 4 * ks + fk;
                    const bool kin = kl < kc;
                    const double bneg = kin ? -Xs[(k0 + kl) * nw + fr] : 0.0;
                    double2 a2 = make_double2(0.0, 0.0);
                    if (kin) a2 = *reinterpret_cast<const double2*>(us + kl * lds + row);
                    dmma(c0.x, c0.y, a2.x, bneg);
                    dmma(c1.x, c1.y, a2.y, bneg);
                }
                if (row < k0) *reinterpret_cast<double2*>(Xs + row * nw + 2 * fk) = c0;
                if (row + 1 < k0) *reinterpret_cast<double2*>(Xs + (row + 1) * nw + 2 * fk) = c1;
            }
        }
        __syncthreads();  // updated right-hand sides visible to the next block's diagonal solve; the stage is free
        if (w == 0 && j + S < nb) {
            const int bn = nb - 1 - (j + S);
            coop_issue(As + stage * stage_doubles, U + (long long)D * bn * KC, Up ? Up + (long long)lds * bn * KC : nullptr, blk_cols(bn),
                       blk_rows(bn), D, bulk, &bars[stage]);
        }
        if (++stage == S) {
            stage = 0;
            par ^= 1u;
        }
    }
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int d = l + 32 * e;
        if (d < D) x[e] = Xs[d * nw + w];
    }
    __syncthreads();  // every warp has its solution before the slab is reused
}

// ------------------------------------------------------------------------------------------------
// metric:  dH/dr and the kinetic lane-partial  sum_e r_e * (dH/dr)_e   (neg_energy = -sum/2)
// ------------------------------------------------------------------------------------------------
// METRIC: AHMC_METRIC_UNIT / _DIAG / _DENSE (one shared matrix), or kMetricDenseChain (chain c's own matrices)
template <int METRIC, int G, int E>
struct MetricOps {
    double Minv[E];  // Diag only
    const double* A; // Dense only: M^-1 (kMetricDenseChain: the chain's own)
    const double* U;
    const double *Ac, *Uc;  // their padded copies for the cooperative products (nullable)
    int D;
    double* coop;    // non-null: dense products are CTA-cooperative through this shared-memory region (matvec_coop)

    __device__ __forceinline__ void load(const MetricDev& m, long long chain, int l, int D_) {
        D = D_;
        coop = nullptr;
        A = m.Minv;
        U = m.cholU;
        Ac = m.Minv_coop;
        Uc = m.cholU_coop;
        if (METRIC == AHMC_METRIC_DIAG) {
            vload<G, E>(Minv, m.Minv + m.chain_stride * chain, l, D);
        } else if (METRIC == kMetricDenseChain) {
            A = m.Minv + m.chain_stride * chain;
            U = m.cholU ? m.cholU + m.chain_stride * chain : nullptr;
        }
    }
    // dr = dH/dr(r)   (hamiltonian.jl:50-68)
    __device__ __forceinline__ void dHdr(const double (&r)[E], double (&dr)[E], double* xs, int l) const {
        if (METRIC == AHMC_METRIC_UNIT) {
#pragma unroll
            for (int e = 0; e < E; ++e) dr[e] = r[e];
        } else if (METRIC == AHMC_METRIC_DIAG) {
#pragma unroll
            for (int e = 0; e < E; ++e) dr[e] = Minv[e] * r[e];
        } else if (METRIC == kMetricDenseChain) {
            matvec_coherent<G, E>(A, D, r, dr, xs, l);
        } else {
            if (G == 32 && coop) matvec_coop<E>(A, Ac, D, r, dr, coop, l);
            else matvec<G, E>(A, D, r, dr, xs, l);
        }
    }
    // r from standard normals z (metric.jl:290-320)
    __device__ __forceinline__ void rand_momentum(double (&r)[E], int l) const {
        if (METRIC == AHMC_METRIC_DIAG) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                int d = l + G * e;
                r[e] = (d < D) ? r[e] / sqrt(Minv[e]) : 0.0;
            }
        } else if (METRIC == AHMC_METRIC_DENSE) {
            if (G == 32 && coop) upper_solve_coop<E>(U, Uc, D, r, coop, l);
            else upper_solve<G, E>(U, D, r, l);
        } else if (METRIC == kMetricDenseChain) {
            upper_solve_coherent<G, E>(U, D, r, l);
        }
    }
};

// ------------------------------------------------------------------------------------------------
// models:  eval(theta) -> g = MINUS grad log pi (what PhasePoint caches), returns log pi (all lanes)
// ------------------------------------------------------------------------------------------------
template <int MODEL, int G, int E>
struct ModelOps {
    double m[E];
    double w[E];
    const double* P;
    const double* Pc;  // DENSE_GAUSS: padded copy of P for the cooperative product (nullable)
    double c0;
    int D;
    double* coop;  // see MetricOps

    __device__ __forceinline__ void load(const ModelDev& md, int l, int D_) {
        D = D_;
        coop = nullptr;
        c0 = md.c0;
        P = md.p1;
        Pc = md.p1_coop;
        if (MODEL == AHMC_MODEL_DIAG_GAUSS) {
            vload<G, E>(m, md.p0, l, D);
            vload<G, E>(w, md.p1, l, D);
        } else if (MODEL == AHMC_MODEL_DENSE_GAUSS) {
            vload<G, E>(m, md.p0, l, D);
        } else if (MODEL == AHMC_MODEL_USER) {
            P = md.p0;  // the user's parameters
        }
    }

    // true: eval_part already returns the finished log pi on every lane (the model needs its own collective anyway);
    // false: it returns this lane's partial sum and log pi = finish(Grp::sum(partial)).
#if defined(AHMC_NVRTC_USER_MODEL) && (defined(AHMC_USER_COORDWISE) || defined(AHMC_USER_GROUPWISE))
    static constexpr bool kLpReduced = MODEL == AHMC_MODEL_FUNNEL;
#else
    static constexpr bool kLpReduced = MODEL == AHMC_MODEL_FUNNEL || MODEL == AHMC_MODEL_USER;
#endif
    __device__ __forceinline__ double finish(double part_sum) const {
        return MODEL == AHMC_MODEL_USER ? part_sum + c0 : fma(-0.5, part_sum, c0);
    }
    __device__ __forceinline__ double eval(const double (&th)[E], double (&g)[E], double* xs, int l) const {
        const double v = eval_part(th, g, xs, l);
        if constexpr (kLpReduced) return v;
        else return finish(Grp<G>::sum(v));
    }
    __device__ __forceinline__ double eval_part(const double (&th)[E], double (&g)[E], double* xs, int l) const {
        double part = 0.0;
        if (MODEL == AHMC_MODEL_STD_NORMAL) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                g[e] = th[e];
                part = fma(th[e], th[e], part);
            }
            return part;
        } else if (MODEL == AHMC_MODEL_DIAG_GAUSS) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                double diff = th[e] - m[e];
                g[e] = diff * w[e];
                part = fma(diff, g[e], part);
            }
            return part;
        } else if (MODEL == AHMC_MODEL_DENSE_GAUSS) {
            double diff[E];
#pragma unroll
            for (int e = 0; e < E; ++e) diff[e] = th[e] - m[e];
            if (G == 32 && coop) matvec_coop<E>(P, Pc, D, diff, g, coop, l);
            else matvec<G, E>(P, D, diff, g, xs, l);
#pragma unroll
            for (int e = 0; e < E; ++e) part = fma(diff[e], g[e], part);
            return part;
        } else if (MODEL == AHMC_MODEL_USER) {
#if defined(AHMC_NVRTC_USER_MODEL)
#if defined(AHMC_USER_COORDWISE)
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int d = l + G * e;
                double gd = 0.0, term = 0.0;
                if (d < D) term = ahmc_user_coord(d, th[e], P, &gd);
                g[e] = -gd;  // PhasePoint caches MINUS the gradient (hamiltonian.jl:45-48)
                part += term;
            }
            return part;
#elif defined(AHMC_USER_GROUPWISE)
            // every call site reaches this with all lanes of the warp converged (the loops around it are steered by
            // warp-wide votes), so the full-warp syncs below and the user's group collectives are well defined
            double* gs = xs + D;
            __syncwarp();
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int d = l + G * e;
                if (d < D) xs[d] = th[e];
            }
            __syncwarp();
            part = ahmc_user_logp_grad_group(xs, gs, D, P, ahmc_group{l, G});
            __syncwarp();
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int d = l + G * e;
                g[e] = (d < D) ? -gs[d] : 0.0;
            }
            return part;
#else
            double* gs = xs + D;  // second slab vector of this group
            __syncwarp();
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int d = l + G * e;
                if (d < D) xs[d] = th[e];
            }
            __syncwarp();
            double lp = 0.0;
            if (l == 0) lp = ahmc_user_logp_grad(xs, gs, D, P);
            __syncwarp();
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int d = l + G * e;
                g[e] = (d < D) ? -gs[d] : 0.0;
            }
            return Grp<G>::bcast(lp, 0) + c0;
#endif
#else
            return 0.0;  // the user-target kernels exist only in run-time compiled modules
#endif
        } else {  // FUNNEL
            double v = Grp<G>::bcast(th[0], 0);
            double ev = exp(-v);
#pragma unroll
            for (int e = 0; e < E; ++e) {
                int d = l + G * e;
                double xe = (d >= 1 && d < D) ? th[e] : 0.0;
                g[e] = xe * ev;  // -d lp / d th_i = th_i e^{-v}
                part = fma(xe, g[e], part);
            }
            double S = Grp<G>::sum(part);
            double Dm1 = (double)(D - 1);
            if (l == 0) g[0] = v / 9.0 - (S - Dm1) * 0.5;  // -(d lp/dv) = v/9 - (S-(D-1))/2
            return c0 - v * v / 18.0 - (S + Dm1 * v) * 0.5;
        }
    }
};

// ------------------------------------------------------------------------------------------------
// one chain's phase point in registers + one exact leapfrog step
// ------------------------------------------------------------------------------------------------
template <int E>
struct ChainState {
    double th[E], r[E], g[E];
    double lp, lk;
};

// dH/dr of the current r and this lane's share of r' dH/dr (neg kinetic energy = -sum/2)
template <int METRIC, int G, int E>
__device__ __forceinline__ double kinetic_part(const MetricOps<METRIC, G, E>& me, const double (&r)[E], double (&dr)[E],
                                               double* xs, int l) {
    me.dHdr(r, dr, xs, l);
    double part = 0.0;
    if (METRIC == AHMC_METRIC_DIAG) {
        // -sum(abs2.(r) .* Minv)/2  (hamiltonian.jl:173-177)
#pragma unroll
        for (int e = 0; e < E; ++e) part = fma(r[e] * r[e], me.Minv[e], part);
    } else {
#pragma unroll
        for (int e = 0; e < E; ++e) part = fma(r[e], dr[e], part);
    }
    return part;
}

// neg kinetic energy and (optionally) dH/dr of the current r
template <int METRIC, int G, int E>
__device__ __forceinline__ double kinetic(const MetricOps<METRIC, G, E>& me, const double (&r)[E], double (&dr)[E],
                                          double* xs, int l) {
    return -0.5 * Grp<G>::sum(kinetic_part<METRIC, G, E>(me, r, dr, xs, l));
}

// One leapfrog step (integrator.jl:235-247) with signed step size eps.  Returns isfinite(z)
// (hamiltonian.jl:141-142), identical on all lanes of the group.  s.lp / s.lk get the -Inf mapping.
// dr receives dH/dr of the final momentum (PhasePoint.lk.gradient).
// temper_mul1/2: multiply r before the first / after the second half kick (1.0 = no tempering).
// TemperedLeapfrog (integrator.jl:198-209): what r is multiplied by before the first / after the second half kick of
// step i (1-based) of an n-step `step` call.  alpha <= 0: plain Leapfrog.
__device__ __forceinline__ void temper_muls(double alpha, int i, int n, double& t1, double& t2) {
    t1 = 1.0;
    t2 = 1.0;
    if (alpha > 0.0) {
        const double sa = sqrt(alpha);
        t1 = (2 * (i - 1) + 1 <= n) ? sa : 1.0 / sa;
        t2 = (2 * (i - 1) + 2 <= n) ? sa : 1.0 / sa;
    }
}

template <int MODEL, int METRIC, int G, int E>
__device__ __forceinline__ void leapfrog_moves(ChainState<E>& s, const ModelOps<MODEL, G, E>& mo,
                                               const MetricOps<METRIC, G, E>& me, double eps, double (&dr)[E],
                                               double* xs, int l, double temper_mul1, double temper_mul2,
                                               double& lp_v, double& lk_part) {
    const double he = 0.5 * eps;
    if (temper_mul1 != 1.0) {
#pragma unroll
        for (int e = 0; e < E; ++e) s.r[e] *= temper_mul1;
    }
#pragma unroll
    for (int e = 0; e < E; ++e) s.r[e] = fma(-he, s.g[e], s.r[e]);  // r - eps/2 .* gradient
    me.dHdr(s.r, dr, xs, l);
#pragma unroll
    for (int e = 0; e < E; ++e) s.th[e] = fma(eps, dr[e], s.th[e]);  // theta + eps .* dH/dr
    lp_v = mo.eval_part(s.th, s.g, xs, l);                           // dH/dtheta
#pragma unroll
    for (int e = 0; e < E; ++e) s.r[e] = fma(-he, s.g[e], s.r[e]);
    if (temper_mul2 != 1.0) {
#pragma unroll
        for (int e = 0; e < E; ++e) s.r[e] *= temper_mul2;
    }
    lk_part = kinetic_part<METRIC, G, E>(me, s.r, dr, xs, l);
}

template <int MODEL, int METRIC, int G, int E>
__device__ __forceinline__ bool leapfrog_step(ChainState<E>& s, const ModelOps<MODEL, G, E>& mo,
                                              const MetricOps<METRIC, G, E>& me, double eps, double (&dr)[E],
                                              double* xs, int l, double temper_mul1 = 1.0,
                                              double temper_mul2 = 1.0) {
    double lp, lk;
    leapfrog_moves<MODEL, METRIC, G, E>(s, mo, me, eps, dr, xs, l, temper_mul1, temper_mul2, lp, lk);
    if constexpr (!ModelOps<MODEL, G, E>::kLpReduced) lp = mo.finish(Grp<G>::sum(lp));
    lk = -0.5 * Grp<G>::sum(lk);
    bool fin = true;
#pragma unroll
    for (int e = 0; e < E; ++e) fin = fin && finite_d(s.g[e]) && finite_d(dr[e]);
    fin = Grp<G>::all(fin) && finite_d(lp) && finite_d(lk);
    s.lp = map_nonfinite(lp);
    s.lk = map_nonfinite(lk);
    return fin;
}

// The same step for a caller that needs the energies only at the step it stops on (the fused trajectory, K1 / K2):
// `isfinite(z)` is decided from the lane partials when that is a proof -- every gradient entry finite and every
// partial of log pi and of the kinetic energy below 2^990, so the 32-term sums are below 2^995 -- and the two
// group reductions run only when `want_energies` (warp-uniform) or some group of the warp is outside the proof.
// Then s.lp / s.lk are exactly leapfrog_step's; otherwise they are left untouched and the step is finite.
template <int MODEL, int METRIC, int G, int E>
__device__ __forceinline__ bool leapfrog_step_lean(ChainState<E>& s, const ModelOps<MODEL, G, E>& mo,
                                                   const MetricOps<METRIC, G, E>& me, double eps, double (&dr)[E],
                                                   double* xs, int l, double temper_mul1, double temper_mul2,
                                                   bool want_energies) {
    double lp, lk;
    leapfrog_moves<MODEL, METRIC, G, E>(s, mo, me, eps, dr, xs, l, temper_mul1, temper_mul2, lp, lk);
    constexpr int T990 = expo_bits(990);
    bool fin = true;
#pragma unroll
    for (int e = 0; e < E; ++e) fin = fin && finite_d(s.g[e]) && finite_d(dr[e]);
    const bool proven = fin && !big_d(lp, T990) && !big_d(lk, T990);
    if (!want_energies && __all_sync(FULL, proven)) return true;
    if constexpr (!ModelOps<MODEL, G, E>::kLpReduced) lp = mo.finish(Grp<G>::sum(lp));
    lk = -0.5 * Grp<G>::sum(lk);
    fin = Grp<G>::all(fin) && finite_d(lp) && finite_d(lk);
    s.lp = map_nonfinite(lp);
    s.lk = map_nonfinite(lk);
    return fin;
}

// ------------------------------------------------------------------------------------------------
// counter-based RNG: Philox4x32-10 (Salmon et al. 2011) keyed by the seed; the 128-bit counter of a draw is
// (chain, (offset << 24) ^ (stream << 60) ^ block), injective while block < 2^24 and offset < 2^36 (DESIGN.md, "Random streams")
// ------------------------------------------------------------------------------------------------
struct Philox {
    static __device__ __forceinline__ void round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
        const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
        uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
        uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
        uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
        c[0] = n0;
        c[1] = n1;
        c[2] = n2;
        c[3] = n3;
    }
    static __device__ __forceinline__ void gen(uint64_t seed, uint64_t ctr_lo, uint64_t ctr_hi, uint32_t (&out)[4]) {
        uint32_t c[4] = {(uint32_t)ctr_lo, (uint32_t)(ctr_lo >> 32), (uint32_t)ctr_hi, (uint32_t)(ctr_hi >> 32)};
        uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
        for (int i = 0; i < 10; ++i) {
            round(c, k0, k1);
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        out[0] = c[0];
        out[1] = c[1];
        out[2] = c[2];
        out[3] = c[3];
    }
    // uniform in (0,1]: 53 random bits plus a half, never 0; the half rounds to even above 2^52, so the all-ones draw is 1.0
    static __device__ __forceinline__ double u01(uint32_t a, uint32_t b) {
        uint64_t x = (((uint64_t)a << 32) | b) >> 11;  // 53 bits
        return ((double)x + 0.5) * (1.0 / 9007199254740992.0);
    }
};

// stream ids for the counter's high word
constexpr uint64_t STREAM_NORMAL = 1, STREAM_EXP = 2, STREAM_DIR = 3;

// D standard normals of (chain, transition) as a group-distributed vector: coordinates e = 2q and e = 2q+1 of a lane
// share ONE Philox block and ONE Box-Muller evaluation (block index = lane + G*q), so a lane with E coordinates
// spends ceil(E/2) blocks.  The stream is a pure function of (seed, offset, chain, D) -- the layout (G) follows from D.
template <int G, int E>
__device__ __forceinline__ void philox_normals(uint64_t seed, uint64_t offset, long long chain, int l, int D,
                                               double (&z)[E]) {
#pragma unroll
    for (int q = 0; q < (E + 1) / 2; ++q) {
        uint32_t o[4];
        Philox::gen(seed, (uint64_t)chain, (offset << 24) ^ (STREAM_NORMAL << 60) ^ (uint64_t)(l + G * q), o);
        const double u1 = Philox::u01(o[0], o[1]), u2 = Philox::u01(o[2], o[3]);
        const double rad = sqrt(-2.0 * log(u1));
        double sn, cs;
        sincospi(2.0 * u2, &sn, &cs);
        z[2 * q] = (l + G * (2 * q) < D) ? rad * cs : 0.0;
        if (2 * q + 1 < E) z[2 * q + 1] = (l + G * (2 * q + 1) < D) ? rad * sn : 0.0;
    }
}

// rand_momentum (metric.jl:290-320) of a chain: standard normals from the tape (D x N, ld = D) or the chain's Philox
// stream of transition `offset`, scaled by the metric
template <int METRIC, int G, int E>
__device__ __forceinline__ void draw_momentum(const MetricOps<METRIC, G, E>& me, const double* normal_tape, uint64_t seed,
                                              uint64_t offset, long long chain, int l, int D, double (&r)[E]) {
    if (normal_tape) vload_nc<G, E>(r, normal_tape + (long long)D * chain, l, D);
    else philox_normals<G, E>(seed, offset, chain, l, D, r);
    me.rand_momentum(r, l);
}

// min(0, x) and min(1, x) with Julia's NaN-propagating min
__device__ __forceinline__ double jl_min0(double x) { return (x != x) ? x : (x < 0.0 ? x : 0.0); }
// mh_accept_ratio's acceptance probability min(1, exp(H - H')) (trajectory.jl:869-877)
__device__ __forceinline__ double mh_accept_ratio(double H0, double H1) {
    const double alpha = exp(H0 - H1);
    return (alpha != alpha) ? alpha : (alpha < 1.0 ? alpha : 1.0);
}

// standard exponential, k-th draw of (chain, transition)
__device__ __forceinline__ double philox_exp(uint64_t seed, uint64_t offset, long long chain, int k) {
    uint32_t o[4];
    Philox::gen(seed, (uint64_t)chain, (offset << 24) ^ (STREAM_EXP << 60) ^ (uint64_t)(k >> 1), o);
    double u = (k & 1) ? Philox::u01(o[2], o[3]) : Philox::u01(o[0], o[1]);
    return -log(u);
}
// direction bit, k-th draw
__device__ __forceinline__ bool philox_bit(uint64_t seed, uint64_t offset, long long chain, int k) {
    uint32_t o[4];
    Philox::gen(seed, (uint64_t)chain, (offset << 24) ^ (STREAM_DIR << 60) ^ (uint64_t)(k >> 7), o);
    return (o[(k >> 5) & 3] >> (k & 31)) & 1u;
}

}  // namespace ahmc

#if defined(AHMC_NVRTC_USER_MODEL) && defined(AHMC_USER_GROUPWISE)
// Collectives of the chain's group for ahmc_user_logp_grad_group (the user's source follows this file).  The G lanes of
// the group call them together; they synchronise only those lanes, so groups sharing a warp may take different paths
// through the user's code.  The sum is Grp::sum's xor butterfly (fixed order; every lane ends with identical bits).
namespace ahmc {
template <int G>
__device__ __forceinline__ double user_group_sum(double v) {
    unsigned m = FULL;
    if constexpr (G < 32) m = Grp<G>::gmask();
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(m, v, o);
    return v;
}
}  // namespace ahmc
__device__ __forceinline__ double ahmc_group_sum(ahmc_group g, double x) {
    switch (g.size) {
        case 4: return ahmc::user_group_sum<4>(x);
        case 8: return ahmc::user_group_sum<8>(x);
        case 16: return ahmc::user_group_sum<16>(x);
        default: return ahmc::user_group_sum<32>(x);
    }
}
// the value x of lane `src` (0..G-1) of the group
__device__ __forceinline__ double ahmc_group_bcast(ahmc_group g, double x, int src) {
    switch (g.size) {
        case 4: return __shfl_sync(ahmc::Grp<4>::gmask(), x, src, 4);
        case 8: return __shfl_sync(ahmc::Grp<8>::gmask(), x, src, 8);
        case 16: return __shfl_sync(ahmc::Grp<16>::gmask(), x, src, 16);
        default: return __shfl_sync(ahmc::FULL, x, src, 32);
    }
}
// shared-memory writes of the group's lanes (to grad, say) become visible to the group
__device__ __forceinline__ void ahmc_group_sync(ahmc_group g) {
    switch (g.size) {
        case 4: __syncwarp(ahmc::Grp<4>::gmask()); break;
        case 8: __syncwarp(ahmc::Grp<8>::gmask()); break;
        case 16: __syncwarp(ahmc::Grp<16>::gmask()); break;
        default: __syncwarp(ahmc::FULL); break;
    }
}
#endif
