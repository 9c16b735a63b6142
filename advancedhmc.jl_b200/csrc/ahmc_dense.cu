// ahmc_dense.cu -- K4: fused leapfrog trajectory for GEMM-shaped operators (Dense-Euclidean metric
// `dH/dr = Minv * r`, src/hamiltonian.jl:60-68, and/or a dense-Gaussian target `grad = -P (theta - mu)`).
//
// The warp-per-chain kernels re-read the D x D matrix once per chain per step (L1-bandwidth bound).  Here a CTA
// owns a TILE of CT chains, keeps the tile's (x, r, g) in registers in the accumulator layout of the fp64 tensor
// instruction, and evaluates  Y[D x CT] = A[D x D] * X[D x CT]  per operator per step with
// `mma.sync.aligned.m8n8k4.f64` (DMMA -- tcgen05 has no f64 kind):
//   * A is streamed from global/L2 in 16-column chunks by `cp.async.bulk` (1-D bulk copies, one per column,
//     completion on an mbarrier; SASS: UBLKCP) into a double-buffered, padded shared-memory stage;
//   * X (the tile's vectors) is staged through shared memory once per product;
//   * A is shared by all CTAs, so after the first touch it is served from L2.
// All targets handled here are Gaussian and the metric Euclidean, so the dynamics are LINEAR: the same magnitude
// proof as the separable fast path applies with the induced infinity norms (K = (1+|eps| |Minv|_inf)(1+|eps| |P|_inf)),
// energies are evaluated once at the end, and a tile that fails a magnitude check is handed, chain by chain, to
// the exact warp-per-chain kernel (`only_mask`) inside the same stream -- no host round trip.
#include "ahmc_kernels.cuh"
#ifndef AHMC_SIMT_EMULATION
#include "ahmc_dispatch.cuh"
#endif

namespace ahmc {

constexpr int kDenseThreads = 256;  // 8 warps
constexpr int kKC = 16;             // columns of A per pipeline stage
// A pipeline:
//   * the padded matrix is stored with the shared-memory stage's leading dimension (Dp + 4, ahmc_kernels.cuh dense_lda), so a
//     16-column chunk is ONE contiguous bulk copy instead of sixteen;
//   * consumers release a stage through an "empty" mbarrier (one arrival per warp) and only the producer thread waits on it,
//     instead of a CTA-wide __syncthreads per chunk;
//   * three stages.  Shared memory: 68 KB per CTA at Dp = 128 (two CTAs per SM still fit), 232,272 of the 232,448 bytes a CTA
//     may have at Dp = 512.
constexpr int kStages = 3;  // the wait is L2 latency per chunk, not pipeline depth
constexpr int kBars = 2 * kStages;  // full[kStages] + empty[kStages]
#ifdef AHMC_SIMT_EMULATION
extern unsigned char* emu_dynamic_smem;  // the block's dynamic shared memory (blocks run one at a time)
#endif

// (mbarrier / bulk-copy / DMMA wrappers: ahmc_device.cuh)

// Y += A * X for the CTA's tile.  A: Dp x Dp column-major (padded, zero-filled) in global memory.
// Xs: CT x Dx doubles in shared memory (chain-major, Dx = Dp + 4).  acc[rb][cb][2]: this thread's accumulators:
// rows 8*(RB*warp + rb) + lane/4, columns 8*cb + 2*(lane%4) + {0,1}.
template <int RB, int CB>
__device__ __forceinline__ void tile_gemm(const double* __restrict__ A, int Dp, const double* Xs, double* As /* kStages stages */,
                                          uint64_t* bars, uint32_t (&phase)[kBars], double (&acc)[RB][CB][2]) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Ds = Dp + 4, Dx = Dp + 4;
    const int nchunks = Dp / kKC;
    const uint32_t chunk_bytes = (uint32_t)(kKC * Ds * sizeof(double));
    auto issue = [&](int c, int stage) {  // global leading dimension == stage leading dimension: one contiguous copy
        mbar_expect_tx(&bars[stage], chunk_bytes);
        bulk_g2s(As + (size_t)stage * kKC * Ds, A + (size_t)c * kKC * Ds, chunk_bytes, &bars[stage]);
    };
    // Bit s of phase[0]: parity of the next "full" phase of stage s (every thread).  Producer thread only -- bit s of
    // phase[1]: parity of the number of fills f of stage s so far; of phase[2]: f > 0.  Fill f >= 1 of a stage waits for
    // the stage's (f-1)-th release: bars[kStages + s] completes one phase per consumption (8 warp arrivals), and at that
    // point it has completed f-1 or f of them, so the parity wait is unambiguous.
    auto refill = [&](int c, int stage) {
        const uint32_t bit = 1u << stage;
        if (phase[2] & bit) mbar_wait(&bars[kStages + stage], ((phase[1] >> stage) & 1u) ^ 1u);
        phase[2] |= bit;
        phase[1] ^= bit;
        issue(c, stage);
    };
    if (tid == 0)
        for (int c = 0; c < kStages && c < nchunks; ++c) refill(c, c);
    const int arow = 8 * RB * warp + (lane >> 2);
    int stage = 0, prev = kStages - 1;
    for (int c = 0; c < nchunks; ++c) {
        mbar_wait(&bars[stage], (phase[0] >> stage) & 1u);
        phase[0] ^= 1u << stage;
        const double* as = As + (size_t)stage * kKC * Ds;
#pragma unroll
        for (int ks = 0; ks < kKC / 4; ++ks) {
            double a[RB], b[CB];
            const int kl = 4 * ks + (lane & 3);
#pragma unroll
            for (int rb = 0; rb < RB; ++rb) a[rb] = as[(size_t)kl * Ds + arow + 8 * rb];
#pragma unroll
            for (int cb = 0; cb < CB; ++cb) b[cb] = Xs[(size_t)(8 * cb + (lane >> 2)) * Dx + c * kKC + kl];
#pragma unroll
            for (int rb = 0; rb < RB; ++rb)
#pragma unroll
                for (int cb = 0; cb < CB; ++cb) dmma(acc[rb][cb][0], acc[rb][cb][1], a[rb], b[cb]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars[kStages + stage]);  // this warp is done with the stage
        // the producer refills the stage of the PREVIOUS chunk: its last readers are at most one chunk behind
        if (tid == 0 && c >= 1 && c - 1 + kStages < nchunks) refill(c - 1 + kStages, prev);
        prev = stage;
        stage = (stage + 1 == kStages) ? 0 : stage + 1;
    }
    __syncthreads();  // every warp is done with Xs; every release of this product has arrived
}

template <int RB, int CB>
__device__ __forceinline__ void tile_to_smem(double* Xs, int Dp, const double (&v)[RB][CB][2]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int Dx = Dp + 4;
#pragma unroll
    for (int rb = 0; rb < RB; ++rb)
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j)
                Xs[(size_t)(8 * cb + 2 * (lane & 3) + j) * Dx + 8 * (RB * warp + rb) + (lane >> 2)] = v[rb][cb][j];
    __syncthreads();
}

struct DenseArgs {
    int D, Dp;
    long long N;
    const double* P;      // Dp x Dp padded precision (nullptr: separable target)
    const double* w;      // D: 1/s^2 for DIAG_GAUSS (nullptr with P == nullptr: std normal)
    const double* mu;     // D or nullptr
    double c0;
    const double* Minv;   // Dp x Dp padded (dense metric) or nullptr
    const double* Mdiag;  // D (diag metric) or nullptr (unit)
    const double* norms;  // [0] = |Minv|_inf (or max Mdiag, or 1), [1] = |P|_inf (or max w, or 1)
    double eps;
    const double* eps_chain;
    int n_steps, fwd;
    const double *th_in, *r_in, *g_in;
    long long ld_in;
    double *th_out, *r_out, *g_out, *dr_out, *lp_out, *lk_out;
    long long ld_out;
    uint32_t* status;
    int32_t* steps_done;
    uint8_t* need_exact;  // per chain: 1 -> the exact warp-per-chain kernel must redo this chain
};

template <int RB, int CB, int MINB = 1>
__global__ void __launch_bounds__(kDenseThreads, MINB) dense_traj_kernel(const DenseArgs a) {
#ifdef AHMC_SIMT_EMULATION
    unsigned char* smem_raw = emu_dynamic_smem;
#else
    extern __shared__ __align__(16) unsigned char smem_raw[];
#endif
    constexpr int CT = 8 * CB;
    const int Dp = a.Dp, D = a.D, Dx = Dp + 4, Ds = Dp + 4;
    double* As = reinterpret_cast<double*>(smem_raw);
    double* Xs = As + (size_t)kStages * kKC * Ds;
    double* red = Xs + (size_t)CT * Dx;                        // [8 warps][CT][2]
    uint64_t* bars = reinterpret_cast<uint64_t*>(red + 8 * CT * 2);
    __shared__ int s_flag;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int i = 0; i < kStages; ++i) {
            mbar_init(&bars[i], 1);
            mbar_init(&bars[kStages + i], kDenseThreads / 32);
        }
        s_flag = 0;
        mbar_fence_init();
    }
    __syncthreads();
    uint32_t phase[kBars] = {};
    const long long tile0 = (long long)blockIdx.x * CT;
    constexpr int T200 = expo_bits(200), T100 = expo_bits(100), T50 = expo_bits(50);

    // this thread's rows / columns
    int row[RB];
    long long col[CB][2];
    bool cval[CB][2];
    double eps_c[CB][2];
    bool susp = false;
#pragma unroll
    for (int rb = 0; rb < RB; ++rb) row[rb] = 8 * (RB * warp + rb) + (lane >> 2);
#pragma unroll
    for (int cb = 0; cb < CB; ++cb)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const long long c = tile0 + 8 * cb + 2 * (lane & 3) + j;
            cval[cb][j] = c < a.N;
            col[cb][j] = cval[cb][j] ? c : a.N - 1;
            double e = a.eps_chain ? __ldg(a.eps_chain + col[cb][j]) : a.eps;
            eps_c[cb][j] = a.fwd ? e : -e;
            susp |= big_d(eps_c[cb][j], T50);
        }
    double x[RB][CB][2], r[RB][CB][2], g[RB][CB][2];
    double muv[RB], wv[RB], mdv[RB];
#pragma unroll
    for (int rb = 0; rb < RB; ++rb) {
        const bool in = row[rb] < D;
        muv[rb] = (a.mu && in) ? __ldg(a.mu + row[rb]) : 0.0;
        wv[rb] = in ? (a.w ? __ldg(a.w + row[rb]) : 1.0) : 0.0;
        mdv[rb] = in ? (a.Mdiag ? __ldg(a.Mdiag + row[rb]) : 1.0) : 0.0;
        susp |= big_d(muv[rb], T200) | big_d(wv[rb], T100) | big_d(mdv[rb], T100);
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                double th = 0.0, rr = 0.0, gg = 0.0;
                if (in) {
                    th = a.th_in[a.ld_in * col[cb][j] + row[rb]];
                    rr = a.r_in[a.ld_in * col[cb][j] + row[rb]];
                    gg = a.g_in[a.ld_in * col[cb][j] + row[rb]];
                }
                susp |= big_d(th, T200) | big_d(rr, T200) | big_d(gg, T200);
                x[rb][cb][j] = th - muv[rb];
                r[rb][cb][j] = fma(-0.5 * eps_c[cb][j], gg, rr);  // first half kick with the cached gradient
            }
    }
    // growth bound: K = (1 + |eps| |Minv|_inf)(1 + |eps| |P|_inf); magnitude check every floor(100 / (exponent(K)+1)) steps
    double emax = 0.0;
#pragma unroll
    for (int cb = 0; cb < CB; ++cb)
#pragma unroll
        for (int j = 0; j < 2; ++j) emax = fmax(emax, fabs(eps_c[cb][j]));
    const double nM = __ldg(a.norms + 0), nP = __ldg(a.norms + 1);
    const double K = (1.0 + emax * nM) * (1.0 + emax * nP);
    int kcheck;
    {
        const int ek = ((__double2hiint(K) >> 20) & 0x7ff) - 1023 + 1;
        if (ek > 100 || !(K >= 1.0) || big_d(nM, T100) || big_d(nP, T100)) susp = true;
        const int kk = 100 / (ek < 1 ? 1 : ek);
        kcheck = kk < 1 ? 1 : kk;
    }
    // kcheck must be uniform across the CTA (per-chain eps differ): take the minimum
    {
        __shared__ int s_k;
        if (tid == 0) s_k = 0x7fffffff;
        __syncthreads();
        atomicMin(&s_k, kcheck);
        __syncthreads();
        kcheck = s_k;
    }

    auto apply_metric = [&](double (&y)[RB][CB][2]) {  // y = Minv * r
        if (a.Minv) {
#pragma unroll
            for (int rb = 0; rb < RB; ++rb)
#pragma unroll
                for (int cb = 0; cb < CB; ++cb) y[rb][cb][0] = y[rb][cb][1] = 0.0;
            tile_to_smem<RB, CB>(Xs, Dp, r);
            tile_gemm<RB, CB>(a.Minv, Dp, Xs, As, bars, phase, y);
        } else {
#pragma unroll
            for (int rb = 0; rb < RB; ++rb)
#pragma unroll
                for (int cb = 0; cb < CB; ++cb)
#pragma unroll
                    for (int j = 0; j < 2; ++j) y[rb][cb][j] = mdv[rb] * r[rb][cb][j];
        }
    };
    auto apply_target = [&]() {  // g = P * x  (minus grad log pi)
        if (a.P) {
#pragma unroll
            for (int rb = 0; rb < RB; ++rb)
#pragma unroll
                for (int cb = 0; cb < CB; ++cb) g[rb][cb][0] = g[rb][cb][1] = 0.0;
            tile_to_smem<RB, CB>(Xs, Dp, x);
            tile_gemm<RB, CB>(a.P, Dp, Xs, As, bars, phase, g);
        } else {
#pragma unroll
            for (int rb = 0; rb < RB; ++rb)
#pragma unroll
                for (int cb = 0; cb < CB; ++cb)
#pragma unroll
                    for (int j = 0; j < 2; ++j) g[rb][cb][j] = wv[rb] * x[rb][cb][j];
        }
    };

    double y[RB][CB][2];
    const int n = a.n_steps;
    int since_check = 0;
    for (int i = 1; i <= n; ++i) {
        apply_metric(y);
#pragma unroll
        for (int rb = 0; rb < RB; ++rb)
#pragma unroll
            for (int cb = 0; cb < CB; ++cb)
#pragma unroll
                for (int j = 0; j < 2; ++j) x[rb][cb][j] = fma(eps_c[cb][j], y[rb][cb][j], x[rb][cb][j]);
        apply_target();
        const double kf = (i < n) ? 1.0 : 0.5;  // merged full kick between steps, half kick at the end
#pragma unroll
        for (int rb = 0; rb < RB; ++rb)
#pragma unroll
            for (int cb = 0; cb < CB; ++cb)
#pragma unroll
                for (int j = 0; j < 2; ++j) r[rb][cb][j] = fma(-kf * eps_c[cb][j], g[rb][cb][j], r[rb][cb][j]);
        if (++since_check >= kcheck || i == n) {
            since_check = 0;
#pragma unroll
            for (int rb = 0; rb < RB; ++rb)
#pragma unroll
                for (int cb = 0; cb < CB; ++cb)
#pragma unroll
                    for (int j = 0; j < 2; ++j) susp |= big_d(x[rb][cb][j], T200) | big_d(r[rb][cb][j], T200);
        }
    }
    // energies: lp = c0 - x'g/2, lk = -r'(Minv r)/2
    apply_metric(y);
    double plp[CB][2], plk[CB][2];
#pragma unroll
    for (int cb = 0; cb < CB; ++cb)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            double s1 = 0.0, s2 = 0.0;
#pragma unroll
            for (int rb = 0; rb < RB; ++rb) {
                s1 = fma(x[rb][cb][j], g[rb][cb][j], s1);
                s2 = fma(r[rb][cb][j], y[rb][cb][j], s2);
            }
            // reduce over the 8 row-lanes that share (lane & 3)
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                s1 += __shfl_xor_sync(FULL, s1, o);
                s2 += __shfl_xor_sync(FULL, s2, o);
            }
            plp[cb][j] = s1;
            plk[cb][j] = s2;
        }
    if ((lane >> 2) == 0) {
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int cc = 8 * cb + 2 * (lane & 3) + j;
                red[(warp * CT + cc) * 2 + 0] = plp[cb][j];
                red[(warp * CT + cc) * 2 + 1] = plk[cb][j];
            }
    }
    if (susp) atomicOr(&s_flag, 1);
    __syncthreads();
    const bool tile_bad = s_flag != 0;
    if (tid < CT) {
        const long long c = tile0 + tid;
        if (c < a.N) {
            a.need_exact[c] = tile_bad ? 1 : 0;
            if (!tile_bad) {
                double s1 = 0.0, s2 = 0.0;
                for (int wv_ = 0; wv_ < 8; ++wv_) {
                    s1 += red[(wv_ * CT + tid) * 2 + 0];
                    s2 += red[(wv_ * CT + tid) * 2 + 1];
                }
                a.lp_out[c] = fma(-0.5, s1, a.c0);
                a.lk_out[c] = -0.5 * s2;
                if (a.status) a.status[c] = 0u;
                if (a.steps_done) a.steps_done[c] = n;
            }
        }
    }
    if (tile_bad) return;
#pragma unroll
    for (int rb = 0; rb < RB; ++rb) {
        if (row[rb] >= D) continue;
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                if (!cval[cb][j]) continue;
                const long long o = a.ld_out * col[cb][j] + row[rb];
                a.th_out[o] = x[rb][cb][j] + muv[rb];
                a.r_out[o] = r[rb][cb][j];
                a.g_out[o] = g[rb][cb][j];
                if (a.dr_out) a.dr_out[o] = y[rb][cb][j];
            }
    }
}

// |A|_inf (max absolute row sum) of a D x D column-major matrix, and a padded Dp x Dp copy (zero filled)
__global__ void pad_norm_kernel(const double* __restrict__ A, int D, int Dp, double* __restrict__ Ap, double* norm) {
    __shared__ double smax[256];
    double best = 0.0;
    for (int rowi = threadIdx.x; rowi < Dp; rowi += blockDim.x) {
        double s = 0.0;
        for (int k = 0; k < Dp; ++k) {
            double v = (rowi < D && k < D) ? A[(size_t)k * D + rowi] : 0.0;
            if (Ap) Ap[(size_t)k * dense_lda(Dp) + rowi] = v;
            s += fabs(v);
        }
        best = (s > best || s != s) ? s : best;
    }
    if (Ap)  // the 4 padding rows of every column travel with the chunk copy: keep them defined
        for (int i = threadIdx.x; i < 4 * Dp; i += blockDim.x) Ap[(size_t)(i >> 2) * dense_lda(Dp) + Dp + (i & 3)] = 0.0;
    smax[threadIdx.x] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        double m = 0.0;
        for (int t = 0; t < blockDim.x; ++t) m = (smax[t] > m || smax[t] != smax[t]) ? smax[t] : m;
        *norm = m;
    }
}
__global__ void vec_norm_kernel(const double* __restrict__ v, int D, double* norm) {  // max |v_d| (1 if v == nullptr)
    if (threadIdx.x == 0) {
        double m = v ? 0.0 : 1.0;
        if (v)
            for (int d = 0; d < D; ++d) {
                double t = fabs(v[d]);
                m = (t > m || t != t) ? t : m;
            }
        *norm = m;
    }
}

bool dense_tile_shape(int D, int* Dp, int* RB, int* CB) {
    if (D < 1 || D > 512) return false;
    *Dp = ((D + 63) / 64) * 64;
    *RB = *Dp / 64;
    *CB = (*RB <= 2) ? 4 : (*RB <= 4 ? 2 : 1);
    return true;
}

#ifndef AHMC_SIMT_EMULATION
cudaError_t launch_pad_norm(const double* A, int D, int Dp, double* Ap, double* norm, cudaStream_t st) {
    pad_norm_kernel<<<1, 256, 0, st>>>(A, D, Dp, Ap, norm);
    return cudaGetLastError();
}
cudaError_t launch_vec_norm(const double* v, int D, double* norm, cudaStream_t st) {
    vec_norm_kernel<<<1, 32, 0, st>>>(v, D, norm);
    return cudaGetLastError();
}

template <int RB, int CB, int MINB = 1>
static cudaError_t launch_dense_t(const DenseArgs& a, cudaStream_t st) {
    constexpr int CT = 8 * CB;
    const int Ds = a.Dp + 4;
    const size_t sm = ((size_t)kStages * kKC * Ds + (size_t)CT * Ds + 8 * CT * 2) * sizeof(double) + 64;
    return launch_kernel(dense_traj_kernel<RB, CB, MINB>, (a.N + CT - 1) / CT, kDenseThreads, sm, st, a);
}

cudaError_t launch_dense_traj(const DenseTrajHost& h, cudaStream_t st, int* n_launches) {
    DenseArgs a{};
    a.D = h.D; a.Dp = h.Dp; a.N = h.N; a.P = h.P; a.w = h.w; a.mu = h.mu; a.c0 = h.c0; a.Minv = h.Minv; a.Mdiag = h.Mdiag;
    a.norms = h.norms; a.eps = h.eps; a.eps_chain = h.eps_chain; a.n_steps = h.n_steps; a.fwd = h.fwd;
    a.th_in = h.th_in; a.r_in = h.r_in; a.g_in = h.g_in; a.ld_in = h.ld_in;
    a.th_out = h.th_out; a.r_out = h.r_out; a.g_out = h.g_out; a.dr_out = h.dr_out; a.lp_out = h.lp_out; a.lk_out = h.lk_out;
    a.ld_out = h.ld_out; a.status = h.status; a.steps_done = h.steps_done; a.need_exact = h.need_exact;
    if (n_launches) *n_launches += 1;
    const int RB = h.Dp / 64;
    switch (RB) {
        case 1: return launch_dense_t<1, 4>(a, st);
        case 2: return launch_dense_t<2, 2, 2>(a, st);  // D <= 128: tiles of 16 chains, two CTAs per SM -- the barrier / copy
                                                         // waits of one hide behind the other
        case 3: return launch_dense_t<3, 2>(a, st);
        case 4: return launch_dense_t<4, 2>(a, st);
        case 5: return launch_dense_t<5, 1>(a, st);
        case 6: return launch_dense_t<6, 1>(a, st);
        case 7: return launch_dense_t<7, 1>(a, st);
        case 8: return launch_dense_t<8, 1>(a, st);
    }
    return cudaErrorInvalidValue;
}
#endif  // AHMC_SIMT_EMULATION

}  // namespace ahmc
