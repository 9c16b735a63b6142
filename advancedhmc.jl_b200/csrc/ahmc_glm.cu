// ahmc_glm.cu -- K6: fused leapfrog trajectory for generalised linear model targets,
//   log pi(theta) = c0 + sum_i l(y_i, x_i' theta) - sum_d prec_d theta_d^2 / 2     (Bernoulli-logit, Poisson-log).
//
// For a TILE of CT chains the linear predictor eta = X theta and the score X' (y - mu(eta)) are two GEMMs with X shared by
// every chain.  A CTA of 8 warps owns the tile and keeps its (theta, r, g) in registers in the accumulator layout of
// `mma.sync.aligned.m8n8k4.f64` (rows = coordinates, columns = chains), as K4 (ahmc_dense.cu) does.  One gradient is ONE
// pass over X:
//   * X is stored row-major with the shared-memory stage's leading dimension (glm_lds), rows beyond n zero, so a chunk of
//     nc rows is one contiguous `cp.async.bulk` (SASS: UBLKCP) completing on the stage's mbarrier;
//   * per chunk, from the same staged rows: eta_c[nc x CT] = X_c theta on DMMA (a warp per 8-row block), the link function
//     in registers (one exp per row and chain), w = y - mu into a small shared tile, one CTA barrier, then
//     g[D x CT] += X_c' w on DMMA with the warps owning row blocks of D;
//   * that barrier also proves every warp is done with the PREVIOUS chunk's stage, so the producer thread refills it right
//     behind the barrier: no "empty" barriers are needed.
// The dynamics are not linear, so there is no magnitude proof: `isfinite(z)` (hamiltonian.jl:141-142) is decided per
// column at every step from the reduced energies, and a column that goes non-finite stops there: its phase point and
// scalars are stored at that step.  It keeps taking part in the products with its results ignored; columns of a GEMM are
// independent, so its NaNs stay in its own column.
#include "ahmc_glm.cuh"
#ifndef AHMC_SIMT_EMULATION
#include "ahmc_dispatch.cuh"
#endif

namespace ahmc {

constexpr int kGlmThreads = 256;  // 8 warps
constexpr int kGlmMaxStages = 3;
#ifdef AHMC_SIMT_EMULATION
extern unsigned char* emu_dynamic_smem;
#endif

// Shared-memory fragment reads.  With lds = 8k + 4 doubles a half-warp's 16 addresses (q * lds + k and k * lds + q with
// q, k in 0..3 -- the A fragment of the eta product and the transposed A fragment of the score product) fall into 16
// different 8-byte bank pairs: lds mod 16 is 4 or 12, and {4q + k} = {12q + k} = 0..15 (mod 16).  The w tile's leading
// dimension nc + 4 and theta's (lds again) are of the same form, so all four fragment patterns are conflict free.
template <int RB, int CB, int FAM>
__global__ void __launch_bounds__(kGlmThreads, 1) glm_traj_kernel(const GlmArgs a) {
#ifdef AHMC_SIMT_EMULATION
    unsigned char* smem_raw = emu_dynamic_smem;
#else
    extern __shared__ __align__(16) unsigned char smem_raw[];
#endif
    constexpr int CT = 8 * CB;
    const int D = a.D, lds = glm_lds(D), Dp = lds - 4, nc = a.nc, ldw = nc + 4, S = a.stages;
    const int nchunks = (a.n + nc - 1) / nc;
    double* Xs = reinterpret_cast<double*>(smem_raw);          // S stages of nc x lds
    double* Ths = Xs + (size_t)S * nc * lds;                   // CT x lds: theta of the tile, chain-major
    double* Ws = Ths + (size_t)CT * lds;                       // 2 x CT x ldw: w = y - mu of a chunk, chain-major
    double* red = Ws + (size_t)2 * CT * ldw;                   // [8 warps][CT][3]: log pi, kinetic, non-finite partials
    uint64_t* bars = reinterpret_cast<uint64_t*>(red + 8 * CT * 3);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, q = lane >> 2, k4 = lane & 3;
    if (tid == 0) {
        for (int s = 0; s < S; ++s) mbar_init(&bars[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    uint32_t phase = 0;  // bit s: parity of the next "full" phase of stage s
    const long long tile0 = (long long)blockIdx.x * CT;
    const uint32_t chunk_bytes = (uint32_t)((size_t)nc * lds * sizeof(double));

    // this thread's rows (coordinates) and columns (chains)
    int row[RB];
    bool ract[RB];  // warp-uniform: the row block holds coordinates
    long long col[CB][2];
    bool cval[CB][2];
    double eps_c[CB][2];
    double prec[RB];
#pragma unroll
    for (int rb = 0; rb < RB; ++rb) {
        row[rb] = 8 * (RB * warp + rb) + q;
        ract[rb] = 8 * (RB * warp + rb) < Dp;
        prec[rb] = row[rb] < D ? __ldg(a.prec + row[rb]) : 0.0;
    }
#pragma unroll
    for (int cb = 0; cb < CB; ++cb)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const long long c = tile0 + 8 * cb + 2 * k4 + j;
            cval[cb][j] = c < a.N;
            col[cb][j] = cval[cb][j] ? c : a.N - 1;  // tail columns shadow the last chain, never store
            const double e = a.eps_chain ? __ldg(a.eps_chain + col[cb][j]) : a.eps;
            eps_c[cb][j] = a.fwd ? e : -e;
        }
    double x[RB][CB][2], r[RB][CB][2], g[RB][CB][2];
#pragma unroll
    for (int rb = 0; rb < RB; ++rb)
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const bool in = row[rb] < D;
                const long long o = a.ld_in * col[cb][j] + row[rb];
                x[rb][cb][j] = in ? a.th_in[o] : 0.0;
                r[rb][cb][j] = in ? a.r_in[o] : 0.0;
                g[rb][cb][j] = (in && a.g_in) ? a.g_in[o] : 0.0;
            }
    auto minv = [&](int rb, int cb, int j) -> double {  // M^-1 of (coordinate, chain); 0 on padding rows
        if (row[rb] >= D) return 0.0;
        return a.Minv ? __ldg(a.Minv + a.chain_stride * col[cb][j] + row[rb]) : 1.0;
    };

    // one pass over X at the tile's x: g = X' (y - mu), lsum = this thread's share of sum_i l_i per column
    auto pass = [&](double (&lsum)[CB][2]) {
#pragma unroll
        for (int rb = 0; rb < RB; ++rb)
#pragma unroll
            for (int cb = 0; cb < CB; ++cb)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    if (ract[rb]) Ths[(size_t)(8 * cb + 2 * k4 + j) * lds + row[rb]] = x[rb][cb][j];
                    g[rb][cb][j] = 0.0;
                }
#pragma unroll
        for (int cb = 0; cb < CB; ++cb) lsum[cb][0] = lsum[cb][1] = 0.0;
        __syncthreads();  // theta staged; every warp is done with the stages and the w tiles of the previous pass
        auto issue = [&](int c, int stage) {
            mbar_expect_tx(&bars[stage], chunk_bytes);
            bulk_g2s(Xs + (size_t)stage * nc * lds, a.Xp + (size_t)c * nc * lds, chunk_bytes, &bars[stage]);
        };
        if (tid == 0)
            for (int c = 0; c < S && c < nchunks; ++c) issue(c, c);
        int stage = 0, prev = S - 1;
        for (int c = 0; c < nchunks; ++c) {
            mbar_wait(&bars[stage], (phase >> stage) & 1u);
            phase ^= 1u << stage;
            const double* xs = Xs + (size_t)stage * nc * lds;
            double* wb = Ws + (size_t)(c & 1) * CT * ldw;
            for (int b = warp; 8 * b < nc; b += kGlmThreads / 32) {  // eta of an 8-row block, then its link function
                double eta[CB][2];
#pragma unroll
                for (int cb = 0; cb < CB; ++cb) eta[cb][0] = eta[cb][1] = 0.0;
                const double* xr = xs + (size_t)(8 * b + q) * lds + k4;
                const double* tr = Ths + (size_t)q * lds + k4;
                for (int ks = 0; ks < Dp / 4; ++ks) {
                    const double av = xr[4 * ks];
#pragma unroll
                    for (int cb = 0; cb < CB; ++cb) dmma(eta[cb][0], eta[cb][1], av, tr[(size_t)8 * cb * lds + 4 * ks]);
                }
                const int i = c * nc + 8 * b + q;
                const bool in = i < a.n;  // rows beyond n contribute exactly zero
                const double yi = in ? __ldg(a.y + i) : 0.0;
#pragma unroll
                for (int cb = 0; cb < CB; ++cb)
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const double e = eta[cb][j];
                        double l, mu;
                        if (FAM == AHMC_GLM_BERNOULLI_LOGIT) {  // one exp per row: t = e^-|eta| serves softplus and sigmoid
                            const double t = exp(-fabs(e));
                            l = yi * e - (fmax(e, 0.0) + log1p(t));
                            mu = (e >= 0.0 ? 1.0 : t) / (1.0 + t);
                            if (e != e) l = mu = e;  // fmax would drop a NaN
                        } else {
                            mu = exp(e);
                            l = yi * e - mu;
                        }
                        lsum[cb][j] += in ? l : 0.0;
                        wb[(size_t)(8 * cb + 2 * k4 + j) * ldw + 8 * b + q] = in ? yi - mu : 0.0;
                    }
            }
            __syncthreads();  // w of this chunk is complete; every warp has left chunk c - 1
            if (tid == 0 && c >= 1 && c - 1 + S < nchunks) issue(c - 1 + S, prev);
            const double* wr = wb + (size_t)q * ldw + k4;
            for (int ks = 0; ks < nc / 4; ++ks) {
                double bv[CB];
#pragma unroll
                for (int cb = 0; cb < CB; ++cb) bv[cb] = wr[(size_t)8 * cb * ldw + 4 * ks];
#pragma unroll
                for (int rb = 0; rb < RB; ++rb) {
                    if (!ract[rb]) continue;
                    const double av = xs[(size_t)(4 * ks + k4) * lds + row[rb]];
#pragma unroll
                    for (int cb = 0; cb < CB; ++cb) dmma(g[rb][cb][0], g[rb][cb][1], av, bv[cb]);
                }
            }
            prev = stage;
            stage = (stage + 1 == S) ? 0 : stage + 1;
        }
    };
    // column sums of (v0, v1) and the OR of `bad`: the 8 row-lanes sharing lane & 3 by shuffles, then the 8 warps through
    // shared memory in warp order -- a fixed order, the same value in every thread of the column
    auto reduce = [&](double (&v0)[CB][2], double (&v1)[CB][2], bool (&bad)[CB][2]) {
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                double s0 = v0[cb][j], s1 = v1[cb][j], s2 = bad[cb][j] ? 1.0 : 0.0;
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                    s0 += __shfl_xor_sync(FULL, s0, o);
                    s1 += __shfl_xor_sync(FULL, s1, o);
                    s2 += __shfl_xor_sync(FULL, s2, o);
                }
                if (q == 0) {
                    double* p = red + (size_t)(warp * CT + 8 * cb + 2 * k4 + j) * 3;
                    p[0] = s0;
                    p[1] = s1;
                    p[2] = s2;
                }
            }
        __syncthreads();
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                double s0 = 0.0, s1 = 0.0, s2 = 0.0;
                for (int w = 0; w < kGlmThreads / 32; ++w) {
                    const double* p = red + (size_t)(w * CT + 8 * cb + 2 * k4 + j) * 3;
                    s0 += p[0];
                    s1 += p[1];
                    s2 += p[2];
                }
                v0[cb][j] = s0;
                v1[cb][j] = s1;
                bad[cb][j] = s2 != 0.0;
            }
        // (the next write to `red` is behind the barriers of the next pass)
    };

    bool alive[CB][2];
#pragma unroll
    for (int cb = 0; cb < CB; ++cb) alive[cb][0] = alive[cb][1] = true;
    double lsum[CB][2], lks[CB][2];
    bool bad[CB][2];
    const int n = a.n_steps;
    // iteration 0 is the pass at the start point: without a cached gradient, and for phasepoint (n == 0), whose energies
    // it also yields
    for (int i = (!a.g_in || n == 0) ? 0 : 1; i <= n; ++i) {
        if (i > 0) {  // integrator.jl:235-247: half kick, drift, gradient, half kick
#pragma unroll
            for (int rb = 0; rb < RB; ++rb)
#pragma unroll
                for (int cb = 0; cb < CB; ++cb)
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const double e = eps_c[cb][j];
                        r[rb][cb][j] = fma(-0.5 * e, g[rb][cb][j], r[rb][cb][j]);
                        x[rb][cb][j] = fma(e, minv(rb, cb, j) * r[rb][cb][j], x[rb][cb][j]);
                    }
        }
        pass(lsum);
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                double lk = 0.0;
                bool nf = false;
#pragma unroll
                for (int rb = 0; rb < RB; ++rb) {
                    g[rb][cb][j] = fma(prec[rb], x[rb][cb][j], -g[rb][cb][j]);  // MINUS the gradient of log pi
                    if (i > 0) r[rb][cb][j] = fma(-0.5 * eps_c[cb][j], g[rb][cb][j], r[rb][cb][j]);
                    const double dr = minv(rb, cb, j) * r[rb][cb][j];
                    lk = fma(r[rb][cb][j], dr, lk);
                    lsum[cb][j] = fma(-0.5 * prec[rb] * x[rb][cb][j], x[rb][cb][j], lsum[cb][j]);
                    nf |= !finite_d(g[rb][cb][j]) | !finite_d(dr);
                }
                lks[cb][j] = lk;
                bad[cb][j] = nf;
            }
        if (i == 0 && n > 0) continue;  // only the gradient of the start point was needed
        reduce(lsum, lks, bad);
#pragma unroll
        for (int cb = 0; cb < CB; ++cb)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                if (!alive[cb][j]) continue;
                const double lp = lsum[cb][j] + a.c0, lk = -0.5 * lks[cb][j];
                const bool fin = !bad[cb][j] && finite_d(lp) && finite_d(lk);
                if (fin && i < n) continue;
                // The chain stops here, finished or non-finite (integrator.jl:252-258 returns the non-finite z): its phase
                // point is stored now, and what its registers do afterwards no longer matters
                alive[cb][j] = false;
                if (!cval[cb][j]) continue;
                const long long c = col[cb][j];
#pragma unroll
                for (int rb = 0; rb < RB; ++rb) {
                    if (row[rb] >= D) continue;
                    const long long o = a.ld_out * c + row[rb];
                    if (a.th_out) a.th_out[o] = x[rb][cb][j];
                    if (a.r_out) a.r_out[o] = r[rb][cb][j];
                    a.g_out[o] = g[rb][cb][j];
                    if (a.dr_out) a.dr_out[o] = minv(rb, cb, j) * r[rb][cb][j];
                }
                if (warp == 0 && q == 0) {
                    a.lp_out[c] = map_nonfinite(lp);
                    a.lk_out[c] = map_nonfinite(lk);
                    if (a.status) a.status[c] = fin ? 0u : AHMC_STATUS_NONFINITE;
                    if (a.steps_done) a.steps_done[c] = i;
                }
            }
    }
}

bool glm_tile_shape(int D, int n, int* RB, int* CB, int* nc, int* stages, size_t* smem) {
    if (D < 1 || D > 256 || n < 1) return false;
    const int lds = glm_lds(D), Dp = lds - 4;
    *RB = (Dp + 63) / 64;
    // tiles of 16 chains at every D: with 32 the D <= 128 form needs more than 255 registers (3 RB x CB x 2 doubles of
    // state per thread plus the fragments), and 4096 chains are 256 CTAs, about two per SM
    *CB = 2;
    const int CT = 8 * *CB;
    const size_t limit = 227 * 1024;
    for (int c = kGlmMaxChunk; c >= 8; c >>= 1)
        for (int s = kGlmMaxStages; s >= 2; --s) {
            const size_t sm = ((size_t)s * c * lds + (size_t)CT * lds + (size_t)2 * CT * (c + 4) + 8 * CT * 3) * sizeof(double) +
                              kGlmMaxStages * sizeof(uint64_t);
            if (sm <= limit) {
                *nc = c;
                *stages = s;
                *smem = sm;
                return true;
            }
        }
    return false;
}

std::string glm_group_source(int family, int D, int n) {
    std::string s = "#define AHMC_USER_GROUPWISE\n#define GLM_N " + std::to_string(n) + "\n#define GLM_D " + std::to_string(D) +
                    "\n#define GLM_LOGIT " + std::to_string(family == AHMC_GLM_BERNOULLI_LOGIT ? 1 : 0) + "\n";
    // G lanes per chain: lane l owns the gradient coordinates d = l + G e in registers; rows are taken G at a time, lane l
    // evaluating eta, l_i and w = y - mu of row c + l, then every lane accumulates its coordinates of x_k w_k
    s += R"GLMSRC(
template <int G>
__device__ __forceinline__ double glm_group(const double* th, double* g, const double* p, int l) {
    constexpr int E = (GLM_D + G - 1) / G;
    const ahmc_group grp{l, G};
    const double* X = p + GLM_D;
    const double* y = X + (long long)GLM_N * GLM_D;
    double acc[E];
    double share = 0.0;
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int d = l + G * e;
        const double t = d < GLM_D ? th[d] : 0.0, pr = d < GLM_D ? p[d] : 0.0;
        acc[e] = -pr * t;
        share -= 0.5 * pr * t * t;
    }
    for (int c = 0; c < GLM_N; c += G) {
        const int i = c + l;
        double w = 0.0;
        if (i < GLM_N) {
            const double* xi = X + (long long)i * GLM_D;
            double eta = 0.0;
            for (int d = 0; d < GLM_D; ++d) eta = fma(xi[d], th[d], eta);
#if GLM_LOGIT
            const double t = exp(-fabs(eta));
            double li = y[i] * eta - (fmax(eta, 0.0) + log1p(t)), mu = (eta >= 0.0 ? 1.0 : t) / (1.0 + t);
            if (eta != eta) li = mu = eta;
#else
            const double mu = exp(eta), li = y[i] * eta - mu;
#endif
            share += li;
            w = y[i] - mu;
        }
        for (int k = 0; k < G; ++k) {
            const double wk = ahmc_group_bcast(grp, w, k);
            if (c + k < GLM_N) {
                const double* xk = X + (long long)(c + k) * GLM_D;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int d = l + G * e;
                    if (d < GLM_D) acc[e] = fma(xk[d], wk, acc[e]);
                }
            }
        }
    }
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int d = l + G * e;
        if (d < GLM_D) g[d] = acc[e];
    }
    return share;
}
__device__ double ahmc_user_logp_grad_group(const double* th, double* g, int D, const double* p, ahmc_group grp) {
    switch (grp.size) {
        case 4: return glm_group<4>(th, g, p, grp.lane);
        case 8: return glm_group<8>(th, g, p, grp.lane);
        case 16: return glm_group<16>(th, g, p, grp.lane);
        default: return glm_group<32>(th, g, p, grp.lane);
    }
}
)GLMSRC";
    return s;
}

#ifndef AHMC_SIMT_EMULATION
template <int RB, int CB>
static cudaError_t launch_glm_t(const GlmArgs& a, size_t sm, cudaStream_t st) {
    const long long blocks = (a.N + 8 * CB - 1) / (8 * CB);
    if (a.family == AHMC_GLM_BERNOULLI_LOGIT)
        return launch_kernel(glm_traj_kernel<RB, CB, AHMC_GLM_BERNOULLI_LOGIT>, blocks, kGlmThreads, sm, st, a);
    return launch_kernel(glm_traj_kernel<RB, CB, AHMC_GLM_POISSON_LOG>, blocks, kGlmThreads, sm, st, a);
}

cudaError_t launch_glm_traj(const GlmArgs& h, cudaStream_t st, int* n_launches) {
    GlmArgs a = h;
    int RB, CB;
    size_t sm;
    if (!glm_tile_shape(a.D, a.n, &RB, &CB, &a.nc, &a.stages, &sm)) return cudaErrorInvalidValue;
    if (n_launches) *n_launches += 1;
    switch (RB) {
        case 1: return launch_glm_t<1, 2>(a, sm, st);
        case 2: return launch_glm_t<2, 2>(a, sm, st);
        case 3: return launch_glm_t<3, 2>(a, sm, st);
        case 4: return launch_glm_t<4, 2>(a, sm, st);
    }
    return cudaErrorInvalidValue;
}
#endif  // AHMC_SIMT_EMULATION

}  // namespace ahmc
