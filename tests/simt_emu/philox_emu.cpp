// philox_emu.cpp -- runs the device's random-stream functions on the CPU: Philox::gen and Philox::u01, philox_normals<G, E>
// for every register layout pick_layout chooses, big_normals (D > 512, tile by tile) and the exponential / direction-bit
// draws, so that tests/test_philox_streams_cpu.py can hold them against the host restatement tests/philox_ref.py.  The
// sources are included unmodified (their host launch code is skipped with AHMC_SIMT_EMULATION).  TEST INFRASTRUCTURE ONLY.
#define AHMC_SIMT_EMULATION 1
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "ahmc_leapfrog.cu"
#include "ahmc_bigd_hmc.cu"

using namespace ahmc;

extern "C" void emu_philox_gen(int64_t n, const uint64_t* seed, const uint64_t* lo, const uint64_t* hi, uint32_t* out) {
    for (int64_t i = 0; i < n; ++i) {
        uint32_t o[4];
        Philox::gen(seed[i], lo[i], hi[i], o);
        for (int w = 0; w < 4; ++w) out[4 * i + w] = o[w];
    }
}

extern "C" double emu_philox_u01(uint32_t a, uint32_t b) { return Philox::u01(a, b); }

extern "C" int emu_pick_layout(int D, int* G, int* E) { return pick_layout(D, G, E) ? 1 : 0; }

// every lane l < G of one chain's group: coordinate l + G e of the draw goes to z[l + G e]; a register past D must hold 0.
// Returns the number of such registers that do not.
template <int G, int E>
static int normals_of(uint64_t seed, uint64_t offset, long long chain, int D, double* z) {
    int bad = 0;
    for (int l = 0; l < G; ++l) {
        double r[E];
        philox_normals<G, E>(seed, offset, chain, l, D, r);
        for (int e = 0; e < E; ++e) {
            const int d = l + G * e;
            if (d < D) z[d] = r[e];
            else bad += r[e] != 0.0;
        }
    }
    return bad;
}

// the normals a D <= 512 launch draws for one chain, under the layout pick_layout chooses; -1 if D has none
extern "C" int emu_philox_normals(uint64_t seed, uint64_t offset, long long chain, int D, double* z) {
    int G, E;
    if (!pick_layout(D, &G, &E)) return -1;
    switch (G * 100 + E) {
        case 401: return normals_of<4, 1>(seed, offset, chain, D, z);
        case 801: return normals_of<8, 1>(seed, offset, chain, D, z);
        case 1601: return normals_of<16, 1>(seed, offset, chain, D, z);
        case 3201: return normals_of<32, 1>(seed, offset, chain, D, z);
        case 3202: return normals_of<32, 2>(seed, offset, chain, D, z);
        case 3204: return normals_of<32, 4>(seed, offset, chain, D, z);
        case 3208: return normals_of<32, 8>(seed, offset, chain, D, z);
        case 3216: return normals_of<32, 16>(seed, offset, chain, D, z);
    }
    return -1;
}

// the normals the D > 512 streaming kernels draw for one chain (big_normals, tile by tile, any D >= 1)
extern "C" int emu_big_normals(uint64_t seed, uint64_t offset, long long chain, int D, double* z) {
    int bad = 0;
    for (int d0 = 0; d0 < D; d0 += kBigTile)
        for (int l = 0; l < 32; ++l) {
            double r[kBigE];
            big_normals(nullptr, seed, offset, chain, d0, l, D, r);
            for (int e = 0; e < kBigE; ++e) {
                const int d = d0 + l + 32 * e;
                if (d < D) z[d] = r[e];
                else bad += r[e] != 0.0;
            }
        }
    return bad;
}

// exponential #k and direction bit #k of (chain, transition offset), for k < n
extern "C" void emu_philox_exp(uint64_t seed, uint64_t offset, long long chain, int n, double* out) {
    for (int k = 0; k < n; ++k) out[k] = philox_exp(seed, offset, chain, k);
}
extern "C" void emu_philox_bits(uint64_t seed, uint64_t offset, long long chain, int n, uint8_t* out) {
    for (int k = 0; k < n; ++k) out[k] = philox_bit(seed, offset, chain, k) ? 1 : 0;
}
