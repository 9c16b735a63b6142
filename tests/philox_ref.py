"""philox_ref.py -- an independent host restatement of the on-device random streams (plain numpy, uint64 arithmetic,
vectorised over chains and draws).  TEST INFRASTRUCTURE ONLY.

The library draws every variate from Philox4x32-10 (Salmon et al. 2011) keyed by the 64-bit seed (k0 = low word,
k1 = high word).  The 128-bit counter of a draw is (lo, hi) = (chain, (offset << 24) ^ (stream << 60) ^ block): chain in
words 0-1, the transition offset in bits 24..59 of the high half, the stream id in bits 60..63 and the block in bits 0..23.
The map is injective while block < 2^24 and offset < 2^36.  Three streams:
  * normals (stream 1): coordinate d of a register layout with G lanes (d = l + G e) uses block l + G floor(e / 2), the
    cosine of the Box-Muller pair for even e and the sine for odd e.  G follows from D (`pick_layout`); above D = 512 the
    G = 32 rule continues tile by tile (block (d mod 32) + 32 floor(floor(d / 32) / 2)), so the first 512 coordinates of a
    D > 512 draw are the D = 512 draw;
  * exponentials / uniforms (stream 2): variate k uses block k >> 1, words (o0, o1) for even k and (o2, o3) for odd k;
  * direction bits (stream 3): bit k is bit k & 31 of word (k >> 5) & 3 of block k >> 7.
The tape builders below turn these streams into the tapes the CPU oracle consumes, so a Philox-mode launch can be checked
chain by chain against the oracle the same way a tape launch is.
"""
from __future__ import annotations

import numpy as np

U64 = np.uint64
MASK32 = U64(0xFFFFFFFF)
_M0, _M1 = U64(0xD2511F53), U64(0xCD9E8D57)
_W0, _W1 = U64(0x9E3779B9), U64(0xBB67AE85)
STREAM_NORMAL, STREAM_EXP, STREAM_DIR = 1, 2, 3
OFFSET_BITS, BLOCK_BITS = 36, 24
LAYOUT_DS = [1, 3, 4, 5, 8, 10, 16, 17, 32, 33, 64, 100, 128, 129, 200, 256, 300, 512]


def _u64(x):
    """a non-negative int (taken modulo 2^64) or an integer array -> uint64"""
    if isinstance(x, (int, np.integer)):
        return U64(int(x) & 0xFFFFFFFFFFFFFFFF)
    return np.asarray(x).astype(U64)


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counter words ctr = (c0, c1, c2, c3) under key words key = (k0, k1); the words broadcast against
    each other.  Returns the four output words as a uint64 array of shape (4, *broadcast shape), each < 2^32."""
    c0, c1, c2, c3 = (_u64(c) & MASK32 for c in ctr)
    k0, k1 = (_u64(k) & MASK32 for k in key)
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(c0, c1, c2, c3, k0, k1)
    c0, c1, c2, c3, k0, k1 = (np.array(v, dtype=U64) for v in (c0, c1, c2, c3, k0, k1))
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0, p1 = _M0 * c0, _M1 * c2  # 32 x 32 -> 64 bits: exact in uint64
            c0, c1, c2, c3 = (p1 >> U64(32)) ^ c1 ^ k0, p1 & MASK32, (p0 >> U64(32)) ^ c3 ^ k1, p0 & MASK32
            k0, k1 = (k0 + _W0) & MASK32, (k1 + _W1) & MASK32
    return np.stack([c0, c1, c2, c3])


def counter(chain, offset, stream, block):
    """the four 32-bit counter words of draw `block` of `stream` for (chain, transition offset), modulo 2^64 like the
    device's uint64 arithmetic"""
    chain, offset, stream, block = _u64(chain), _u64(offset), _u64(stream), _u64(block)
    with np.errstate(over="ignore"):
        hi = (offset << U64(24)) ^ (stream << U64(60)) ^ block
    return chain & MASK32, chain >> U64(32), hi & MASK32, hi >> U64(32)


def key(seed):
    s = _u64(seed)
    return s & MASK32, s >> U64(32)


def block_words(seed, offset, chain, stream, block):
    """output words (4, *shape) of Philox block `block` of `stream` for (seed, offset, chain)"""
    return philox4x32_10(counter(chain, offset, stream, block), key(seed))


def u01(a, b):
    """uniform from two 32-bit words: the top 53 bits of (a << 32 | b), plus a half, times 2^-53 -- the same IEEE
    operations as the device, so bit-identical.  The conversion is exact; the + 0.5 rounds (to even) once the 53-bit
    integer reaches 2^52, so the range is (0, 1], with 1.0 for the all-ones block only."""
    x = ((_u64(a) << U64(32)) | _u64(b)) >> U64(11)
    return (x.astype(np.float64) + 0.5) * (1.0 / 9007199254740992.0)


def pick_layout(D):
    """(G, E): lanes per chain and coordinates per lane of the register-resident layouts (D <= 512)"""
    if D < 1 or D > 512:
        raise ValueError(f"no register layout for D={D}")
    for lim, G, E in [(4, 4, 1), (8, 8, 1), (16, 16, 1), (32, 32, 1), (64, 32, 2), (128, 32, 4), (256, 32, 8), (512, 32, 16)]:
        if D <= lim:
            return G, E


def layout_rule(D):
    """(block, component) of every coordinate d < D of a normal draw: component 0 takes the cosine, 1 the sine"""
    d = np.arange(D, dtype=np.int64)
    if D <= 512:
        G, _ = pick_layout(D)
        l, e = d % G, d // G
        return l + G * (e // 2), e % 2
    return big_rule(D)


def big_rule(D):
    """the D > 512 rule (G = 32 continued tile by tile), defined for any D"""
    d = np.arange(D, dtype=np.int64)
    return d % 32 + 32 * ((d // 32) // 2), (d // 32) % 2


def box_muller(o):
    """(cos, sin) normals of a block's words o = (o0, o1, o2, o3): sqrt(-2 log u1) (cos, sin)(2 pi u2)"""
    u1, u2 = u01(o[0], o[1]), u01(o[2], o[3])
    rad = np.sqrt(-2.0 * np.log(u1))
    return rad * np.cos(np.pi * (2.0 * u2)), rad * np.sin(np.pi * (2.0 * u2))


def normals(seed, offset, chain, D):
    """the standard normals of a momentum draw: shape (len(chain), D) for an array of chains, (D,) for one chain"""
    ch = np.atleast_1d(np.asarray(chain, dtype=np.int64))
    blk, comp = layout_rule(D)
    o = block_words(seed, offset, ch[:, None], STREAM_NORMAL, blk[None, :])
    cs, sn = box_muller(o)
    z = np.where(comp[None, :] == 0, cs, sn)
    return z[0] if np.ndim(chain) == 0 else z


def exp_uniform(seed, offset, chain, k):
    """uniform #k of the exponential stream of (chain, transition offset); chain and k broadcast"""
    k = np.asarray(k, dtype=np.int64)
    o = block_words(seed, offset, chain, STREAM_EXP, k >> 1)
    odd = (k & 1) == 1
    return np.where(odd, u01(o[2], o[3]), u01(o[0], o[1]))


def dir_bit(seed, offset, chain, k):
    """direction bit #k of (chain, transition offset) as uint8; chain and k broadcast"""
    k = np.asarray(k, dtype=np.int64)
    o = block_words(seed, offset, chain, STREAM_DIR, k >> 7)
    word = np.choose((k >> 5) & 3, list(o))  # o has shape (4, *shape); pick word (k >> 5) & 3 elementwise
    return ((word >> (k & 31).astype(U64)) & U64(1)).astype(np.uint8)


# ---------------------------------------------------------------------------------------------- oracle tapes
def normal_tape(seed, offset, N, D):
    """(D, N) normals: the oracle's layout of what a Philox-mode refresh draws for chains 0..N-1"""
    return np.asfortranarray(normals(seed, offset, np.arange(N), D).T)


def static_exp_tape(seed, offset, N):
    """(N,) the static EndPointTS transition's Exp(1) draw: -log of uniform #0"""
    return -np.log(exp_uniform(seed, offset, np.arange(N), 0))


def static_unif_tape(seed, offset, N):
    """(N,) the static MultinomialTS transition's `randcat` uniform: uniform #0 (words o0, o1 of block 0)"""
    return exp_uniform(seed, offset, np.arange(N), 0)


def nuts_exp_tape(seed, offset, N, n_exp, sampler="multinomial"):
    """(N, n_exp) the NUTS exponential tape: MultinomialTS draws -log u_k; SliceTS draws -log u_0 for the slice variable
    and then the uniforms u_k themselves (the convention of the tape form, trajectory.jl:144-145, 178-183, 202)"""
    u = exp_uniform(seed, offset, np.arange(N)[:, None], np.arange(n_exp)[None, :])
    t = -np.log(u)
    if sampler == "slice":
        t[:, 1:] = u[:, 1:]
    return t


def dir_tape(seed, offset, N, n_dir):
    """(N, n_dir) uint8 direction bits"""
    return dir_bit(seed, offset, np.arange(N)[:, None], np.arange(n_dir)[None, :])
