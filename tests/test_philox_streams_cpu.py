"""CPU checks of the on-device random streams: the host restatement (tests/philox_ref.py) against Random123's known answers
for Philox4x32-10, the counter map's injectivity inside its bounds (and the collision beyond them), the coordinate -> block
rule of every register layout, and the device source itself -- Philox::gen, philox_normals<G, E> for every layout,
big_normals and the exponential / direction-bit draws -- run on the CPU (tests/simt_emu/philox_emu.cpp) against the
restatement.  The GPU side is tests/test_philox_streams.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import philox_ref as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "simt_emu")
CSRC = os.path.join(ROOT, "advancedhmc.jl_b200", "csrc")
SEEDS = [0, 1, 2026, 2**32 + 17, 0xDEADBEEFCAFEF00D]  # seeds >= 2^32: key word k1 != 0
OFFSETS = [0, 1, 2**35 + 3, 2**36 - 1]

# Random123 known-answer vectors for Philox4x32-10 (kat_vectors): counter words, key words, output words
KAT = [
    ([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0], [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]),
]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = tmp_path_factory.mktemp("simt_philox") / "libphilox_emu.so"
    cmd = ["g++", "-O1", "-shared", "-fPIC", "-std=c++20", "-pthread", "-ffp-contract=off", "-w", "-I", os.path.join(EMU, "include"),
           "-I", CSRC, "-I", os.path.join(ROOT, "include"), os.path.join(EMU, "simt_emu.cpp"), os.path.join(EMU, "philox_emu.cpp"),
           "-o", str(out)]
    pr = subprocess.run(cmd, capture_output=True, text=True)
    assert pr.returncode == 0, pr.stderr[-2000:]
    lib = C.CDLL(str(out))
    lib.emu_philox_u01.restype = C.c_double
    lib.emu_philox_u01.argtypes = [C.c_uint32, C.c_uint32]
    for f in (lib.emu_philox_normals, lib.emu_big_normals):
        f.argtypes = [C.c_uint64, C.c_uint64, C.c_longlong, C.c_int, C.c_void_p]
    lib.emu_philox_exp.argtypes = [C.c_uint64, C.c_uint64, C.c_longlong, C.c_int, C.c_void_p]
    lib.emu_philox_bits.argtypes = [C.c_uint64, C.c_uint64, C.c_longlong, C.c_int, C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ---------------------------------------------------------------------------------------------- the restatement
@pytest.mark.parametrize("ctr,key,want", KAT)
def test_restatement_matches_random123_known_answers(ctr, key, want):
    got = P.philox4x32_10(ctr, key)
    assert [int(v) for v in got] == want


def test_u01_is_the_top_53_bits_plus_a_half():
    assert P.u01(0, 0) == 2.0**-54
    assert P.u01(0, 0x7FF) == 2.0**-54  # the 11 low bits are dropped
    assert P.u01(0, 0x800) == 1.5 * 2.0**-53
    assert P.u01(0x80000000, 0) == 0.5 + 2.0**-54
    # above 2^52 the half rounds to even: the all-ones block maps to 1.0 (exp draw 0, Box-Muller radius 0), never above
    assert P.u01(0xFFFFFFFF, 0xFFFFFFFF) == 1.0
    rng = np.random.default_rng(0)
    a, b = rng.integers(0, 2**32, 10_000, dtype=np.uint64), rng.integers(0, 2**32, 10_000, dtype=np.uint64)
    u = P.u01(a, b)
    assert (u > 0).all() and (u <= 1).all()
    x = ((a << np.uint64(32)) | b) >> np.uint64(11)
    small = x < 2**52
    assert np.array_equal(u[small], (x[small].astype(np.float64) + 0.5) * 2.0**-53)


def _pack(chain, offset, stream, block):
    c0, c1, c2, c3 = P.counter(chain, offset, stream, block)
    return [tuple(int(w) for w in ws) for ws in zip(np.ravel(c0), np.ravel(c1), np.ravel(c2), np.ravel(c3))]


def test_counter_map_is_injective_inside_its_bounds():
    """chains < 2^20, offsets < 2^36, blocks < 2^24, streams {normal, exp, dir}: distinct arguments, distinct counters --
    on random samples and on every combination of boundary values"""
    rng = np.random.default_rng(11)
    n = 20_000
    args = set()
    for s in (P.STREAM_NORMAL, P.STREAM_EXP, P.STREAM_DIR):
        ch = rng.integers(0, 2**20, n)
        of = rng.integers(0, 2**36, n)
        bl = rng.integers(0, 2**24, n)
        args |= {(int(c), int(o), s, int(b)) for c, o, b in zip(ch, of, bl)}
        # neighbours of the random samples: one step along each coordinate
        args |= {(int(c), int(o) ^ 1, s, int(b)) for c, o, b in zip(ch[:2000], of[:2000], bl[:2000])}
        args |= {(int(c), int(o), s, int(b) ^ 1) for c, o, b in zip(ch[:2000], of[:2000], bl[:2000])}
    edge_c, edge_o, edge_b = [0, 1, 2**20 - 1], [0, 1, 2**35, 2**36 - 2, 2**36 - 1], [0, 1, 2**23, 2**24 - 2, 2**24 - 1]
    args |= {(c, o, s, b) for c in edge_c for o in edge_o for b in edge_b for s in (1, 2, 3)}
    a = np.array(sorted(args), dtype=np.int64)
    ctrs = _pack(a[:, 0], a[:, 1], a[:, 2], a[:, 3])
    assert len(ctrs) == len(args) > 60_000 and len(set(ctrs)) == len(args)
    assert _pack(2**20 - 1, 2**36 - 1, P.STREAM_DIR, 2**24 - 1) == [(2**20 - 1, 0, 0xFFFFFFFF, 0x3FFFFFFF | (P.STREAM_DIR << 28))]


def test_counter_map_collides_beyond_its_bounds():
    """why both bounds exist: offset 3 * 2^36 puts 3 into the stream bits (the normal stream there IS the exp stream at
    offset 0), and block 2^24 is the next offset's block 0"""
    for chain, block in [(0, 0), (5, 77), (2**20 - 1, 2**24 - 1)]:
        assert _pack(chain, 3 * 2**36, P.STREAM_NORMAL, block) == _pack(chain, 0, P.STREAM_EXP, block)
        assert _pack(chain, 2**36, P.STREAM_EXP, block) == _pack(chain, 0, P.STREAM_DIR, block)
    assert _pack(3, 9, P.STREAM_EXP, 2**24) == _pack(3, 8, P.STREAM_EXP, 0)
    # and so do the variates: the D = 8 draw (G = 8: blocks 0..7, cosines only) at offset 3 * 2^36 is Box-Muller of the
    # words that give exponentials 0..15 at offset 0
    blk, comp = P.layout_rule(8)
    assert np.array_equal(blk, np.arange(8)) and (comp == 0).all()
    o = P.block_words(7, 0, 4, P.STREAM_EXP, np.arange(8))
    assert np.array_equal(P.normals(7, 3 * 2**36, 4, 8), P.box_muller(o)[0])
    assert np.array_equal(P.u01(o[0], o[1]), P.exp_uniform(7, 0, 4, np.arange(0, 16, 2)))


# ---------------------------------------------------------------------------------------------- layout rule
@pytest.mark.parametrize("D", P.LAYOUT_DS)
def test_layout_rule_is_injective_and_uses_ceil_E_over_2_blocks_per_lane(D):
    G, E = P.pick_layout(D)
    blk, comp = P.layout_rule(D)
    pairs = set(zip(blk.tolist(), comp.tolist()))
    assert len(pairs) == D  # no two coordinates share a (block, component)
    assert blk.max() < G * ((E + 1) // 2)
    # a cosine and its sine sit on the same lane: the sine of block b is coordinate (cosine's) + G
    d = np.arange(D)
    cos_of = {b: dd for b, c, dd in zip(blk, comp, d) if c == 0}
    for b, c, dd in zip(blk, comp, d):
        if c == 1:
            assert dd == cos_of[b] + G


def test_big_rule_extends_the_512_layout():
    b512, c512 = P.layout_rule(512)
    for D in (513, 1000, 1537, 4096):
        b, c = P.big_rule(D)
        assert np.array_equal(b[:512], b512) and np.array_equal(c[:512], c512)
        assert len(set(zip(b.tolist(), c.tolist()))) == D
        assert b.max() < (D + 1) // 2 + 32 and b.max() < 2**24
    # the D > 512 draw of chain c: its first 512 coordinates are the D = 512 draw
    z = P.normals(2**33 + 1, 5, np.arange(3), 1200)
    assert np.array_equal(z[:, :512], P.normals(2**33 + 1, 5, np.arange(3), 512))


# ---------------------------------------------------------------------------------------------- device source on the CPU
def test_device_philox_gen_matches_known_answers_and_restatement(emu):
    rng = np.random.default_rng(3)
    n = 4096
    seeds = np.concatenate([rng.integers(0, 2**63, n // 2, dtype=np.uint64) * np.uint64(2), rng.integers(0, 2**32, n // 2, dtype=np.uint64)])
    lo = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    hi = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2)
    for (c, k, want) in KAT:
        seeds[:1] = k[0] | (k[1] << 32)
        lo[:1] = c[0] | (c[1] << 32)
        hi[:1] = c[2] | (c[3] << 32)
        out = np.zeros((n, 4), dtype=np.uint32)
        emu.emu_philox_gen(C.c_int64(n), _p(seeds), _p(lo), _p(hi), _p(out))
        assert out[0].tolist() == want
        m32 = np.uint64(0xFFFFFFFF)
        ref = P.philox4x32_10((lo & m32, lo >> np.uint64(32), hi & m32, hi >> np.uint64(32)), (seeds & m32, seeds >> np.uint64(32)))
        assert np.array_equal(out.T.astype(np.uint64), ref)


def test_device_u01_matches_restatement_bit_for_bit(emu):
    rng = np.random.default_rng(4)
    words = [(0, 0), (0xFFFFFFFF, 0xFFFFFFFF), (0, 0x7FF), (0x80000000, 0), (0xFFFFFFFF, 0xFFFFF7FF)]
    words += [tuple(int(x) for x in rng.integers(0, 2**32, 2)) for _ in range(2000)]
    for a, b in words:
        assert emu.emu_philox_u01(a, b) == float(P.u01(a, b))


@pytest.mark.parametrize("D", P.LAYOUT_DS)
def test_device_philox_normals_match_restatement_for_every_layout(emu, D):
    for seed in SEEDS[1:4]:
        for offset in OFFSETS:
            for chain in (0, 1, 4099, 2**20 - 1):
                z = np.full(D, np.nan)
                assert emu.emu_philox_normals(seed, offset, chain, D, _p(z)) == 0  # registers past D hold 0
                want = P.normals(seed, offset, chain, D)
                assert np.abs(z - want).max() < 1e-13, (seed, offset, chain, np.abs(z - want).max())


@pytest.mark.parametrize("D", [1, 100, 512, 513, 1000, 1537, 2100])
def test_device_big_normals_match_restatement_and_the_512_draw(emu, D):
    for seed, offset, chain in [(2026, 0, 0), (2**32 + 17, 1, 7), (0xDEADBEEFCAFEF00D, 2**35 + 3, 2**20 - 1)]:
        z = np.full(D, np.nan)
        assert emu.emu_big_normals(seed, offset, chain, D, _p(z)) == 0
        blk, comp = P.big_rule(D)
        o = P.block_words(seed, offset, chain, P.STREAM_NORMAL, blk)
        cs, sn = P.box_muller(o)
        want = np.where(comp == 0, cs, sn)
        assert np.abs(z - want).max() < 1e-13
        if D > 512:  # the first 512 coordinates of a D > 512 draw are the D = 512 register-layout draw
            z512 = np.zeros(512)
            emu.emu_philox_normals(seed, offset, chain, 512, _p(z512))
            assert np.array_equal(z[:512], z512)
        else:  # D = 1, 100 and 512 have a layout whose rule the big rule restricts to
            assert np.abs(z - P.normals(seed, offset, chain, D)).max() < 1e-13


def test_device_exponentials_and_direction_bits_match_restatement(emu):
    n = 1500  # several 128-bit blocks of direction bits, hundreds of exponential blocks
    for seed in SEEDS:
        for offset in OFFSETS:
            for chain in (0, 3, 2**20 - 1):
                e = np.zeros(n)
                emu.emu_philox_exp(seed, offset, chain, n, _p(e))
                # -log of the same uniform; host libm and numpy may differ by an ulp in log
                assert np.abs(e - -np.log(P.exp_uniform(seed, offset, chain, np.arange(n)))).max() < 1e-13
                b = np.zeros(n, dtype=np.uint8)
                emu.emu_philox_bits(seed, offset, chain, n, _p(b))
                assert np.array_equal(b, P.dir_bit(seed, offset, chain, np.arange(n)))
