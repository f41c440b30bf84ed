"""The host restatement of the engines' in-kernel draws (oracle/philox.py) on the CPU: Random123's known-answer vectors,
the float32 word -> uniform maps at their edges, the `uniforms` layout, and the zero Exp(1) draws the RAW head used to
make.  tests/test_gpu_sampling.py holds every engine to this restatement."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import philox as P

F32 = np.float32


@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox4x32_10_known_answer_vectors(ctr, key, want):
    """Random123's kat_vectors for philox4x32 with 10 rounds, as scalars and broadcast over an array."""
    got = P.philox4x32_10(*ctr, *key)
    assert tuple(int(v) for v in got) == want
    arr = P.philox4x32_10(np.full(3, ctr[0], np.uint64), *ctr[1:], *key)
    assert all(a.dtype == np.uint32 and (a == w).all() for a, w in zip(arr, want))


def test_philox_counter_lanes_and_key_words_are_not_interchangeable():
    base = [int(v) for v in P.philox4x32_10(1, 2, 3, 4, 5, 6)]
    for args in ((2, 1, 3, 4, 5, 6), (1, 2, 4, 3, 5, 6), (1, 2, 3, 4, 6, 5), (1, 2, 3, 5, 5, 6), (1, 2, 3, 4, 5, 7)):
        assert [int(v) for v in P.philox4x32_10(*args)] != base, args


def test_u01_edges_in_float32():
    """((float)(x >> 8) + 0.5f) * 2^-24: exact midpoints below 2^23, ties to even above, and exactly 1.0 at the top word."""
    m = np.array([0, 1, 2 ** 22, 2 ** 23 - 1], dtype=np.uint64)
    assert np.array_equal(P.u01((m << np.uint64(8)).astype(np.uint32)), ((m.astype(np.float64) + 0.5) / 2 ** 24).astype(F32))
    assert P.u01(0x000000ff) == F32(2.0 ** -25) and P.u01(0) == F32(2.0 ** -25)     # the low 8 bits are ignored
    assert P.u01(0x80000000) == F32(0.5)                                                    # 8388608.5 -> 8388608 (even)
    assert P.u01(0xfffffe00) == P.u01(0xfffffd00) == F32(1.0 - 2.0 ** -23)                # ties to the even neighbour
    assert P.u01(0xffffff00) == P.u01(0xffffffff) == F32(1.0)                              # 16777215.5 -> 2^24
    top = P.u01(np.arange(0xfff00000, 0x100000000, 0x100, dtype=np.uint64).astype(np.uint32))
    assert (top == F32(1.0)).sum() == 1 and top.dtype == F32
    # the RAW head's open map changes the top word only
    assert P.u01_open(0xffffffff) == F32(1.0 - 2.0 ** -24) and -np.log(P.u01_open(0xffffffff)) > 0
    w = np.random.RandomState(0).randint(0, 2 ** 32, 100_000, dtype=np.uint64).astype(np.uint32)
    w[:2] = 0xffffff00, 0
    keep = (w >> np.uint32(8)) != np.uint32(0xffffff)
    assert np.array_equal(P.u01_open(w)[keep], P.u01(w)[keep]) and (P.u01_open(w) < 1).all()


def test_u_ref_range_is_one_rounding_of_the_exact_fma():
    """u01 * (1 - 2e-5f) + 1e-5f is one FFMA on the device.  Its exact value fits a float64, so the restatement's
    float64 evaluation rounds once, like the FFMA; it stays inside the reference's [1e-5, 1 - 1e-5] at both ends."""
    w = np.concatenate([np.array([0, 0xff, 0x80000000, 0xfffffe00, 0xffffff00, 0xffffffff], np.uint64),
                        np.random.RandomState(1).randint(0, 2 ** 32, 2000, dtype=np.uint64)]).astype(np.uint32)
    u = P.u01(w)
    for ui in u:
        exact = Fraction(float(ui)) * Fraction(float(P.U_SPAN)) + Fraction(float(P.U_LO))
        assert Fraction(float(np.float64(ui) * np.float64(P.U_SPAN) + np.float64(P.U_LO))) == exact
    r = P.u_ref_range(w)
    assert r.dtype == F32 and r.min() >= F32(1e-5) and r.max() <= F32(1.0 - 1e-5)
    assert P.u_ref_range(0xffffffff) == F32(1.0 - 1e-5)
    assert P.u_ref_range(0) == F32(np.float64(F32(1e-5)) + 2.0 ** -25 * np.float64(F32(1.0) - F32(2e-5)))


def test_mol_uniforms_layout_and_keying():
    """Row t = [B x 10 mixture | B logistic] (helpers.replay_uniforms' layout): mixture draw k of fold f is word k of the
    blocks 0, 1, 2 keyed (t, seg_first + f, block, offset) under (seed low, seed high); the logistic draw is word 10.
    A shard (seg_first = f0) is the same columns of the whole job, cut as bench.py and vocoder.py cut them."""
    seed, off, B, S = (5 << 32) | 7, 3, 6, 4
    U = P.mol_uniforms(seed, off, 0, B, S)
    assert U.shape == (S, 11 * B) and U.dtype == F32
    for t, f in ((0, 0), (3, 5), (2, 1)):
        r = [P.philox4x32_10(t, f, b, off, 7, 5) for b in range(3)]
        words = [int(v) for blk in r for v in blk]
        want = P.u_ref_range(np.array(words[:11], np.uint32))
        assert np.array_equal(U[t, 10 * f:10 * f + 10], want[:10]) and U[t, 10 * B + f] == want[10]
    f0, n = 2, 3
    part = P.mol_uniforms(seed, off, f0, n, S)
    assert np.array_equal(part, np.concatenate([U[:, 10 * f0:10 * (f0 + n)], U[:, 10 * B + f0:10 * B + f0 + n]], 1))
    # every input of the key matters
    for other in (P.mol_uniforms(seed & 0xffffffff, off, 0, B, S), P.mol_uniforms(seed, 0, 0, B, S),
                  P.mol_uniforms(seed, off, 1, B, S)[:, :10]):
        assert not np.array_equal(other[:, :other.shape[1]], U[:, :other.shape[1]])


def test_raw_expo_keying_and_strictly_positive_draws():
    seed, off = (5 << 32) | 7, 3
    e, words = P.raw_expo(seed, off, 4, 2, 3)
    assert e.shape == words.shape == (3, 2, 512) and e.dtype == F32
    x, y, z, w = P.philox4x32_10(2, 5, 16 + 489 // 4, off, 7, 5)
    assert words[2, 1, 489] == (x, y, z, w)[489 % 4]
    assert (e > 0).all() and np.isfinite(e).all()


def test_seed_220_draws_a_zero_exponential_at_fold_0_step_29_class_489():
    """seed 220, offset 0, seg_first 0: word y of Philox block 16 + 122 at (step 29, fold 0) has x >> 8 == 0xffffff.
    u01 maps it to 1.0, so -logf(u01) was -0.0; u01_open gives the smallest Exp(1) draw instead."""
    e, words = P.raw_expo(220, 0, 0, 1, 30)
    assert words[29, 0, 489] >> 8 == 0xffffff and P.u01(words[29, 0, 489]) == F32(1.0)
    z = -np.log(P.u01(words[29, 0, 489]))
    assert z == 0 and np.signbit(z)
    assert e[29, 0, 489] == (-np.log(np.float64(F32(1.0 - 2.0 ** -24)))).astype(F32) > 0
    assert P.zero_draw_events(220, 0, 0, 1, 30) == [(0, 29, 489)]


def test_bench_cfg3_zero_draw_events():
    """bench.py --workload cfg3 (RAW head, seed 0, offset 0, 19 folds x 12,100 steps) meets the u01 == 1 word 7 times."""
    assert P.zero_draw_events(0, 0, 0, 19, 12100) == [(1, 3034, 257), (4, 9754, 214), (13, 3351, 159), (15, 439, 411),
                                                      (17, 3659, 167), (17, 10339, 331), (18, 3755, 211)]
