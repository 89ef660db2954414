"""oracle/philox.py, the numpy restatement of the in-kernel Langevin noise, on its own: the published known-answer
vectors of Philox4x32-10, where the seed, step and slot words go, and the Box-Muller transforms at the ends of the
uniform range.  (The draws of the kernels themselves are compared with it in test_gpu_langevin_noise.)"""
import numpy as np
import pytest

from oracle import philox as P

# Random123's known-answer vectors for philox4x32-10: (counter c0..c3, key k0 k1) -> output words
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("counter,key,want", KAT, ids=["zeros", "ones", "pi"])
def test_philox_known_answers(counter, key, want):
    got = tuple(int(w) for w in P.philox4x32_10(counter, key))
    assert got == want, [f"{w:08x}" for w in got]


def test_philox_vectorised_equals_one_at_a_time():
    rng = np.random.default_rng(0)
    c = rng.integers(0, 2**32, size=(4, 64), dtype=np.uint64)
    k = rng.integers(0, 2**32, size=(2, 64), dtype=np.uint64)
    batch = np.stack(P.philox4x32_10(tuple(c), tuple(k)))
    for j in range(64):
        one = P.philox4x32_10(tuple(int(x) for x in c[:, j]), tuple(int(x) for x in k[:, j]))
        assert tuple(int(w) for w in one) == tuple(int(w) for w in batch[:, j])


SEED, STEP, SLOT = 0x1234_5678_9ABC_DEF1 & (2**62 - 1), 0x0000_0007_0000_0003, 0x0000_0002_0000_0005


def test_words_land_in_their_halves():
    """key = (seed lo, seed hi), counter = (slot lo, slot hi, step lo, step hi): the draw equals the transform of the
    Philox block of exactly those words, in both precisions."""
    lo, hi = (lambda x: x & 0xFFFFFFFF), (lambda x: x >> 32)
    block = P.philox4x32_10((lo(SLOT), hi(SLOT), lo(STEP), hi(STEP)), (lo(SEED), hi(SEED)))
    np.testing.assert_array_equal(P.normal3_f32(SEED, STEP, SLOT), P.box_muller_f32(block))
    block2 = P.philox4x32_10((lo(SLOT), hi(SLOT) | 0x80000000, lo(STEP), hi(STEP)), (lo(SEED), hi(SEED)))
    np.testing.assert_array_equal(P.normal3_f64(SEED, STEP, SLOT), P.box_muller_f64(block, block2))


@pytest.mark.parametrize("normal", [P.normal3_f32, P.normal3_f64], ids=["fp32", "fp64"])
def test_every_word_changes_the_draw(normal):
    """Each of the six 32-bit words (both seed words, both step words, both slot words) changes every component."""
    base = normal(SEED, STEP, SLOT)
    for seed, step, slot in [(SEED ^ 1, STEP, SLOT), (SEED ^ (1 << 32), STEP, SLOT), (SEED, STEP ^ 1, SLOT),
                             (SEED, STEP ^ (1 << 32), SLOT), (SEED, STEP, SLOT ^ 1), (SEED, STEP, SLOT ^ (1 << 32))]:
        assert np.all(normal(seed, step, slot) != base), (seed, step, slot)
    # the step and slot words are not interchangeable
    assert np.all(normal(SEED, SLOT, STEP) != base)


def test_langevin_noise_layout():
    """Step k of a call keyed on first_step + position + k, atom i of replica r on slot r * N + i; the step wraps mod 2^64."""
    seed, R, N = 2**62 - 1, 2, 5
    for dtype, normal in ((np.float32, P.normal3_f32), (np.float64, P.normal3_f64)):
        z = P.langevin_noise(seed, 3, R, N, dtype, position=4, first_step=2**32 - 2)
        assert z.shape == (3, R, N, 3) and z.dtype == dtype
        for k in range(3):
            for r in range(R):
                np.testing.assert_array_equal(z[k, r], normal(seed, 2**32 - 2 + 4 + k + 1, np.arange(N, dtype=np.uint64) + r * N))
        wrap = P.langevin_noise(seed, 2, 1, N, dtype, first_step=2**64 - 1)
        np.testing.assert_array_equal(wrap[0], normal(seed, 0, np.arange(N, dtype=np.uint64))[None])
        np.testing.assert_array_equal(wrap[1], normal(seed, 1, np.arange(N, dtype=np.uint64))[None])
        # a later call continues the stream of an earlier one
        np.testing.assert_array_equal(P.langevin_noise(seed, 5, R, N, dtype)[3:], P.langevin_noise(seed, 2, R, N, dtype, position=3))
    import torch

    np.testing.assert_array_equal(P.langevin_noise(7, 1, 1, 4, torch.float64), P.langevin_noise(7, 1, 1, 4, np.float64))
    np.testing.assert_array_equal(P.langevin_noise(7, 1, 1, 4, torch.float32), P.langevin_noise(7, 1, 1, 4, np.float32))


def test_uniforms_and_extreme_words():
    """The uniforms stay inside (0, 1) at the extreme words, and the draws stay finite and bounded there."""
    assert P._uniform_f32(np.uint64(0)) == np.float32(2.0**-25)
    assert P._uniform_f32(np.uint64(0xFFFFFFFF)) == np.float32(1.0)  # (2^24 - 1) + 0.5 rounds to 2^24 in fp32: u = 1
    assert P.u53(0, 0) == 2.0**-54 and P.u53(0xFFFFFFFF, 0xFFFFFFFF) == 1.0 - 2.0**-54
    for w in (0, 0xFFFFFFFF):
        for block in [(w, w, w, w), (w, 0, w, 0), (0, w, 0, w)]:
            x = P.box_muller_f32(tuple(np.uint64(b) for b in block))
            assert np.all(np.isfinite(x)) and np.abs(x).max() <= 6.0, (block, x)
            y = P.box_muller_f64(tuple(np.uint64(b) for b in block), tuple(np.uint64(b) for b in block))
            assert np.all(np.isfinite(y)) and np.abs(y).max() <= 9.0, (block, y)
    # u = 1 (all ones): log u = 0, so r = 0 and the draw is exactly zero; u smallest: the largest radius
    assert np.all(P.box_muller_f32((np.uint64(0xFFFFFFFF),) * 4)[..., :2] == 0)
    r_max = P.box_muller_f32((np.uint64(0), np.uint64(0), np.uint64(0), np.uint64(0)))[0]
    np.testing.assert_allclose(r_max, np.sqrt(-2 * np.log(2.0**-25)), rtol=1e-6)


def test_moments():
    """A sanity check of the restatement (the exact comparison with the kernels is what matters)."""
    for dtype in (np.float32, np.float64):
        z = P.langevin_noise(11, 4, 2, 50000, dtype).reshape(-1).astype(np.float64)
        assert abs(z.mean()) < 0.005 and abs(z.std() - 1) < 0.005 and abs((z**4).mean() - 3) < 0.05
