"""CPU: the host reference of the noise the LM step draws itself (``philox4x32_10`` / ``step_noise_ref`` in tests/util.py),
against the published Philox4x32-10 known answers and the element layout of ``lm_noise_kernel``."""
import numpy as np
import pytest

from tests.util import exp1_ref64, f32_ulp, philox4x32_10, step_noise_ref, step_words

# Random123's known-answer vectors for philox4x32_10 (kat_vectors): counter, key -> output
KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT, ids=["zero", "ones", "pi"])
def test_philox_known_answers(ctr, key, want):
    got = philox4x32_10(np.array(ctr, dtype=np.uint64), np.array(key, dtype=np.uint64))
    assert got.dtype == np.uint32
    assert [int(v) for v in got] == list(want), [hex(int(v)) for v in got]


def test_philox_vectorised_equals_one_by_one():
    rng = np.random.default_rng(5)
    ctr = rng.integers(0, 2 ** 32, size=(37, 4), dtype=np.uint64)
    key = rng.integers(0, 2 ** 32, size=(37, 2), dtype=np.uint64)
    batch = philox4x32_10(ctr, key)
    for i in range(37):
        assert np.array_equal(batch[i], philox4x32_10(ctr[i], key[i]))


@pytest.mark.parametrize("seed,ctr", [(0, 0), (2 ** 62 - 1, 1), (0x1234_5678_9ABC_DEF1, 2 ** 32 + 5)])
def test_step_layout(seed, ctr):
    """Element i is word i % 4 of block i // 4, counter (q lo, q hi, ctr lo, ctr hi), key (seed lo, seed hi); a prefix of a
    longer draw is the shorter draw."""
    n = 2025 * 3 + 2
    w = step_words(seed, ctr, n)
    assert w.shape == (n,) and w.dtype == np.uint32
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64)
    for q in (0, 1, 506, (n - 1) // 4):
        block = philox4x32_10(np.array([q, 0, ctr & 0xFFFFFFFF, ctr >> 32], dtype=np.uint64), key)
        for j in range(4):
            if 4 * q + j < n:
                assert w[4 * q + j] == block[j]
    assert np.array_equal(step_words(seed, ctr, 5), w[:5])
    # the high word of the block index reaches the counter
    q = 2 ** 32 + 3
    far = philox4x32_10(np.array([q & 0xFFFFFFFF, q >> 32, ctr & 0xFFFFFFFF, ctr >> 32], dtype=np.uint64), key)
    near = philox4x32_10(np.array([3, 0, ctr & 0xFFFFFFFF, ctr >> 32], dtype=np.uint64), key)
    assert not np.array_equal(far, near)
    m, x = step_noise_ref(seed, ctr, n)
    assert np.array_equal(m, w >> np.uint32(8))
    assert np.array_equal(x, -np.log((m.astype(np.float64) + 1) / 2 ** 24))


def test_streams_differ_by_seed_counter_and_element():
    a = step_words(7, 0, 4096)
    for other in (step_words(8, 0, 4096), step_words(7, 1, 4096), step_words(7 + 2 ** 32, 0, 4096), step_words(7, 2 ** 32, 4096)):
        assert (a != other).mean() > 0.99
    assert np.unique(a).size > 4090


def test_reference_draws_look_exponential():
    """The fp64 draws of the reference over 2^20 elements: mean and variance 1 within 6 standard errors."""
    _, x = step_noise_ref(11, 3, 1 << 20)
    n = x.size
    assert x.min() > 0
    assert abs(x.mean() - 1) < 6 / np.sqrt(n)
    assert abs(x.var() - 1) < 6 * np.sqrt(8 / n)


def test_exp1_ref64_edges():
    assert exp1_ref64(np.array([2 ** 24 - 1]))[0] == 0.0
    assert exp1_ref64(np.array([0]))[0] == pytest.approx(24 * np.log(2), rel=1e-15)
    assert f32_ulp(np.array([1.0]))[0] == 2.0 ** -23
    assert f32_ulp(np.array([2.0 ** -24]))[0] == 2.0 ** -47
