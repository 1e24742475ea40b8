"""The host restatement of the device Philox stream (tests/_philox.py) against the Random123 known-answer vectors,
and the properties the perf-mode tests rely on: a keep rate of one half, streams and steps that differ, and the
layout of the keep bits."""
import numpy as np

from tests import _philox as P


def _words(r):
    return [int(np.asarray(w).reshape(-1)[0]) for w in r]


def test_philox4x32_10_known_answers():
    # Random123 kat_vectors: philox4x32 10 rounds
    assert _words(P.philox4x32_10((0, 0, 0, 0), (0, 0))) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    ones = 0xFFFFFFFF
    assert _words(P.philox4x32_10((ones,) * 4, (ones, ones))) == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    assert _words(P.philox4x32_10((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0))) == \
        [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def test_vectorised_call_matches_scalar_calls():
    ctr = np.array([0, 1, 2**32 - 1, 12345], dtype=np.uint64)
    got = P.philox4x32_10((ctr, 7, 3, 0), (0xdeadbeef, 0x1234))
    for i, c in enumerate(ctr):
        assert [int(w[i]) for w in got] == _words(P.philox4x32_10((int(c), 7, 3, 0), (0xdeadbeef, 0x1234)))


def test_keep_mask_bit_layout():
    """Element idx = m*H + n is bit idx & 31 of word idx >> 5; words come four to a Philox call whose counter is
    (word >> 2 split into 32-bit halves, (step << 8) | stream split into halves), keyed (seed lo, seed hi)."""
    seed, step, sid, n, H = (7 << 32) | 99, 3, 5, 7, 50          # H % 32 != 0: rows straddle words
    m = P.keep_mask(seed, step, sid, n, H)
    assert m.shape == (n, H) and m.dtype == np.uint8
    for idx in (0, 31, 32, 49, 50, 127, 128, 200, n * H - 1):
        w = idx >> 5
        r = _words(P.philox4x32_10((w >> 2, 0, (step << 8) | sid, 0), (99, 7)))
        assert m.reshape(-1)[idx] == (r[w & 3] >> (idx & 31)) & 1, idx


def test_keep_rate_and_distinct_streams():
    seed = 1234
    masks = {(step, k): P.keep_mask(seed, step, k, 300, 100) for step in (0, 1) for k in range(8)}
    for m in masks.values():
        assert abs(m.mean() - 0.5) < 0.01
    keys = list(masks)
    for i, a in enumerate(keys):
        for b in keys[i + 1:]:
            agree = (masks[a] == masks[b]).mean()
            assert abs(agree - 0.5) < 0.01, (a, b, agree)        # independent streams agree on about half the bits
    assert not np.array_equal(P.keep_mask(seed, 0, 0, 4, 32), P.keep_mask(seed + 1, 0, 0, 4, 32))


def test_td3_noise_is_standard_normal_times_std():
    z = P.td3_noise(77, 0, 4000, 33, 0.5)
    assert z.shape == (4000, 33) and np.isfinite(z).all()
    assert abs(z.mean()) < 0.01 and abs(z.std() - 0.5) < 0.01
    assert not np.array_equal(z, P.td3_noise(77, 1, 4000, 33, 0.5))
    # element (m, n) depends on m*A + n only: the same counter gives the same draw whatever the shape
    np.testing.assert_array_equal(P.td3_noise(77, 0, 33, 4000, 0.5).reshape(-1), z.reshape(-1))
