"""Host-side checks of the REINFORCE policy's sampled slates: the C symbols, the record size, the refusals of
DiscreteActor.sample_topk before any device work, and the float64 restatement (tests/_policy_sample_oracle.py) against
brute-force Plackett-Luce probabilities and against its own sharded merge.  No kernel is launched."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest
import torch
from scipy import stats

import recnn_b200
from recnn_b200 import _lib
from tests import _policy_sample_oracle as PS
from tests import _policy_topk_oracle as TK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("recnn_discrete_sample_topk", "recnn_discrete_sample_topk_sets", "recnn_vocab_sample_topk_record_floats",
               "recnn_discrete_shard_sample_topk", "recnn_discrete_shard_sample_topk_sets",
               "recnn_discrete_shard_sample_topk_finish")


def test_new_symbols_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES
        assert getattr(L, name) is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))


def test_record_size():
    L = _lib.lib()
    # header, M and S planes, k key / logit / id planes, two seed words
    assert L.recnn_vocab_sample_topk_record_floats(40, 10) == 4 + 32 * 40 + 2
    assert L.recnn_vocab_sample_topk_record_floats(1, 64) == 4 + 194 + 2
    for n, k in [(40, 0), (40, 65), (0, 10)]:
        assert L.recnn_vocab_sample_topk_record_floats(n, k) == 0


def test_python_refusals_happen_before_device_work():
    L = _lib.lib()
    torch.manual_seed(0)
    m = recnn_b200.nn.DiscreteActor(6, 10, 8)
    st = torch.zeros(3, 6)
    k0 = L.recnn_b200_launch_count()
    for k in (0, 11, 65, 2.0, True, None):
        with pytest.raises(ValueError, match="k must be"):
            m.sample_topk(st, k)
    for seed in (1.0, "3", True, -1, 2 ** 64, np.float32(2)):
        with pytest.raises(ValueError, match="seed"):
            m.sample_topk(st, 2, seed=seed)
    with pytest.raises(ValueError, match="state"):
        m.sample_topk(torch.zeros(3, 5), 2)
    for ex in (torch.zeros(3, 2), torch.zeros(2, 2, dtype=torch.int64), torch.zeros(3, 257, dtype=torch.int64),
               torch.zeros(3, dtype=torch.int64), torch.zeros(3, 2, dtype=torch.bool), [[1, 2]] * 3):
        with pytest.raises(ValueError, match="exclude"):
            m.sample_topk(st, 2, exclude=ex)
    with pytest.raises(ValueError, match="exclude_rows"):
        m.sample_topk(st, 2, exclude_rows=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(_lib.RecnnError, match="CUDA only"):
        m.sample_topk(st, 2, exclude=torch.zeros(3, 256, dtype=torch.int64), seed=2 ** 64 - 1)
    assert L.recnn_b200_launch_count() == k0


def test_uniforms_lie_strictly_inside_the_unit_interval_and_bound_the_noise():
    u = PS.uniforms(7, np.arange(64), 4096)
    assert u.min() > 0 and u.max() < 1
    assert (u * 2 ** 24 % 2 == 1).all()                      # (2 m + 1) 2^-24: exact in fp32
    assert np.array_equal(u.astype(np.float32).astype(np.float64), u)
    # the extreme u of the construction: the noise stays below the pruning bound
    assert -np.log(-np.log(1 - 2.0 ** -24)) < PS.G_MAX
    with np.errstate(divide="ignore"):
        g32 = -np.log(-np.log(np.float32(1 - 2.0 ** -24)))
    assert g32 < PS.G_MAX
    # rows and items key distinct noise: no more repeats than 2^23 equally likely values give (birthday: n^2 / 2^24)
    assert u.size - len(np.unique(u)) < 1.2 * u.size ** 2 / 2 ** 24


def _small_policy_logits(seed=3, items=12):
    rng = np.random.default_rng(seed)
    return rng.normal(0, 1.0, items)


def _chi2(counts, probs):
    probs = np.asarray(probs, dtype=np.float64)
    expected = probs / probs.sum() * counts.sum()
    return stats.chisquare(counts, expected).pvalue


def check_distribution(ids, z, exclude=()):
    """ids [R, >= 2] drawn from rows with logits z: the first-position and ordered-pair frequencies against
    Plackett-Luce over the eligible items, by chi-square (fixed seeds: deterministic)."""
    p = np.exp(z - z.max())
    p[list(exclude)] = 0.0
    p /= p.sum()
    I = len(z)
    first = np.bincount(ids[:, 0], minlength=I)
    assert first[list(exclude)].sum() == 0
    elig = p > 0
    assert _chi2(first[elig], p[elig]) > 1e-3, first
    pl = PS.plackett_luce(p, 2)
    pairs = np.bincount(ids[:, 0] * I + ids[:, 1], minlength=I * I)
    cells = sorted(pl)
    assert pairs.sum() == sum(pairs[a * I + b] for a, b in cells)
    assert _chi2(np.array([pairs[a * I + b] for a, b in cells]), [pl[c] for c in cells]) > 1e-3
    for r in range(min(len(ids), 1000)):
        assert len(set(ids[r].tolist())) == ids.shape[1]


@pytest.mark.parametrize("exclude", [(), (2, 7)], ids=["all", "excluded"])
def test_restatement_is_plackett_luce(exclude):
    """12 items, 3 draws, 2^17 rows of one policy's logits: each row's slate is one Plackett-Luce draw."""
    z1 = _small_policy_logits()
    R = 1 << 17
    z = np.tile(z1, (R, 1))
    ex = None if not exclude else np.tile(np.array(exclude), (R, 1))
    _, ids, _ = PS.sample_topk(z, 3, seed=2024, exclude=ex)
    check_distribution(ids, z1, exclude)
    # the third position too: ordered triples against brute force
    p = np.exp(z1 - z1.max())
    p[list(exclude)] = 0.0
    p /= p.sum()
    pl = PS.plackett_luce(p, 3)
    key = ids[:, 0] * 144 + ids[:, 1] * 12 + ids[:, 2]
    counts = np.bincount(key, minlength=12 ** 3)
    cells = sorted(pl, key=lambda c: -pl[c])[:60]           # the likeliest triples, each expected > ~100 times
    rest = R - sum(counts[a * 144 + b * 12 + c] for a, b, c in cells)
    obs = np.array([counts[a * 144 + b * 12 + c] for a, b, c in cells] + [rest])
    exp = np.array([pl[c] for c in cells] + [1 - sum(pl[c] for c in cells)])
    assert _chi2(obs, exp) > 1e-3


def test_restatement_depends_on_the_global_row_and_seed_only():
    rng = np.random.default_rng(5)
    z = rng.normal(0, 2, (30, 500))
    _, a, _ = PS.sample_topk(z, 10, 99)
    _, b, _ = PS.sample_topk(z[10:], 10, 99, row0=10)
    assert np.array_equal(a[10:], b)
    _, c, _ = PS.sample_topk(z, 10, 100)
    assert (c != a).any(1).mean() > 0.9
    # with huge logit gaps the noise cannot reorder: the slate is the top-k
    big = np.argsort(-z, 1)
    zz = np.zeros_like(z)
    np.put_along_axis(zz, big, -100.0 * np.arange(500)[None, :], 1)
    _, d, _ = PS.sample_topk(zz, 10, 1)
    assert np.array_equal(d, TK.topk(zz, 10)[1])


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_restatement_sharded_merge_equals_the_unsharded_slate(world):
    """1,003 and 100 items (13 per rank at W = 8: k = 64 exceeds every block), with exclusions on shard edges."""
    for items in (1003, 100):
        rng = np.random.default_rng(world + items)
        z = rng.normal(0, 2, (25, items))
        edges = sorted({e for lo, hi in TK.item_plan(items, world) for e in (lo - 1, lo, hi - 1) if 0 <= e < items})
        ex = np.full((25, 3), -1)
        ex[:, 0] = edges[-1]
        ex[:, 1] = edges[0]
        for k in (1, 10, 64):
            for e in (None, ex):
                v1, i1, _ = PS.sample_topk(z, k, 31 + k, e)
                vw, iw = PS.shard_sample_topk(z, k, world, 31 + k, e)
                assert np.array_equal(iw, i1)
                np.testing.assert_allclose(vw, v1, rtol=1e-12)
                if e is not None:
                    assert not any(np.isin(i1[r], ex[r][ex[r] >= 0]).any() for r in range(25))
