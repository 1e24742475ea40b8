"""Host restatement of the device RNG of perf mode (recnn_b200/csrc/common.cuh: Philox, philox_keep_bits32; the
EPI_LINEAR noise draw of tc_gemm.cuh / gemm_simt.cuh), vectorised in numpy with uint64 arithmetic.

A step without ``batch["dropout_masks"]`` draws its dropout keep bits and TD3's target-policy noise on the device,
keyed on the engine's seed (``torch.initial_seed()`` when the engine is created) and on ``rng_step`` (0 for the first
step, +1 per step).  These functions give the same bits on the host, so a perf-mode step can be replayed through the
oracle."""
from __future__ import annotations

import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)

# mask slot k of a step is Philox stream k (include/recnn_b200.h: masks in the reference's call order)
DDPG_STREAMS = {"value": (0, 1), "policy": (2, 3), "policy_value": (4, 5)}
TD3_STREAMS = {"value1": (0, 1), "value2": (2, 3), "policy": (4, 5), "policy_value1": (6, 7)}
NOISE_STREAM = 15


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) on arrays: ctr = 4 words, key = 2 words (each an int or a uint32 array;
    they broadcast).  Returns the 4 output words as uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _LO for c in ctr)
    k0, k1 = (np.asarray(k, dtype=np.uint64) & _LO for k in key)
    for _ in range(10):
        p0 = _M0 * c0                       # < 2^64: exact in uint64
        p1 = _M1 * c2
        hi0, lo0 = p0 >> _S32, p0 & _LO
        hi1, lo1 = p1 >> _S32, p1 & _LO
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + _W0) & _LO
        k1 = (k1 + _W1) & _LO
    return tuple(np.asarray(c, dtype=np.uint32) for c in (c0, c1, c2, c3))


def _philox_seeded(seed, ctr_lo, ctr_hi):
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    ctr_lo = np.asarray(ctr_lo, dtype=np.uint64)
    ctr_hi = np.uint64(int(ctr_hi) & 0xFFFFFFFFFFFFFFFF)
    return philox4x32_10((ctr_lo & _LO, ctr_lo >> _S32, ctr_hi & _LO, ctr_hi >> _S32),
                         (seed & 0xFFFFFFFF, seed >> 32))


def keep_mask(seed, step, stream_id, n_rows, H):
    """uint8 [n_rows, H] dropout keep mask of stream ``stream_id`` at rng step ``step``: element (m, n) has
    idx = m*H + n and keeps iff bit idx & 31 of word idx >> 5 is set; word w is output word w & 3 of the Philox
    call with counter (w >> 2, (step << 8) | stream_id)."""
    n_words = (n_rows * H + 31) // 32
    calls = np.arange((n_words + 3) // 4, dtype=np.uint64)
    r = _philox_seeded(seed, calls, (int(step) << 8) | int(stream_id))
    words = np.stack(r, axis=1).reshape(-1)[:n_words]
    idx = np.arange(n_rows * H, dtype=np.uint64)
    bits = (words[(idx >> np.uint64(5)).astype(np.int64)].astype(np.uint64) >> (idx & np.uint64(31))) & np.uint64(1)
    return bits.astype(np.uint8).reshape(n_rows, H)


def step_masks(seed, step, n_rows, H, algo):
    """The 6 (DDPG) / 8 (TD3) masks a perf-mode step draws, in mask-slot order."""
    return [keep_mask(seed, step, k, n_rows, H) for k in range(6 if algo == "ddpg" else 8)]


def td3_noise(seed, step, n_rows, A, std):
    """float64 [n_rows, A]: TD3's target-policy noise before clipping, as the EPI_LINEAR epilogue draws it on stream
    15.  Element (m, n) uses the Philox call with counter (m*A + n, (step << 8) | 15); u1 = (float(r.x) + 1) * 2^-32 and
    u2 = float(r.y) * 2^-32 are formed in fp32 as on the device, z = sqrt(-2 ln u1) cos(2 pi u2) * std in float64."""
    idx = np.arange(n_rows * A, dtype=np.uint64)
    rx, ry, _, _ = _philox_seeded(seed, idx, (int(step) << 8) | NOISE_STREAM)
    two_m32 = np.float32(2.3283064365386963e-10)
    u1 = (rx.astype(np.float32) + np.float32(1.0)) * two_m32
    u2 = ry.astype(np.float32) * two_m32
    z = np.sqrt(-2.0 * np.log(u1.astype(np.float64))) * np.cos(6.283185307179586 * u2.astype(np.float64)) * float(std)
    return z.reshape(n_rows, A)
