"""wgmma 3xTF32 GEMM (recnn_gemm_tf32x3) against float64 numpy and against the exact-fp32
CUDA-core GEMM (recnn_gemm_fp32), all four operand-major combinations, ragged shapes."""
import numpy as np
import pytest
import torch

from recnn_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pad4(n):
    return (n + 3) // 4 * 4


def _make(rows, cols, rng, scale=1.0):
    """fp32 [rows, cols] stored with a row pitch that is a multiple of 4 floats (TMA)."""
    ld = _pad4(cols)
    host = (rng.standard_normal((rows, cols)) * scale).astype(np.float32)
    dev = torch.zeros(rows, ld, device=DEV)
    dev[:, :cols] = torch.from_numpy(host).to(DEV)
    return host, dev, ld


def _run(kind, M, N, K, a_mn, b_mn, seed=0, tile_n=0, scale_b=1.0):
    rng = np.random.default_rng(seed)
    a_h, a_d, lda = _make(K, M, rng) if a_mn else _make(M, K, rng)
    b_h, b_d, ldb = _make(K, N, rng, scale_b) if b_mn else _make(N, K, rng, scale_b)
    ldc = _pad4(N)
    c_d = torch.full((M, ldc), float("nan"), device=DEV)
    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    if kind == "tc":
        _lib.check(L.recnn_gemm_tf32x3(M, N, K, a_d.data_ptr(), lda, int(a_mn), b_d.data_ptr(), ldb, int(b_mn),
                                       c_d.data_ptr(), ldc, tile_n, st))
    else:
        _lib.check(L.recnn_gemm_fp32(M, N, K, a_d.data_ptr(), lda, int(a_mn), b_d.data_ptr(), ldb, int(b_mn),
                                     c_d.data_ptr(), ldc, st))
    torch.cuda.synchronize()
    A = (a_h.T if a_mn else a_h).astype(np.float64)
    B = (b_h.T if b_mn else b_h).astype(np.float64)
    want = A @ B.T
    got = c_d[:, :N].cpu().numpy().astype(np.float64)
    return got, want


SHAPES = [
    (128, 256, 16), (128, 256, 64), (128, 64, 48), (128, 128, 200),
    (300, 256, 1290),          # ragged M, K with a zero-filled tail block
    (4096, 256, 1290), (4096, 256, 256), (4096, 128, 256), (1000, 100, 77),
]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
def test_tf32x3_matches_float64(M, N, K, a_mn, b_mn):
    got, want = _run("tc", M, N, K, a_mn, b_mn, seed=M + N + K)
    assert np.isfinite(got).all()
    # Error model of the split: hi is the truncated operand, lo = rna(x - hi); the dropped lo*lo
    # term is <= 2^-20 (1e-6) of each product, so the max over ~1e5-1e6 outputs of a length-K sum of
    # unit-variance products sits at a few 1e-6 * sqrt(K) -- about 5x plain fp32 accumulation and
    # ~250x better than one TF32 pass (1e-3).
    err = np.abs(got - want).max() / np.sqrt(K)
    print("max abs err / sqrt(K) = %.3g" % err)
    assert err < 8e-6, "max abs err / sqrt(K) = %.3g" % err
    rel = np.abs(got - want).max() / np.abs(want).max()
    assert rel < 8e-6, rel


@pytest.mark.parametrize("M,N,K", [(300, 256, 1290), (257, 130, 333)])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
def test_fp32_simt_matches_float64(M, N, K, a_mn, b_mn):
    got, want = _run("simt", M, N, K, a_mn, b_mn, seed=1)
    assert np.abs(got - want).max() / np.abs(want).max() < 3e-6


def test_tf32_operand_truncation_semantics():
    """The split assumes kind::tf32 reads a raw fp32 word by ignoring its low 13 mantissa bits.
    If the hardware rounded instead, hi (as read) + lo (as computed) != x for about half of all
    inputs and the error would be ~2^-11 (5e-4) relative, not ~1e-7."""
    got, want = _run("tc", 256, 256, 512, False, False, seed=7)
    err = np.abs(got - want).max() / np.sqrt(512)
    assert err < 8e-6, err


def test_accumulation_is_not_truncated_over_long_k():
    """The tensor core's fp32 accumulate rounds toward zero; unchunked, all-positive operands would
    lose ~2.2e-8 * K of the sum (-9e-5 at K=4096).  With 64-wide chunks drained into round-to-nearest
    register sums the bias stays ~1e-6 whatever K is."""
    rng = np.random.default_rng(11)
    M = N = 256
    for K in (64, 4096):
        a = rng.uniform(0.5, 1.0, (M, K)).astype(np.float32)
        b = rng.uniform(0.5, 1.0, (N, K)).astype(np.float32)
        a_d, b_d = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
        c_d = torch.empty(M, N, device=DEV)
        _lib.check(_lib.lib().recnn_gemm_tf32x3(M, N, K, a_d.data_ptr(), K, 0, b_d.data_ptr(), K, 0, c_d.data_ptr(), N,
                                               0, torch.cuda.current_stream().cuda_stream))
        want = a.astype(np.float64) @ b.astype(np.float64).T
        rel = (c_d.cpu().numpy() - want) / want
        assert abs(rel.mean()) < 5e-7 and np.abs(rel).max() < 2e-6, (K, rel.mean(), np.abs(rel).max())


@pytest.mark.parametrize("tile_n", [64, 128])
def test_tile_widths_agree(tile_n):
    got, want = _run("tc", 512, 256, 320, False, False, seed=3, tile_n=tile_n)
    assert np.abs(got - want).max() / np.abs(want).max() < 8e-6


def test_wide_dynamic_range():
    """gradient-like operand (1e-6 scale) times activation-like operand: relative accuracy holds."""
    got, want = _run("tc", 256, 256, 4096, True, True, seed=5, scale_b=1e-6)
    assert np.abs(got - want).max() / np.abs(want).max() < 8e-6


# ----------------------------------------------------------------------------- tile widths / worker counts agree bit for bit
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(128, 64, 16), (128, 256, 64), (128, 256, 96), (300, 256, 1290), (4096, 256, 1290),
                                   (4096, 128, 256), (1000, 100, 77), (256, 1290, 4096)])
def test_tile_shapes_are_bit_identical(M, N, K, a_mn, b_mn):
    """64-wide tiles run four split groups (16 worker warps, 16 accumulator columns per thread), 128-wide tiles two
    (8 warps, 64 columns): same MMA sequence and the same order of chunk additions per element, so the two kernels
    must agree bit for bit (K = 16 / 64 / 96 leave some groups without a k-block), and both meet the accuracy bar."""
    got64, ref = _run("tc", M, N, K, a_mn, b_mn, seed=3, tile_n=64)
    got128, _ = _run("tc", M, N, K, a_mn, b_mn, seed=3, tile_n=128)
    assert np.array_equal(got64, got128)
    assert np.abs(got64 - ref).max() / np.abs(ref).max() < 2e-6
