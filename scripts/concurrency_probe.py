"""How much do the 3xTF32 GEMMs slow each other down when they run side by side?  (diagnostic for the intra-step stream overlap)

K concurrent layer-1 GEMMs [4096x1292]x[1292x256] on K streams inside one CUDA graph, per configuration:
    tile 128 (64 CTAs each) / tile 64 (128 CTAs each);  distinct A operands / the SAME A operand;
    A fresh from HBM (L2 flushed) / A L2-resident (written just before).
Prints the device time of the group."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from recnn_b200 import _lib  # noqa: E402

dev = torch.device("cuda:0")
L = _lib.lib()
M, N, K, LD = 4096, 256, 1290, 1292
A = [torch.randn(M, LD, device=dev) for _ in range(4)]
W = [torch.randn(N, LD, device=dev) for _ in range(4)]
C = [torch.empty(M, N, device=dev) for _ in range(4)]
flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
streams = [torch.cuda.Stream(dev) for _ in range(4)]


def gemm(i, ai, tile, stream):
    _lib.check(L.recnn_gemm_tf32x3(M, N, K, A[ai].data_ptr(), LD, 0, W[i].data_ptr(), LD, 0, C[i].data_ptr(), N, tile,
                                   stream.cuda_stream))


def build(k, tile, same_a, chain=1):
    def body():
        cur = torch.cuda.current_stream(dev)
        for i in range(k):
            streams[i].wait_stream(cur)
            for _ in range(chain):
                gemm(i, 0 if same_a else i, tile, streams[i])
        for i in range(k):
            cur.wait_stream(streams[i])
    body()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    return g


def timed(g, warm_l2, reps=15):
    ts = []
    for _ in range(reps):
        flush.zero_()
        if warm_l2:
            for a in A[:warm_l2]:
                a.add_(0.0)          # rewrite the operands that will be read: they sit in L2 as after the gather
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


for tile in (128, 64):
    for k in (1, 2, 3):
        for same in (False, True):
            if k == 1 and same:
                continue
            g1 = build(k, tile, same, chain=1)
            g4 = build(k, tile, same, chain=4)
            row = []
            for warm in (0, 1 if same else k):
                t1, t4 = timed(g1, warm), timed(g4, warm)
                row.append("%s: 1 GEMM/stream %.1f us, 4 chained %.1f us (%.1f per GEMM)" % ("L2-warm A" if warm else "cold A", t1, t4, t4 / 4))
            print("tile %3d  %d concurrent  %s | %s" % (tile, k, "same A    " if same else "distinct A", " | ".join(row)))


# one GEMM over all rows vs two concurrent GEMMs over half the rows each (same CTAs, same unique bytes)
def build_split(parts, tile):
    rows = M // parts

    def body():
        cur = torch.cuda.current_stream(dev)
        for i in range(parts):
            streams[i].wait_stream(cur)
            for _ in range(4):
                _lib.check(L.recnn_gemm_tf32x3(rows, N, K, A[0][i * rows:].data_ptr(), LD, 0, W[i].data_ptr(), LD, 0,
                                               C[0][i * rows:].data_ptr(), N, tile, streams[i].cuda_stream))
        for i in range(parts):
            cur.wait_stream(streams[i])
    body()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    return g


for parts in (1, 2, 4):
    g = build_split(parts, 128)
    print("tile 128: M=4096 as %d concurrent GEMM(s) of %d rows, 4 chained: cold %.1f us, L2-warm %.1f us per chain step"
          % (parts, M // parts, timed(g, 0) / 4, timed(g, 1) / 4))
