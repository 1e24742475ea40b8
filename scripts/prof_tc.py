"""One wgmma 3xTF32 GEMM at the layer-1 shape, a few launches (for ncu)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from recnn_b200 import _lib
L = _lib.lib(); DEV = "cuda:0"
M, N, K = 4096, 256, 1290
tile = int(sys.argv[1]) if len(sys.argv) > 1 else 128
ld = (K + 3) // 4 * 4
A = torch.randn(M, ld, device=DEV); B = torch.randn(N, ld, device=DEV); C = torch.empty(M, N, device=DEV)
st = torch.cuda.current_stream().cuda_stream
for _ in range(4):
    _lib.check(L.recnn_gemm_tf32x3(M, N, K, A.data_ptr(), ld, 0, B.data_ptr(), ld, 0, C.data_ptr(), N, tile, st))
torch.cuda.synchronize()
print("done")
