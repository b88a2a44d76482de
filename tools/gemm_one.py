"""Run the GEMM kernel a few times on one shape (a short target for a profiler)."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neuronx_distributed_b200 import ops
M, N, K = (int(x) for x in (sys.argv[1:4] if len(sys.argv) > 3 else (4096, 12288, 4096)))
a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16); b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
e = ops._ext.ext()
for _ in range(3):
    e.gemm_bf16(a, b, out, False, True, False)
torch.cuda.synchronize()
print("done")
