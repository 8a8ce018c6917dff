"""One launch of rl_gemm_bf16_tn per shape (for a profiler capture): the actor's and the learner's fc forward shapes.
    python tools/gemm_once.py"""
import sys

import torch

sys.path.insert(0, __file__.rsplit('/', 2)[0])
from parl_b200 import kernels as K  # noqa: E402

dev = torch.device('cuda', 0)
bf = torch.bfloat16
torch.manual_seed(0)
for M, N, Kd in [(4096, 512, 5184), (204800, 512, 5184)]:
    a = (torch.randn(M, Kd, device=dev) * 0.1).to(bf)
    b = (torch.randn(N, Kd, device=dev) * 0.1).to(bf)
    bias = torch.randn(N, device=dev)
    o = torch.empty(M, N, device=dev, dtype=bf)
    K.gemm_bf16_tn(a, b, bias, relu=True, out=o)
    torch.cuda.synchronize()
print('done')
