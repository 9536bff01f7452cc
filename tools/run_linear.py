"""Launch the dense-layer kernels once at bench shapes (for profiler captures)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from emernerf_b200 import _ops

n = 524288
for k, o, act in ((64, 64, 1), (177, 64, 1)):
    x = torch.randn(n, k, device="cuda", requires_grad=True)
    w = (torch.randn(o, k, device="cuda") / k ** 0.5).requires_grad_(True)
    b = torch.zeros(o, device="cuda", requires_grad=True)
    for _ in range(3):
        y = _ops.linear(x, w, b, act)
        y.backward(torch.ones_like(y))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); y = _ops.linear(x, w, b, act); e1.record(); torch.cuda.synchronize()
    print(k, o, "fwd ms", e0.elapsed_time(e1))

