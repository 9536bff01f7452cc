"""Time the wgmma weight-gradient entry point at the benchmark's shapes (CUDA events, 5 repetitions)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from emernerf_b200 import _lib, _ops

n = int(sys.argv[1]) if len(sys.argv) > 1 else 524288
name = "emer_linear_tc_bwd_weight"
for k, ldx in ((64, 64), (64, 128), (128, 128), (40, 40)):
    x = torch.randn(n, ldx, device="cuda")
    dz = torch.randn(n, 64, device="cuda")
    _ops._need_cuda(x)
    dw, db = torch.zeros(64, k, device="cuda"), torch.zeros(64, device="cuda")
    ts = []
    for it in range(6):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.call(name, _ops._ptr(x), ldx, _ops._ptr(dz), 64, _ops._ptr(dw), _ops._ptr(db), n, k, 64, _ops._stream())
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = min(ts[1:])
    print(f"k={k:3d} ldx={ldx:3d} {name:30s} {ms * 1e3:7.1f} us  {n * (k + 64) * 4 / ms / 1e6:7.1f} GB/s of algorithmic bytes")
