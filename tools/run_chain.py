"""Launch the fused field chain (forward + backward) at the benchmark's shapes, for profiler captures and CUDA-event timing.

    python tools/run_chain.py [n_points] [reps]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from emernerf_b200 import _ops

n = int(sys.argv[1]) if len(sys.argv) > 1 else 524288
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
S, c = 64, 49
g = torch.Generator().manual_seed(0)
rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
enc = rnd(n, 40, scale=0.5).requires_grad_(True)
rb = rnd(n // S, 128, scale=0.3).requires_grad_(True)
ws = [rnd(64, 40, scale=0.2), rnd(64, scale=0.1), rnd(64, 64, scale=0.15), rnd(64, scale=0.1), rnd(64, 64 + c, scale=0.12),
      rnd(64, 128 + c, scale=0.1), rnd(3, 64, scale=0.2), rnd(3, scale=0.1)]
ws = [w.requires_grad_(True) for w in ws]
g_s, g_c = rnd(n), rnd(n, 3)
ev = lambda: torch.cuda.Event(enable_timing=True)
for it in range(reps):
    e = [ev() for _ in range(3)]
    e[0].record()
    sigma, rgb, _, _ = _ops.field_chain(enc, rb, S, ws[:4], ws[4:])
    e[1].record()
    torch.autograd.grad((sigma * g_s).sum() + (rgb * g_c).sum(), [enc, rb] + ws)
    e[2].record()
    torch.cuda.synchronize()
    print(f"rep {it}: forward {e[0].elapsed_time(e[1]):.3f} ms   backward (data + weight gradients + torch glue) {e[1].elapsed_time(e[2]):.3f} ms")
with torch.no_grad():
    for it in range(3):
        e = [ev() for _ in range(2)]
        e[0].record()
        _ops.field_chain(enc, rb, S, ws[:4], ws[4:])
        e[1].record()
        torch.cuda.synchronize()
        print(f"inference rep {it}: forward without saves {e[0].elapsed_time(e[1]):.3f} ms")
