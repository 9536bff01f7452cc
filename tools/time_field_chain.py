"""Time the fused field chain's three kernels one by one at the benchmark's shape, with CUDA events.

    python tools/time_field_chain.py [--n 524288] [--reps 30] [--warmup 5] [--dump DIR]

emer_field_fwd (with the training saves), emer_field_bwd and emer_field_wgrad are launched on seeded inputs with
k_enc = 40, n_feat = 64 and the colour head, 64 samples per ray: the static benchmark's chain.  Each kernel is
timed alone over --reps launches after --warmup; the median, and the bytes each launch must move (from the shapes),
are printed.  --dump DIR writes the forward's outputs (sigma, rgb and the saves hb, hg, h1) as DIR/<name>.npy, so the
forward of two builds can be compared bit for bit.
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from emernerf_b200 import _lib, _ops

K_ENC, N_FEAT, S, RAY_COLS = 40, 64, 64, 49


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=524288)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--dump", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_field_chain: no CUDA device")
    n, R = args.n, (args.n + S - 1) // S
    g = torch.Generator().manual_seed(args.seed)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
    enc = rnd(n, K_ENC, scale=0.5)
    rb = rnd(R, 128, scale=0.3)
    wb0, bb0, wb1, bb1 = rnd(64, K_ENC, scale=0.2), rnd(64, scale=0.1), rnd(N_FEAT, 64, scale=0.15), rnd(N_FEAT, scale=0.1)
    w0, w1, w2, b2 = rnd(64, RAY_COLS + 64, scale=0.12), rnd(64, 128 + RAY_COLS, scale=0.1), rnd(3, 64, scale=0.2), rnd(3, scale=0.1)
    d_rgb, d_sigma = rnd(n, 3), rnd(n)
    f32 = dict(dtype=torch.float32, device="cuda")
    sigma, rgb = torch.empty(n, **f32), torch.empty((n, 3), **f32)
    hb, hg, h1 = torch.empty((n, 64), **f32), torch.empty((n, 128), **f32), torch.empty((n, 64), **f32)
    dz2, dz1, d1, dzb = torch.empty((n, 3), **f32), torch.empty((n, 64), **f32), torch.empty((n, 128), **f32), torch.empty((n, 64), **f32)
    d_enc, d_rb = torch.empty((n, K_ENC), **f32), torch.zeros((R, 128), **f32)
    w1hg = torch.cat([w1[:, :64], w1[:, 64 + RAY_COLS:]], dim=1)
    w0g = w0[:, RAY_COLS:].contiguous()
    dwb0, dbb0, dwb1, dbb1 = (torch.zeros_like(t) for t in (wb0, bb0, wb1, bb1))
    dw0, dw1, dw2, db2 = (torch.zeros_like(t) for t in (w0, w1, w2, b2))
    P, st = _ops._ptr, _ops._stream()
    _ops._need_cuda(enc)

    def fwd():
        _lib.call("emer_field_fwd", P(enc), K_ENC, K_ENC, P(wb0), P(bb0), P(wb1), P(bb1), N_FEAT, P(w0[:, RAY_COLS:]),
                  w0.stride(0), P(w1[:, :64]), P(w1[:, 64 + RAY_COLS:]), w1.stride(0), P(w2), P(b2), P(rb), S, P(sigma),
                  P(rgb), P(hb), P(hg), P(h1), None, n, st)

    def bwd():
        _lib.call("emer_field_bwd", P(d_rgb), P(rgb), P(d_sigma), P(sigma), None, None, P(hb), P(hg), P(h1), P(wb0),
                  K_ENC, P(wb1), N_FEAT, P(w0g), 64, P(w1hg), P(w1hg[:, 64:]), 128, P(w2), P(dz2), P(dz1), P(d1),
                  P(dzb), P(d_enc), K_ENC, P(d_rb), S, n, st)

    def wgrad():
        _lib.call("emer_field_wgrad", P(enc), K_ENC, K_ENC, P(hb), P(hg), P(h1), P(dz2), P(dz1), P(d1), P(dzb), None,
                  N_FEAT, P(dwb0), P(dbb0), P(dwb1), P(dbb1), P(dw0[:, RAY_COLS:]), dw0.stride(0), P(dw1),
                  P(dw1[:, 64 + RAY_COLS:]), dw1.stride(0), P(dw2), P(db2), n, st)

    # bytes each launch must move (fp32 rows; per-ray and weight traffic is under 1 %)
    row_bytes = {
        "field_fwd_kernel": 4 * (K_ENC + 1 + 3 + 64 + 128 + 64),
        "field_bwd_kernel": 4 * (3 + 3 + 1 + 1 + 64 + 128 + 64) + 4 * (3 + 64 + 128 + 64 + K_ENC),
        "field_wgrad_kernel": 4 * (K_ENC + 64 + 128 + 64 + 3 + 64 + 128 + 64),
    }
    fwd()
    bwd()
    torch.cuda.synchronize()
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        for name, t in dict(sigma=sigma, rgb=rgb, hb=hb, hg=hg, h1=h1).items():
            np.save(os.path.join(args.dump, f"{name}.npy"), t.cpu().numpy())
    print(f"N = {n}, k_enc = {K_ENC}, n_feat = {N_FEAT}, colour head, {S} samples per ray; "
          f"{torch.cuda.get_device_name()}; median of {args.reps} launches")
    for name, fn in (("field_fwd_kernel", fwd), ("field_bwd_kernel", bwd), ("field_wgrad_kernel", wgrad)):
        for _ in range(args.warmup):
            fn()
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = statistics.median(times)
        b = row_bytes[name] * n
        print(f"{name:20s} {ms:7.3f} ms  (min {min(times):.3f}, max {max(times):.3f})  {b / 1e9:6.3f} GB  "
              f"{b / ms / 1e6:7.0f} GB/s")


if __name__ == "__main__":
    main()
