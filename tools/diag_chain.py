"""Per-tensor errors of the fused chain's forward saves and backward against fp64 (needs a CUDA device)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch
from emernerf_b200 import _ops
from test_gpu_kernels import _chain_reference
DEV = "cuda"

def err(a, b):
    a, b = a.detach().double(), b.detach().double()
    d = (a - b).abs()
    i = int(d.reshape(a.shape[0], -1).amax(1).argmax())
    return f"{float(d.max() / b.abs().max().clamp_min(1e-12)):.2e}@row{i}"

for (k_enc, n_feat, n, S, c) in [(64, 64, 128 * 300, 64, 49), (64, 64, 128 * 20, 64, 49), (40, 64, 128 * 300, 64, 49), (40, 64, 128 * 1200, 64, 49)]:
    gen = torch.Generator().manual_seed(k_enc + n)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=gen) * scale).to(DEV)
    R = (n + S - 1) // S
    enc = rnd(n, k_enc, scale=0.5).requires_grad_(True)
    rb = rnd(R, 128, scale=0.3).requires_grad_(True)
    ws = [rnd(64, k_enc, scale=0.2), rnd(64, scale=0.1), rnd(n_feat, 64, scale=0.15), rnd(n_feat, scale=0.1),
          rnd(64, 64 + c, scale=0.12), rnd(64, 128 + c, scale=0.1), rnd(3, 64, scale=0.2), rnd(3, scale=0.1)]
    ws = [w.requires_grad_(True) for w in ws]
    sigma, rgb, geo, sem = _ops.field_chain(enc, rb, S, ws[:4], ws[4:], want_geo=True)
    want = _chain_reference(enc.detach(), rb.detach(), S, *[w.detach() for w in ws], c)
    saved = sigma.grad_fn.saved_tensors          # enc2, hb, hg, h1, rgb, sigma, ...
    print(f"== k_enc={k_enc} n={n}: fwd sigma {err(sigma, want[0])} rgb {err(rgb, want[1])} geo {err(geo, want[2])} "
          f"hb {err(saved[1], want[4])} h0 {err(saved[2][:, :64], want[5])} h1 {err(saved[3], want[6])}")
    g_s, g_c, g_g = rnd(n), rnd(n, 3), rnd(n, 64, scale=0.1)
    loss = (sigma * g_s).sum() + (rgb * g_c).sum() + (geo * g_g).sum()
    got = torch.autograd.grad(loss, [enc, rb] + ws)
    enc64, rb64 = enc.detach().double().requires_grad_(True), rb.detach().double().requires_grad_(True)
    ws64 = [w.detach().double().requires_grad_(True) for w in ws]
    r = _chain_reference(enc64, rb64, S, *ws64, c)
    loss64 = (r[0] * g_s).sum() + (r[1] * g_c).sum() + (r[2] * g_g).sum()
    want_g = torch.autograd.grad(loss64, [enc64, rb64] + ws64)
    print("   bwd " + "  ".join(f"{nm} {err(a, b)}" for nm, a, b in
                                zip(["enc", "rb", "wb0", "bb0", "wb1", "bb1", "w0", "w1", "w2", "b2"], got, want_g)))
