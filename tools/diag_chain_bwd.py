"""Step through _FieldChain.backward's kernel sequence, comparing every intermediate with fp64 (needs a CUDA device)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch
from emernerf_b200 import _ops
from emernerf_b200._ops import _layer_bwd_data, _layer_bwd_weight
DEV = "cuda"

def err(a, b):
    a, b = a.detach().double(), b.detach().double()
    d = (a - b).abs().reshape(a.shape[0], -1).amax(1)
    bad = int((d > 1e-4 * b.abs().max()).sum())
    return f"{float(d.max() / b.abs().max().clamp_min(1e-12)):.2e} (rows off: {bad}, first {d.argmax().item()})"

for rep in range(2):
  for n in (128 * 300, 128 * 1200):
    gen = torch.Generator().manual_seed(n + rep)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=gen) * scale).to(DEV)
    f32 = dict(dtype=torch.float32, device=DEV)
    h1 = torch.relu(rnd(n, 64)); hg = torch.cat([torch.relu(rnd(n, 64)), rnd(n, 64)], 1).contiguous(); hb = torch.relu(rnd(n, 64))
    enc = rnd(n, 40, scale=0.5)
    w2, w1hg, w0g, wb1, wb0 = rnd(3, 64, scale=0.2), rnd(64, 128, scale=0.1), rnd(64, 64, scale=0.12), rnd(64, 64, scale=0.15), rnd(64, 40, scale=0.2)
    dz2 = rnd(n, 3)
    d = lambda t: t.double()
    # 1. narrow wgrad + bwd data
    dw2, db2 = _layer_bwd_weight(h1, 64, dz2, 3, w2, True, n)
    dz1 = torch.empty((n, 64), **f32)
    _layer_bwd_data(dz2, 3, w2, dz1, 64, n, h1, 64, 64)
    dz1_w = (d(dz2) @ d(w2)) * (h1 > 0)
    print(f"n={n} rep={rep}\n  dz1 (narrow bwd)        {err(dz1, dz1_w)}   dw2 {err(dw2, d(dz2).T @ d(h1))}")
    # 2. wgrad 128
    dw1hg, _ = _layer_bwd_weight(hg, 128, dz1, 64, w1hg, False, n)
    print(f"  dw1hg (tc wgrad k128)   {err(dw1hg, d(dz1).T @ d(hg))}")
    # 3. bwd data 64 -> 128 with relu on first 64
    D1 = torch.empty((n, 128), **f32)
    _layer_bwd_data(dz1, 64, w1hg, D1, 128, n, hg, 128, 64)
    D1_w = d(dz1) @ d(w1hg)
    D1_w[:, :64] *= (hg[:, :64] > 0)
    print(f"  D1 (tc bwd 64->128)     {err(D1, D1_w)}")
    dz0 = D1[:, :64]
    dw0g, _ = _layer_bwd_weight(hg[:, 64:], 128, dz0, 128, w0g, False, n)
    print(f"  dw0g (tc wgrad strided) {err(dw0g, d(dz0).T @ d(hg[:, 64:]))}")
    before = D1.clone()
    _layer_bwd_data(dz0, 128, w0g, D1[:, 64:], 128, n, None, 0, 0, accumulate=True)
    acc_w = d(before)
    acc_w[:, 64:] += d(before[:, :64]) @ d(w0g)
    print(f"  D1 after accumulate     {err(D1, acc_w)}")
    dfe = D1[:, 64:]
    dwb1, dbb1 = _layer_bwd_weight(hb, 64, dfe, 128, wb1, True, n)
    print(f"  dwb1 (tc wgrad, dz ld128) {err(dwb1, d(dfe).T @ d(hb))}  dbb1 {err(dbb1[:, None], d(dfe).sum(0)[:, None])}")
    dzb = torch.empty((n, 64), **f32)
    _layer_bwd_data(dfe, 128, wb1, dzb, 64, n, hb, 64, 64)
    print(f"  dzb (tc bwd 64->64, relu) {err(dzb, (d(dfe) @ d(wb1)) * (hb > 0))}")
    dwb0, _ = _layer_bwd_weight(enc, 40, dzb, 64, wb0, True, n)
    print(f"  dwb0 (tc wgrad k40)     {err(dwb0, d(dzb).T @ d(enc))}")
    d_enc = torch.empty((n, 40), **f32)
    _layer_bwd_data(dzb, 64, wb0, d_enc, 40, n, None, 0, 0)
    print(f"  d_enc (tc bwd 64->40)   {err(d_enc, d(dzb) @ d(wb0))}")
