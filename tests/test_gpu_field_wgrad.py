"""emer_field_wgrad (csrc/field_wgrad.cu): the fused field chain's five weight gradients in one launch, against fp64
dZ^T X and column sums, with the bars of test_gpu_kernels.py::test_tc_weight_gradient_row_major_operands."""
import pytest
import torch

from helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
RAY_COLS = 49           # [dir | emb] columns of the colour head's first two layers, in front of their geo blocks

CASES = [(k, f, sem, head, 64 * 1500 + 21, ld)
         for k, ld in ((32, 32), (40, 48), (64, 64))
         for f, sem in ((64, False), (128, True), (128, False))
         for head in (True, False)]
CASES += [(40, 64, False, True, 524288, 40), (64, 128, True, True, 524288, 64), (32, 128, True, False, 524288, 32)]


@pytest.mark.parametrize("k_enc,n_feat,sem,head,n,ld_enc", CASES)
def test_field_weight_gradients(k_enc, n_feat, sem, head, n, ld_enc):
    """Every output accumulates into a non-zero buffer; the head's blocks land in strided column blocks of [64, 113] /
    [64, 177] buffers whose other columns stay as they were; without dz2 the head's outputs are not touched, without
    d_sem neither are dWb1's rows 64.. nor dbb1[64:]; ragged last tile, enc rows with a stride wider than k_enc."""
    from emernerf_b200 import _lib, _ops

    g = torch.Generator(device=DEV).manual_seed(n + 7 * k_enc + n_feat + 3 * sem + head)
    r = lambda *s: torch.randn(*s, device=DEV, generator=g)
    enc = r(n, ld_enc)[:, :k_enc]
    hb, hg, h1, dz1, d1, dzb = r(n, 64), r(n, 128), r(n, 64), r(n, 64), r(n, 128), r(n, 64)
    dz2 = r(n, 3) if head else None
    d_sem = r(n, 64) if sem else None
    dwb0, dbb0, dwb1, dbb1 = r(64, k_enc), r(64), r(n_feat, 64), r(n_feat)
    w0, w1, dw2, db2 = r(64, RAY_COLS + 64), r(64, 128 + RAY_COLS), r(3, 64), r(3)
    before = {k: v.clone() for k, v in dict(dwb0=dwb0, dbb0=dbb0, dwb1=dwb1, dbb1=dbb1, w0=w0, w1=w1, dw2=dw2, db2=db2).items()}
    _ops._need_cuda(enc)
    P = _ops._ptr
    _lib.call("emer_field_wgrad", P(enc), ld_enc, k_enc, P(hb), P(hg), P(h1), P(dz2), P(dz1), P(d1), P(dzb), P(d_sem),
              n_feat, P(dwb0), P(dbb0), P(dwb1), P(dbb1), P(w0[:, RAY_COLS:]), w0.stride(0), P(w1),
              P(w1[:, 64 + RAY_COLS:]), w1.stride(0), P(dw2), P(db2), n, _ops._stream())
    torch.cuda.synchronize()

    d = lambda t: t.double()
    b = {k: d(v) for k, v in before.items()}
    dF, geo = d(d1[:, 64:]), d(hg[:, 64:])
    checks = [(dwb0, b["dwb0"] + d(dzb).T @ d(enc)), (dbb0, b["dbb0"] + d(dzb).sum(0)),
              (dwb1[:64], b["dwb1"][:64] + dF.T @ d(hb)), (dbb1[:64], b["dbb1"][:64] + dF.sum(0))]
    if sem:
        checks += [(dwb1[64:], b["dwb1"][64:] + d(d_sem).T @ d(hb)), (dbb1[64:], b["dbb1"][64:] + d(d_sem).sum(0))]
    elif n_feat == 128:
        assert torch.equal(dwb1[64:], before["dwb1"][64:]) and torch.equal(dbb1[64:], before["dbb1"][64:])
    if head:
        checks += [(w0[:, RAY_COLS:], b["w0"][:, RAY_COLS:] + d(d1[:, :64]).T @ geo),
                   (w1[:, :64], b["w1"][:, :64] + d(dz1).T @ d(hg[:, :64])),
                   (w1[:, 64 + RAY_COLS:], b["w1"][:, 64 + RAY_COLS:] + d(dz1).T @ geo),
                   (dw2, b["dw2"] + d(dz2).T @ d(h1)), (db2, b["db2"] + d(dz2).sum(0))]
        assert torch.equal(w0[:, :RAY_COLS], before["w0"][:, :RAY_COLS])
        assert torch.equal(w1[:, 64:64 + RAY_COLS], before["w1"][:, 64:64 + RAY_COLS])
    else:
        for k, v in dict(w0=w0, w1=w1, dw2=dw2, db2=db2).items():
            assert torch.equal(v, before[k]), k
    tol = 2e-5 if n < 200000 else 5e-5               # fp32 accumulation over thousands of row tiles + one partial sum per CTA
    for i, (got, want) in enumerate(checks):
        assert rel_err(got, want) < tol, (i, rel_err(got, want))
