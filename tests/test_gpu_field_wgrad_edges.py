"""emer_field_wgrad (csrc/field_wgrad.cu) at the row counts where its producer / consumer pipeline has the fewest tiles
per CTA: one tile, fewer tiles than ring stages, exactly as many, one more, and a grid of every SM with three or four
tiles each.  All six kernel instantiations, with and without d_sem.  The row buffers are views of taller buffers whose
rows past N (and enc's columns past k_enc) are NaN, so a read past the last row shows up; every output accumulates
into a non-zero buffer.  Bars of test_gpu_field_wgrad.py, against fp64."""
import pytest
import torch

from helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
RAY_COLS = 49
TR, STAGES = 16, 3            # rows per tile, ring depth (field_wgrad.cu)
PAD = 40                      # NaN rows behind every row buffer

NS = [1, 15, 16, 17, 47, 48, 49, "sms*48-1", "sms*48+1"]


def _rows(spec):
    if isinstance(spec, int):
        return spec
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sms * TR * STAGES + (1 if spec.endswith("+1") else -1)


@pytest.mark.parametrize("sem", [False, True])
@pytest.mark.parametrize("head", [True, False])
@pytest.mark.parametrize("k_enc,ld_enc", [(32, 36), (40, 48), (64, 64)])
@pytest.mark.parametrize("n_spec", NS)
def test_field_wgrad_few_tiles(n_spec, k_enc, ld_enc, head, sem):
    from emernerf_b200 import _lib, _ops

    n = _rows(n_spec)
    n_feat = 128 if sem else 64
    g = torch.Generator(device=DEV).manual_seed(n + 7 * k_enc + 3 * sem + head)

    def rows(w, ld=None):
        buf = torch.full((n + PAD, ld or w), float("nan"), device=DEV)
        buf[:n, :w] = torch.randn(n, w, device=DEV, generator=g)
        return buf[:n, :w] if ld else buf[:n]

    r = lambda *s: torch.randn(*s, device=DEV, generator=g)
    enc = rows(k_enc, ld_enc)
    hb, hg, h1, dz1, d1, dzb = rows(64), rows(128), rows(64), rows(64), rows(128), rows(64)
    dz2 = rows(3) if head else None
    d_sem = rows(64) if sem else None
    dwb0, dbb0, dwb1, dbb1 = r(64, k_enc), r(64), r(n_feat, 64), r(n_feat)
    w0, w1, dw2, db2 = r(64, RAY_COLS + 64), r(64, 128 + RAY_COLS), r(3, 64), r(3)
    outs = dict(dwb0=dwb0, dbb0=dbb0, dwb1=dwb1, dbb1=dbb1, w0=w0, w1=w1, dw2=dw2, db2=db2)
    before = {k: v.clone() for k, v in outs.items()}
    _ops._need_cuda(enc)
    P = _ops._ptr
    _lib.call("emer_field_wgrad", P(enc), ld_enc, k_enc, P(hb), P(hg), P(h1), P(dz2), P(dz1), P(d1), P(dzb), P(d_sem),
              n_feat, P(dwb0), P(dbb0), P(dwb1), P(dbb1), P(w0[:, RAY_COLS:]), w0.stride(0), P(w1),
              P(w1[:, 64 + RAY_COLS:]), w1.stride(0), P(dw2), P(db2), n, _ops._stream())
    torch.cuda.synchronize()

    for k, v in outs.items():
        assert torch.isfinite(v).all(), k
    d = lambda t: t.double()
    b = {k: d(v) for k, v in before.items()}
    dF, geo = d(d1[:, 64:]), d(hg[:, 64:])
    checks = [(dwb0, b["dwb0"] + d(dzb).T @ d(enc)), (dbb0, b["dbb0"] + d(dzb).sum(0)),
              (dwb1[:64], b["dwb1"][:64] + dF.T @ d(hb)), (dbb1[:64], b["dbb1"][:64] + dF.sum(0))]
    if sem:
        checks += [(dwb1[64:], b["dwb1"][64:] + d(d_sem).T @ d(hb)), (dbb1[64:], b["dbb1"][64:] + d(d_sem).sum(0))]
    if head:
        checks += [(w0[:, RAY_COLS:], b["w0"][:, RAY_COLS:] + d(d1[:, :64]).T @ geo),
                   (w1[:, :64], b["w1"][:, :64] + d(dz1).T @ d(hg[:, :64])),
                   (w1[:, 64 + RAY_COLS:], b["w1"][:, 64 + RAY_COLS:] + d(dz1).T @ geo),
                   (dw2, b["dw2"] + d(dz2).T @ d(h1)), (db2, b["db2"] + d(dz2).sum(0))]
        assert torch.equal(w0[:, :RAY_COLS], before["w0"][:, :RAY_COLS])
        assert torch.equal(w1[:, 64:64 + RAY_COLS], before["w1"][:, 64:64 + RAY_COLS])
    else:
        for k in ("w0", "w1", "dw2", "db2"):
            assert torch.equal(outs[k], before[k]), k
    for i, (got, want) in enumerate(checks):
        assert rel_err(got, want) < 2e-5, (i, rel_err(got, want))
