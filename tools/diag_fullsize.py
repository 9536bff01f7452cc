"""Where does the end-to-end difference at the benchmarked configuration come from?  (needs a CUDA device)

Stage-by-stage comparison of the drop-in on cuda:0 with the CPU oracle for the full-size static model
(tests/golden/full_cases.py), evaluation mode: every proposal level in isolation (fed with the ORACLE's previous
edges / CDF), the chained levels, and the field + compositing at the oracle's samples.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)

import full_cases as fc  # noqa: E402
from helpers import GOLDEN_DIR, Golden, rel_err  # noqa: E402
from emernerf_b200 import _ops  # noqa: E402
from emernerf_b200.radiance_fields import RadianceField, build_density_field  # noqa: E402
from emernerf_b200.radiance_fields.encodings import HashEncoder  # noqa: E402
from emernerf_b200.radiance_fields.render_utils import render_rays, rendering  # noqa: E402
from emernerf_b200.third_party.nerfacc_prop_net import PropNetEstimator  # noqa: E402
from oracle import adapters, hotpath, nerfacc_ref as nf  # noqa: E402

DEV = "cuda"
variant = sys.argv[1] if len(sys.argv) > 1 else "static"
ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField, build_density_field=build_density_field)
field, props = fc.build_models(ns, variant)
g = Golden.__new__(Golden)
g.case, g.z = variant, np.load(os.path.join(GOLDEN_DIR, f"full_{variant}.npz"))
field.load_state_dict(g.tensors("sd/field"), strict=False)
[p.load_state_dict(g.tensors(f"sd/prop{i}"), strict=False) for i, p in enumerate(props)]
batch = g.tensors("in/pixel")
R = batch["origins"].shape[0]
net = props[-1]
psd, pspec = adapters.cpu_state_dict(net), adapters.spec_from_module(net)
s_min, s_max = hotpath.s_bounds("uniform_lindisp", fc.NEAR, fc.FAR)

# ---- oracle, level by level
cdf = torch.tensor([[0.0, 1.0]]).repeat(R, 1)
s = cdf.clone()
orc = []
for n in fc.PROP_SAMPLES:
    iv, _ = nf.importance_sampling(nf.RayIntervals(s), cdf, n, False)
    t = hotpath._s_to_t("uniform_lindisp", iv.vals, fc.NEAR, fc.FAR)
    pos = batch["origins"][:, None, :] + batch["viewdirs"][:, None, :] * (t[:, :-1] + t[:, 1:])[..., None] / 2.0
    sig = hotpath.density_field_forward(psd, pspec, pos)["density"].squeeze(-1)
    trans, _ = nf.render_transmittance_from_density(t[:, :-1], t[:, 1:], sig)
    new_cdf = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1)
    orc.append((s, cdf, iv.vals, t, sig, new_cdf))
    s, cdf = iv.vals, new_cdf
iv, _ = nf.importance_sampling(nf.RayIntervals(s), cdf, fc.NUM_SAMPLES, False)
t_final = hotpath._s_to_t("uniform_lindisp", iv.vals, fc.NEAR, fc.FAR)

net_d = net.to(DEV)
lin = [m for m in net_d.base_mlp if isinstance(m, torch.nn.Linear)]
o_d, d_d = batch["origins"].to(DEV), batch["viewdirs"].to(DEV)


def level(prev_s, prev_cdf, n):
    return _ops.prop_level(prev_s.to(DEV), prev_cdf.to(DEV), n, None, s_min, s_max, "uniform_lindisp", o_d, d_d,
                           net_d.aabb, True, net_d.xyz_encoder.desc, net_d.xyz_encoder.tcnn_encoding.params,
                           lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias)


print("== each level in isolation (fed with the oracle's previous edges / CDF)")
for i, (ps, pc, s_w, t_w, sig_w, cdf_w) in enumerate(orc):
    s_g, t_g, cdf_g = level(ps, pc, fc.PROP_SAMPLES[i])
    # generic path: DensityField.forward on the oracle's points
    pos = o_d[:, None, :] + d_d[:, None, :] * (t_w.to(DEV)[:, :-1] + t_w.to(DEV)[:, 1:])[..., None] / 2.0
    with torch.no_grad():
        sig_gen = net_d(pos)["density"].squeeze(-1)
    print(f"level {i}: s exact {torch.equal(s_g.cpu(), s_w)}  t exact {torch.equal(t_g.cpu(), t_w)}  "
          f"cdf max|d| {float((cdf_g.cpu() - cdf_w).abs().max()):.3e}  "
          f"sigma(generic path) rel {rel_err(sig_gen, sig_w):.3e}  max sigma {float(sig_w.max()):.3e}  "
          f"max sigma*dt {float((sig_w * (t_w[:, 1:] - t_w[:, :-1])).max()):.3e}")

print("== chained levels on the GPU (its own CDFs)")
ps, pc = orc[0][0], orc[0][1]
for i, n in enumerate(fc.PROP_SAMPLES):
    s_g, t_g, cdf_g = level(ps, pc, n)
    d_t = (t_g.cpu() - orc[i][3]).abs()
    print(f"level {i}: edges differing {int((t_g.cpu() != orc[i][3]).sum())}/{t_g.numel()}  max |dt| {float(d_t.max()):.3e} "
          f"max rel {float((d_t / orc[i][3]).max()):.3e}  cdf max|d| {float((cdf_g.cpu() - orc[i][5]).abs().max()):.3e}")
    ps, pc = s_g, cdf_g
s_f, t_f = _ops.pdf_resample(ps.to(DEV), pc.to(DEV), fc.NUM_SAMPLES, None, s_min, s_max, "uniform_lindisp")
d_t = (t_f.cpu() - t_final).abs()
print(f"final: edges differing {int((t_f.cpu() != t_final).sum())}/{t_f.numel()}  max |dt| {float(d_t.max()):.3e}  "
      f"max rel {float((d_t / t_final).max()):.3e}  median rel {float((d_t / t_final).median()):.3e}")

print("== field + compositing at the ORACLE's samples")
field_d = field.to(DEV).eval()
fsd, fspec = adapters.cpu_state_dict(field), adapters.spec_from_module(field)
S = fc.NUM_SAMPLES
t0, t1 = t_final[:, :-1].contiguous(), t_final[:, 1:].contiguous()


def query_cpu(a, b):
    d = batch["viewdirs"][:, None, :].repeat_interleave(S, dim=-2)
    sub = {k: v[..., None].repeat_interleave(S, dim=-1) for k, v in batch.items()
           if k not in ("viewdirs", "origins", "pixel_coords")}
    sub["pixel_coords"] = batch["pixel_coords"]
    pos = batch["origins"][:, None, :] + d * (a + b)[..., None] / 2.0
    r = hotpath.radiance_field_forward(fsd, fspec, pos, d, sub, training=False)
    r["density"] = r["density"].squeeze(-1)
    return r


def query_gpu(a, b):
    bd = {k: v.to(DEV) for k, v in batch.items()}
    d = bd["viewdirs"][:, None, :].expand(-1, S, -1)
    sub = {k: v.unsqueeze(-1).expand(*v.shape, S) for k, v in bd.items() if k not in ("viewdirs", "origins", "pixel_coords")}
    sub["pixel_coords"] = bd["pixel_coords"]
    pos = bd["origins"][:, None, :] + d * (a + b)[..., None] / 2.0
    r = field_d(pos, d, sub)
    r["density"] = r["density"].squeeze(-1)
    return r


with torch.no_grad():
    want = hotpath.rendering(t0, t1, query_cpu(t0, t1), False)
    got = rendering(t0.to(DEV), t1.to(DEV), query_gpu)
for k in ("rgb", "depth", "opacity", "density"):
    print(f"  {k}: rel {rel_err(got[k], want[k]):.3e}")
print(f"  weights: rel {rel_err(got['extras']['weights'], want['extras']['weights']):.3e}")

print("== end to end (eval), fused levels vs generic levels")
est = PropNetEstimator(None, None).to(DEV).eval()
props_d = [p.to(DEV).eval() for p in props]
ref = g.nested("eval/out")
for fused in (True, False):
    est.fused_levels = fused
    with torch.no_grad():
        out = render_rays(field_d, est, props_d, {k: v.to(DEV) for k, v in batch.items()}, fc.render_cfg())
    print(f"  fused_levels={fused}: " + "  ".join(f"{k} {rel_err(out[k], ref[k]):.3e}" for k in ("rgb", "depth", "opacity")))
    tv = out["extras"]["t_vals"].cpu()
    dd = (tv - ref["extras"]["t_vals"]).abs() / ref["extras"]["t_vals"]
    print(f"     t_vals: max rel {float(dd.max()):.3e}  rays with any edge off by >1e-5 rel: {int((dd > 1e-5).any(-1).sum())}/{R}")
    per_ray = ((out["depth"].cpu() - ref["depth"]).abs() / ref["depth"].abs().max()).squeeze(-1)
    print(f"     depth: rays above 1e-4: {int((per_ray > 1e-4).sum())}/{R}; worst rays {per_ray.topk(5).indices.tolist()}")
