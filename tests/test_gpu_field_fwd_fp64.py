"""emer_field_fwd and emer_flow_field_fwd (csrc/field_fused.cu) through the C ABI, every element of every output and
save against an fp64 restatement of include/emer_b200.h, in every forward kernel the library builds, at the edges of the
persistent tile walk.

Kernels and cases.  field_fwd_kernel<k_enc, n_feat> for k_enc in {32, 40, 64}, n_feat in {64, 128} (one query per
row), each in training (every save), inference (saves NULL) and want_geo (save_hg only); the plain functions
flow_field_fwd_k40_f64, flow_field_fwd_k40_f128, flow_field_fwd_k64_f64 and flow_field_fwd_k64_f128 (three queries
per row, FLOW_KERNELS below), each with and without the colour head, in training and inference.  Sizes n in {1, 63,
64, 65, 192 SMs (one tile per warpgroup of the full grid), 192 SMs + 1, 3 * 192 SMs + 37}; the first four take the
min(SMs, ceil(tiles / 3)) grid's other branch.  S in {1, 33, 64, 128}, with ragged last rays.  Three input regimes:
*init* (encodings U(+-1e-4), the hash tables' initial scale, and nn.Linear's init), *trained* (per-row scales
10^U(-3, 1) mixed in every tile; feats[:, 0] - 1 spans [-25, 95], past the backward's e^15 clamp and fp32 exp's
overflow; colour logits span [-110, 40], where expf(-z) overflows and the sigmoid is exactly 0 or 1) and *cancel*
(ray_bias cancels geo W0g^T and the h1 pre-activation to 1e-3 of their size in half the units, so h0 and h1 sit at zero;
every 11th encoding row is exactly zero).  Every case has one geometry column (and one semantic column) whose weights
are zero and whose bias is an odd subnormal: the blend rounds there, and only a fused multiply-add changes its result.
enc is a 32-byte-aligned column view of a wider NaN buffer with NaN rows past n (3n); every output is a row view of a
NaN- or -7.0-filled buffer with 8 guard rows in front and 72 behind.

Error bound (u = 2^-24, per element, propagated stage by stage; the fp64 values are the reference's):
* Magnitudes: M_x = |x| + e_x; a layer z = W x + b has S_z = |W| M_x and M_z = S_z + |b|.
* Errors: e_z = |W| e_x + gamma_K S_z + 2 u M_z + 2^-126.  ReLU is 1-Lipschitz, so e passes through it whichever side
  of zero the kernel lands on.  The ray bias is b of the head's layers 0 and 1; layer 1 is one K = 128 product over
  [h0 | geo] (its accumulator carries across stages 2 and 3).
* gamma_K, 3xTF32 on the tensor core.  The truncating split leaves |x - hi - lo| <= 2^-20 |x| (tc_common.cuh), and
  mma3 drops lo*lo (<= 2^-20 |x| |w|): the three products miss x w by at most 3 * 2^-20 |x| |w|.  Accumulation: Hopper
  does not document how wgmma sums; the model assumed is the worst published for NVIDIA tensor cores -- the products of
  tf32 operands are exact, the eight of one k step and the accumulator are aligned to the largest exponent with
  truncation and no guard bits, and the sum is truncated back to fp32 -- so each of the 3K/8 wgmma calls of a product
  errs by at most 9 ulp of its largest term, <= 9 * 2^-23 S_z.  gamma_K = 3 * 2^-20 + (3K/8 + 1) * 9 * 2^-23 (the +1:
  the sum of the three products exceeds S_z by at most a factor 1 + 2^-9).  This constant was fixed before the first
  GPU run.
* sigma = expf(f0 - 1): the subtraction rounds (u |f0 - 1|) and expf is within 2 ulp (4 u), so
  |d sigma| <= sigma64 (exp(e_s) (1 + 4 u) - 1), e_s = e_f0 + u (|f0 - 1| + e_f0).  Where sigma64 exp(-e_s) (1 - 4 u)
  exceeds FLT_MAX the kernel must give +inf; where sigma64 exp(e_s) (1 + 4 u) is below it, a finite value.
* rgb = 1 / (1 + expf(-z)): the sigmoid's largest derivative over [z - e_z, z + e_z] times e_z, plus 8 u rgb (expf, the
  add, the divide), plus 2^-126 (where expf(-z) overflows to inf and rgb is 0).
* The blend ((F_c + 0.5 F_f) + 0.5 F_b) / 2: the 0.5 products and the halving are exact, the two adds round, so
  (e_c + e_f / 2 + e_b / 2) / 2 + u (M_c + M_f / 2 + M_b / 2) + 2^-126.

Checks per case: every element of sigma, rgb, save_hb (3N rows for three queries), save_hg = [h0 | geo], save_h1 and
save_sem within its bound (a NaN, i.e. an element never written over a NaN fill, fails); every element outside rows
[0, n) -- and save_hg's h0 half when the colour head is skipped -- bit for bit the fill; a second launch bit-identical.
Besides: a NaN encoding row per tile gives NaN in that row's outputs and leaves every other row bit-identical (a row
read from the wrong tile shows here); the three-query kernels' blended features equal the one-query kernel's per-query
features blended by torch in fp32, bit for bit; k_enc = 32 is refused for three queries.

The unmarked companion runs the same reference and bounds against tests/cabi_emulator.py, and against a torch
emulation of the kernel's arithmetic (the bit-mask split, the three products, fp32 accumulation per 8-wide k step, the
fp32 bias adds and the blend), and shows that each mutation in MUTATIONS fails at least one of the checks above.

Measured on an H100 80GB HBM3 (700 W power limit), the largest error / bound over the GPU cases, init / trained /
cancel: hb 0.45 / 0.19 / 0.059, geo 0.031 / 0.11 / 0.023, sem 0.044 / 0.036 / 0.035, sigma 0.052 / 0.10 / 0.035,
h0 0.010 / 0.078 / 0.0093, h1 0.0053 / 0.021 / 0.0053, rgb 0.0021 / 0.25 / 0.0017 (one and three queries within 1.5x
of each other); the whole file ran in 24 s there.  The emulation's maxima are 2 to 4 times lower (hb 0.43 / 0.11 /
0.021, geo 0.016 / 0.036 / 0.012, rgb 0.0011 / 0.21 / 0.0009), as a truncating accumulator would make them.  hb and
rgb are tight; the deeper layers sit 10 to 100 times below their bound because it charges every wgmma its worst case
and adds the stages' bounds, while the mutations, each 2^-11-sized or larger, still exceed it."""
import ctypes
import math

import pytest
import torch

import cabi_emulator

DEV = "cuda"
U = 2.0 ** -24
TINY = 2.0 ** -126
FLT_MAX = torch.finfo(torch.float32).max
C = 49                                     # the head's per-ray input columns: direction encoding (33) + embedding (16)
G, T = 8, 72                               # guard rows in front of / behind every output
SUB = (7, 64 + 5)                          # feature columns with zero weights and an odd subnormal bias
Q1 = [(k, f) for k in (32, 40, 64) for f in (64, 128)]
FLOW_KERNELS = {(40, 64): "flow_field_fwd_k40_f64", (40, 128): "flow_field_fwd_k40_f128",
                (64, 64): "flow_field_fwd_k64_f64", (64, 128): "flow_field_fwd_k64_f128"}
MODES = {1: ("train", "infer", "geo"), 3: ("train", "infer", "density_train", "density_infer")}
SAVES = {"train": ("hb", "hg", "h1"), "infer": (), "geo": ("hg",), "density_train": ("hb", "hg"),
         "density_infer": ("hg",)}
REGIMES = ("init", "trained", "cancel")
S_LIST = (1, 33, 64, 128)
SIZES = ("1", "63", "64", "65", "wg1", "wg1+1", "wg3+37")


def gamma(K):
    return 3 * 2.0 ** -20 + (3 * K // 8 + 1) * 9 * 2.0 ** -23


def size_of(label, sms):
    return {"wg1": 192 * sms, "wg1+1": 192 * sms + 1, "wg3+37": 3 * 192 * sms + 37}.get(label) or int(label)


def _cases():
    out = []
    for Q, insts in ((1, Q1), (3, list(FLOW_KERNELS))):
        for i, (k, f) in enumerate(insts):
            for m, mode in enumerate(MODES[Q]):
                for j, size in enumerate(SIZES):
                    out.append((Q, k, f, mode, size, S_LIST[(i + j) % 4], REGIMES[(i + m + j) % 3]))
    return out


CASES = _cases()


def _head(mode):
    return not mode.startswith("density")


# ------------------------------------------------------------------------------------------------- fp64 reference
def _lin(x, ex, w, b, K):
    """x W^T + b in fp64 and its error bound (the module docstring's model)."""
    S = (x.abs() + ex) @ w.abs().T
    z = x @ w.T + b
    return z, ex @ w.abs().T + gamma(K) * S + 2 * U * (S + b.abs()) + TINY


def _chain64(x, Q, n, S, nf, head):
    """{buffer: (fp64 value, bound)} of include/emer_b200.h's formula (sigma also carries its lower factor)."""
    d = {k: v.double() for k, v in x.items() if v is not None}
    k = d["enc"].shape[1]
    out, hbs, ehbs, F, eF = {}, [], [], [], []
    for q in range(Q):
        X = d["enc"][q * n:(q + 1) * n]
        z, e = _lin(X, torch.zeros_like(X), d["wb0"], d["bb0"], k)
        hbs.append(z.clamp_min(0.0))
        ehbs.append(e)
        f, ef = _lin(hbs[-1], e, d["wb1"], d["bb1"], 64)
        F.append(f)
        eF.append(ef)
    if Q == 1:
        feat, ef = F[0], eF[0]
    else:                                    # radiance_field.py: (dynamic + 0.5 * warped[0] + 0.5 * warped[1]) / 2.0
        feat = ((F[0] + 0.5 * F[1]) + 0.5 * F[2]) / 2.0
        M = [f.abs() + e for f, e in zip(F, eF)]
        ef = (eF[0] + eF[1] / 2 + eF[2] / 2) / 2 + U * (M[0] + M[1] / 2 + M[2] / 2) + TINY
    out["hb"] = (torch.cat(hbs), torch.cat(ehbs))
    geo, eg = feat[:, :64], ef[:, :64]
    out["geo"] = (geo, eg)
    if nf == 128:
        out["sem"] = (feat[:, 64:], ef[:, 64:])
    f0, e0 = feat[:, 0], ef[:, 0]
    es = e0 + U * ((f0 - 1.0).abs() + e0)
    sig = torch.exp(f0 - 1.0)
    out["sigma"] = (sig, sig * (torch.exp(es) * (1 + 4 * U) - 1.0) + TINY, torch.exp(-es) * (1 - 4 * U))
    if head:
        rb = d["rb"][torch.arange(n, device=geo.device) // S]
        w0, w1 = d["w0"], d["w1"]
        z0, e0 = _lin(geo, eg, w0[:, C:], rb[:, :64], 64)
        h0 = z0.clamp_min(0.0)
        z1, e1 = _lin(torch.cat([h0, geo], 1), torch.cat([e0, eg], 1), torch.cat([w1[:, :64], w1[:, 64 + C:]], 1),
                      rb[:, 64:], 128)
        h1 = z1.clamp_min(0.0)
        zl, el = _lin(h1, e1, d["w2"], d["b2"], 64)
        s = torch.sigmoid(zl)
        xi = torch.minimum(torch.maximum(torch.zeros_like(zl), zl - el), zl + el)
        sx = torch.sigmoid(xi)
        out.update(h0=(h0, e0), h1=(h1, e1), rgb=(s, sx * (1 - sx) * el + 8 * U * s + TINY))
    return out


# ------------------------------------------------------------------------------------------------- inputs, buffers
def _affine(t, lo, hi):
    """a, b with a t + b spanning [lo, hi] over t (a single row sits at lo)."""
    spread = (t.max() - t.min()).clamp_min(1e-3 * (float(t.abs().max()) + 1.0))
    a = (hi - lo) / spread
    return a, lo - a * t.min()


def _ray_mean(v, n, S):
    R = (n + S - 1) // S
    ray = torch.arange(n, device=v.device) // S
    s = torch.zeros(R, v.shape[1], dtype=v.dtype, device=v.device).index_add_(0, ray, v)
    return s / torch.bincount(ray, minlength=R)[:, None].to(v.dtype)


def _inputs(Q, k, nf, n, S, regime, seed, dev):
    """The kernel's inputs as fp32 tensors (enc and rb views of NaN-padded buffers)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, device=dev, dtype=torch.float64)
    nrm = lambda *s: torch.randn(*s, generator=g, device=dev, dtype=torch.float64)
    uni = lambda lim, *s: (rnd(*s) * 2 - 1) * lim
    R, rows = (n + S - 1) // S, Q * n
    if regime == "trained":
        x = dict(wb0=nrm(64, k) / k ** 0.5, bb0=nrm(64) * 0.1, wb1=nrm(nf, 64) / 8, bb1=nrm(nf) * 0.1,
                 w0=nrm(64, 64 + C) / (64 + C) ** 0.5, w1=nrm(64, 128 + C) / (128 + C) ** 0.5)
        b0, b1 = nrm(64) * 0.1, nrm(64) * 0.1
        enc = nrm(rows, k) * 10.0 ** (4 * rnd(rows, 1) - 3)
    else:                                  # nn.Linear's init: U(+-1 / sqrt(fan_in)) for weights and biases
        x = dict(wb0=uni(k ** -0.5, 64, k), bb0=uni(k ** -0.5, 64), wb1=uni(1 / 8, nf, 64), bb1=uni(1 / 8, nf),
                 w0=uni((64 + C) ** -0.5, 64, 64 + C), w1=uni((128 + C) ** -0.5, 64, 128 + C))
        b0, b1 = uni((64 + C) ** -0.5, 64), uni((128 + C) ** -0.5, 64)
        if regime == "init":
            enc = uni(1e-4, rows, k)
        else:                              # cancel: each ray's rows close to one encoding, every 11th row zero
            ray = (torch.arange(rows, device=dev) % n) // S
            enc = (nrm(R, k) * 0.5)[ray] * (1 + 1e-4 * nrm(rows, k))
            enc[::11] = 0.0
    x["w2"], x["b2"] = uni(1 / 8, 3, 64), uni(1 / 8, 3)
    for col, m in zip(SUB, (3, 5)):
        if col < nf:
            x["wb1"][col] = 0.0
            x["bb1"][col] = m * 2.0 ** -149
    v = uni(1.0, R, C)                     # per-ray inputs of the head: direction encoding and embedding
    x["rb"] = torch.cat([b0 + v @ x["w0"][:, :C].T, b1 + v @ x["w1"][:, 64:64 + C].T], 1)
    x["enc"] = enc
    f32 = lambda: {key: val.float().double() for key, val in x.items()}

    if regime == "trained":                # feats[:, 0] - 1 over [-25, 95]
        r = nrm(64)
        ref = _chain64(f32(), Q, n, S, nf, False)
        hb = ref["hb"][0]
        t = hb[:n] @ r if Q == 1 else ((hb[:n] @ r + 0.5 * (hb[n:2 * n] @ r)) + 0.5 * (hb[2 * n:] @ r)) / 2
        a, b = _affine(t, -24.0, 96.0)
        x["wb1"][0], x["bb1"][0] = a * r, b
    if regime == "cancel":                 # pre-activations of h0 (even units), then of h1 (odd units) cancelled
        ev, od = slice(0, 64, 2), slice(1, 64, 2)
        geo = _chain64(f32(), Q, n, S, nf, False)["geo"][0]
        pre0 = _ray_mean(geo, n, S) @ x["w0"][:, C:].T
        x["rb"][:, ev] = -pre0[:, ev] * (1 + uni(1e-3, R, 32))
        ref = _chain64(f32(), Q, n, S, nf, True)
        pre1 = _ray_mean(ref["h0"][0] @ x["w1"][:, :64].T + geo @ x["w1"][:, 64 + C:].T, n, S)
        x["rb"][:, 64 + 1::2] = -pre1[:, od] * (1 + uni(1e-3, R, 32))
    if regime == "trained":                # colour logits over [-110, 40]
        h1 = _chain64(f32(), Q, n, S, nf, True)["h1"][0]
        r2 = nrm(3, 64)
        for c in range(3):
            a, b = _affine(h1 @ r2[c], -110.0, 40.0)
            x["w2"][c], x["b2"][c] = a * r2[c], b
    out = {key: val.float() for key, val in x.items() if key not in ("enc", "rb")}
    eb = torch.full((rows + T, k + 16), float("nan"), device=dev)
    eb[:rows, 8:8 + k] = enc.float()
    rbb = torch.full((R + 8, 128), float("nan"), device=dev)
    rbb[:R] = x["rb"].float()
    out["enc"], out["rb"] = eb[:rows, 8:8 + k], rbb[:R]
    return out


def _outputs(Q, n, nf, mode, fill, dev):
    """{name: NaN- or fill-padded buffer}; the kernel writes rows [G, G + rows) of each."""
    saves = list(SAVES[mode]) or (["hg"] if Q == 3 else [])          # (three queries blend in save_hg)
    names = ["sigma"] + (["rgb"] if _head(mode) else []) + saves + (["sem"] if nf == 128 else [])
    cols = dict(sigma=1, rgb=3, hb=64, hg=128, h1=64, sem=64)
    return {m: torch.full((G + (Q * n if m == "hb" else n) + T, cols[m]), fill, device=dev) for m in names}


def _rows(o, name, Q, n):
    return o[name][G:G + (Q * n if name == "hb" else n)]


def _launch(call, stream, Q, x, o, k, nf, S, n, enc=None):
    P = lambda t: ctypes.c_void_p(0 if t is None else t.data_ptr())
    V = lambda m: _rows(o, m, Q, n) if m in o else None
    enc = x["enc"] if enc is None else enc
    w0, w1 = x["w0"], x["w1"]
    head = "rgb" in o
    call("emer_field_fwd" if Q == 1 else "emer_flow_field_fwd", P(enc), enc.stride(0), k, P(x["wb0"]), P(x["bb0"]),
         P(x["wb1"]), P(x["bb1"]), nf, P(w0[:, C:]), w0.stride(0), P(w1[:, :64]), P(w1[:, 64 + C:]), w1.stride(0),
         P(x["w2"]), P(x["b2"]), P(x["rb"] if head else None), S, P(V("sigma")), P(V("rgb")), P(V("hb")), P(V("hg")),
         P(V("h1")), P(V("sem")), n, stream)


# ------------------------------------------------------------------------------------------------- checks
def _bits(t):
    return t.contiguous().view(torch.int32)


def _failures(o, ref, Q, n, fill):
    """(failed checks as "kind: what", {buffer: largest error / bound})."""
    fails, ratios = [], {}
    fb = _bits(torch.tensor([fill]))[0].item()
    head = "rgb" in o
    for name, buf in o.items():
        rows = Q * n if name == "hb" else n
        guard = torch.cat([_bits(buf[:G]).flatten(), _bits(buf[G + rows:]).flatten()])
        if bool((guard != fb).any()):
            fails.append(f"sentinel: {name} written outside rows [0, {rows})")
        if name == "hg" and not head and bool((_bits(buf[G:G + rows, :64]) != fb).any()):
            fails.append("sentinel: save_hg's h0 half written without the colour head")

    def bound(label, got, want, b):
        if got.numel() == 0:
            return
        err = (got.double() - want).abs()
        ratios[label] = max(ratios.get(label, 0.0), float((err / b).nan_to_num(math.inf).max()))
        bad = ~(err <= b)
        if bool(bad.any()):
            i = int(bad.flatten().nonzero()[0])
            fails.append(f"bound: {label} {int(bad.sum())} elements, first flat {i}: got {got.flatten()[i].item()!r} "
                         f"want {want.flatten()[i].item()!r} +- {b.flatten()[i].item():.3g}")

    got = {m: _rows(o, m, Q, n) for m in o}
    for m in ("hb", "h1", "sem", "rgb"):
        if m in got:
            bound(m, got[m], *ref[m])
    if "hg" in got:
        bound("geo", got["hg"][:, 64:], *ref["geo"])
        if head:
            bound("h0", got["hg"][:, :64], *ref["h0"])
    s, (sig, b, lo) = got["sigma"][:, 0].double(), ref["sigma"]
    must_inf, must_fin = sig * lo > FLT_MAX, sig + b < FLT_MAX
    if not bool((s[must_inf] == math.inf).all()):
        fails.append("bound: sigma finite where exp(f0 - 1) overflows fp32")
    if bool(torch.isinf(s[must_fin]).any()):
        fails.append("bound: sigma inf where exp(f0 - 1) is within fp32")
    fin = ~must_inf & ~(torch.isinf(s) & ~must_fin)
    bound("sigma", s[fin], sig[fin], b[fin])
    return fails, ratios


def _blend32(f):
    """The reference's blend in fp32 torch: (dynamic + 0.5 * warped[0] + 0.5 * warped[1]) / 2.0."""
    return (f[0] + 0.5 * f[1] + 0.5 * f[2]) / 2.0


def _report(tag, ratios):
    print(f"RATIO {tag} " + " ".join(f"{m}={r:.3g}" for m, r in sorted(ratios.items())))


def _ids(cases):
    return [f"Q{Q}-k{k}-f{f}-{m}-n{s}-S{S}-{r}" for Q, k, f, m, s, S, r in cases]


# ------------------------------------------------------------------------------------------------- GPU
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(Q, k, nf, mode, n, S, x, fill, enc=None):
    from emernerf_b200 import _lib, _ops

    o = _outputs(Q, n, nf, mode, fill, DEV)
    _ops._need_cuda(x["enc"])
    _launch(_lib.call, _ops._stream(), Q, x, o, k, nf, S, n, enc=enc)
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("Q,k,nf,mode,size,S,regime", CASES, ids=_ids(CASES))
def test_field_fwd_vs_fp64(Q, k, nf, mode, size, S, regime):
    """Every element within its bound, nothing written outside rows [0, n), a second launch bit-identical."""
    n = size_of(size, _sms())
    fill = (float("nan"), -7.0)[(n + k + nf + S) % 2]
    x = _inputs(Q, k, nf, n, S, regime, seed=n + 7 * k + nf + S + Q, dev=DEV)
    a = _run(Q, k, nf, mode, n, S, x, fill)
    b = _run(Q, k, nf, mode, n, S, x, fill)
    torch.cuda.synchronize()
    fails, ratios = _failures(a, _chain64(x, Q, n, S, nf, _head(mode)), Q, n, fill)
    _report(f"{regime} Q{Q}", ratios)
    assert not fails, fails
    for m in a:
        assert torch.equal(_bits(a[m]), _bits(b[m])), m


@pytest.mark.gpu
@pytest.mark.parametrize("Q,k,nf", [(1, k, f) for k, f in Q1] + [(3, k, f) for k, f in FLOW_KERNELS])
def test_field_fwd_rows_are_independent(Q, k, nf):
    """One NaN encoding row per tile (for three queries, in the query tile % 3): that row's sigma, rgb and saves are
    NaN, as torch.relu keeps NaN; every other element of every buffer is bit-identical to the launch without them."""
    n, S = 192 * _sms() + 1, 64
    x = _inputs(Q, k, nf, n, S, "trained", seed=5 + k + nf + Q, dev=DEV)
    clean = _run(Q, k, nf, "train", n, S, x, -7.0)
    tiles = torch.arange((n + 63) // 64)
    row = (tiles * 64 + (37 * tiles) % 64).clamp(max=n - 1)
    qrow = (tiles % Q) * n + row
    x["enc"][qrow.to(DEV)] = float("nan")
    dirty = _run(Q, k, nf, "train", n, S, x, -7.0)
    torch.cuda.synchronize()
    for m in clean:
        a, b = _rows(clean, m, Q, n), _rows(dirty, m, Q, n)
        bad = torch.zeros(a.shape[0], dtype=torch.bool, device=DEV)
        bad[(qrow if m == "hb" else row).to(DEV)] = True
        assert not bool(a.isnan().any()), m
        # (the SUB columns' weights are zero: whether the tensor core's NaN * 0 is NaN is not at stake here)
        skip = {"hg": 64 + SUB[0], "sem": SUB[1] - 64}.get(m)
        assert bool(b[bad][:, [c for c in range(a.shape[1]) if c != skip]].isnan().all()), m
        assert torch.equal(a[~bad], b[~bad]), m
        assert torch.equal(_bits(clean[m][:G]), _bits(dirty[m][:G])), m
        assert torch.equal(_bits(clean[m][G + a.shape[0]:]), _bits(dirty[m][G + a.shape[0]:])), m


@pytest.mark.gpu
@pytest.mark.parametrize("k,nf", list(FLOW_KERNELS))
def test_flow_blend_is_the_reference_expression_bit_for_bit(k, nf):
    """The three-query kernel's blended geometry and semantic features equal the one-query kernel's features of each
    third of enc, blended by torch in fp32, bit for bit: both kernels run field_fwd_body's MMA sequence, and the blend
    keeps the reference's operation order without contraction (the subnormal columns of SUB round differently under a
    fused multiply-add)."""
    n, S = 192 * _sms() + 1, 64
    x = _inputs(3, k, nf, n, S, "trained", seed=9 + k + nf, dev=DEV)
    flow = _run(3, k, nf, "train", n, S, x, float("nan"))
    per = [_run(1, k, nf, "train", n, S, x, float("nan"), enc=x["enc"][q * n:(q + 1) * n]) for q in range(3)]
    torch.cuda.synchronize()
    geo = _blend32([_rows(o, "hg", 1, n)[:, 64:] for o in per])
    assert geo[:, SUB[0]].abs().max().item() < TINY and bool((geo[:, SUB[0]] != 0).all())
    assert torch.equal(_rows(flow, "hg", 3, n)[:, 64:], geo)
    if nf == 128:
        assert torch.equal(_rows(flow, "sem", 3, n), _blend32([_rows(o, "sem", 1, n) for o in per]))


@pytest.mark.gpu
def test_flow_field_fwd_refuses_k_enc_32():
    x = _inputs(3, 32, 64, 64, 64, "init", seed=1, dev=DEV)
    with pytest.raises(RuntimeError, match="k_enc=32 must be 40 or 64"):
        _run(3, 32, 64, "train", 64, 64, x, -7.0)


# ------------------------------------------------------------------------------------------------- CPU companion
MASK = -8192                                # 0xFFFFE000: tc::split keeps sign, exponent and 10 mantissa bits


def _split(v):
    hi = (v.view(torch.int32) & MASK).view(torch.float32)
    return hi, ((v - hi).view(torch.int32) & MASK).view(torch.float32)


def _mma(acc, a, w, products=("hh", "lh", "hl")):
    """acc (+)= a w^T as the kernel's wgmma k steps: three products of the split operands per 8-wide step, each step's
    eight exact products and the accumulator summed and rounded to fp32 once."""
    (ah, al), (bh, bl) = _split(a), _split(w)
    ops = {"hh": (ah, bh), "lh": (al, bh), "hl": (ah, bl)}
    for ks in range(0, a.shape[1], 8):
        for p in products:
            A, B = ops[p]
            s = A[:, ks:ks + 8].double() @ B[:, ks:ks + 8].double().T
            acc = s.float() if acc is None else (acc.double() + s).float()
    return acc


def _emulate(x, Q, n, S, nf, o, mut=None, enc=None):
    """field_fwd_body<k_enc, nf, Q> in torch: whole 64-row tiles whose rows past n read row n - 1, fp32 everywhere the
    kernel rounds, stores of rows [0, n) into the buffers of ``o``.  ``mut`` names one entry of MUTATIONS."""
    enc = x["enc"] if enc is None else enc
    npad = -(-n // 64) * 64
    rows = torch.arange(npad).clamp(max=n - 1)
    keep = npad if mut == "store_last_tile" else n

    def store(m, v, r0=0):
        if m in o:
            o[m][G + r0:G + r0 + keep, :v.shape[1]] = v[:keep]

    feat = None
    for q in range(Q):
        hb = torch.relu(_mma(None, enc[q * n + rows], x["wb0"]) + x["bb0"])
        store("hb", hb, q * n)
        F = _mma(None, hb, x["wb1"], ("hh",) if mut == "1xtf32_stage1" else ("hh", "lh", "hl")) + x["bb1"]
        if q == 0:
            feat = F
        elif mut == "blend_fma":
            feat = (feat.double() + 0.5 * F.double()).float()
        else:
            feat = feat + 0.5 * F
        if q == Q - 1 and Q > 1:
            feat = feat * 0.5
    geo = feat[:, :64]
    o["sigma"][G:G + keep, 0] = torch.exp(geo[:, 0] - 1.0)[:keep]
    if "sem" in o:
        o["sem"][G:G + keep] = feat[:keep, 64:]
    if "hg" in o:
        o["hg"][G:G + keep, 64:] = geo[:keep]
    if "rgb" not in o:
        return
    ray = rows // S
    if mut == "last_ray_prev_bias" and n % S and n > S:
        ray = torch.where(ray == (n - 1) // S, ray - 1, ray)
    rb = x["rb"][ray]
    stage2 = ("hh", "hl") if mut == "drop_alo_bhi_stage2" else ("hh", "lh", "hl")
    d0 = _mma(None, geo, x["w0"][:, C:], stage2)
    d1 = _mma(None, geo, x["w1"][:, 64 + C:], stage2)
    h0 = torch.relu(d0 + rb[:, :64])
    store("hg", h0)
    h1 = torch.relu(_mma(d1, h0, x["w1"][:, :64]) + rb[:, 64:])
    store("h1", h1)
    z = _mma(None, h1, x["w2"]) + x["b2"]
    store("rgb", 1.0 / (1.0 + torch.exp(-z)))


# mutation of the emulation -> the kind of check it must fail
MUTATIONS = {
    "1xtf32_stage1": "bound",               # feats from hi * hi alone
    "drop_alo_bhi_stage2": "bound",         # the head's first products without alo * bhi
    "blend_fma": "blend",                   # acc + 0.5 F rounded once, as a fused multiply-add would
    "last_ray_prev_bias": "bound",          # the ragged last ray reads the previous ray's bias
    "store_last_tile": "sentinel",          # the whole last tile stored, past row n
}
CPU_SIZES = (1, 65, 64 * 3 + 37)


def _cpu_cases():
    out = []
    for Q, insts in ((1, Q1), (3, list(FLOW_KERNELS))):
        for i, (k, f) in enumerate(insts):
            for m, mode in enumerate(MODES[Q]):
                for j, n in enumerate(CPU_SIZES):
                    out.append((Q, k, f, mode, n, S_LIST[(i + j + m) % 4], REGIMES[(i + m + j) % 3]))
    return out


CPU_CASES = _cpu_cases()


def _emulation_failures(Q, k, nf, mode, n, S, regime, mut=None):
    fill = (float("nan"), -7.0)[(n + k + nf + S) % 2]
    x = _inputs(Q, k, nf, n, S, regime, seed=n + 7 * k + nf + S + Q, dev="cpu")
    o = _outputs(Q, n, nf, mode, fill, "cpu")
    _emulate(x, Q, n, S, nf, o, mut)
    fails, ratios = _failures(o, _chain64(x, Q, n, S, nf, _head(mode)), Q, n, fill)
    if Q == 3:
        per = []
        for q in range(3):
            p = _outputs(1, n, nf, "train", fill, "cpu")
            _emulate(x, 1, n, S, nf, p, enc=x["enc"][q * n:(q + 1) * n])
            per.append(p)
        want = _blend32([_rows(p, "hg", 1, n)[:, 64:] for p in per])
        if not torch.equal(_rows(o, "hg", 3, n)[:, 64:], want):
            fails.append("blend: the blended geometry features differ from the reference expression's")
    return fails, ratios


@pytest.mark.parametrize("Q,k,nf,mode,n,S,regime", [c for c in CPU_CASES if c[0] == 1],
                         ids=_ids([c for c in CPU_CASES if c[0] == 1]))
def test_emulator_vs_fp64(Q, k, nf, mode, n, S, regime):
    """tests/cabi_emulator.py's emer_field_fwd within the same bounds, on the same buffer layout."""
    fill = (float("nan"), -7.0)[(n + k + nf + S) % 2]
    x = _inputs(Q, k, nf, n, S, regime, seed=n + 7 * k + nf + S + Q, dev="cpu")
    o = _outputs(Q, n, nf, mode, fill, "cpu")
    _launch(lambda name, *a: getattr(cabi_emulator, name)(*a), None, Q, x, o, k, nf, S, n)
    fails, ratios = _failures(o, _chain64(x, Q, n, S, nf, True), Q, n, fill)
    _report(f"{regime} emulator", ratios)
    assert not fails, fails


@pytest.mark.parametrize("Q,k,nf,mode,n,S,regime", CPU_CASES, ids=_ids(CPU_CASES))
def test_kernel_emulation_within_bounds(Q, k, nf, mode, n, S, regime):
    """The kernel's arithmetic, emulated, passes every check the GPU cases make."""
    fails, ratios = _emulation_failures(Q, k, nf, mode, n, S, regime)
    _report(f"{regime} emulation Q{Q}", ratios)
    assert not fails, fails


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_mutation_fails_a_check(mut):
    """Each mutation of the emulation fails a check of its kind in at least one case (all regimes, both query counts,
    a ragged last tile and ray)."""
    kinds = set()
    for Q, k, nf in ((1, 40, 128), (3, 64, 128)):
        for regime in REGIMES:
            fails, _ = _emulation_failures(Q, k, nf, "train", 64 * 2 + 37, 64, regime, mut)
            kinds |= {f.split(":")[0] for f in fails}
    assert MUTATIONS[mut] in kinds, (mut, kinds)
