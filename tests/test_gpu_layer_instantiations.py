"""Every compiled instantiation of the dense-layer kernels (csrc/linear_tc.cu, wgrad_mn.cu, linear_simt.cu), of the hash
grid (grid.cu), the proposal level (prop_level.cu) and the small accumulation (composite.cu), each against a plain fp64
restatement of its entry point in include/emer_b200.h, and the layer dispatch of _ops on both sides of every boundary.

Case tables: one per templated kernel.  The instantiation a row launches follows from its shape by the library's
dispatch rule, restated here (``wgrad_key``, ``tc_nb``, ...; ``_key`` form, e.g. ``emer::wg::wgrad_kernel<16,1>``).
``test_every_template_instantiation_has_a_case`` (no GPU needed) lists the ``__global__`` template instantiations of the
built library and fails for one that no row -- here or in the suites named by ``elsewhere()`` -- launches, so a kernel
instantiation added later without a test case fails the suite.

Layer cases call the C ABI directly: row counts 1, 37, 64 k + r and one with more tiles than the persistent grid has
warpgroups; inputs are column views of wider buffers whose other columns are NaN (a kernel that reads past its columns
fails); outputs are views of NaN-filled buffers whose NaN bits outside [0, ncols) must survive bit for bit; accumulating
outputs (dW, db, ``accumulate = 1``) start from non-zero values.

Bars, relative to the max-abs of the fp64 result: 2e-5 for per-row products and for reductions over up to 2e5 rows,
5e-5 beyond (the bars of test_gpu_kernels.py).  3xTF32 and FFMA land near 1e-6; one dropped product of a 3xTF32 stage
gives tf32's ~5e-4."""
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

from helpers import rel_err

DEV = "cuda"
NONE, RELU, SIGMOID = 0, 1, 2
NAN = float("nan")
# 4225 tiles of 64 rows: more than the 2112 warpgroups of a 132-SM grid at its 8-CTA occupancy limit, so every
# warpgroup of tc_linear_kernel's persistent loop walks at least two tiles
N_BIG = 64 * 4224 + 45
ROWS = (1, 37, 64 * 150 + 29, N_BIG)


def _key(symbol: str) -> str:
    """``void emer::wg::wgrad_kernel<(int)16, (int)1>(emer::wg::Params)`` (cu++filt) and ``void
    emer::wg::wgrad_kernel<16, 1>(emer::wg::Params)`` -> ``emer::wg::wgrad_kernel<16,1>``."""
    s = re.sub(r"\((?:int|bool)\)", "", symbol)
    s = re.sub(r"\bfalse\b", "0", re.sub(r"\btrue\b", "1", s))
    if s.startswith("void "):
        s = s[5:]
    return s.split("(", 1)[0].replace(" ", "")


def _tol(n: int) -> float:
    return 2e-5 if n <= 200000 else 5e-5


# ============================================================================ case tables
# tc_linear_kernel<BWD>: the output walks 64-column blocks, then one run_block<NB> tail for NB = n_pad % 64.  Forward:
# output width n_out, reduction k.  Backward (data): output width k, reduction n_out; the resident panels limit a
# 256-wide output to a reduction of at most 96.
TC_FWD = [  # (k, n_out, act)
    (40, 16, RELU),          # n_pad 16: the NB = 16 block alone
    (64, 24, NONE),          # 32
    (33, 40, SIGMOID),       # 48
    (64, 64, RELU),          # 64
    (100, 80, NONE),         # 64 + 16
    (17, 90, SIGMOID),       # 64 + 32
    (128, 176, RELU),        # 2 x 64 + 48
    (96, 256, NONE),         # n_pad 256, the widest MMA: 4 x 64
    (90, 250, SIGMOID),      # n_pad 256 with six padded columns
]
TC_BWD = [  # (k, n_out, act, relu_cols, accumulate)
    (16, 64, NONE, 0, 0),          # n_pad 16
    (8, 40, RELU, 8, 1),           # 16
    (30, 64, SIGMOID, 0, 1),       # 32
    (40, 33, RELU, 24, 0),         # 48
    (64, 128, NONE, 64, 0),        # 64
    (100, 64, RELU, 64, 1),        # 64 + 48
    (150, 48, SIGMOID, 100, 0),    # 2 x 64 + 32
    (200, 70, NONE, 150, 1),       # 3 x 64 + 16
    (256, 96, NONE, 200, 1),       # n_pad 256
    (250, 64, RELU, 250, 0),       # n_pad 256 with six padded columns
]


def tc_nb(ncols: int) -> int:
    """The run_block<NB> width of the last block of an output ``ncols`` wide (linear_tc.cu: tc_linear_kernel)."""
    t = (ncols + 15) // 16 * 16 % 64
    return t if t else 64


# wgrad_kernel<NP, MB>: NP = n_out rounded up to 16 / 32 / 64 / 128, MB = ceil(k / 64) warpgroups, capped at 4
WG_NOUT = {16: (9, 16), 32: (17, 32), 64: (36, 64), 128: (68, 128)}
WG_K = {1: (40, 64), 2: (65, 128), 3: (136, 192), 4: (193, 256)}
WGRAD = [(np_, mb, WG_K[mb][(i + j) % 2], WG_NOUT[np_][(i + j) % 2])
         for i, np_ in enumerate(WG_NOUT) for j, mb in enumerate(WG_K)]           # (NP, MB, k, n_out)


def wgrad_key(k: int, n_out: int) -> str:
    np_ = 16 if n_out <= 16 else 32 if n_out <= 32 else 64 if n_out <= 64 else 128
    return f"emer::wg::wgrad_kernel<{np_},{min((k + 63) // 64, 4)}>"


# narrow layers (n_out <= 8, k <= 256).  X / dX views start ``off`` floats into their buffer rows.
NARROW_FWD = [  # (k, n_out, act, x_off, ldx, path)  path: 16-byte vector loads or the scalar loop
    (64, 2, RELU, 4, 72, "vec"),
    (256, 8, NONE, 4, 264, "vec"),           # a full shared-memory panel (NARROW_MAX_K x NARROW_MAX_OUT)
    (4, 5, SIGMOID, 0, 8, "vec"),
    (1, 4, NONE, 0, 4, "scalar"),            # k = 1
    (37, 7, RELU, 4, 44, "scalar"),          # k % 4 != 0
    (64, 3, NONE, 1, 70, "scalar"),          # misaligned X
    (255, 1, SIGMOID, 4, 260, "scalar"),
    (256, 6, NONE, 1, 260, "scalar"),        # misaligned X, full panel
]


def narrow_fwd_path(k, x_off, ldx):
    return "vec" if k % 4 == 0 and x_off % 4 == 0 and ldx % 4 == 0 else "scalar"


NARROW_DATA = [  # (k, n_out, relu_cols, dx_off, lddx, store)  store: float4 only, float4 + scalar tail, scalar only
    (64, 3, 64, 4, 72, "vec"),
    (256, 2, 256, 4, 264, "vec"),
    (1, 1, 1, 4, 8, "tail"),                 # k = 1 inside an 8-float row: columns 5..7 are the caller's
    (3, 8, 0, 4, 12, "tail"),
    (37, 5, 20, 4, 48, "tail"),
    (255, 7, 100, 4, 264, "tail"),
    (30, 6, 30, 0, 30, "scalar"),            # dense rows, lddx = k = 30
    (64, 4, 0, 1, 70, "scalar"),             # misaligned dX
]


def narrow_store(k, dx_off, lddx):
    if dx_off % 4 or lddx % 4:
        return "scalar"
    return "vec" if k % 4 == 0 else "tail"


NARROW_WGRAD = [  # (k, n_out, x_off, ldx, dz_off, lddz, bias)
    (64, 3, 4, 72, 0, 4, True),              # vec4<4, true>: dZ rows padded to 4 floats
    (256, 4, 4, 264, 4, 12, False),
    (4, 1, 0, 4, 0, 4, True),
    (64, 2, 4, 72, 0, 2, True),              # vec4<4, false>: unpadded dZ rows
    (128, 4, 4, 136, 1, 12, True),           # misaligned dZ
    (256, 3, 0, 256, 0, 3, False),
    (37, 3, 4, 44, 0, 4, True),              # scalar: k % 4 != 0
    (64, 5, 4, 72, 0, 8, True),              # scalar: n_out > 4
    (64, 2, 1, 70, 0, 4, True),              # scalar: misaligned X
    (256, 8, 4, 264, 0, 8, True),
    (1, 6, 0, 1, 0, 6, True),                # k = 1
]


def narrow_wgrad_key(k, n_out, x_off, ldx, dz_off, lddz):
    """emer_linear_narrow_bwd_weight's choice (linear_simt.cu)."""
    if n_out <= 4 and k % 4 == 0 and ldx % 4 == 0 and x_off % 4 == 0:
        dz_vec = lddz % 4 == 0 and dz_off % 4 == 0
        return f"emer::narrow_wgrad_vec4_kernel<4,{int(dz_vec)}>"
    return "emer::narrow_wgrad_kernel"


# the FP32-FMA kernels: gemm_rows_kernel<BWD> (forward, data gradient), wgrad_kernel (weight gradient)
SIMT_FWD = [(130, 70, NONE), (257, 300, RELU), (5, 65, SIGMOID)]                       # (k, n_out, act)
SIMT_DATA = [(130, 70, NONE, 0), (257, 300, RELU, 1), (65, 5, SIGMOID, 0), (300, 129, SIGMOID, 1), (64, 64, RELU, 0),
             (9, 3, NONE, 1)]                                                           # (k, n_out, act, accumulate)
SIMT_WGRAD = [(130, 70, NONE, True), (257, 300, RELU, True), (65, 5, SIGMOID, False)]  # (k, n_out, act, bias)

# hash grid <D, F>: level configs (levels, base, max resolution, log2 table size, features) with dense and hashed levels
GRID_CASES = {(3, 1): (4, 16, 96, 12, 1), (3, 2): (4, 8, 64, 11, 2), (3, 4): (4, 8, 64, 10, 4),
              (4, 1): (4, 4, 32, 12, 1), (4, 2): (3, 4, 24, 9, 2), (4, 4): (4, 4, 32, 10, 4)}
GRID_G = {1: 8, 2: 4, 4: 1}                      # levels per CTA group (grid.cu: level_group<F>)


def grid_keys(D, F):
    G = GRID_G[F]
    return {f"emer::grid_fwd_kernel<{D},{F},{G}>", f"emer::grid_bwd_table_kernel<{D},{F},{G}>",
            f"emer::grid_bwd_dx_kernel<{D},{F}>"}


# proposal levels: (levels, features, previous level, n).  "uniform": the first level, [0, 1] with a flat CDF;
# "real": the output of a 128-interval level of the same network (m1 = 129), as the benchmark's second level
PROP_CASES = [(8, 1, "uniform", 128), (8, 1, "real", 64), (8, 1, "real", 256), (4, 1, "uniform", 32),
              (4, 1, "real", 256), (4, 2, "uniform", 32), (4, 2, "real", 64)]


def prop_key(levels, feats):
    lf = levels * feats
    return f"emer::prop_level_kernel<{lf if feats == 1 and lf in (4, 8) else 0}>"


ACC_CHANNELS = (1, 2, 3, 4)                       # accumulate_small_fwd_kernel<C>
FIELD_FWD = [(k, f) for k in (32, 40, 64) for f in (64, 128)]        # field_fwd_kernel<k_enc, n_feat>


def case_keys():
    """Every kernel the case tables of this file launch."""
    keys = {"emer::tc::tc_linear_kernel<0>", "emer::tc::tc_linear_kernel<1>", "emer::gemm_rows_kernel<0>",
            "emer::gemm_rows_kernel<1>", "emer::wgrad_kernel", "emer::narrow_fwd_kernel", "emer::narrow_bwd_data_kernel"}
    keys |= {wgrad_key(k, n_out) for _, _, k, n_out in WGRAD}
    keys |= {narrow_wgrad_key(*c[:6]) for c in NARROW_WGRAD}
    for D, F in GRID_CASES:
        keys |= grid_keys(D, F)
    keys |= {prop_key(l, f) for l, f, _, _ in PROP_CASES}
    keys |= {f"emer::accumulate_small_fwd_kernel<{c}>" for c in ACC_CHANNELS}
    keys |= {f"emer::ff::field_fwd_kernel<{k},{f}>" for k, f in FIELD_FWD}
    return keys


def elsewhere():
    """Template instantiations the case tables of other suites launch against their own references."""
    import test_gpu_field_chain
    import test_gpu_field_wgrad
    import test_gpu_prop_level_grad

    out = {f"emer::ff::field_bwd_kernel<{k},{f}>": "test_gpu_field_chain.py" for k, f in test_gpu_field_chain.INSTANCES}
    out.update({f"emer::fw::field_wgrad_kernel<{c[0]},{int(c[3])}>": "test_gpu_field_wgrad.py"
                for c in test_gpu_field_wgrad.CASES})
    out.update({f"emer::grid_indices_kernel<{d}>": "test_gpu_kernels.py::test_grid_corner_indices_bit_exact"
                for d in (3, 4)})
    out.update({f"emer::prop_level_bwd_kernel<{c[0]}>": "test_gpu_prop_level_grad.py::test_level_backward_vs_fp64"
                for c in test_gpu_prop_level_grad.CASES.values()})
    return out


# ============================================================================ the instantiation guard (no GPU)
def _tool(name):
    p = shutil.which(name)
    if p:
        return p
    p = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return p if os.path.exists(p) else None


def test_every_template_instantiation_has_a_case():
    """The ``__global__`` template instantiations in libemer_b200.so (cuobjdump -symbols | cu++filt) are exactly the
    ones the case tables launch, and the tables reach every run-time branch a symbol cannot show: each run_block<NB>
    tail of tc_linear_kernel in both directions with n_pad = 256 among them, both load paths of narrow_fwd_kernel, the
    three store forms of narrow_bwd_data_kernel."""
    from emernerf_b200 import _lib

    dump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if dump is None or filt is None:
        pytest.skip("cuobjdump / cu++filt not found")
    lib = _lib.lib_path()
    if not os.path.exists(lib):
        pytest.skip("libemer_b200.so is not built")
    listing = subprocess.run([dump, "-symbols", lib], capture_output=True, text=True, check=True).stdout
    mangled = [ln.split()[-1] for ln in listing.splitlines() if "STO_ENTRY" in ln]
    assert mangled, "no kernel entry symbols in " + lib
    names = subprocess.run([filt], input="\n".join(mangled) + "\n", capture_output=True, text=True,
                           check=True).stdout.split("\n")
    templates = {_key(s) for s in names if "<" in s}
    assert "emer::wg::wgrad_kernel<16,1>" in templates, sorted(templates)
    covered = case_keys() | set(elsewhere())
    assert not sorted(templates - covered), f"instantiations without a test case: {sorted(templates - covered)}"
    stale = sorted(k for k in covered if "<" in k and k not in templates)
    assert not stale, f"case rows for instantiations the library does not have: {stale}"

    assert {tc_nb(n_out) for _, n_out, _ in TC_FWD} == {16, 32, 48, 64}
    assert {tc_nb(k) for k, *_ in TC_BWD} == {16, 32, 48, 64}
    assert any((n_out + 15) // 16 * 16 == 256 for _, n_out, _ in TC_FWD)
    assert any((k + 15) // 16 * 16 == 256 for k, *_ in TC_BWD)
    assert {(np_, mb) for np_, mb, _, _ in WGRAD} == {(p, m) for p in (16, 32, 64, 128) for m in (1, 2, 3, 4)}
    for np_, mb, k, n_out in WGRAD:
        assert wgrad_key(k, n_out) == f"emer::wg::wgrad_kernel<{np_},{mb}>"
    for k, _, _, x_off, ldx, path in NARROW_FWD:
        assert narrow_fwd_path(k, x_off, ldx) == path
    assert {c[5] for c in NARROW_FWD} == {"vec", "scalar"}
    for k, _, _, dx_off, lddx, store in NARROW_DATA:
        assert narrow_store(k, dx_off, lddx) == store
    assert {c[5] for c in NARROW_DATA} == {"vec", "tail", "scalar"}
    assert {n for _, n, *_ in NARROW_FWD} == set(range(1, 9)) == {n for _, n, *_ in NARROW_DATA}
    assert {c[2] for c in SIMT_FWD} == {c[2] for c in SIMT_DATA} == {c[2] for c in SIMT_WGRAD} == {NONE, RELU, SIGMOID}
    assert {c[3] for c in SIMT_DATA} == {0, 1}


# ============================================================================ GPU helpers
def _operand(n, cols, ld, off, gen, fill=None):
    """[n, cols] view at column ``off`` of an [n, ld] buffer whose other columns are NaN."""
    buf = torch.full((n, ld), NAN, device=DEV)
    buf[:, off:off + cols] = torch.randn(n, cols, device=DEV, generator=gen) if fill is None else fill
    return buf, buf[:, off:off + cols]


def _flat(shape, gen):
    """A non-zero accumulation target [shape] inside a flat buffer with four NaN floats on each side."""
    numel = math.prod(shape)
    buf = torch.full((numel + 8,), NAN, device=DEV)
    buf[4:4 + numel] = torch.randn(numel, device=DEV, generator=gen)
    return buf, buf[4:4 + numel].view(shape)


def _canary_intact(before, after, view):
    """Every float of ``after`` outside ``view`` is bit-identical to ``before``."""
    keep = torch.ones(after.shape, dtype=torch.bool, device=DEV)
    if after.dim() == 2:
        off = (view.data_ptr() - after.data_ptr()) // 4
        keep[:, off:off + view.shape[1]] = False
    else:
        off = (view.data_ptr() - after.data_ptr()) // 4
        keep[off:off + view.numel()] = False
    return torch.equal(before.view(torch.int32)[keep], after.view(torch.int32)[keep])


def _p(t):
    from emernerf_b200 import _ops

    return _ops._ptr(t)


def _call(name, *args):
    from emernerf_b200 import _lib, _ops

    _ops._need_cuda(torch.empty(0, device=DEV))
    _lib.call(name, *args, _ops._stream())


def _act64(z, act):
    return torch.relu(z) if act == RELU else torch.sigmoid(z) if act == SIGMOID else z


def _dz64(dy, y, act):
    """dY * act'(Y), the derivative through the stored output as the kernels take it."""
    dy, y = dy.double(), y.double()
    return dy * (y > 0) if act == RELU else dy * (y * (1.0 - y)) if act == SIGMOID else dy


def _stored_output(n, cols, act, gen):
    """What a layer with activation ``act`` stores: ReLU outputs with about half exact zeros, sigmoid outputs in (0, 1)."""
    z = torch.randn(n, cols, device=DEV, generator=gen)
    return torch.relu(z) if act == RELU else torch.sigmoid(z) if act == SIGMOID else z


def ref_fwd(x, w, b, act):
    """Y = act(X W^T + b)."""
    z = x.double() @ w.double().T
    return _act64(z if b is None else z + b.double(), act)


def ref_bwd_data(dy, y, act, w, relu_src=None, relu_cols=0, dx0=None):
    """dX = (dY * act'(Y)) W, then dX[:, :relu_cols] *= (relu_src > 0), added to dX0 when accumulating."""
    dx = _dz64(dy, y, act) @ w.double()
    if relu_src is not None and relu_cols:
        dx[:, :relu_cols] *= (relu_src[:, :relu_cols] > 0).double()
    return dx if dx0 is None else dx0.double() + dx


def ref_bwd_weight(x, dz, dw0, db0):
    """dW += dZ^T X, db += column sums of dZ."""
    dz = dz.double()
    return dw0.double() + dz.T @ x.double(), None if db0 is None else db0.double() + dz.sum(0)


ERRORS = {}


def _record(family, err, tol):
    ERRORS[family] = max(ERRORS.get(family, 0.0), err)
    print(f"maxerr {family} {err:.2e} (bar {tol:.0e})")
    assert err < tol, (family, err, tol)


def _ids(rows):
    return [f"n{n}" for n in rows]


# ============================================================================ tensor-core layers
@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("k,n_out,act", TC_FWD)
def test_tc_forward(k, n_out, act, n):
    g = torch.Generator(device=DEV).manual_seed(k * 1000 + n_out + n)
    xb, x = _operand(n, k, k + 12, 4, g)
    w = torch.randn(n_out, k, device=DEV, generator=g) / k ** 0.5
    b = torch.randn(n_out, device=DEV, generator=g)
    yb, y = _operand(n, n_out, n_out + 9, 4, g, fill=NAN)
    y0 = yb.clone()
    _call("emer_linear_tc_fwd", _p(x), xb.shape[1], _p(w), _p(b), _p(y), yb.shape[1], n, k,
                                     n_out, act)
    assert _canary_intact(y0, yb, y)
    _record(f"tc_fwd_NB{tc_nb(n_out)}", rel_err(y, ref_fwd(x, w, b, act)), 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("k,n_out,act,relu_cols,accumulate", TC_BWD)
def test_tc_backward_data(k, n_out, act, relu_cols, accumulate, n):
    g = torch.Generator(device=DEV).manual_seed(k * 1000 + n_out + n + 7)
    dyb, dy = _operand(n, n_out, n_out + 8, 4, g)
    yb, y = _operand(n, n_out, n_out + 4, 0, g, fill=_stored_output(n, n_out, act, g)) if act else (None, None)
    w = torch.randn(n_out, k, device=DEV, generator=g) / n_out ** 0.5
    rb, relu_src = _operand(n, k, k + 3, 1, g) if relu_cols else (None, None)
    if relu_cols:
        relu_src[:, ::5] = 0.0                                  # exact zeros: masked (the test is > 0)
    dxb, dx = _operand(n, k, k + 8, 4, g, fill=None if accumulate else NAN)
    dx0, dxb0 = dx.clone(), dxb.clone()
    _call(
        "emer_linear_tc_bwd_data", _p(dy), dyb.shape[1], _p(y), 0 if yb is None else yb.shape[1], act, _p(w), _p(dx),
        dxb.shape[1], _p(relu_src), 0 if rb is None else rb.shape[1], relu_cols, n, k, n_out, accumulate)
    assert _canary_intact(dxb0, dxb, dx)
    want = ref_bwd_data(dy, y if act else dy, act, w, relu_src, relu_cols, dx0 if accumulate else None)
    _record(f"tc_bwd_data_NB{tc_nb(k)}", rel_err(dx, want), 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("np_,mb,k,n_out", WGRAD)
def test_tc_weight_gradient_instantiations(np_, mb, k, n_out, n):
    """emer_linear_tc_bwd_weight in each wgrad_kernel<NP, MB>: 16-byte-aligned strided X and dZ (NaN between the rows'
    columns), dW and db accumulated onto non-zero values inside NaN guards."""
    g = torch.Generator(device=DEV).manual_seed(np_ * 100 + mb * 10 + n)
    ldx, lddz = 4 + (k + 3) // 4 * 4 + 4, 4 + (n_out + 3) // 4 * 4
    xb, x = _operand(n, k, ldx, 4, g)
    zb, dz = _operand(n, n_out, lddz, 4, g)
    dwb, dw = _flat((n_out, k), g)
    dbb, db = _flat((n_out,), g)
    dw0, db0, dwb0, dbb0 = dw.clone(), db.clone(), dwb.clone(), dbb.clone()
    _call("emer_linear_tc_bwd_weight", _p(x), ldx, _p(dz), lddz, _p(dw), _p(db), n, k, n_out)
    assert _canary_intact(dwb0, dwb, dw) and _canary_intact(dbb0, dbb, db)
    want_w, want_b = ref_bwd_weight(x, dz, dw0, db0)
    _record(f"tc_wgrad_NP{np_}", rel_err(dw, want_w), _tol(n))
    _record(f"tc_wgrad_db_NP{np_}", rel_err(db, want_b), _tol(n))


# ============================================================================ narrow layers (n_out <= 8)
@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("k,n_out,act,x_off,ldx,path", NARROW_FWD)
def test_narrow_forward(k, n_out, act, x_off, ldx, path, n):
    g = torch.Generator(device=DEV).manual_seed(k * 31 + n_out + n)
    xb, x = _operand(n, k, ldx, x_off, g)
    w = torch.randn(n_out, k, device=DEV, generator=g) / k ** 0.5
    b = torch.randn(n_out, device=DEV, generator=g)
    yb, y = _operand(n, n_out, n_out + 5, 2, g, fill=NAN)
    y0 = yb.clone()
    _call("emer_linear_narrow_fwd", _p(x), ldx, _p(w), _p(b), _p(y), yb.shape[1], n, k, n_out,
                                     act)
    assert _canary_intact(y0, yb, y)
    _record(f"narrow_fwd_{path}", rel_err(y, ref_fwd(x, w, b, act)), 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("k,n_out,relu_cols,dx_off,lddx,store", NARROW_DATA)
def test_narrow_backward_data(k, n_out, relu_cols, dx_off, lddx, store, n):
    """dX of a narrow layer writes columns [0, k) of its rows and nothing else: with k % 4 != 0 the last 16-byte group
    is stored column by column (the columns behind k belong to the caller)."""
    g = torch.Generator(device=DEV).manual_seed(k * 31 + n_out + n + 3)
    dzb, dz = _operand(n, n_out, n_out + 3, 1, g)
    w = torch.randn(n_out, k, device=DEV, generator=g)
    rb, relu_src = _operand(n, k, k + 2, 2, g) if relu_cols else (None, None)
    if relu_cols:
        relu_src[:, ::3] = 0.0
    dxb, dx = _operand(n, k, lddx, dx_off, g, fill=NAN)
    dxb0 = dxb.clone()
    _call("emer_linear_narrow_bwd_data", _p(dz), dzb.shape[1], _p(w), _p(dx), lddx,
                                     _p(relu_src), 0 if rb is None else rb.shape[1], relu_cols, n, k, n_out)
    assert _canary_intact(dxb0, dxb, dx), "wrote outside columns [0, k)"
    _record(f"narrow_bwd_data_{store}", rel_err(dx, ref_bwd_data(dz, dz, NONE, w, relu_src, relu_cols)), 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("k,n_out,x_off,ldx,dz_off,lddz,bias", NARROW_WGRAD)
def test_narrow_weight_gradient_instantiations(k, n_out, x_off, ldx, dz_off, lddz, bias, n):
    g = torch.Generator(device=DEV).manual_seed(k * 31 + n_out + n + 5)
    xb, x = _operand(n, k, ldx, x_off, g)
    zb, dz = _operand(n, n_out, lddz, dz_off, g)
    dwb, dw = _flat((n_out, k), g)
    dbb, db = _flat((n_out,), g) if bias else (None, None)
    dw0, dwb0 = dw.clone(), dwb.clone()
    db0, dbb0 = (db.clone(), dbb.clone()) if bias else (None, None)
    want_key = narrow_wgrad_key(k, n_out, x_off, ldx, dz_off, lddz)
    _call("emer_linear_narrow_bwd_weight", _p(x), ldx, _p(dz), lddz, _p(dw), _p(db), n, k,
                                     n_out)
    assert _canary_intact(dwb0, dwb, dw) and (not bias or _canary_intact(dbb0, dbb, db))
    want_w, want_b = ref_bwd_weight(x, dz, dw0, db0)
    fam = want_key.split("::")[-1].replace(",", "_")
    _record(f"{fam}_dW", rel_err(dw, want_w), _tol(n))
    if bias:
        _record(f"{fam}_db", rel_err(db, want_b), _tol(n))


# ============================================================================ FP32-FMA layers
@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("k,n_out,act", SIMT_FWD)
def test_simt_forward(k, n_out, act, n):
    g = torch.Generator(device=DEV).manual_seed(k + n_out * 7 + n)
    xb, x = _operand(n, k, k + 5, 3, g)
    w = torch.randn(n_out, k, device=DEV, generator=g) / k ** 0.5
    b = torch.randn(n_out, device=DEV, generator=g)
    yb, y = _operand(n, n_out, n_out + 6, 2, g, fill=NAN)
    y0 = yb.clone()
    _call("emer_linear_fwd", _p(x), xb.shape[1], _p(w), _p(b), _p(y), yb.shape[1], n, k, n_out,
                                     act)
    assert _canary_intact(y0, yb, y)
    _record("gemm_rows_fwd", rel_err(y, ref_fwd(x, w, b, act)), 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("k,n_out,act,accumulate", SIMT_DATA)
def test_simt_backward_data(k, n_out, act, accumulate, n):
    g = torch.Generator(device=DEV).manual_seed(k + n_out * 7 + n + 1)
    dyb, dy = _operand(n, n_out, n_out + 4, 1, g)
    yb, y = _operand(n, n_out, n_out + 2, 2, g, fill=_stored_output(n, n_out, act, g)) if act else (None, None)
    w = torch.randn(n_out, k, device=DEV, generator=g) / n_out ** 0.5
    dxb, dx = _operand(n, k, k + 7, 3, g, fill=None if accumulate else NAN)
    dx0, dxb0 = dx.clone(), dxb.clone()
    _call("emer_linear_bwd_data", _p(dy), dyb.shape[1], _p(y), 0 if yb is None else yb.shape[1],
                                     act, _p(w), _p(dx), dxb.shape[1], n, k, n_out, accumulate)
    assert _canary_intact(dxb0, dxb, dx)
    want = ref_bwd_data(dy, y if act else dy, act, w, dx0=dx0 if accumulate else None)
    _record("gemm_rows_bwd_data", rel_err(dx, want), 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS, ids=_ids(ROWS))
@pytest.mark.parametrize("k,n_out,act,bias", SIMT_WGRAD)
def test_simt_weight_gradient(k, n_out, act, bias, n):
    """emer_linear_bwd_weight with the activation derivative applied to dY through the stored output."""
    g = torch.Generator(device=DEV).manual_seed(k + n_out * 7 + n + 2)
    xb, x = _operand(n, k, k + 3, 1, g)
    dyb, dy = _operand(n, n_out, n_out + 2, 2, g)
    yb, y = _operand(n, n_out, n_out + 1, 1, g, fill=_stored_output(n, n_out, act, g)) if act else (None, None)
    dwb, dw = _flat((n_out, k), g)
    dbb, db = _flat((n_out,), g) if bias else (None, None)
    dw0, dwb0 = dw.clone(), dwb.clone()
    db0, dbb0 = (db.clone(), dbb.clone()) if bias else (None, None)
    _call("emer_linear_bwd_weight", _p(x), xb.shape[1], _p(dy), dyb.shape[1], _p(y),
                                     0 if yb is None else yb.shape[1], act, _p(dw), _p(db), n, k, n_out)
    assert _canary_intact(dwb0, dwb, dw) and (not bias or _canary_intact(dbb0, dbb, db))
    want_w, want_b = ref_bwd_weight(x, _dz64(dy, y if act else dy, act), dw0, db0)
    _record("simt_wgrad_dW", rel_err(dw, want_w), _tol(n))
    if bias:
        _record("simt_wgrad_db", rel_err(db, want_b), _tol(n))


# ============================================================================ dispatch boundaries of _ops
F_TC, F_SIMT, F_NAR = "emer_linear_tc_fwd", "emer_linear_fwd", "emer_linear_narrow_fwd"
D_TC, D_SIMT, D_NAR = "emer_linear_tc_bwd_data", "emer_linear_bwd_data", "emer_linear_narrow_bwd_data"
W_TC, W_SIMT, W_NAR = "emer_linear_tc_bwd_weight", "emer_linear_bwd_weight", "emer_linear_narrow_bwd_weight"
BOUNDARIES = [  # id, rows (0 = TC_MIN_ROWS, -1 = one below), k, n_out, X layout, (forward, data, weight gradient)
    ("rows_below_tc", -1, 64, 64, "dense", (F_SIMT, D_SIMT, W_SIMT)),
    ("rows_at_tc", 0, 64, 64, "dense", (F_TC, D_TC, W_TC)),
    ("n_out_8_narrow", 37, 64, 8, "dense", (F_NAR, D_NAR, W_NAR)),
    ("n_out_9_tc", 37, 64, 9, "dense", (F_TC, D_TC, W_SIMT)),           # n_out % 4 != 0: FFMA weight gradient
    ("n_out_12_tc", 37, 64, 12, "dense", (F_TC, D_TC, W_TC)),
    ("k_256_narrow", 37, 256, 4, "dense", (F_NAR, D_NAR, W_NAR)),
    ("k_257_narrow_out", 37, 257, 4, "dense", (F_TC, D_SIMT, W_SIMT)),   # data gradient 272 columns wide > one MMA
    ("k_256_wide", 37, 256, 64, "dense", (F_TC, D_TC, W_TC)),
    ("k_257_wide", 37, 257, 64, "dense", (F_TC, D_SIMT, W_SIMT)),
    ("n_out_128", 37, 64, 128, "dense", (F_TC, D_TC, W_TC)),
    ("n_out_132", 37, 64, 132, "dense", (F_TC, D_TC, W_SIMT)),           # n_out > 128: no tc weight gradient
    ("n_out_256", 37, 96, 256, "dense", (F_TC, D_TC, W_SIMT)),           # n_pad 256, panels 193 KB
    ("n_out_257", 37, 64, 257, "dense", (F_SIMT, D_TC, W_SIMT)),         # n_out > 256
    ("panels_overflow", 37, 97, 256, "dense", (F_SIMT, D_TC, W_SIMT)),   # forward panels 257 KB > 227 KB
    ("x_misaligned", 37, 64, 64, "offset1", (F_TC, D_TC, W_SIMT)),
    ("x_rows_unpadded", 37, 30, 64, "dense", (F_TC, D_TC, W_SIMT)),      # ldx = 30 < pad4(k) = 32
    ("x_rows_padded", 37, 30, 64, "pad4", (F_TC, D_TC, W_TC)),           # ldx = 32
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", BOUNDARIES, ids=[b[0] for b in BOUNDARIES])
def test_linear_dispatch_boundaries(case):
    """_ops.linear on each side of a dispatch boundary: the entry points it launches, and Y, dX, dW, db against fp64."""
    from emernerf_b200 import _lib, _ops

    _, rows, k, n_out, layout, (want_f, want_d, want_w) = case
    n = _ops.TC_MIN_ROWS + rows
    g = torch.Generator(device=DEV).manual_seed(k * 7 + n_out)
    pad = {"dense": 0, "offset1": 8, "pad4": (k + 3) // 4 * 4 - k}[layout]
    base = torch.randn(n, k + pad, device=DEV, generator=g).requires_grad_(True)
    x = base[:, 1:1 + k] if layout == "offset1" else base[:, :k]
    w = (torch.randn(n_out, k, device=DEV, generator=g) / k ** 0.5).requires_grad_(True)
    b = torch.randn(n_out, device=DEV, generator=g).requires_grad_(True)
    dy = torch.randn(n, n_out, device=DEV, generator=g)
    rec = []
    _lib.set_profile(lambda name, args: name.startswith("emer_linear"), rec)
    try:
        y = _ops.linear(x, w, b, NONE)
        fwd = [r[0] for r in rec]
        y.backward(dy)
        bwd = sorted(r[0] for r in rec[len(fwd):])
    finally:
        _lib.set_profile(None, None)
    assert fwd == [want_f] and bwd == sorted([want_d, want_w]), (fwd, bwd)
    x64, w64, b64 = (t.detach().double().requires_grad_(True) for t in (base, w, b))
    xs64 = x64[:, 1:1 + k] if layout == "offset1" else x64[:, :k]
    y64 = xs64 @ w64.T + b64
    y64.backward(dy.double())
    _record("dispatch_y", rel_err(y, y64), 2e-5)
    _record("dispatch_dx", rel_err(base.grad, x64.grad), 2e-5)
    _record("dispatch_dw", rel_err(w.grad, w64.grad), 2e-5)
    _record("dispatch_db", rel_err(b.grad, b64.grad), 2e-5)


CHAINS = [  # id, rows, widths, entry points launched
    ("tc_hidden_narrow_head", 37, (40, 64, 5), {F_TC, F_NAR, D_NAR, W_NAR, D_TC, W_TC}),
    ("tc_hidden_tc_head", 37, (40, 64, 9), {F_TC, D_TC, W_TC, W_SIMT}),
    ("below_tc_rows", -1, (40, 64, 9), {F_SIMT, D_SIMT, W_SIMT}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CHAINS, ids=[c[0] for c in CHAINS])
def test_mlp_chain_dispatch(case):
    """A two-layer ReLU head through _ops.mlp_chain: the hidden layer's ReLU mask reaches dX through the data-gradient
    kernel's epilogue (narrow, tc) or the separate mask (FFMA).  The fp64 side uses the kernel's own mask (a
    pre-activation within rounding distance of zero may take the other subgradient)."""
    from emernerf_b200 import _lib, _ops

    _, rows, (k0, h, n_out), want = case
    n = _ops.TC_MIN_ROWS + rows
    g = torch.Generator(device=DEV).manual_seed(n_out + rows)
    x = torch.randn(n, k0, device=DEV, generator=g).requires_grad_(True)
    ws = [(torch.randn(h, k0, device=DEV, generator=g) / k0 ** 0.5).requires_grad_(True),
          (torch.randn(n_out, h, device=DEV, generator=g) / h ** 0.5).requires_grad_(True)]
    bs = [torch.randn(h, device=DEV, generator=g).requires_grad_(True),
          torch.randn(n_out, device=DEV, generator=g).requires_grad_(True)]
    dy = torch.randn(n, n_out, device=DEV, generator=g)
    rec = []
    _lib.set_profile(lambda name, args: name.startswith("emer_linear"), rec)
    try:
        y = _ops.mlp_chain(x, ws, bs, NONE)
        hidden = y.grad_fn.saved_tensors[1].detach().clone()
        y.backward(dy)
    finally:
        _lib.set_profile(None, None)
    assert {r[0] for r in rec} == want, {r[0] for r in rec}
    leaves = [t.detach().double().requires_grad_(True) for t in [x] + ws + bs]
    x64, w0, w1, b0, b1 = leaves
    h64 = (x64 @ w0.T + b0) * (hidden > 0).double()
    y64 = h64 @ w1.T + b1
    y64.backward(dy.double())
    _record("chain_y", rel_err(y, y64), 2e-5)
    for got, want64 in zip([x] + ws + bs, leaves):
        _record("chain_grads", rel_err(got.grad, want64.grad), 2e-5)


# ============================================================================ hash grid, proposal level, accumulation
@pytest.mark.gpu
@pytest.mark.parametrize("n", (1, 3001))
@pytest.mark.parametrize("D,F", list(GRID_CASES))
def test_grid_instantiations_vs_oracle(D, F, n):
    """grid_fwd / grid_bwd_table / grid_bwd_dx <D, F> against tcnn_ref, as test_gpu_kernels.py's grid test."""
    from emernerf_b200 import _ops
    from emernerf_b200.grid_desc import GridDesc
    from oracle import hotpath, tcnn_ref

    cfg = hotpath.hash_encoder_config(*GRID_CASES[(D, F)])
    desc, geom = GridDesc(D, cfg), tcnn_ref.grid_geometry(D, cfg)
    g = torch.Generator().manual_seed(D * 10 + F + n)
    x = torch.rand(n, D, generator=g)
    x[: n // 8] = torch.rand(n // 8, D, generator=g).round()          # exact cell corners 0 / 1
    params = torch.randn(geom.n_params, generator=g)
    dy = torch.randn(n, geom.n_output_dims, generator=g)
    xo, po = x.clone().requires_grad_(True), params.clone().requires_grad_(True)
    yo = tcnn_ref.grid_forward(xo, po, geom)
    yo.backward(dy)
    xg, pg = x.to(DEV).requires_grad_(True), params.to(DEV).requires_grad_(True)

    def run():
        yg = _ops.grid_encode(xg, pg, desc)
        yg.backward(dy.to(DEV))
        return yg

    yg = run()
    assert (yg.detach().cpu() - yo).abs().max().item() <= 1e-6 * yo.abs().max().item()
    _record(f"grid_{D}d_f{F}_table_grad", rel_err(pg.grad, po.grad), 2e-5)
    _record(f"grid_{D}d_f{F}_x_grad", rel_err(xg.grad, xo.grad), 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("levels,feats,prev,n", PROP_CASES)
def test_prop_level_instantiations_vs_oracle(levels, feats, prev, n):
    """emer_prop_level in each prop_level_kernel<LF> (<0>: the generic loops, e.g. 4 levels x 2 features) against the
    oracle: s / t edges bit-exact, the CDF within 2e-5, as test_fused_proposal_level_vs_oracle.  A "real" previous level
    is this network's own 128-interval output -- m1 = 129 edges with a non-uniform CDF, as the benchmark's second
    level -- and n = 256 fills PL_MAX_EDGES = 257."""
    from emernerf_b200 import _ops
    from emernerf_b200.radiance_fields import build_density_field
    from oracle import adapters, hotpath
    from oracle import nerfacc_ref as nf

    torch.manual_seed(levels * 10 + feats)
    net = build_density_field(n_input_dims=3, n_levels=levels, max_resolution=96 if levels == 4 else 512,
                              log2_hashmap_size=12 if levels == 4 else 15, n_features_per_level=feats, unbounded=True)
    net.set_aabb([-20.0, -20.0, -5.0, 20.0, 20.0, 10.0])
    gen = torch.Generator().manual_seed(n + levels)
    with torch.no_grad():
        p = net.xyz_encoder.tcnn_encoding.params
        p.copy_(torch.randn(p.shape, generator=gen) * 0.5)
    R = 300
    origins = torch.randn(R, 3, generator=gen) * 2.0
    dirs = torch.randn(R, 3, generator=gen)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    jit = torch.rand(R, 1, generator=gen)
    s_min, s_max = hotpath.s_bounds("uniform_lindisp", 0.1, 1000.0)
    net = net.to(DEV)
    lin = [m for m in net.base_mlp if isinstance(m, torch.nn.Linear)]
    rest = (origins.to(DEV), dirs.to(DEV), net.aabb, True, net.xyz_encoder.desc, net.xyz_encoder.tcnn_encoding.params,
            lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias)
    prev_s = torch.tensor([[0.0, 1.0]]).repeat(R, 1)
    prev_cdf = prev_s.clone()
    if prev == "real":
        s1, _, c1 = _ops.prop_level(prev_s.to(DEV), prev_cdf.to(DEV), 128, jit.to(DEV), s_min, s_max,
                                    "uniform_lindisp", *rest)
        prev_s, prev_cdf = s1.cpu(), c1.cpu()
        assert prev_s.shape[1] == 129 and not torch.equal(prev_cdf, prev_s)
    (s_got, t_got, cdf_got) = _ops.prop_level(
        prev_s.to(DEV), prev_cdf.to(DEV), n, jit.to(DEV), s_min, s_max, "uniform_lindisp", *rest)

    iv, _ = nf.importance_sampling(nf.RayIntervals(prev_s), prev_cdf, n, True, jitter=jit)
    t = hotpath._s_to_t("uniform_lindisp", iv.vals, 0.1, 1000.0)
    pos = origins[:, None, :] + dirs[:, None, :] * (t[:, :-1] + t[:, 1:])[..., None] / 2.0
    sd = adapters.cpu_state_dict(net)
    sig = hotpath.density_field_forward(sd, adapters.spec_from_module(net), pos)["density"].squeeze(-1)
    trans, _ = nf.render_transmittance_from_density(t[:, :-1], t[:, 1:], sig)
    cdf_want = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], -1)
    assert torch.equal(s_got.cpu(), iv.vals) and torch.equal(t_got.cpu(), t)
    assert torch.equal(cdf_got[:, -1].cpu(), torch.ones(R))
    _record(f"prop_level_{prop_key(levels, feats).split('<')[1][:-1]}_cdf", rel_err(cdf_got, cdf_want), 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("C", ACC_CHANNELS)
def test_accumulate_small_channel_instantiations(C):
    """accumulate_small_fwd_kernel<C> (sum_s w[r, s] v[r, s, c] for C <= 4) against fp64."""
    from emernerf_b200 import _ops

    g = torch.Generator(device=DEV).manual_seed(C)
    w = torch.rand(257, 64, device=DEV, generator=g)
    v = torch.randn(257, 64, C, device=DEV, generator=g)
    out = _ops.accumulate(w, v)
    _record("accumulate_small", rel_err(out, (w.double()[..., None] * v.double()).sum(1)), 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("k_enc,n_feat", FIELD_FWD)
def test_field_forward_instantiations(k_enc, n_feat):
    """field_fwd_kernel<k_enc, n_feat> under no_grad (inference: no saved activations) against test_gpu_kernels.py's
    fp64 restatement of the chain, ragged last tile and last ray."""
    from emernerf_b200 import _ops
    from test_gpu_kernels import _chain_reference

    gen = torch.Generator().manual_seed(k_enc + n_feat)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=gen) * scale).to(DEV)
    n, S, c = 64 * 300 + 37, 64, 49
    enc, rb = rnd(n, k_enc, scale=0.5), rnd((n + S - 1) // S, 128, scale=0.3)
    ws = [rnd(64, k_enc, scale=0.2), rnd(64, scale=0.1), rnd(n_feat, 64, scale=0.15), rnd(n_feat, scale=0.1),
          rnd(64, 64 + c, scale=0.12), rnd(64, 128 + c, scale=0.1), rnd(3, 64, scale=0.2), rnd(3, scale=0.1)]
    with torch.no_grad():
        (sigma, rgb, geo, sem) = _ops.field_chain(enc, rb, S, ws[:4], ws[4:], want_geo=True)
    want = _chain_reference(enc, rb, S, *ws, c)
    _record("field_fwd", max(rel_err(sigma, want[0]), rel_err(rgb, want[1]), rel_err(geo, want[2]),
                             rel_err(sem, want[3]) if n_feat == 128 else 0.0), 2e-5)
    assert (sem is None) == (n_feat == 64)
