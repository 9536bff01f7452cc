"""torch.autograd wrappers over the C ABI (include/emer_b200.h).

Mirrors the calling conventions of the reference's binding shim
(third_party/tcnn_modules.py:115-208,235-263): inputs are cast to fp32 and made contiguous here,
``ctx.set_materialize_grads(False)``, ``None`` gradients for inputs that do not need one.  All
tensors must live on a CUDA device -- there is no CPU path.
"""
from __future__ import annotations

import ctypes
import math
import weakref
from typing import Callable, Dict, Optional, Sequence, Tuple

import torch
from torch import Tensor

from . import _lib
from .grid_desc import GridDesc

import os

ACT_NONE, ACT_RELU, ACT_SIGMOID = 0, 1, 2
# Dense layers run on the wgmma tensor-core kernels (3xTF32, fp32-accurate).  "simt" selects the
# fp32 CUDA-core kernels of linear_simt.cu (the bit-faithful checker); both are sm_90a code in the
# same library -- this is a debugging switch, not a backend dispatch.
LINEAR_IMPL = os.environ.get("EMER_LINEAR", "tc")
LINEAR_WGRAD_IMPL = os.environ.get("EMER_LINEAR_WGRAD", "tc")      # "simt": the FFMA weight gradient; anything else: the
                                                                   # tensor-core one (csrc/wgrad_mn.cu)
SKIP_BWD_IMPL = os.environ.get("EMER_SKIP_BWD", "stack")   # "stack": one stacked product; "add": two + add
TC_MIN_ROWS = int(os.environ.get("EMER_TC_MIN_ROWS", "1024"))   # below: the FP32-FMA kernels (tiny per-ray heads are launch-bound either way)
STOT_KINDS = {"uniform": 0, "lindisp": 1, "sqrt": 2, "log": 3, "uniform_lindisp": 4, "uniform_lindisp_0": 5}


def _stream() -> ctypes.c_void_p:
    """torch's current stream ON THE DEVICE OF THE OP'S TENSORS (see _need_cuda / _lib.DEVICE)."""
    return ctypes.c_void_p(torch.cuda.current_stream(_lib.DEVICE).cuda_stream)


def _ptr(t: Optional[Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def on_device(t: Tensor) -> bool:
    """Whether ``t`` lives where the kernels run.  The fused-path selectors ask through this one predicate (the
    CPU harness of tests/cabi_emulator.py answers for them; the product has no CPU path, see _need_cuda)."""
    return t.is_cuda


def _need_cuda(*ts: Tensor) -> None:
    """Every forward op starts here: all tensors on ONE CUDA device, which becomes the device the launch (and its
    stream lookup) is guarded to -- a model on cuda:1 works while the current device is cuda:0.  (Backward nodes run
    under autograd's own device guard.)"""
    dev = None
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("emernerf_b200 ops need CUDA tensors (there is no CPU fallback)")
        if dev is None:
            dev = t.device.index
        elif t.device.index != dev:
            raise RuntimeError(f"emernerf_b200 op got tensors on cuda:{dev} and cuda:{t.device.index}")
    if dev is not None:
        _lib.DEVICE = dev


# ----------------------------------------------------------------------------- gradient sinks
# ``emernerf_b200.optim.FusedAdam`` owns one persistent, pre-zeroed flat gradient buffer per parameter group and
# registers every parameter's slice here.  A library backward that produces a parameter gradient looks its parameter
# up (by storage address) and ACCUMULATES into the slice -- the scatter / weight-gradient kernels add with atomics anyway
# -- instead of allocating and zero-filling a fresh tensor that autograd would then copy or add: for the 122 MB hash
# table that is a 122 MB memset per backward.  It returns None for that input (autograd has nothing left to do) and
# tells the optimizer the parameter was touched.  Without a registered sink (the reference's own torch.optim.Adam) the
# ordinary autograd path runs.
_GRAD_SINKS: Dict[int, Tuple[Tensor, Callable, "weakref.ref"]] = {}


def register_grad_sink(param: Tensor, sink: Tensor, on_touch: Callable) -> None:
    if sink.shape != param.shape or sink.dtype != torch.float32 or not sink.is_contiguous():
        raise ValueError("grad sink must be a contiguous fp32 tensor of the parameter's shape")
    _GRAD_SINKS[param.data_ptr()] = (sink, on_touch, weakref.ref(param))


def clear_grad_sinks() -> None:
    _GRAD_SINKS.clear()


def _grad_sink(t: Optional[Tensor]):
    """(sink, touch) for a registered parameter's storage, else None."""
    if t is None or not _GRAD_SINKS:
        return None
    e = _GRAD_SINKS.get(t.data_ptr())
    if e is None:
        return None
    sink, on_touch, ref = e
    p = ref()
    if p is None or p.data_ptr() != t.data_ptr() or sink.shape != t.shape:
        return None
    touched = getattr(on_touch, "__self__", None)
    is_touched = (lambda: id(p) in touched._touched) if hasattr(touched, "_touched") else None
    return sink, (lambda: on_touch(p)), is_touched


# ----------------------------------------------------------------------------- weight gradients on a side stream
# (EMER_WGRAD_STREAM=0 turns it off.)  With FusedAdam's gradient sinks the fused chain's weight-gradient kernels run on a side stream, forked where the dZ buffers are
# complete.  The main stream goes on to the hash-grid scatter and -- multi-GPU -- to the reduce-scatter of the table
# gradients, which no weight gradient feeds; the optimizer (or the reduction of the MLP gradients) joins the side stream
# first (:func:`join_side_streams`).  Captured into the step's CUDA graph this becomes two parallel branches.
WGRAD_STREAM = os.environ.get("EMER_WGRAD_STREAM", "1") == "1"
# proposal levels on the steps that update the proposal networks: "fused" = emer_prop_level + emer_prop_level_bwd,
# "layers" = the modular autograd path (contract, grid, two layers, trunc_exp, composite)
PROP_TRAIN = os.environ.get("EMER_PROP_TRAIN", "fused")
_SIDE: Dict[int, "torch.cuda.Stream"] = {}
_PENDING: Dict[int, bool] = {}
_AFTER_JOIN: list = []          # small updates of buffers the main stream also writes: run there, after the join


class _on_side_stream:
    """Context: launch on the device's side stream after everything enqueued so far on the current stream; tensors
    listed are marked as used there (the caching allocator must not hand their memory out early)."""

    def __init__(self, device, *tensors):
        self.dev, self.tensors = device, [t for t in tensors if t is not None]

    def __enter__(self):
        idx = self.dev.index
        if idx not in _SIDE:
            _SIDE[idx] = torch.cuda.Stream(device=self.dev)
        side, main = _SIDE[idx], torch.cuda.current_stream(self.dev)
        side.wait_stream(main)
        for t in self.tensors:
            t.record_stream(side)
        _PENDING[idx] = True
        self.ctx = torch.cuda.stream(side)
        self.ctx.__enter__()
        return side

    def __exit__(self, *exc):
        return self.ctx.__exit__(*exc)


_BEFORE_FIELD: list = []        # streams whose work the field forward needs (a deferred parameter all-gather)


def join_before_field() -> None:
    """Called by RadianceField.forward: the current stream waits for work that only the FIELD's parameters depend on
    (DataParallel's deferred all-gather runs beside the proposal sampling of the next step)."""
    while _BEFORE_FIELD:
        torch.cuda.current_stream().wait_stream(_BEFORE_FIELD.pop())


def join_side_streams() -> None:
    """The current stream waits for weight gradients still running on a side stream (no-op when there are none)."""
    for idx, pending in list(_PENDING.items()):
        if pending:
            torch.cuda.current_stream(idx).wait_stream(_SIDE[idx])
            _PENDING[idx] = False
    while _AFTER_JOIN:
        _AFTER_JOIN.pop(0)()


def _f32c(t: Tensor) -> Tensor:
    if t.dtype != torch.float32:
        t = t.to(torch.float32)
    return t if t.is_contiguous() else t.contiguous()


def _rows(t: Tensor, k: int) -> Tuple[Tensor, int]:
    """View as [N, k] rows with unit inner stride; returns (2-D tensor, row stride)."""
    t2 = t.reshape(-1, k)
    if t2.dtype != torch.float32:
        t2 = t2.to(torch.float32)
    if t2.stride(1) != 1 or (t2.shape[0] > 1 and t2.stride(0) < k):
        t2 = t2.contiguous()
    return t2, (t2.stride(0) if t2.shape[0] > 1 else k)


# ----------------------------------------------------------------------------- hash grid
class _GridEncode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, params: Tensor, desc: GridDesc):
        ctx.set_materialize_grads(False)
        _need_cuda(x, params)
        x = _f32c(x)
        params = _f32c(params)
        n = x.shape[0]
        y = torch.empty((n, desc.n_output_dims), dtype=torch.float32, device=x.device)
        _lib.call("emer_grid_fwd", ctypes.byref(desc.c), _ptr(x), _ptr(params), _ptr(y), n, _stream())
        ctx.save_for_backward(x, params)
        ctx.desc = desc
        return y

    @staticmethod
    def backward(ctx, dy):
        if dy is None:
            return None, None, None
        x, params = ctx.saved_tensors
        desc = ctx.desc
        dy = _f32c(dy)
        need_x, need_p = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        sink = _grad_sink(params) if need_p else None
        if sink is not None:
            dparams = sink[0]                     # the optimizer's pre-zeroed slice: scatter straight into it
        else:
            dparams = torch.zeros_like(params) if need_p else None
        dx = torch.empty_like(x) if need_x else None
        if need_x or need_p:
            _lib.call("emer_grid_bwd", ctypes.byref(desc.c), _ptr(x), _ptr(params), _ptr(dy), _ptr(dparams),
                      _ptr(dx), x.shape[0], _stream())
        if sink is not None:
            sink[1]()
            dparams = None
        return dx, dparams, None


def grid_encode(x: Tensor, params: Tensor, desc: GridDesc) -> Tensor:
    """[N, D] -> [N, L*F] multi-resolution hash-grid features."""
    if x.dim() != 2 or x.shape[1] != desc.n_dims:
        raise ValueError(f"grid_encode expects [N, {desc.n_dims}], got {tuple(x.shape)}")
    if params.numel() != desc.n_params:
        raise ValueError(f"grid params have {params.numel()} floats, level table needs {desc.n_params}")
    return _GridEncode.apply(x, params, desc)


@torch.no_grad()
def grid_indices(x: Tensor, desc: GridDesc) -> Tensor:
    _need_cuda(x)
    x = _f32c(x)
    out = torch.empty((x.shape[0], desc.n_levels, 2 ** desc.n_dims), dtype=torch.int32, device=x.device)
    _lib.call("emer_grid_indices", ctypes.byref(desc.c), _ptr(x), _ptr(out), x.shape[0], _stream())
    return out


# ----------------------------------------------------------------------------- contraction
class _Contract(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos: Tensor, aabb: Tensor, time: Optional[Tensor], unbounded: bool, selector: bool = True):
        ctx.set_materialize_grads(False)
        _need_cuda(pos, aabb)
        pos = _f32c(pos)
        aabb = _f32c(aabb.reshape(-1))
        n = pos.shape[0]
        out_dim = 3 if time is None else 4
        ctx.time_shape = None if time is None else time.shape
        if time is not None:
            time = _f32c(time.reshape(-1))
            if time.shape[0] != n:
                raise ValueError("time must have one value per point")
        out = torch.empty((n, out_dim), dtype=torch.float32, device=pos.device)
        _lib.call("emer_contract_fwd", _ptr(pos), _ptr(aabb), _ptr(time), _ptr(out), out_dim, int(unbounded), int(selector),
                  n, _stream())
        ctx.save_for_backward(pos, aabb)
        ctx.out_dim, ctx.unbounded, ctx.selector = out_dim, bool(unbounded), bool(selector)
        return out

    @staticmethod
    def backward(ctx, dout):
        if dout is None:
            return None, None, None, None, None
        pos, aabb = ctx.saved_tensors
        dout = _f32c(dout)
        need_pos = ctx.needs_input_grad[0]
        need_t = ctx.out_dim == 4 and ctx.needs_input_grad[2]
        if not (need_pos or need_t):
            return None, None, None, None, None
        dpos = torch.empty_like(pos)
        dtime = torch.empty(pos.shape[0], dtype=torch.float32, device=pos.device) if need_t else None
        _lib.call("emer_contract_bwd", _ptr(pos), _ptr(aabb), _ptr(dout), _ptr(dpos), _ptr(dtime), ctx.out_dim,
                  int(ctx.unbounded), int(ctx.selector), pos.shape[0], _stream())
        if dtime is not None:
            dtime = dtime.view(ctx.time_shape)
        return (dpos if need_pos else None), None, dtime, None, None


def contract(pos: Tensor, aabb: Tensor, time: Optional[Tensor] = None, unbounded: bool = True) -> Tensor:
    """[N,3] world positions -> [N,3] (or [N,4] with the time column) grid coordinates in [0,1]."""
    return _Contract.apply(pos, aabb, time, unbounded, True)


def contract_raw(pos: Tensor, aabb: Tensor) -> Tensor:
    """The bare inf-norm contraction of nerf_utils.py:13-28 (no in-cube selector)."""
    return _Contract.apply(pos, aabb, None, True, False)


# ----------------------------------------------------------------------------- trunc_exp(x - 1)
class _TruncExpM1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor):
        _need_cuda(x)
        shape = x.shape
        x2 = _f32c(x).reshape(-1)
        y = torch.empty_like(x2)
        _lib.call("emer_trunc_exp_fwd", _ptr(x2), 1, _ptr(y), x2.numel(), _stream())
        ctx.save_for_backward(x2)
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        (x2,) = ctx.saved_tensors
        dy2 = _f32c(dy).reshape(-1)
        dx = torch.empty_like(x2)
        _lib.call("emer_trunc_exp_bwd", _ptr(x2), 1, _ptr(dy2), _ptr(dx), x2.numel(), _stream())
        return dx.view(dy.shape)


def density_activation(x: Tensor) -> Tensor:
    """trunc_exp(x - 1): exp forward, exp(clamp(.,15)) backward (nerf_utils.py:59-75)."""
    return _TruncExpM1.apply(x)


# ----------------------------------------------------------------------------- dense layers
def _pad4(v: int) -> int:
    return (v + 3) // 4 * 4


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


_SMEM_MAX = 227 * 1024


def _tc_fits(kred: int, ncols: int) -> bool:
    """Whether tc_linear_kernel can take a layer with reduction width ``kred`` and output width ``ncols``
    (csrc/linear_tc.cu, launch<>): the output width padded to 16 is at most 256, and the resident hi/lo weight panels
    (reduction width padded to 32) plus the bias fit shared memory.  Wider layers run on the CUDA-core kernels."""
    n_pad, kred_pad = _round_up(ncols, 16), _round_up(kred, 32)
    return n_pad <= 256 and 2 * (kred_pad // 4) * n_pad * 16 + n_pad * 4 <= _SMEM_MAX


def _tc_wgrad_fits(k: int, n_out: int) -> bool:
    """Same for the tensor-core weight gradient (emer_linear_tc_bwd_weight, csrc/wgrad_mn.cu)."""
    return k <= 256 and n_out <= 128


def _tc_rows_ok(n: int) -> bool:
    return LINEAR_IMPL == "tc" and n >= TC_MIN_ROWS


def _aligned(t: Tensor, ld: int) -> bool:
    return ld % 4 == 0 and t.data_ptr() % 16 == 0


def _narrow_ok(k: int, n_out: int) -> bool:
    return LINEAR_IMPL != "simt" and n_out <= 8 and k <= 256


def _layer_fwd(x2: Tensor, ldx: int, w: Tensor, b: Optional[Tensor], y: Tensor, ldy: int, n: int, act: int) -> None:
    n_out, k = w.shape
    if _narrow_ok(k, n_out):
        _lib.call("emer_linear_narrow_fwd", _ptr(x2), ldx, _ptr(w), _ptr(b), _ptr(y), ldy, n, k, n_out, act, _stream())
        return
    name = "emer_linear_tc_fwd" if (_tc_rows_ok(n) and _tc_fits(k, n_out)) else "emer_linear_fwd"
    _lib.call(name, _ptr(x2), ldx, _ptr(w), _ptr(b), _ptr(y), ldy, n, k, n_out, act, _stream())


def _layer_bwd_data(dz: Tensor, lddz: int, w: Tensor, dx: Tensor, lddx: int, n: int,
                    relu_src: Optional[Tensor], ld_relu: int, relu_cols: int) -> None:
    """dx[n, k] = dz[n, n_out] @ w, then dx[:, :relu_cols] *= (relu_src > 0) (the dZ of the layer below)."""
    n_out, k = w.shape
    if _narrow_ok(k, n_out):
        _lib.call("emer_linear_narrow_bwd_data", _ptr(dz), lddz, _ptr(w), _ptr(dx), lddx, _ptr(relu_src), ld_relu,
                  relu_cols, n, k, n_out, _stream())
    elif _tc_rows_ok(n) and _tc_fits(n_out, k):
        _lib.call("emer_linear_tc_bwd_data", _ptr(dz), lddz, None, 0, ACT_NONE, _ptr(w), _ptr(dx), lddx,
                  _ptr(relu_src), ld_relu, relu_cols, n, k, n_out, 0, _stream())
    else:
        _lib.call("emer_linear_bwd_data", _ptr(dz), lddz, None, 0, ACT_NONE, _ptr(w), _ptr(dx), lddx, n, k, n_out, 0,
                  _stream())
        if relu_src is not None:
            dx[:, :relu_cols].mul_(relu_src[:, :relu_cols] > 0)


def _layer_bwd_weight(x2: Tensor, ldx: int, dz: Tensor, lddz: int, w: Tensor, has_bias: bool, n: int,
                      w_sink=None, b_sink=None):
    """(dW, db) of one layer.  With gradient sinks (``_grad_sink`` of the weight / bias parameter) the kernels
    accumulate into the optimizer's buffers and the returned entries are None."""
    n_out, k = w.shape
    dw = w_sink[0] if w_sink is not None else torch.zeros_like(w)
    if not has_bias:
        db = None
    elif b_sink is not None:
        db = b_sink[0]
    else:
        db = torch.zeros(n_out, dtype=torch.float32, device=w.device)
    tc = (_tc_rows_ok(n) and LINEAR_WGRAD_IMPL != "simt" and _tc_wgrad_fits(k, n_out) and n_out % 4 == 0
          and _aligned(x2, ldx) and _aligned(dz, lddz) and _pad4(k) <= ldx)
    if _narrow_ok(k, n_out):
        _lib.call("emer_linear_narrow_bwd_weight", _ptr(x2), ldx, _ptr(dz), lddz, _ptr(dw), _ptr(db), n, k, n_out,
                  _stream())
    elif tc:
        _lib.call("emer_linear_tc_bwd_weight", _ptr(x2), ldx, _ptr(dz), lddz, _ptr(dw), _ptr(db), n, k, n_out,
                  _stream())
    else:
        _lib.call("emer_linear_bwd_weight", _ptr(x2), ldx, _ptr(dz), lddz, None, 0, ACT_NONE, _ptr(dw), _ptr(db), n, k,
                  n_out, _stream())
    if w_sink is not None:
        w_sink[1]()
        dw = None
    if has_bias and b_sink is not None:
        b_sink[1]()
        db = None
    return dw, db


class _MLPChain(torch.autograd.Function):
    """A whole head: Linear -> ReLU -> ... -> Linear [-> out_act], optionally with the chain input
    concatenated in front of layer ``skip_layer`` (radiance_fields/mlp.py:38-46).  Hidden activations
    are written once (they are needed by the backward pass), the skip concatenation is assembled in
    place (the previous layer writes straight into the concat buffer), and in the backward pass every
    data-gradient kernel applies the ReLU mask of the layer below in its epilogue, so no
    activation-derivative pass ever runs on its own."""

    @staticmethod
    def forward(ctx, x: Tensor, catbuf: Optional[Tensor], skip_layer: int, out_act: int, has_bias: bool,
                *params: Tensor):
        ctx.set_materialize_grads(False)
        ws = [_f32c(w) for w in (params[0::2] if has_bias else params)]
        bs = [_f32c(b) for b in params[1::2]] if has_bias else [None] * len(ws)
        _need_cuda(x, *ws)
        ctx.sinks = [(_grad_sink(w), _grad_sink(b)) for w, b in zip(ws, bs)]
        k0 = ws[0].shape[1]
        lead = x.shape[:-1]
        x2, ldx = _rows(x, k0)
        n = x2.shape[0]
        dev = x.device
        L = len(ws)
        inputs, lds, outs = [], [], []
        cur, ld = x2, ldx
        cat = None               # [n, pad4(h + k0)] buffer of the skip concatenation [hidden | x]
        shared = False           # ... which is the caller's: x already sits behind the hidden columns
        for i, (w, b) in enumerate(zip(ws, bs)):
            n_out, k = w.shape
            if i == skip_layer and i > 0:
                # layer i-1 wrote cat[:, :h]; the chain input goes behind it
                h = ws[i - 1].shape[0]
                if not shared:
                    cat[:, h:h + k0].copy_(x2)
                cur, ld = cat[:, :h + k0], cat.shape[1]
            if cur.shape[1] != k:
                raise ValueError(f"mlp layer {i}: input width {cur.shape[1]} != weight width {k}")
            act = ACT_RELU if i < L - 1 else out_act
            if i + 1 == skip_layer and i + 1 < L:
                shared = (catbuf is not None and catbuf.dim() == 2 and catbuf.is_contiguous()
                          and catbuf.dtype == torch.float32 and tuple(catbuf.shape) == (n, _pad4(n_out + k0))
                          and x2.data_ptr() == catbuf.data_ptr() + 4 * n_out and ldx == catbuf.shape[1])
                if shared:
                    cat = catbuf
                else:
                    cat = torch.empty((n, _pad4(n_out + k0)), dtype=torch.float32, device=dev)
                    if cat.shape[1] > n_out + k0:
                        cat[:, n_out + k0:].zero_()
                y, ldy = cat[:, :n_out], cat.shape[1]
            else:
                y = torch.empty((n, n_out), dtype=torch.float32, device=dev)
                ldy = n_out
            _layer_fwd(cur, ld, w, b, y, ldy, n, act)
            inputs.append(cur)
            lds.append(ld)
            outs.append(y)
            cur, ld = y, ldy
        ctx.save_for_backward(*inputs, outs[-1], *ws)
        ctx.meta = (skip_layer, out_act, has_bias, L, lds, k0, x.shape)
        return outs[-1].view(*lead, -1)

    @staticmethod
    def backward(ctx, dy):
        skip_layer, out_act, has_bias, L, lds, k0, x_shape = ctx.meta
        n_grads = _CHAIN_ARGS + (2 * L if has_bias else L)
        if dy is None:
            return (None,) * n_grads
        saved = ctx.saved_tensors
        inputs, y_last, ws = saved[:L], saved[L], saved[L + 1:]
        n = inputs[0].shape[0]
        n_last = ws[-1].shape[0]
        dev = y_last.device
        dz, lddz = _rows(dy, n_last)
        if out_act == ACT_SIGMOID:
            dz = dz * (y_last * (1.0 - y_last))
            lddz = n_last
        elif out_act == ACT_RELU:
            dz = dz * (y_last > 0)
            lddz = n_last
        elif not dz.is_contiguous() and dz.shape[0] > 1 and lddz % 4 != 0:
            dz, lddz = dz.contiguous(), n_last
        need_x = ctx.needs_input_grad[0]
        grads_w = [None] * L
        grads_b = [None] * L
        dx = None
        dx_skip = None
        # Skip in front of layer 1 (the reference's heads): dX = dZ0 W0 + dZ1 W1[:, h:] is ONE product
        # [dZ0 | dZ1] [W0 ; W1[:, h:]], so dZ1 and dZ0 are written side by side into ``gcat`` and the skip
        # layer's data gradient only computes its hidden columns: no [n, k0] partial result, no add pass.
        h0, n1 = ws[0].shape[0], (ws[1].shape[0] if L > 1 else 0)
        stacked = (SKIP_BWD_IMPL == "stack" and skip_layer == 1 and L >= 3 and need_x and h0 % 4 == 0
                   and n1 % 4 == 0 and h0 + n1 <= 128 and k0 <= 128)
        gcat = torch.empty((n, h0 + n1), dtype=torch.float32, device=dev) if stacked else None
        for i in range(L - 1, -1, -1):
            w = ws[i]
            n_out, k = w.shape
            inp, ld = inputs[i], lds[i]
            w_idx = _CHAIN_ARGS + (2 * i if has_bias else i)
            if ctx.needs_input_grad[w_idx] or (has_bias and ctx.needs_input_grad[w_idx + 1]):
                grads_w[i], grads_b[i] = _layer_bwd_weight(inp, ld, dz, lddz, w, has_bias, n, *ctx.sinks[i])
            if i == 0 and not need_x:
                break
            if stacked and i == 2:
                # dZ1 = relu'(h1) * (dZ2 W2)  ->  gcat[:, h0:]
                d_inp = gcat[:, h0:]
                _layer_bwd_data(dz, lddz, w, d_inp, gcat.shape[1], n, inp, ld, n1)
                dz, lddz = d_inp, gcat.shape[1]
            elif stacked and i == 1:
                # dZ0 = relu'(h0) * (dZ1 W1[:, :h0])  ->  gcat[:, :h0]
                d_inp = gcat[:, :h0]
                _layer_bwd_data(dz, lddz, w[:, :h0].contiguous(), d_inp, gcat.shape[1], n, inp, ld, h0)
                dz, lddz = d_inp, gcat.shape[1]
            elif stacked and i == 0:
                w_stack = torch.cat([w, ws[1][:, h0:h0 + k0]], dim=0)
                d_inp = torch.empty((n, _pad4(k0)), dtype=torch.float32, device=dev)
                _layer_bwd_data(gcat, gcat.shape[1], w_stack, d_inp, d_inp.shape[1], n, None, 0, 0)
                dx = d_inp[:, :k0]
            elif i > 0:
                d_inp = torch.empty((n, _pad4(k)), dtype=torch.float32, device=dev)
                h = ws[i - 1].shape[0]          # first h columns of this layer's input are ReLU outputs
                _layer_bwd_data(dz, lddz, w, d_inp, d_inp.shape[1], n, inp, ld, h)
                if i == skip_layer:
                    dx_skip = d_inp[:, h:h + k0]
                dz, lddz = d_inp[:, :h], d_inp.shape[1]
            else:
                d_inp = torch.empty((n, _pad4(k)), dtype=torch.float32, device=dev)
                _layer_bwd_data(dz, lddz, w, d_inp, d_inp.shape[1], n, None, 0, 0)
                dx = d_inp[:, :k]
        if need_x:
            if dx_skip is not None:
                # sum into the skip slice of the [n, pad4] gradient buffer: rows stay 16-byte aligned for
                # the consumer (no re-padding copy downstream)
                dx = dx_skip.add_(dx)
            dx = dx.reshape(x_shape)
        out = [dx if need_x else None] + [None] * (_CHAIN_ARGS - 1)
        for i in range(L):
            out.append(grads_w[i])
            if has_bias:
                out.append(grads_b[i])
        return tuple(out)


_CHAIN_ARGS = 5           # x, catbuf, skip_layer, out_act, has_bias come before the parameters


def mlp_chain(x: Tensor, weights, biases=None, out_act: int = ACT_NONE, skip_layer: int = -1,
              catbuf: Optional[Tensor] = None) -> Tensor:
    """Evaluate a ReLU MLP head.  ``weights[i]``: [n_out_i, k_i] (nn.Linear layout); ``skip_layer``: the
    layer in front of which [hidden, x] is concatenated (-1: none).  ``catbuf`` (optional): the
    [n, pad4(hidden + k)] buffer whose columns [hidden, hidden + k) ARE x (see :func:`field_tail`); the layer
    before the skip then writes its output into the front columns and the concatenation is free."""
    if x.shape[-1] != weights[0].shape[1]:
        raise ValueError(f"mlp: input width {x.shape[-1]} != first layer width {weights[0].shape[1]}")
    if biases is None:
        return _MLPChain.apply(x, catbuf, skip_layer, out_act, False, *weights)
    flat = []
    for w, b in zip(weights, biases):
        flat += [w, b]
    return _MLPChain.apply(x, catbuf, skip_layer, out_act, True, *flat)


def linear(x: Tensor, w: Tensor, b: Optional[Tensor], act: int = ACT_NONE) -> Tensor:
    """act(x @ w.T + b) over the last dimension."""
    if x.shape[-1] != w.shape[1]:
        raise ValueError(f"linear: input width {x.shape[-1]} != weight width {w.shape[1]}")
    return mlp_chain(x, [w], None if b is None else [b], act)


def cat_pad4(parts, dim_check: bool = True) -> Tensor:
    """torch.cat along the last dim into rows padded to a multiple of 4 floats (16-byte aligned rows
    for the tensor-core loaders); returns the [..., total] view of the padded buffer."""
    total = sum(p.shape[-1] for p in parts)
    cat = torch.cat(parts, dim=-1)
    pad = _pad4(total) - total
    if pad == 0:
        return cat
    return torch.nn.functional.pad(cat, (0, pad))[..., :total]


# ----------------------------------------------------------------------------- field tail
FT_DIR = 33


class _FieldTail(torch.autograd.Function):
    """feats [R, S, >=G], per-ray dirs [R, 3], per-ray embedding index [R] -> (sigma [R, S],
    rgb_in [R, S, G+33+E] laid out [geo | dir encoding | embedding] in rows padded to 16 bytes)."""

    @staticmethod
    def forward(ctx, feats: Tensor, dirs: Tensor, idx: Optional[Tensor], emb: Optional[Tensor], g_dim: int,
                front: int):
        ctx.set_materialize_grads(False)
        _need_cuda(feats, dirs)
        r, s_, width_in = feats.shape
        f2, ldf = _rows(feats, width_in)
        dirs = _f32c(dirs)
        e_dim = 0 if emb is None else emb.shape[1]
        embc = None if emb is None else _f32c(emb)
        idxc = None if idx is None else idx.to(torch.int64).contiguous()
        width = g_dim + FT_DIR + e_dim
        # ``front`` spare columns ahead of every row: the colour head writes its first hidden layer there, which
        # makes this buffer the [hidden | input] skip concatenation without a copy (see _MLPChain)
        ld = _pad4(front + width)
        buf = torch.empty((r * s_, ld), dtype=torch.float32, device=feats.device)
        out = buf[:, front:front + width]
        sigma = torch.empty((r, s_), dtype=torch.float32, device=feats.device)
        _lib.call("emer_field_tail_fwd", _ptr(f2), ldf, g_dim, _ptr(dirs), _ptr(idxc), _ptr(embc), e_dim, _ptr(out), ld,
                  _ptr(sigma), r, s_, _stream())
        ctx.save_for_backward(f2, idxc)
        ctx.meta = (ldf, g_dim, e_dim, width, _pad4(width), r, s_, width_in, None if emb is None else emb.shape)
        ctx.mark_non_differentiable(buf)
        return sigma, out.view(r, s_, width), buf

    @staticmethod
    def backward(ctx, d_sigma, d_rgb_in, _d_buf=None):
        f2, idxc = ctx.saved_tensors
        ldf, g_dim, e_dim, width, ld, r, s_, width_in, emb_shape = ctx.meta
        n = r * s_
        if d_rgb_in is None:
            g2 = torch.zeros((n, ld), dtype=torch.float32, device=f2.device)
        else:
            # INVARIANT: the kernel adds d_sigma's contribution to column 0 of this buffer IN PLACE.  rgb_in has exactly one
            # consumer (mlp_chain, whose backward hands over a buffer it allocated for this purpose and never reads
            # again), so nothing else can observe the mutation; a tensor hook or retain_grad() on rgb_in would see the
            # combined gradient.  field_tail() is not exported for other uses.
            g2 = d_rgb_in.reshape(n, width)
            if g2.stride(1) != 1 or g2.stride(0) % 4 != 0 or g2.data_ptr() % 16 != 0:
                g2 = torch.nn.functional.pad(g2, (0, ld - width))
        ldg = g2.stride(0)
        d_emb = None
        if emb_shape is not None and ctx.needs_input_grad[3]:
            d_emb = torch.zeros(emb_shape, dtype=torch.float32, device=f2.device)
        ds = None if d_sigma is None else _f32c(d_sigma)
        _lib.call("emer_field_tail_bwd", _ptr(f2), ldf, _ptr(g2), ldg, g_dim, _ptr(ds), _ptr(idxc), _ptr(d_emb), e_dim, r,
                  s_, _stream())
        d_feats = g2[:, :g_dim]
        if width_in > g_dim:
            d_feats = torch.nn.functional.pad(d_feats, (0, width_in - g_dim))
        return d_feats.reshape(r, s_, width_in), None, None, d_emb, None, None


def field_tail(feats: Tensor, dirs: Tensor, idx: Optional[Tensor], emb: Optional[Tensor], g_dim: int, front: int = 0):
    """(sigma, rgb_in) -- or (sigma, rgb_in, catbuf) with ``front`` > 0, where rgb_in = catbuf[:, front:front+width]
    and catbuf is handed to :func:`mlp_chain` so that the head's skip concatenation needs no copy."""
    if front % 4:
        raise ValueError("field_tail: front must be a multiple of 4 (16-byte aligned rows)")
    sigma, rgb_in, buf = _FieldTail.apply(feats, dirs, idx, emb, g_dim, front)
    return (sigma, rgb_in, buf) if front else (sigma, rgb_in)


# ----------------------------------------------------------------------------- fused field chain
FIELD_CHAIN = os.environ.get("EMER_FIELD_CHAIN", "fused")      # "layers": the per-layer path (A/B and debugging switch)
CHAIN_BWD = os.environ.get("EMER_CHAIN_BWD", "fused")          # "layers": data gradients layer by layer (A/B switch)
CHAIN_K_ENC = (32, 40, 64)


def _tc_bwd_data_acc(dz: Tensor, lddz: int, w: Tensor, dx: Tensor, lddx: int, n: int) -> None:
    """dx[n, k] += dz[n, n_out] @ w on the tensor-core layer kernel (accumulating form)."""
    n_out, k = w.shape
    _lib.call("emer_linear_tc_bwd_data", _ptr(dz), lddz, None, 0, ACT_NONE, _ptr(w), _ptr(dx), lddx, None, 0, 0, n, k,
              n_out, 1, _stream())


class _FieldChain(torch.autograd.Function):
    """enc [N, k_enc] -> (sigma [N], rgb [N, 3], geo [N, 64] | None, sem [N, 64] | None): base MLP, density and the
    colour head in one kernel (``emer_field_fwd``, csrc/field_fused.cu).  ``ray_bias`` [R, 128] carries the per-ray
    input columns of the colour head and its first two biases (see :func:`field_chain`).

    Backward: the data gradients come from one kernel (``emer_field_bwd``) or -- ragged rays, batches below
    ``TC_MIN_ROWS``, ``EMER_CHAIN_BWD=layers`` -- from a walk over the saved activations with the layer kernels
    ([h0 | geo] side by side, so layer 1 of the head is one 64 -> 128 product and the skip gradient accumulates in
    place).  Either way the five layers' weight gradients then come from one ``emer_field_wgrad`` launch over the
    buffers the data path left.  ``d_ray_bias`` is the per-ray sum of the two hidden-layer gradients, which hands the
    per-ray weight columns, the biases and the embedding their gradients through ordinary autograd."""

    @staticmethod
    def forward(ctx, enc: Tensor, ray_bias: Tensor, samples: int, want_geo: bool, wb0: Tensor, bb0: Tensor, wb1: Tensor,
                bb1: Tensor, w0: Tensor, w1: Tensor, w2: Tensor, b2: Tensor):
        ctx.set_materialize_grads(False)
        _need_cuda(enc, ray_bias, wb0, wb1, w0, w1, w2)
        enc2, ld_enc = _rows(enc, enc.shape[-1])
        n, k_enc = enc2.shape
        if ld_enc % 8 or enc2.data_ptr() % 32:          # the kernel reads its rows 32 bytes at a time
            enc2, ld_enc = enc2.contiguous(), k_enc
        n_feat = wb1.shape[0]
        n_ray_cols = w0.shape[1] - 64                   # [dir | emb] columns in front of geo (radiance_field.py:647)
        ws = [_f32c(t) for t in (wb0, bb0, wb1, bb1, w0, w1, w2, b2)]
        wb0c, bb0c, wb1c, bb1c, w0c, w1c, w2c, b2c = ws
        rb = _f32c(ray_bias)
        if rb.shape != ((n + samples - 1) // samples, 128):
            raise ValueError(f"field_chain: ray_bias {tuple(rb.shape)} for {n} points x {samples} samples per ray")
        dev = enc.device
        train = any(ctx.needs_input_grad)          # (False under torch.no_grad(): no saves, inference traffic only)
        f32 = dict(dtype=torch.float32, device=dev)
        sigma = torch.empty(n, **f32)
        rgb = torch.empty((n, 3), **f32)
        hb = torch.empty((n, 64), **f32) if train else None
        hg = torch.empty((n, 128), **f32) if (train or want_geo) else None
        h1 = torch.empty((n, 64), **f32) if train else None
        sem = torch.empty((n, 64), **f32) if n_feat == 128 else None
        w0g = w0c[:, n_ray_cols:]
        w1h, w1g = w1c[:, :64], w1c[:, 64 + n_ray_cols:]
        _lib.call("emer_field_fwd", _ptr(enc2), ld_enc, k_enc, _ptr(wb0c), _ptr(bb0c), _ptr(wb1c), _ptr(bb1c), n_feat,
                  _ptr(w0g), w0c.shape[1], _ptr(w1h), _ptr(w1g), w1c.shape[1], _ptr(w2c), _ptr(b2c), _ptr(rb), samples,
                  _ptr(sigma), _ptr(rgb), _ptr(hb), _ptr(hg), _ptr(h1), _ptr(sem), n, _stream())
        geo = hg[:, 64:] if want_geo else None
        if train:
            ctx.sinks = {k: _grad_sink(t) for k, t in zip(("wb0", "bb0", "wb1", "bb1", "w0", "w1", "w2", "b2"), ws)}
            ctx.save_for_backward(enc2, hb, hg, h1, rgb, sigma, wb0c, wb1c, w0c, w1c, w2c)
            ctx.meta = (samples, n_ray_cols, n_feat, enc.shape, ld_enc)
        return sigma, rgb, geo, sem

    @staticmethod
    def backward(ctx, d_sigma, d_rgb, d_geo, d_sem):
        enc2, hb, hg, h1, rgb, sigma, wb0, wb1, w0, w1, w2 = ctx.saved_tensors
        samples, n_ray_cols, n_feat, enc_shape, ld_enc = ctx.meta
        n, k_enc = enc2.shape
        dev = enc2.device
        f32 = dict(dtype=torch.float32, device=dev)
        none = (None,) * 12
        if d_sigma is None and d_rgb is None and d_geo is None and d_sem is None:
            return none
        n_rays = (n + samples - 1) // samples
        sk = ctx.sinks
        w1hg = torch.cat([w1[:, :64], w1[:, 64 + n_ray_cols:]], dim=1)            # [64, 128] = [hidden | geo] columns
        w0g = w0[:, n_ray_cols:].contiguous()
        D1 = torch.empty((n, 128), **f32)          # [dZ0 | dF] side by side (row stride 128)
        dz2 = dz1 = d_rb = d_enc = None
        c = lambda g, w: None if g is None else _f32c(g.reshape(n, w))
        d_geo, d_sem = c(d_geo, 64), c(d_sem, 64)
        if CHAIN_BWD == "fused" and samples % 32 == 0 and _tc_rows_ok(n):
            # ---- the whole data path in one kernel (csrc/field_fused.cu: field_bwd_kernel)
            d_rgb2 = c(d_rgb, 3)
            d_sig = None if d_sigma is None else _f32c(d_sigma).reshape(n)
            dz2 = torch.empty((n, 3), **f32) if d_rgb is not None else None
            dz1 = torch.empty((n, 64), **f32)
            dzb = torch.empty((n, 64), **f32)
            if ctx.needs_input_grad[0]:
                d_enc = torch.empty((n, k_enc), **f32)
            d_rb = torch.zeros((n_rays, 128), **f32) if d_rgb is not None else None
            _lib.call("emer_field_bwd", _ptr(d_rgb2), _ptr(rgb), _ptr(d_sig), _ptr(sigma), _ptr(d_geo), _ptr(d_sem), _ptr(hb),
                      _ptr(hg), _ptr(h1), _ptr(wb0), k_enc, _ptr(wb1), n_feat, _ptr(w0g), 64, _ptr(w1hg), _ptr(w1hg[:, 64:]),
                      128, _ptr(w2), _ptr(dz2), _ptr(dz1), _ptr(D1), _ptr(dzb), _ptr(d_enc), k_enc, _ptr(d_rb), samples, n,
                      _stream())
        else:
            # ---- layer by layer on the same buffers (ragged rays, tiny batches, EMER_CHAIN_BWD=layers)
            if d_rgb is not None:
                dz2 = _f32c(d_rgb.reshape(n, 3)) * (rgb * (1.0 - rgb))
                dz1 = torch.empty((n, 64), **f32)
                _layer_bwd_data(dz2, 3, w2, dz1, 64, n, h1, 64, 64)                   # relu'(h1) applied
                _layer_bwd_data(dz1, 64, w1hg, D1, 128, n, hg, 128, 64)               # [relu'(h0) dH0 | dGeo(layer 1)]
                dz0 = D1[:, :64]
                if _tc_rows_ok(n):
                    _tc_bwd_data_acc(dz0, 128, w0g, D1[:, 64:], 128, n)              # dGeo += dZ0 W0g
                else:
                    _lib.call("emer_linear_bwd_data", _ptr(dz0), 128, None, 0, ACT_NONE, _ptr(w0g), _ptr(D1[:, 64:]), 128,
                              n, 64, 64, 1, _stream())
                if n_rays * samples - n:                   # ragged last ray: sum what is there
                    d_rb = torch.zeros((n_rays, 128), **f32)
                    d_rb[:, :64].index_add_(0, torch.arange(n, device=dev) // samples, dz0)
                    d_rb[:, 64:].index_add_(0, torch.arange(n, device=dev) // samples, dz1)
                else:
                    d_rb = torch.cat([D1.view(n_rays, samples, 128)[:, :, :64].sum(1),
                                      dz1.view(n_rays, samples, 64).sum(1)], dim=1)
            else:
                D1[:, 64:].zero_()
            dgeo = D1[:, 64:]
            if d_geo is not None:
                dgeo += d_geo
            if d_sigma is not None:
                # trunc_exp backward (nerf_utils.py:72-75): g * exp(clamp(x, max=15)), x = feats[:, 0] - 1 = log(sigma)
                dgeo[:, 0] += _f32c(d_sigma).reshape(n) * torch.clamp(sigma, max=3269017.25)
            # [dF | d_sem]: the gradient of the base MLP's output (zeros for an absent semantic half)
            if n_feat == 128:
                dfe = torch.cat([D1[:, 64:], torch.zeros((n, 64), **f32) if d_sem is None else d_sem], dim=1)
            else:
                dfe = D1[:, 64:]
            dzb = torch.empty((n, 64), **f32)
            _layer_bwd_data(dfe, 128, wb1, dzb, 64, n, hb, 64, 64)
            if ctx.needs_input_grad[0]:
                d_enc = torch.empty((n, _pad4(k_enc)), **f32)
                _layer_bwd_data(dzb, 64, wb0, d_enc, d_enc.shape[1], n, None, 0, 0)
                d_enc = d_enc[:, :k_enc]

        shapes = dict(wb0=wb0.shape, bb0=(64,), wb1=wb1.shape, bb1=(n_feat,), w0=w0.shape, w1=w1.shape, w2=w2.shape,
                      b2=(3,))
        keys = list(shapes) if dz2 is not None else ["wb0", "bb0", "wb1", "bb1"]
        side = WGRAD_STREAM and all(v is not None for v in sk.values())

        def weight_gradients(deferred):
            """The five layers' X^T dZ in one emer_field_wgrad launch, accumulated into the optimizer's buffers (or
            into zeros shaped like the parameters, returned to autograd).  ``deferred``: the side stream's list of
            updates to run after the join -- the head's w0 / w1 gradients then go to zeros and are added there,
            because autograd adds the per-ray columns' gradient to the same buffers on the main stream with an
            in-place add of the whole tensor, which would race the kernel's atomics."""
            out, grads = {}, {}
            for k in keys:
                s = sk[k]
                if s is None:
                    out[k] = grads[k] = torch.zeros(shapes[k], **f32)
                elif deferred is not None and k in ("w0", "w1"):
                    out[k] = torch.zeros(shapes[k], **f32)
                    deferred.append(lambda dst=s[0], src=out[k]: dst.add_(src))
                else:
                    out[k] = s[0]
            o = lambda k: _ptr(out[k]) if k in out else None
            if dz2 is not None:        # the head's geo / hidden column blocks; the per-ray ones come through ray_bias
                w0g_d, ld_w0, w1g_d, ld_w1 = out["w0"][:, n_ray_cols:], out["w0"].stride(0), out["w1"][:, 64 + n_ray_cols:], out["w1"].stride(0)
            else:
                w0g_d, ld_w0, w1g_d, ld_w1 = None, 0, None, 0
            _lib.call("emer_field_wgrad", _ptr(enc2), ld_enc, k_enc, _ptr(hb), _ptr(hg), _ptr(h1), _ptr(dz2),
                      _ptr(dz1), _ptr(D1), _ptr(dzb), _ptr(d_sem), n_feat, o("wb0"), o("bb0"), o("wb1"), o("bb1"),
                      _ptr(w0g_d), ld_w0, o("w1"), _ptr(w1g_d), ld_w1, o("w2"), o("b2"), n, _stream())
            for k in keys:
                if sk[k] is not None:
                    sk[k][1]()
            return tuple(grads.get(k) for k in ("wb0", "bb0", "wb1", "bb1", "w0", "w1", "w2", "b2"))

        if side:
            # every weight gradient lands in the optimizer's buffers: nothing autograd waits for, so the kernel may
            # run beside the hash-grid scatter / the table's reduce-scatter (joined by FusedAdam.step /
            # DataParallel.reduce)
            with _on_side_stream(dev, enc2, hb, hg, h1, dz2, dz1, D1, dzb, d_sem):
                dwb0, dbb0, dwb1, dbb1, dw0, dw1, dw2, db2 = weight_gradients(_AFTER_JOIN)
        else:
            dwb0, dbb0, dwb1, dbb1, dw0, dw1, dw2, db2 = weight_gradients(None)
        if d_enc is not None:
            d_enc = d_enc.reshape(enc_shape)
        return d_enc, d_rb, None, None, dwb0, dbb0, dwb1, dbb1, dw0, dw1, dw2, db2


def field_chain_usable(k_enc: int, n_feat: int, width: int, head: Sequence[Tuple[int, int]]) -> bool:
    """Whether ``emer_field_fwd`` is specialised for this model: 64-wide base / head layers, a 64-d geometry feature
    (+ optional 64-d semantic half), a 3-layer colour head with the skip in front of layer 1."""
    if FIELD_CHAIN != "fused" or LINEAR_IMPL != "tc":
        return False
    if k_enc not in CHAIN_K_ENC or n_feat not in (64, 128) or width != 64 or len(head) != 3:
        return False
    (o0, i0), (o1, i1), (o2, i2) = head
    return o0 == 64 and o1 == 64 and o2 == 3 and i2 == 64 and i0 >= 64 and i1 == 64 + i0


def field_chain(enc: Tensor, ray_bias: Tensor, samples: int, base, head, want_geo: bool = False):
    """``base`` = (wb0, bb0, wb1, bb1), ``head`` = (w0, w1, w2, b2) with the reference's column order
    ([dir | emb | geo] for layer 0, [hidden | dir | emb | geo] for layer 1, radiance_field.py:647, mlp.py:42-43);
    ``ray_bias`` [R, 128] = [b0 + w0[:, :c] v | b1 + w1[:, 64:64+c] v] for the per-ray input columns v."""
    return _FieldChain.apply(enc, ray_bias, samples, want_geo, *base, *head)


# ----------------------------------------------------------------------------- flow variants' dynamic branch
# "fused": RadianceField.forward runs the flow configs' temporal aggregation through flow_warp, one dynamic-table gather
# over the stacked [current | forward | backward] coordinates and emer_flow_field_fwd / _bwd; "layers": the per-layer path
FLOW_BRANCH = os.environ.get("EMER_FLOW_BRANCH", "layers")
FLOW_K_ENC = (40, 64)           # emer_flow_field_*: the dynamic grid's L*F (40: the shipped configs)


class _FlowWarp(torch.autograd.Function):
    """(pos [N,3], flow [N,6], noise [N] | None, t [N]) -> the [2N, 4] grid coordinates of both flow warps
    (``emer_flow_warp_fwd``); the backward hands d_flow to the flow MLP (time and noise take no gradient)."""

    @staticmethod
    def forward(ctx, pos: Tensor, flow: Tensor, noise: Optional[Tensor], t: Tensor, aabb: Tensor, time_diff,
                unbounded: bool):
        ctx.set_materialize_grads(False)
        _need_cuda(pos, flow, t, aabb)
        pos2, flow2 = _f32c(pos.reshape(-1, 3)), _f32c(flow.reshape(-1, 6))
        n = pos2.shape[0]
        t2 = _f32c(t.reshape(-1))
        nz, ldn = (None, 0) if noise is None else _rows(noise.reshape(n, 1), 1)
        box = _f32c(aabb.reshape(-1))
        # the model's time step is a 0-d device tensor when it comes from the registered timesteps: read on the device
        if isinstance(time_diff, Tensor):
            td = _f32c(time_diff.reshape(1))
        else:
            td = torch.full((1,), float(time_diff), dtype=torch.float32, device=pos2.device)
        coords = torch.empty((2 * n, 4), dtype=torch.float32, device=pos2.device)
        _lib.call("emer_flow_warp_fwd", _ptr(pos2), _ptr(flow2), _ptr(nz), ldn, _ptr(t2), _ptr(box), _ptr(td),
                  int(unbounded), _ptr(coords), n, _stream())
        ctx.save_for_backward(pos2, flow2, nz, box)
        ctx.meta = (ldn, int(unbounded), flow.shape)
        return coords

    @staticmethod
    def backward(ctx, d_coords):
        if d_coords is None or not ctx.needs_input_grad[1]:
            return (None,) * 7
        pos2, flow2, nz, box = ctx.saved_tensors
        ldn, unbounded, flow_shape = ctx.meta
        n = pos2.shape[0]
        d_flow = torch.empty((n, 6), dtype=torch.float32, device=pos2.device)
        _lib.call("emer_flow_warp_bwd", _ptr(pos2), _ptr(flow2), _ptr(nz), ldn, _ptr(box), unbounded,
                  _ptr(_f32c(d_coords)), _ptr(d_flow), n, _stream())
        return None, d_flow.view(flow_shape), None, None, None, None, None


def flow_warp(pos: Tensor, flow: Tensor, noise: Optional[Tensor], t: Tensor, aabb: Tensor, time_diff,
              unbounded: bool) -> Tensor:
    """Rows [0, N): contract(pos + flow[..., :3] noise) | clamp(t + time_diff noise, 0, 1); rows [N, 2N): the backward
    warp with flow[..., 3:] and -time_diff (radiance_field.py:449-452).  ``noise`` None: 1 (the eval renders)."""
    return _FlowWarp.apply(pos, flow, noise, t, aabb, time_diff, unbounded)


class _GridEncodeRows(torch.autograd.Function):
    """grid_encode of the stacked rows [x_fixed ; x_var] in one gather; the backward scatters all rows into the table and
    computes the input gradient of the x_var rows only (x_fixed takes none)."""

    @staticmethod
    def forward(ctx, x_fixed: Tensor, x_var: Tensor, params: Tensor, desc: GridDesc):
        ctx.set_materialize_grads(False)
        _need_cuda(x_fixed, x_var, params)
        x = torch.cat([_f32c(x_fixed), _f32c(x_var)])
        params = _f32c(params)
        n = x.shape[0]
        y = torch.empty((n, desc.n_output_dims), dtype=torch.float32, device=x.device)
        _lib.call("emer_grid_fwd", ctypes.byref(desc.c), _ptr(x), _ptr(params), _ptr(y), n, _stream())
        ctx.save_for_backward(x, params)
        ctx.desc, ctx.n0 = desc, x_fixed.shape[0]
        return y

    @staticmethod
    def backward(ctx, dy):
        if dy is None:
            return None, None, None, None
        x, params = ctx.saved_tensors
        desc, n0 = ctx.desc, ctx.n0
        dy = _f32c(dy)
        need_x, need_p = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        sink = _grad_sink(params) if need_p else None
        dparams = sink[0] if sink is not None else (torch.zeros_like(params) if need_p else None)
        if need_p:
            _lib.call("emer_grid_bwd", ctypes.byref(desc.c), _ptr(x), _ptr(params), _ptr(dy), _ptr(dparams), _ptr(None),
                      x.shape[0], _stream())
        dx = None
        if need_x:
            dx = torch.empty((x.shape[0] - n0, x.shape[1]), dtype=torch.float32, device=x.device)
            _lib.call("emer_grid_bwd", ctypes.byref(desc.c), _ptr(x[n0:]), _ptr(params), _ptr(dy[n0:]), _ptr(None),
                      _ptr(dx), dx.shape[0], _stream())
        if sink is not None:
            sink[1]()
            dparams = None
        return None, dx, dparams, None


def grid_encode_rows(x_fixed: Tensor, x_var: Tensor, params: Tensor, desc: GridDesc) -> Tensor:
    """[N0 + N1, L*F] features of the rows [x_fixed ; x_var] (each [., D]); only x_var takes an input gradient."""
    return _GridEncodeRows.apply(x_fixed, x_var, params, desc)


class _FlowFieldChain(torch.autograd.Function):
    """enc [3N, k_enc] = [current | forward-warped | backward-warped] encodings -> (sigma [N], rgb [N, 3] | None,
    geo [N, 64], sem [N, 64] | None) of the blended features (F_c + 0.5 F_f + 0.5 F_b) / 2: base MLP per query, blend,
    density and colour head in one kernel (``emer_flow_field_fwd``).  ``ray_bias`` None: density only (the lidar pass).

    Backward: ``emer_flow_field_bwd`` for the data path (d_enc for all 3N rows), then the weight gradients from
    ``emer_field_wgrad``: the colour head and the base MLP over the current N rows in one launch, the base MLP over the
    2N warped rows in a second (density only: the base MLP over all 3N rows in one)."""

    @staticmethod
    def forward(ctx, enc: Tensor, ray_bias: Optional[Tensor], samples: int, wb0: Tensor, bb0: Tensor, wb1: Tensor,
                bb1: Tensor, w0: Tensor, w1: Tensor, w2: Tensor, b2: Tensor):
        ctx.set_materialize_grads(False)
        _need_cuda(enc, wb0, wb1, w0, w1, w2)
        enc2, ld_enc = _rows(enc, enc.shape[-1])
        if ld_enc % 8 or enc2.data_ptr() % 32:
            enc2, ld_enc = enc2.contiguous(), enc2.shape[1]
        n3, k_enc = enc2.shape
        n = n3 // 3
        n_feat = wb1.shape[0]
        n_ray_cols = w0.shape[1] - 64
        ws = [_f32c(t) for t in (wb0, bb0, wb1, bb1, w0, w1, w2, b2)]
        wb0c, bb0c, wb1c, bb1c, w0c, w1c, w2c, b2c = ws
        head = ray_bias is not None
        rb = _f32c(ray_bias) if head else None
        if head and rb.shape != ((n + samples - 1) // samples, 128):
            raise ValueError(f"flow_field_chain: ray_bias {tuple(rb.shape)} for {n} points x {samples} samples per ray")
        dev = enc.device
        train = any(ctx.needs_input_grad)
        f32 = dict(dtype=torch.float32, device=dev)
        sigma = torch.empty(n, **f32)
        rgb = torch.empty((n, 3), **f32) if head else None
        hb = torch.empty((n3, 64), **f32) if train else None
        hg = torch.empty((n, 128), **f32)                 # the geometry half carries the blend
        h1 = torch.empty((n, 64), **f32) if (train and head) else None
        sem = torch.empty((n, 64), **f32) if n_feat == 128 else None
        _lib.call("emer_flow_field_fwd", _ptr(enc2), ld_enc, k_enc, _ptr(wb0c), _ptr(bb0c), _ptr(wb1c), _ptr(bb1c), n_feat,
                  _ptr(w0c[:, n_ray_cols:]), w0c.shape[1], _ptr(w1c[:, :64]), _ptr(w1c[:, 64 + n_ray_cols:]), w1c.shape[1],
                  _ptr(w2c), _ptr(b2c), _ptr(rb), samples, _ptr(sigma), _ptr(rgb), _ptr(hb), _ptr(hg), _ptr(h1), _ptr(sem),
                  n, _stream())
        if train:
            ctx.sinks = {k: _grad_sink(t) for k, t in zip(("wb0", "bb0", "wb1", "bb1", "w0", "w1", "w2", "b2"), ws)}
            ctx.save_for_backward(enc2, hb, hg, h1, rgb, sigma, wb0c, wb1c, w0c, w1c, w2c)
            ctx.meta = (samples, n_ray_cols, n_feat, enc.shape, ld_enc, head)
        return sigma, rgb, hg[:, 64:], sem

    @staticmethod
    def backward(ctx, d_sigma, d_rgb, d_geo, d_sem):
        enc2, hb, hg, h1, rgb, sigma, wb0, wb1, w0, w1, w2 = ctx.saved_tensors
        samples, n_ray_cols, n_feat, enc_shape, ld_enc, head = ctx.meta
        n3, k_enc = enc2.shape
        n = n3 // 3
        dev = enc2.device
        f32 = dict(dtype=torch.float32, device=dev)
        if d_sigma is None and d_rgb is None and d_geo is None and d_sem is None:
            return (None,) * 11
        n_rays = (n + samples - 1) // samples
        w1hg = torch.cat([w1[:, :64], w1[:, 64 + n_ray_cols:]], dim=1)            # [64, 128] = [hidden | geo] columns
        w0g = w0[:, n_ray_cols:].contiguous()
        c = lambda g, w: None if g is None else _f32c(g.reshape(n, w))
        d_geo, d_sem = c(d_geo, 64), c(d_sem, 64)
        d_rgb2 = c(d_rgb, 3) if head else None
        d_sig = None if d_sigma is None else _f32c(d_sigma).reshape(n)
        D1 = torch.empty((n3, 128), **f32)         # rows [0, n): [dZ0 | dF_c]; rows [n, 3n): [unused | dF_f, dF_b]
        dz2 = torch.empty((n, 3), **f32) if d_rgb2 is not None else None
        dz1 = torch.empty((n, 64), **f32) if head else None
        dzb = torch.empty((n3, 64), **f32)
        d_enc = torch.empty((n3, k_enc), **f32) if ctx.needs_input_grad[0] else None
        d_sem_q = torch.empty((n3, 64), **f32) if d_sem is not None else None
        ray_sums = dz2 is not None and samples % 32 == 0
        d_rb = torch.zeros((n_rays, 128), **f32) if ray_sums else None
        _lib.call("emer_flow_field_bwd", _ptr(d_rgb2), _ptr(rgb), _ptr(d_sig), _ptr(sigma), _ptr(d_geo), _ptr(d_sem),
                  _ptr(hb), _ptr(hg if head else None), _ptr(h1), _ptr(wb0), k_enc, _ptr(wb1), n_feat, _ptr(w0g), 64,
                  _ptr(w1hg), _ptr(w1hg[:, 64:]), 128, _ptr(w2), _ptr(dz2), _ptr(dz1), _ptr(D1), _ptr(dzb), _ptr(d_enc),
                  k_enc, _ptr(d_rb), _ptr(d_sem_q), samples, n, _stream())
        if dz2 is not None and not ray_sums:            # ragged rays: the per-ray sums of [dZ0 | dZ1] on the host side
            ray = torch.arange(n, device=dev) // samples
            d_rb = torch.zeros((n_rays, 128), **f32)
            d_rb[:, :64].index_add_(0, ray, D1[:n, :64])
            d_rb[:, 64:].index_add_(0, ray, dz1)

        sk = ctx.sinks
        shapes = dict(wb0=wb0.shape, bb0=(64,), wb1=wb1.shape, bb1=(n_feat,), w0=w0.shape, w1=w1.shape, w2=w2.shape,
                      b2=(3,))
        keys = list(shapes) if dz2 is not None else ["wb0", "bb0", "wb1", "bb1"]
        out, grads = {}, {}
        for k in keys:
            if sk[k] is None:
                out[k] = grads[k] = torch.zeros(shapes[k], **f32)
            else:
                out[k] = sk[k][0]
        o = lambda k: _ptr(out[k]) if k in out else None
        rows = lambda t, r0: None if t is None else t[r0:]

        def wgrad(r0: int, rn: int, with_head: bool):
            if with_head:
                w0g_d, ld_w0, w1g_d, ld_w1 = out["w0"][:, n_ray_cols:], out["w0"].stride(0), out["w1"][:, 64 + n_ray_cols:], out["w1"].stride(0)
                hd = (hg, h1, dz2, dz1)
            else:
                w0g_d, ld_w0, w1g_d, ld_w1 = None, 0, None, 0
                hd = (None, None, None, None)
            _lib.call("emer_field_wgrad", _ptr(enc2[r0:]), ld_enc, k_enc, _ptr(hb[r0:]), _ptr(hd[0]), _ptr(hd[1]),
                      _ptr(hd[2]), _ptr(hd[3]), _ptr(D1[r0:]), _ptr(dzb[r0:]), _ptr(rows(d_sem_q, r0)), n_feat, o("wb0"),
                      o("bb0"), o("wb1"), o("bb1"), _ptr(w0g_d), ld_w0, o("w1") if with_head else None, _ptr(w1g_d),
                      ld_w1, o("w2") if with_head else None, o("b2") if with_head else None, rn, _stream())

        if dz2 is not None:
            wgrad(0, n, True)                           # colour head + base MLP over the current rows
            wgrad(n, 2 * n, False)                      # base MLP over the warped rows
        else:
            wgrad(0, n3, False)
        for k in keys:
            if sk[k] is not None:
                sk[k][1]()
        g = tuple(grads.get(k) for k in ("wb0", "bb0", "wb1", "bb1", "w0", "w1", "w2", "b2"))
        if d_enc is not None:
            d_enc = d_enc.reshape(enc_shape)
        return (d_enc, d_rb, None) + g


def flow_field_chain(enc: Tensor, ray_bias: Optional[Tensor], samples: int, base, head):
    """The three-query chain of the flow variants: ``enc`` [3N, k_enc] stacked [current | forward | backward]
    encodings, ``base`` / ``head`` / ``ray_bias`` as :func:`field_chain`; ``ray_bias`` None: density only.
    Returns (sigma [N], rgb [N, 3] | None, geo [N, 64], sem [N, 64] | None) of the blended features."""
    return _FlowFieldChain.apply(enc, ray_bias, samples, *base, *head)


# ----------------------------------------------------------------------------- sampling
@torch.no_grad()
def pdf_resample(vals: Tensor, cdfs: Tensor, n: int, bias: Optional[Tensor], s_min: float, s_max: float,
                 kind: str, want_bins: bool = False):
    """Inverse-CDF resampling of [R, m1] edges into n intervals; returns (s_edges, t_edges[, bins])."""
    _need_cuda(vals, cdfs)
    vals, cdfs = _f32c(vals), _f32c(cdfs)
    r, m1 = cdfs.shape
    out_s = torch.empty((r, n + 1), dtype=torch.float32, device=vals.device)
    out_t = torch.empty_like(out_s)
    bins = torch.empty((r, n + 1), dtype=torch.int32, device=vals.device) if want_bins else None
    if bias is not None:
        bias = _f32c(bias.reshape(-1))
        if bias.shape[0] != r:
            raise ValueError("bias must have one value per ray")
    _lib.call("emer_pdf_resample", _ptr(vals), _ptr(cdfs), m1, n, _ptr(bias), float(s_min), float(s_max),
              STOT_KINDS[kind], _ptr(out_s), _ptr(out_t), _ptr(bins), r, _stream())
    return (out_s, out_t, bins) if want_bins else (out_s, out_t)


@torch.no_grad()
def prop_level(prev_s: Tensor, prev_cdf: Tensor, n: int, bias: Optional[Tensor], s_min: float, s_max: float, kind: str,
               origins: Tensor, dirs: Tensor, aabb: Tensor, unbounded: bool, desc: GridDesc, table: Tensor,
               w0: Tensor, b0: Tensor, w1: Tensor, b1: Tensor, want_sigma: bool = False):
    """One proposal level in one launch (no autograd): returns (s_edges, t_edges, cdf), each [R, n+1] -- and, with
    ``want_sigma``, the level's densities [R, n] (what ``emer_prop_level_bwd`` starts from)."""
    _need_cuda(prev_s, prev_cdf, origins, dirs, table)
    prev_s, prev_cdf = _f32c(prev_s), _f32c(prev_cdf)
    r, m1 = prev_cdf.shape
    dev = prev_s.device
    out_s = torch.empty((r, n + 1), dtype=torch.float32, device=dev)
    out_t = torch.empty_like(out_s)
    out_cdf = torch.empty_like(out_s)
    sigma = torch.empty((r, n), dtype=torch.float32, device=dev) if want_sigma else None
    if bias is not None:
        bias = _f32c(bias.reshape(-1))
    # every converted tensor is bound to a local that outlives the launch: a temporary copy made by _f32c would be
    # freed (and its block reused by the next temporary) before the kernel is even enqueued
    o, d, box = _f32c(origins), _f32c(dirs), _f32c(aabb.reshape(-1))
    tab, w0c, b0c, w1c, b1c = _f32c(table), _f32c(w0), _f32c(b0), _f32c(w1.reshape(-1)), _f32c(b1.reshape(-1))
    if o.shape != (r, 3) or d.shape != (r, 3):
        raise ValueError(f"prop_level: origins / dirs must be [{r}, 3], got {tuple(o.shape)} / {tuple(d.shape)}")
    _lib.call("emer_prop_level", ctypes.byref(desc.c), _ptr(prev_s), _ptr(prev_cdf), m1, n, _ptr(bias), float(s_min),
              float(s_max), STOT_KINDS[kind], _ptr(o), _ptr(d), _ptr(box), int(unbounded), _ptr(tab), _ptr(w0c),
              _ptr(b0c), _ptr(w1c), _ptr(b1c), _ptr(out_s), _ptr(out_t), _ptr(out_cdf), _ptr(sigma), r, _stream())
    if want_sigma:
        return out_s, out_t, out_cdf, sigma
    return out_s, out_t, out_cdf


class _PropLevelTrain(torch.autograd.Function):
    """A proposal level on the steps that update the proposal networks: the same single launch as the no-grad steps
    forward (so both kinds of step draw bit-identical samples), and a backward that is one launch for the MLP
    (``emer_prop_level_bwd``: recomputes the grid features and hidden units instead of saving [N, 64] activations) plus
    the grid scatter.  Only ``cdf`` carries gradient (the sample positions are drawn without,
    third_party/nerfacc_prop_net.py:147-170 of the reference)."""

    @staticmethod
    def forward(ctx, table, w0, b0, w1, b1, prev_s, prev_cdf, n, bias, s_min, s_max, kind, origins, dirs, aabb,
                unbounded, desc):
        out_s, out_t, out_cdf, sigma = prop_level(prev_s, prev_cdf, n, bias, s_min, s_max, kind, origins, dirs, aabb,
                                                  unbounded, desc, table, w0, b0, w1, b1, want_sigma=True)
        ctx.save_for_backward(table, w0, b0, w1, b1, out_t, sigma, origins, dirs, aabb)
        ctx.desc, ctx.unbounded, ctx.n = desc, bool(unbounded), n
        ctx.sinks = [_grad_sink(t) for t in (table, w0, b0, w1, b1)]
        ctx.mark_non_differentiable(out_s, out_t)
        return out_s, out_t, out_cdf

    @staticmethod
    def backward(ctx, _ds, _dt, d_cdf):
        table, w0, b0, w1, b1, t_edges, sigma, origins, dirs, aabb = ctx.saved_tensors
        desc, n = ctx.desc, ctx.n
        r = t_edges.shape[0]
        dev = t_edges.device
        none = (None,) * 12
        if d_cdf is None:
            return (None,) * 5 + none
        _need_cuda(d_cdf, table)
        d_cdf = _f32c(d_cdf)
        lf = desc.n_output_dims
        xc = torch.empty((r * n, 3), dtype=torch.float32, device=dev)
        d_enc = torch.empty((r * n, lf), dtype=torch.float32, device=dev)
        outs = []
        for t, sink in zip((table, w0, b0, w1, b1), ctx.sinks):
            if sink is not None:
                outs.append(sink[0])
            else:
                outs.append(torch.zeros(t.shape, dtype=torch.float32, device=dev))
        d_table, d_w0, d_b0, d_w1, d_b1 = outs
        tsink = ctx.sinks[0]
        if tsink is not None and tsink[2] is not None and not tsink[2]():
            d_table.zero_()                    # L2 write-allocate before the scatter (see _GridEncode.backward)
        o, d, box = _f32c(origins), _f32c(dirs), _f32c(aabb.reshape(-1))
        tab, w0c, b0c, w1c = _f32c(table), _f32c(w0), _f32c(b0), _f32c(w1.reshape(-1))
        _lib.call("emer_prop_level_bwd", ctypes.byref(desc.c), _ptr(t_edges), _ptr(sigma), _ptr(d_cdf), n, _ptr(o), _ptr(d),
                  _ptr(box), int(ctx.unbounded), _ptr(tab), _ptr(w0c), _ptr(b0c), _ptr(w1c), _ptr(xc), _ptr(d_enc),
                  _ptr(d_w0), _ptr(d_b0), _ptr(d_w1), _ptr(d_b1), r, _stream())
        _lib.call("emer_grid_bwd", ctypes.byref(desc.c), _ptr(xc), _ptr(tab), _ptr(d_enc), _ptr(d_table), None, r * n,
                  _stream())
        grads = []
        for g, sink in zip(outs, ctx.sinks):
            if sink is not None:
                sink[1]()
                grads.append(None)
            else:
                grads.append(g)
        return tuple(grads) + none


def prop_level_train_usable(desc: GridDesc) -> bool:
    return PROP_TRAIN == "fused" and desc.n_dims == 3 and desc.n_feat == 1 and desc.n_output_dims in (4, 8)


def prop_level_train(prev_s: Tensor, prev_cdf: Tensor, n: int, bias: Optional[Tensor], s_min: float, s_max: float,
                     kind: str, origins: Tensor, dirs: Tensor, aabb: Tensor, unbounded: bool, desc: GridDesc,
                     table: Tensor, w0: Tensor, b0: Tensor, w1: Tensor, b1: Tensor):
    """(s_edges, t_edges, cdf) of one proposal level, ``cdf`` differentiable w.r.t. the table and the MLP."""
    return _PropLevelTrain.apply(table, w0, b0, w1, b1, prev_s, prev_cdf, n, bias, s_min, s_max, kind, origins, dirs,
                                 aabb, unbounded, desc)


# ----------------------------------------------------------------------------- interlevel (proposal) loss
INTERLEVEL = os.environ.get("EMER_INTERLEVEL", "fused")       # "torch": the op-by-op restatement in nerfacc_prop_net.py


class _InterlevelLoss(torch.autograd.Function):
    """mean_k max(dq_k - dP_k, 0)^2 / (dP_k + 1e-5) of one proposal level against the blurred final-level histogram
    (third_party/nerfacc_prop_net.py:182-240 of the reference); differentiable w.r.t. the level's CDF only -- the
    target is detached there too."""

    @staticmethod
    def forward(ctx, prop_cdf: Tensor, s: Tensor, cdf: Tensor, prop_s: Tensor, pulse_width: float):
        _need_cuda(prop_cdf, s, cdf, prop_s)
        pc, sc, cc, ps = _f32c(prop_cdf), _f32c(s), _f32c(cdf), _f32c(prop_s)
        r, m = sc.shape
        n1 = pc.shape[1]
        total = torch.zeros(1, dtype=torch.float32, device=pc.device)
        grad = torch.empty_like(pc) if ctx.needs_input_grad[0] else None
        _lib.call("emer_interlevel_loss", _ptr(sc), _ptr(cc), m, _ptr(ps), _ptr(pc), n1, float(pulse_width), _ptr(total),
                  _ptr(grad), r, _stream())
        ctx.count = float(r * (n1 - 1))
        if grad is not None:
            ctx.save_for_backward(grad)
        return (total / ctx.count).reshape(())

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * (g / ctx.count), None, None, None, None


def interlevel_loss_usable(s: Tensor, prop_s: Tensor) -> bool:
    return (INTERLEVEL == "fused" and on_device(s) and s.dim() == 2 and prop_s.dim() == 2 and 2 <= s.shape[1] <= 129
            and 2 <= prop_s.shape[1] <= 257)


def interlevel_loss(s: Tensor, cdf: Tensor, prop_s: Tensor, prop_cdf: Tensor, pulse_width: float) -> Tensor:
    if cdf.shape != s.shape or prop_cdf.shape != prop_s.shape or prop_s.shape[0] != s.shape[0]:
        raise ValueError(f"interlevel_loss: edges / cdf shapes {tuple(s.shape)} {tuple(cdf.shape)} "
                         f"{tuple(prop_s.shape)} {tuple(prop_cdf.shape)}")
    return _InterlevelLoss.apply(prop_cdf, s, cdf.detach(), prop_s, pulse_width)


# ----------------------------------------------------------------------------- embedding rows
class _GatherRows(torch.autograd.Function):
    """``table[idx]`` for a small table hit by many repeated indices (the appearance embedding: 8192 rays over a few
    hundred rows).  The backward of torch's advanced indexing / nn.Embedding sorts the indices first -- a 64-bit radix
    sort, ~12 launches; one pass of atomic adds needs neither."""

    @staticmethod
    def forward(ctx, table: Tensor, idx: Tensor):
        ctx.save_for_backward(idx)
        ctx.rows = table.shape
        return table.index_select(0, idx)

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        out = torch.zeros(ctx.rows, dtype=g.dtype, device=g.device)
        out.index_add_(0, idx, g.contiguous())
        return out, None


def gather_rows(table: Tensor, idx: Tensor) -> Tensor:
    return _GatherRows.apply(table, idx.reshape(-1).long())


# ----------------------------------------------------------------------------- volume rendering
class _Composite(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t0: Tensor, t1: Tensor, sigma: Tensor, want_cdf: bool):
        _need_cuda(t0, t1, sigma)
        t0, t1, sigma = _f32c(t0), _f32c(t1), _f32c(sigma)
        r, s = sigma.shape
        dev = sigma.device
        weights = torch.empty((r, s), dtype=torch.float32, device=dev)
        trans = torch.empty_like(weights)
        opacity = torch.empty((r, 1), dtype=torch.float32, device=dev)
        depth = torch.empty_like(opacity)
        median = torch.empty_like(opacity)
        cdf = torch.empty((r, s + 1), dtype=torch.float32, device=dev) if want_cdf else None
        _lib.call("emer_composite_fwd", _ptr(t0), _ptr(t1), _ptr(sigma), _ptr(weights), _ptr(trans), _ptr(opacity),
                  _ptr(depth), _ptr(median), _ptr(cdf), r, s, _stream())
        ctx.save_for_backward(t0, t1, sigma, weights, trans)
        ctx.mark_non_differentiable(median)
        if cdf is None:
            cdf = torch.empty(0, device=dev)
            ctx.mark_non_differentiable(cdf)
        ctx.want_cdf = want_cdf
        return weights, trans, opacity, depth, median, cdf

    @staticmethod
    def backward(ctx, g_w, g_t, g_o, g_d, _g_m, g_cdf):
        t0, t1, sigma, weights, trans = ctx.saved_tensors
        r, s = sigma.shape
        if ctx.want_cdf and g_cdf is not None:
            # cdf[:, :S] = 1 - trans  ->  d trans -= g_cdf[:, :S]
            extra = -g_cdf[:, :s]
            g_t = extra if g_t is None else g_t + extra
        if g_w is None and g_t is None and g_o is None and g_d is None:
            return None, None, None, None
        c = lambda g: None if g is None else _f32c(g)
        g_w, g_t, g_o, g_d = c(g_w), c(g_t), c(g_o), c(g_d)
        dsigma = torch.empty_like(sigma)
        _lib.call("emer_composite_bwd", _ptr(t0), _ptr(t1), _ptr(sigma), _ptr(weights), _ptr(trans), _ptr(g_w),
                  _ptr(g_t), _ptr(g_o), _ptr(g_d), _ptr(dsigma), r, s, _stream())
        return None, None, dsigma, None


def composite(t0: Tensor, t1: Tensor, sigma: Tensor, want_cdf: bool = False):
    """weights, trans [R,S]; opacity, depth, median_depth [R,1]; cdf [R,S+1] (or an empty tensor)."""
    return _Composite.apply(t0, t1, sigma, want_cdf)


ACC_MAX_CHANNELS = 256          # csrc/composite.cu: 32 lanes x ACC_MAX_PER_LANE


class _Accumulate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, w: Tensor, v: Tensor):
        ctx.set_materialize_grads(False)
        _need_cuda(w, v)
        w, v = _f32c(w), _f32c(v)
        r, s = w.shape
        c = v.shape[-1]
        out = torch.empty((r, c), dtype=torch.float32, device=w.device)
        _lib.call("emer_accumulate_fwd", _ptr(w), _ptr(v), _ptr(out), r, s, c, _stream())
        ctx.save_for_backward(w, v)
        return out

    @staticmethod
    def backward(ctx, g):
        if g is None:
            return None, None
        w, v = ctx.saved_tensors
        r, s = w.shape
        c = v.shape[-1]
        g = _f32c(g)
        dw = torch.empty_like(w) if ctx.needs_input_grad[0] else None
        dv = torch.empty_like(v) if ctx.needs_input_grad[1] else None
        _lib.call("emer_accumulate_bwd", _ptr(w), _ptr(v), _ptr(g), _ptr(dw), _ptr(dv), r, s, c, _stream())
        return dw, dv


def accumulate(w: Tensor, v: Tensor) -> Tensor:
    """sum_s w[R,S] * v[R,S,C] -> [R,C]."""
    if v.dim() == 2:
        v = v.unsqueeze(-1)
    if v.shape[:2] != w.shape:
        raise ValueError(f"accumulate: weights {tuple(w.shape)} vs values {tuple(v.shape)}")
    if v.shape[-1] > ACC_MAX_CHANNELS:
        # one launch handles up to 256 channels (a warp per ray, 8 per lane); wider features go in slices
        return torch.cat([_Accumulate.apply(w, v[..., c:c + ACC_MAX_CHANNELS])
                          for c in range(0, v.shape[-1], ACC_MAX_CHANNELS)], dim=-1)
    return _Accumulate.apply(w, v)


# ----------------------------------------------------------------------------- the body of `rendering` (csrc/render.cu)
# differentiable inputs of emer_render_* (per sample: [R,S] or [R,S,3|C]; per ray: rgb_sky [R,3], dino_sky / dino_pe
# [R,C]) and the outputs a training pass can differentiate; every other output is evaluation-only
RENDER_INPUTS = ("sigma", "sigma_s", "sigma_d", "rgb", "rgb_s", "rgb_d", "shadow", "rgb_sky", "dino", "dino_s", "dino_d",
                 "dino_sky", "dino_pe")
RENDER_TRAIN_OUTPUTS = ("weights", "trans", "opacity", "depth", "median_depth", "rgb", "shadow_ratio", "dino",
                        "dino_pe_free")
RENDER_DECOMPOSITION = ("static_opacity", "dynamic_opacity", "static_depth", "dynamic_depth", "static_rgb",
                        "dynamic_rgb", "shadow_reduced_static_rgb", "shadow_only_static_rgb", "shadow", "forward_flow",
                        "backward_flow", "static_dino", "dynamic_dino")
RENDER_MAX_CHANNELS = 256       # csrc/render.cu: 32 lanes x RENDER_MAX_PER_LANE


def _render_in(t0: Tensor, t1: Tensor, ins: Dict[str, Tensor], flows) -> "_lib.EmerRenderIn":
    r, s = ins["sigma"].shape
    dino = ins.get("dino") if ins.get("dino") is not None else ins.get("dino_s")
    c = _lib.EmerRenderIn(t0=t0.data_ptr(), t1=t1.data_ptr(), n_rays=r, n_samples=s,
                          n_dino=0 if dino is None else dino.shape[-1], ld_flow=3)
    for k in RENDER_INPUTS:
        if ins.get(k) is not None:
            setattr(c, k, ins[k].data_ptr())
    if flows is not None:
        (f, ld), (b, _) = flows
        c.fwd_flow, c.bwd_flow, c.ld_flow = f.data_ptr(), b.data_ptr(), ld
    return c


def _render_fwd(t0: Tensor, t1: Tensor, ins: Dict[str, Tensor], flows, decomposition: bool) -> Dict[str, Tensor]:
    """One emer_render_fwd launch; returns every output the inputs define (the decomposition when asked for)."""
    r, s = ins["sigma"].shape
    dev = ins["sigma"].device
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)    # noqa: E731
    two = ins.get("sigma_s") is not None
    blend_rgb = ins.get("rgb") is None and ins.get("rgb_s") is not None
    dino = ins.get("dino") if ins.get("dino") is not None else ins.get("dino_s")
    out = {"weights": new(r, s), "trans": new(r, s), "opacity": new(r, 1), "depth": new(r, 1),
           "median_depth": new(r, 1)}
    if ins.get("rgb") is not None or blend_rgb:
        out["rgb"] = new(r, 3)
    if ins.get("shadow") is not None and blend_rgb:
        out["shadow_ratio"] = new(r, 1)
    if dino is not None:
        c = dino.shape[-1]
        out["dino"] = new(r, c)
        if ins.get("dino_pe") is not None:
            out["dino_pe_free"] = new(r, c)
    if decomposition and two:
        for k in ("static_opacity", "dynamic_opacity", "static_depth", "dynamic_depth"):
            out[k] = new(r, 1)
        if blend_rgb:
            out["static_rgb"], out["dynamic_rgb"] = new(r, 3), new(r, 3)
            if ins.get("shadow") is not None:
                out["shadow_reduced_static_rgb"], out["shadow_only_static_rgb"] = new(r, 3), new(r, 3)
                out["shadow"] = new(r, 1)
            if flows is not None:
                out["forward_flow"], out["backward_flow"] = new(r, 3), new(r, 3)
        if ins.get("dino") is None and ins.get("dino_s") is not None:
            out["static_dino"], out["dynamic_dino"] = new(r, dino.shape[-1]), new(r, dino.shape[-1])
    cout = _lib.EmerRenderOut(**{k: v.data_ptr() for k, v in out.items()})
    _lib.call("emer_render_fwd", ctypes.byref(_render_in(t0, t1, ins, flows)), ctypes.byref(cout), _stream())
    return out


class _Render(torch.autograd.Function):
    """The training outputs of emer_render_fwd (RENDER_TRAIN_OUTPUTS, None where the inputs define none) and their
    backward in one emer_render_bwd launch; t0 / t1 are constants, as in _Composite."""

    @staticmethod
    def forward(ctx, t0: Tensor, t1: Tensor, *ins):
        ctx.set_materialize_grads(False)
        named = dict(zip(RENDER_INPUTS, ins))
        out = _render_fwd(t0, t1, named, None, False)
        ctx.save_for_backward(t0, t1, out["weights"], out["trans"], *ins)
        ctx.mark_non_differentiable(out["median_depth"])
        return tuple(out.get(k) for k in RENDER_TRAIN_OUTPUTS)

    @staticmethod
    def backward(ctx, *grads):
        t0, t1, weights, trans, *ins = ctx.saved_tensors
        named = dict(zip(RENDER_INPUTS, ins))
        need = ctx.needs_input_grad[2:]
        if all(g is None for g in grads) or not any(need):
            return (None,) * (2 + len(RENDER_INPUTS))
        g = _lib.EmerRenderGrad()
        upstream = []           # holds the fp32 copies while the struct points at them
        for k, gr in zip(RENDER_TRAIN_OUTPUTS, grads):
            if gr is not None and k != "median_depth":
                upstream.append(_f32c(gr))
                setattr(g, "g_" + k, upstream[-1].data_ptr())
        d = [torch.empty_like(x) if (x is not None and n) else None for x, n in zip(ins, need)]
        for k, dk in zip(RENDER_INPUTS, d):
            if dk is not None:
                setattr(g, "d_" + k, dk.data_ptr())
        _lib.call("emer_render_bwd", ctypes.byref(_render_in(t0, t1, named, None)), _ptr(weights), _ptr(trans),
                  ctypes.byref(g), _stream())
        return (None, None, *d)


def render_usable(n_channels: int) -> bool:
    return n_channels <= RENDER_MAX_CHANNELS


def render(t0: Tensor, t1: Tensor, ins: Dict[str, Optional[Tensor]], flows=None,
           decomposition: bool = False) -> Dict[str, Tensor]:
    """The body of ``rendering`` in one emer_render_fwd launch (and one emer_render_bwd in the backward).

    ``ins``: the RENDER_INPUTS present (the rest None or missing), sigma / sigma_s / sigma_d / shadow [R,S], rgb /
    rgb_s / rgb_d [R,S,3], dino / dino_s / dino_d [R,S,C], rgb_sky [R,3], dino_sky / dino_pe [R,C].  ``flows``:
    (forward, backward) [R,S,3] flows, read in place when they are column slices of wider rows; only the decomposition
    uses them.  Returns the RENDER_TRAIN_OUTPUTS the inputs define (opacity, depth, median_depth, rgb, shadow_ratio
    [R,1] or [R,3]; dino, dino_pe_free [R,C]) and, with ``decomposition``, the RENDER_DECOMPOSITION outputs, which
    have no gradient: ask for them only where nothing needs one."""
    sigma = ins["sigma"]
    if sigma.dim() != 2:
        raise ValueError(f"render: sigma must be [R, S], got {tuple(sigma.shape)}")
    r, s = sigma.shape
    _need_cuda(t0, t1, *[v for v in ins.values() if v is not None], *(flows or ()))
    shapes = {"sigma_s": (r, s), "sigma_d": (r, s), "shadow": (r, s), "rgb": (r, s, 3), "rgb_s": (r, s, 3),
              "rgb_d": (r, s, 3), "rgb_sky": (r, 3)}
    cins = {}
    for k in RENDER_INPUTS:
        v = ins.get(k)
        if v is None:
            continue
        if k in ("shadow", "sigma_s", "sigma_d") and v.dim() == 3:
            v = v.squeeze(-1)
        want = shapes.get(k)
        if k in ("dino", "dino_s", "dino_d"):
            want = (r, s, v.shape[-1])
        elif k in ("dino_sky", "dino_pe"):
            want = (r, v.shape[-1])
        if want is not None and tuple(v.shape) != want:
            raise ValueError(f"render: {k} must be {want}, got {tuple(v.shape)}")
        cins[k] = _f32c(v)
    for a, b in (("sigma_s", "sigma_d"), ("rgb_s", "rgb_d"), ("dino_s", "dino_d")):
        if (a in cins) != (b in cins):
            raise ValueError(f"render: {a} and {b} come together")
    if ("rgb_s" in cins or "dino_s" in cins) and "sigma_s" not in cins:
        raise ValueError("render: static / dynamic colours or features need static and dynamic densities")
    dino = cins.get("dino", cins.get("dino_s"))
    c = 0 if dino is None else dino.shape[-1]
    for k in ("dino_s", "dino_d", "dino_sky", "dino_pe"):
        if k in cins and cins[k].shape[-1] != c:
            raise ValueError(f"render: {k} has {cins[k].shape[-1]} channels, the features {c}")
    if not 0 <= c <= RENDER_MAX_CHANNELS:
        raise ValueError(f"render: {c} feature channels (at most {RENDER_MAX_CHANNELS})")
    t0, t1 = _f32c(t0), _f32c(t1)
    if decomposition:
        if torch.is_grad_enabled() and any(v.requires_grad for v in ins.values() if v is not None):
            raise ValueError("render: the decomposition outputs have no gradient; ask for them without grad")
        rows = None
        if flows is not None:
            rows = [_rows(f, 3) for f in flows]
            if rows[0][1] != rows[1][1] or rows[0][0].shape[0] != r * s:
                rows = [(_f32c(f).reshape(-1, 3), 3) for f in flows]
        return _render_fwd(t0, t1, cins, rows, True)
    outs = _Render.apply(t0, t1, *[cins.get(k) for k in RENDER_INPUTS])
    return {k: v for k, v in zip(RENDER_TRAIN_OUTPUTS, outs) if v is not None}


# ----------------------------------------------------------------------------- training losses (csrc/losses.cu)
LOSS_KINDS = {"l1": 0, "l2": 1, "smooth_l1": 2, "depth_l1": 3, "depth_l2": 4, "depth_smooth_l1": 5, "sky_bce": 6,
              "sparsity": 7, "entropy": 8}
RAY_LOSS_KINDS = {"line_of_sight": 0, "sky_weights": 1, "sight": 2}
LOSS_WORKSPACE_BYTES = 16384    # EMER_LOSS_WORKSPACE_BYTES
_LOSS_WS: Dict[object, Tensor] = {}


def _workspace(cache: Dict[object, Tensor], dev: torch.device, nbytes: int, what: str) -> Tensor:
    """The device's entry of ``cache`` (one per kernel family: losses, metrics, occupancy): a workspace zeroed once and
    left zeroed by every call (the last CTA resets its ticket), so it is shared by all of the family's calls on the
    device's stream and by graph replays.  Created outside graph capture."""
    ws = cache.get(dev)
    if ws is None:
        if dev.type == "cuda" and torch.cuda.is_current_stream_capturing():
            raise RuntimeError(f"emernerf_b200 {what}: run each call once before capturing it in a CUDA graph")
        ws = torch.zeros(nbytes // 4, dtype=torch.int32, device=dev)
        cache[dev] = ws
    return ws


class _PointwiseLoss(torch.autograd.Function):
    """post * mean(pre * term(a, b)) for one of LOSS_KINDS; b is a constant (target / mask) except for the entropy
    loss, where it is the static density and gets a gradient."""

    @staticmethod
    def forward(ctx, a: Tensor, b: Optional[Tensor], kind: int, p0: float, p1: float, pre: float, post: float):
        ctx.set_materialize_grads(False)
        _need_cuda(a, b)
        ac = _f32c(a)
        bc = None if b is None else _f32c(b)
        if bc is not None and bc.numel() != ac.numel():
            raise ValueError(f"pointwise loss: {tuple(a.shape)} vs {tuple(b.shape)}")
        out = torch.empty(2, dtype=torch.float32, device=ac.device)
        _lib.call("emer_pointwise_loss_fwd", kind, _ptr(ac), _ptr(bc), ac.numel(), p0, p1, pre, post, _ptr(out),
                  _ptr(_workspace(_LOSS_WS, ac.device, LOSS_WORKSPACE_BYTES, "losses")), _stream())
        ctx.save_for_backward(ac, bc, out)
        ctx.args = (kind, p0, p1, pre, post)
        ctx.shapes = (a.shape, None if b is None else b.shape)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        need_a = ctx.needs_input_grad[0]
        need_b = ctx.needs_input_grad[1] and ctx.args[0] == LOSS_KINDS["entropy"]
        if g is None or not (need_a or need_b):
            return None, None, None, None, None, None, None
        a, b, out = ctx.saved_tensors
        kind, p0, p1, pre, post = ctx.args
        da = torch.empty_like(a) if need_a else None
        db = torch.empty_like(b) if need_b else None
        _lib.call("emer_pointwise_loss_bwd", kind, _ptr(a), _ptr(b), a.numel(), p0, p1, pre, post, _ptr(out),
                  _ptr(_f32c(g)), _ptr(da), _ptr(db), _stream())
        return (None if da is None else da.view(ctx.shapes[0]), None if db is None else db.view(ctx.shapes[1]),
                None, None, None, None, None)


def pointwise_loss(kind: str, a: Tensor, b: Optional[Tensor], p0: float = 0.0, p1: float = 0.0, pre: float = 1.0,
                   post: float = 1.0) -> Tensor:
    """0-d loss value; see EMER_LOSS_* in include/emer_b200.h for what ``kind`` computes and what p0 / p1 are."""
    return _PointwiseLoss.apply(a, b, LOSS_KINDS[kind], float(p0), float(p1), float(pre), float(post))


class _RayLoss(torch.autograd.Function):
    """Per-ray sums over [R, S] rows (EMER_RAY_LOSS_*); differentiable w.r.t. the weights only."""

    @staticmethod
    def forward(ctx, w: Tensor, t: Optional[Tensor], gt: Tensor, kind: int, consts: Tuple[float, float, float],
                pre: float, post: float):
        ctx.set_materialize_grads(False)
        _need_cuda(w, t, gt)
        wc, gc = _f32c(w), _f32c(gt)
        tc = None if t is None else _f32c(t)
        r, s = wc.shape
        if gc.numel() != r or (tc is not None and tc.shape != wc.shape):
            raise ValueError(f"ray loss: weights {tuple(w.shape)}, t {None if t is None else tuple(t.shape)}, "
                             f"per-ray {tuple(gt.shape)}")
        out = torch.empty(2, dtype=torch.float32, device=wc.device)
        _lib.call("emer_ray_loss_fwd", kind, _ptr(wc), _ptr(tc), _ptr(gc), r, s, *consts, pre, post, _ptr(out),
                  _ptr(_workspace(_LOSS_WS, wc.device, LOSS_WORKSPACE_BYTES, "losses")), _stream())
        ctx.save_for_backward(wc, tc, gc, out)
        ctx.args = (kind, consts, pre, post)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        if g is None or not ctx.needs_input_grad[0]:
            return None, None, None, None, None, None, None
        w, t, gt, out = ctx.saved_tensors
        kind, consts, pre, post = ctx.args
        dw = torch.empty_like(w)
        _lib.call("emer_ray_loss_bwd", kind, _ptr(w), _ptr(t), _ptr(gt), w.shape[0], w.shape[1], *consts, pre, post,
                  _ptr(out), _ptr(_f32c(g)), _ptr(dw), _stream())
        return dw, None, None, None, None, None, None


def _sight_consts(epsilon: float) -> Tuple[float, float, float]:
    """(epsilon, 2 sigma^2, 1 / sqrt(2 pi sigma^2)), sigma = epsilon / 3, in double as the reference's Python forms
    them; ctypes rounds each once to fp32, as torch rounds a Python scalar."""
    sigma = float(epsilon) / 3
    return float(epsilon), 2 * sigma**2, 1 / (math.sqrt(2 * math.pi * sigma**2))


def line_of_sight_loss(weights: Tensor, t_vals: Tensor, gt_depth: Tensor, epsilon: float, pre: float = 1.0,
                       post: float = 1.0) -> Tensor:
    """post * mean(pre * compute_line_of_sight_loss(gt_depth, weights, t_vals, epsilon)); t_vals and gt_depth are
    constants."""
    return _RayLoss.apply(weights, t_vals.detach(), gt_depth.detach(), RAY_LOSS_KINDS["line_of_sight"],
                          _sight_consts(epsilon), float(pre), float(post))


def line_of_sight_sum(weights: Tensor, t_vals: Tensor, gt_depth: Tensor, epsilon: float) -> Tensor:
    """mean_r empty_r + mean_r near_r of compute_line_of_sight_loss (before its ray mask), a 0-d tensor."""
    return _RayLoss.apply(weights, t_vals.detach(), gt_depth.detach(), RAY_LOSS_KINDS["sight"], _sight_consts(epsilon),
                          1.0, 1.0)


def sky_weights_loss(weights: Tensor, sky_mask: Tensor, post: float = 1.0) -> Tensor:
    """post * mean_r(sum_s weights^2 * sky_mask_r)."""
    return _RayLoss.apply(weights, None, sky_mask.detach(), RAY_LOSS_KINDS["sky_weights"], (0.0, 0.0, 0.0), 1.0,
                          float(post))


class _CycleLoss(torch.autograd.Function):
    """coef * 0.5 * mean((f + fpb)^2 + (b + bpf)^2) over [..., 3] flows, and the four maximum row norms
    (emer_cycle_loss_*).  Column slices of wider rows are read in place; f and b are constants."""

    @staticmethod
    def forward(ctx, f: Tensor, b: Tensor, fpb: Tensor, bpf: Tensor, coef: float):
        ctx.set_materialize_grads(False)
        _need_cuda(f, b, fpb, bpf)
        if not (f.shape == b.shape == fpb.shape == bpf.shape) or f.dim() == 0 or f.shape[-1] != 3:
            raise ValueError(f"flow cycle loss: flows of shapes {tuple(f.shape)}, {tuple(b.shape)}, "
                             f"{tuple(fpb.shape)}, {tuple(bpf.shape)}; all must be the same [..., 3]")
        if f.numel() == 0:
            raise ValueError("flow cycle loss: no samples (the maximum flow norms of an empty batch are undefined)")
        rows = [_rows(t, 3) for t in (f, b, fpb, bpf)]
        args = [a for r in rows for a in (_ptr(r[0]), r[1])]
        n = rows[0][0].shape[0]
        out = torch.empty(6, dtype=torch.float32, device=rows[0][0].device)
        _lib.call("emer_cycle_loss_fwd", *args, n, coef, _ptr(out),
                  _ptr(_workspace(_LOSS_WS, out.device, LOSS_WORKSPACE_BYTES, "losses")), _stream())
        ctx.save_for_backward(*(r[0] for r in rows), out)
        ctx.lds = [r[1] for r in rows]
        ctx.coef, ctx.shape = coef, fpb.shape
        stats = out[2:]
        ctx.mark_non_differentiable(stats)
        return out[0], stats

    @staticmethod
    def backward(ctx, g, _g_stats):
        need_fpb, need_bpf = ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        if g is None or not (need_fpb or need_bpf):
            return None, None, None, None, None
        f, b, fpb, bpf, out = ctx.saved_tensors
        n = f.shape[0]
        d_fpb = torch.empty(n, 3, dtype=torch.float32, device=f.device) if need_fpb else None
        d_bpf = torch.empty(n, 3, dtype=torch.float32, device=f.device) if need_bpf else None
        args = [a for t, ld in zip((f, b, fpb, bpf), ctx.lds) for a in (_ptr(t), ld)]
        _lib.call("emer_cycle_loss_bwd", *args, n, ctx.coef, _ptr(out), _ptr(_f32c(g)), _ptr(d_fpb), _ptr(d_bpf),
                  _stream())
        view = lambda d: None if d is None else d.view(ctx.shape)
        return None, None, view(d_fpb), view(d_bpf), None


def cycle_loss(forward_flow: Tensor, backward_flow: Tensor, forward_pred_backward_flow: Tensor,
               backward_pred_forward_flow: Tensor, coef: float) -> Tuple[Tensor, Tensor]:
    """(0-d loss value, [4] maximum row norms of the four flows in argument order; no gradient)."""
    return _CycleLoss.apply(forward_flow.detach(), backward_flow.detach(), forward_pred_backward_flow,
                            backward_pred_forward_flow, float(coef))
