"""The layer's dense transform `x W^T (+ b)` (reference: nn/dense/linear.py:121-127, F.linear).

Two back ends, same fp32-level accuracy:
  * "tf32x3" (default on shapes it supports): the hand-written wgmma/TMA 3xTF32 GEMMs of
    csrc/gemm_tf32x3.cu -- forward, grad-input and the split-K grad-weight product all read x, g
    and W exactly as they lie in HBM; each k-step issues the two correction products of the split as
    one BF16 MMA (bf16(a_lo) bf16(b_hi) + bf16(a_hi) bf16(b_lo)) next to the TF32 a_hi b_hi, still
    fp32-class (at most 2^-17 + 2^-22 of |a b| per term);
  * "cublas": torch.nn.functional.linear in strict fp32 (what the reference runs) -- used for
    shapes outside the kernel's limits (reduction dim % 32, output width in {64,128,256k}) and for
    non-fp32 inputs.  A plain library GEMM, not a fallback of the aggregation path.
`set_backend("cublas")` forces the library path (A/B measurements in bench.py).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from . import ops
from ._lib import check, lib

_BACKEND = "tf32x3"
DEFAULT_GEMM_MODE = 1   # library default of b200mp_set_option("gemm_mode") (accepted; the sm_90a kernel has one configuration)
DEFAULT_GEMM_PREFETCH = 0   # library default of b200mp_set_option("gemm_prefetch") (k-blocks ahead, 0 = off)
_B_SPLIT = False            # True: pass W unsplit and let the kernel split its B tiles (w_lo == NULL in the C ABI)


def set_b_split(on: bool) -> None:
    global _B_SPLIT
    _B_SPLIT = bool(on)


def get_b_split() -> bool:
    return _B_SPLIT


def set_backend(name: str) -> None:
    global _BACKEND
    if name not in ("tf32x3", "cublas"):
        raise ValueError("backend must be 'tf32x3' or 'cublas'")
    _BACKEND = name


def get_backend() -> str:
    return _BACKEND


def _width_ok(n: int) -> bool:
    return n in (64, 128) or (n > 0 and n % 256 == 0)


def supported(x: Tensor, weight: Tensor) -> bool:
    if not (x.is_cuda and x.dtype == torch.float32 and weight.dtype == torch.float32 and x.dim() == 2):
        return False
    n, k = weight.shape
    # forward: K % 32, width N;  grad_input: reduction N % 32, width K;  grad_weight: N % 128, width K
    return k % 32 == 0 and n % 128 == 0 and _width_ok(n) and _width_ok(k) and x.size(0) < 2**31


def split_tf32(w: Tensor):
    w = w.detach().contiguous()
    hi, lo = torch.empty_like(w), torch.empty_like(w)
    ops._timed("split_tf32", 1, lib().b200mp_split_tf32, w.data_ptr(), hi.data_ptr(), lo.data_ptr(), w.numel(), ops._stream())
    return hi, lo


def split_tf32_transposed(w: Tensor):
    """(rn_tf32(w^T), w^T - rn_tf32(w^T)), both [cols, rows] contiguous."""
    w = w.detach().contiguous()
    rows, cols = w.shape
    hi = torch.empty((cols, rows), dtype=w.dtype, device=w.device)
    lo = torch.empty_like(hi)
    ops._timed("split_tf32_transposed", 1, lib().b200mp_split_tf32_transposed, w.data_ptr(), hi.data_ptr(), lo.data_ptr(),
               rows, cols, ops._stream())
    return hi, lo


def prepare_weight(weight: Tensor):
    """(w_hi, w_lo) for the kernels; (w, None) when the kernel splits B tiles itself."""
    n, k = weight.shape
    if _B_SPLIT and n % 128 == 0 and k % 128 == 0:
        return weight.detach().contiguous(), None
    return split_tf32(weight)


def linear_forward(x: Tensor, w_hi: Tensor, w_lo: Optional[Tensor], out: Tensor = None) -> Tensor:
    m, k = x.shape
    n = w_hi.size(0)
    if out is None:
        y = torch.empty((m, n), dtype=torch.float32, device=x.device)
    else:
        if out.shape != (m, n) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError("out must be a contiguous fp32 [M, N] tensor")
        y = out
    ops._timed("linear_tf32x3", 1, lib().b200mp_linear_tf32x3, x.data_ptr(), w_hi.data_ptr(), ops._p(w_lo),
               y.data_ptr(), m, n, k, ops._stream())
    return y


def linear_grad_input(g: Tensor, w_hi: Tensor, w_lo: Optional[Tensor]) -> Tensor:
    m, n = g.shape
    k = w_hi.size(1)
    gx = torch.empty((m, k), dtype=torch.float32, device=g.device)
    ops._timed("linear_grad_input_tf32x3", 1, lib().b200mp_linear_grad_input_tf32x3, g.data_ptr(), w_hi.data_ptr(),
               ops._p(w_lo), gx.data_ptr(), m, n, k, ops._stream())
    return gx


def linear_grad_input_w(g: Tensor, weight: Tensor, w_hi: Tensor, w_lo: Optional[Tensor]) -> Tensor:
    """gx = g W.  Widths that are multiples of 128 split W^T once per call and run the K-major pair form, whose B tiles
    need no transposing in the kernel; other widths (64) read W MN-major.  Both give the same bits."""
    m, n = g.shape
    k = weight.size(1)
    if k % 128 != 0:
        return linear_grad_input(g, w_hi, w_lo)
    wt_hi, wt_lo = split_tf32_transposed(weight)
    gx = torch.empty((m, k), dtype=torch.float32, device=g.device)
    ops._timed("linear_grad_input_tf32x3", 1, lib().b200mp_gemm_pair_tf32x3, g.data_ptr(), n, None, 0, wt_hi.data_ptr(),
               wt_lo.data_ptr(), 0, None, 0, gx.data_ptr(), k, None, 0, m, ops._stream())
    return gx


_WS = {}


def linear_grad_weight(g: Tensor, x: Tensor) -> Tensor:
    m, n = g.shape
    k = x.size(1)
    gw = torch.empty((n, k), dtype=torch.float32, device=g.device)
    nbytes = lib().b200mp_linear_grad_weight_workspace_bytes(m, n, k)
    key = (g.device, nbytes)
    ws = _WS.get(key)
    if ws is None:
        _WS.clear()
        ws = _WS[key] = torch.empty(nbytes, dtype=torch.uint8, device=g.device)
    ops._timed("linear_grad_weight_tf32x3", 2, lib().b200mp_linear_grad_weight_tf32x3, g.data_ptr(), x.data_ptr(),
               gw.data_ptr(), m, n, k, ws.data_ptr(), ws.numel(), ops._stream())
    return gw


def gemm_pair(a1: Tensor, a2: Optional[Tensor], b_hi: Tensor, b_lo: Optional[Tensor], b_layout: int, n1: int, n2: int = 0,
              bias: Optional[Tensor] = None, relu: bool = False, out1: Optional[Tensor] = None):
    """[c1 | c2] = act([a1 | a2] . B + bias) on the wgmma kernel (b200mp_gemm_pair_tf32x3)."""
    m, k1 = a1.shape
    k2 = 0 if a2 is None else a2.size(1)
    c1 = out1 if out1 is not None else torch.empty((m, n1), dtype=torch.float32, device=a1.device)
    c2 = torch.empty((m, n2), dtype=torch.float32, device=a1.device) if n2 else None
    if bias is not None and (bias.dtype != torch.float32 or not bias.is_contiguous()):
        bias = bias.detach().float().contiguous()
    ops._timed("gemm_pair_tf32x3", 1, lib().b200mp_gemm_pair_tf32x3, a1.data_ptr(), k1, ops._p(a2), k2, b_hi.data_ptr(),
               ops._p(b_lo), int(b_layout), ops._p(bias), int(bool(relu)), c1.data_ptr(), n1, ops._p(c2), n2, m, ops._stream())
    return c1, c2


def _pair_ok(x: Tensor, n: int, *ks: int) -> bool:
    return (_BACKEND == "tf32x3" and x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.size(0) > 0
            and n % 128 == 0 and all(k % 32 == 0 for k in ks) and x.size(0) < 2**31)


class _LinearTF32x3(torch.autograd.Function):
    """y = act(x W^T + b): bias (and ReLU) in the GEMM epilogue; backward: mask (ReLU), the two wgmma products and a
    deterministic column sum for the bias."""

    @staticmethod
    def forward(ctx, x: Tensor, weight: Tensor, bias: Optional[Tensor], relu: bool):
        x = x.contiguous()
        w_hi, w_lo = prepare_weight(weight)
        n = weight.size(0)
        if (bias is not None or relu) and n % 128 == 0:
            y, _ = gemm_pair(x, None, w_hi, w_lo, 0, n, bias=None if bias is None else bias.detach(), relu=relu)
        else:
            y = linear_forward(x, w_hi, w_lo)
            if bias is not None:
                y = y + bias
            if relu:
                y = y.relu_()
        ctx.relu, ctx.has_bias = relu, bias is not None
        ctx.save_for_backward(x, weight, w_hi, w_lo, y if relu else None)
        return y

    @staticmethod
    def backward(ctx, g: Tensor):
        x, weight, w_hi, w_lo, y = ctx.saved_tensors
        g = g.contiguous()
        if ctx.relu:
            g = g * (y > 0)
        gx = linear_grad_input_w(g, weight, w_hi, w_lo) if ctx.needs_input_grad[0] else None
        gw = linear_grad_weight(g, x) if ctx.needs_input_grad[1] else None
        gb = ops.column_sum(g) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb, None


def linear(x: Tensor, weight: Tensor, bias=None, relu: bool = False) -> Tensor:
    """act(x W^T + b) with fp32 accuracy; tensor cores where the shape allows (bias / ReLU in the epilogue)."""
    if _BACKEND == "tf32x3" and supported(x, weight):
        return _LinearTF32x3.apply(x, weight, bias, relu)
    y = F.linear(x, weight.to(x.dtype), None if bias is None else bias.to(x.dtype))
    return y.relu() if relu else y


class _LinearPair(torch.autograd.Function):
    """y = act(a W_a^T + b W_b^T + bias) in ONE launch (two A streams into one accumulator); backward: both input
    gradients from one read of g (two outputs of one launch), the weight gradients by the split-K kernel."""

    @staticmethod
    def forward(ctx, a: Tensor, w_a: Tensor, b: Tensor, w_b: Tensor, bias: Optional[Tensor], relu: bool):
        a, b = a.contiguous(), b.contiguous()
        w_hi, w_lo = split_tf32(torch.cat([w_a.detach(), w_b.detach()], dim=1))          # [N, Ka + Kb]
        y, _ = gemm_pair(a, b, w_hi, w_lo, 0, w_a.size(0), bias=None if bias is None else bias.detach(), relu=relu)
        ctx.relu, ctx.has_bias = relu, bias is not None
        ctx.save_for_backward(a, b, w_hi, w_lo, y if relu else None)
        return y

    @staticmethod
    def backward(ctx, g: Tensor):
        a, b, w_hi, w_lo, y = ctx.saved_tensors
        g = g.contiguous()
        if ctx.relu:
            g = g * (y > 0)
        ka, kb = a.size(1), b.size(1)
        ga = gb_ = None
        need_a, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[2]
        if need_a or need_b:
            if ka % 128 == 0 and kb % 128 == 0 and g.size(1) % 32 == 0:
                ga, gb_ = gemm_pair(g, None, w_hi, w_lo, 1, ka, kb)                        # g . [W_a | W_b]
            else:
                ga, gb_ = g @ (w_hi[:, :ka] + w_lo[:, :ka]), g @ (w_hi[:, ka:] + w_lo[:, ka:])
        gwa = _mm_tn(g, a) if ctx.needs_input_grad[1] else None
        gwb = _mm_tn(g, b) if ctx.needs_input_grad[3] else None
        gbias = ops.column_sum(g) if (ctx.has_bias and ctx.needs_input_grad[4]) else None
        return (ga if need_a else None), gwa, (gb_ if need_b else None), gwb, gbias, None


def linear_pair(a: Tensor, w_a: Tensor, b: Tensor, w_b: Tensor, bias: Optional[Tensor] = None, relu: bool = False) -> Tensor:
    """act(a W_a^T + b W_b^T + bias): SAGEConv's lin_l(aggregated) + lin_r(x) (sage_conv.py:134-141)."""
    if _pair_ok(a, w_a.size(0), a.size(1), b.size(1)) and b.dtype == torch.float32 and w_a.dtype == torch.float32:
        return _LinearPair.apply(a, w_a, b, w_b, bias, relu)
    y = F.linear(a, w_a.to(a.dtype), None if bias is None else bias.to(a.dtype)) + F.linear(b, w_b.to(b.dtype))
    return y.relu() if relu else y


def matmul(a: Tensor, w: Tensor) -> Tensor:
    """a [M, K] @ w [K, N] (w row-major), differentiable."""
    return _MM.apply(a, w)


class _MatmulPair(torch.autograd.Function):
    """y = a W_a + b W_b + bias with W_* stored [K, N] (RGCNConv: [H | x] . [W_1;..;W_R; root], rgcn_conv.py:257-280)."""

    @staticmethod
    def forward(ctx, a: Tensor, w_a: Tensor, b: Tensor, w_b: Tensor, bias: Optional[Tensor]):
        a, b = a.contiguous(), b.contiguous()
        w_hi, w_lo = split_tf32(torch.cat([w_a.detach(), w_b.detach()], dim=0))          # [Ka + Kb, N]
        y, _ = gemm_pair(a, b, w_hi, w_lo, 1, w_a.size(1), bias=None if bias is None else bias.detach())
        ctx.has_bias = bias is not None
        ctx.save_for_backward(a, b, w_hi, w_lo)
        return y

    @staticmethod
    def backward(ctx, g: Tensor):
        a, b, w_hi, w_lo = ctx.saved_tensors
        g = g.contiguous()
        ka, kb = a.size(1), b.size(1)
        ga = gb_ = None
        need_a, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[2]
        if need_a or need_b:
            if ka % 128 == 0 and kb % 128 == 0 and g.size(1) % 32 == 0:
                ga, gb_ = gemm_pair(g, None, w_hi, w_lo, 0, ka, kb)                        # g . [W_a; W_b]^T
            else:
                w = w_hi + w_lo
                ga, gb_ = g @ w[:ka].t(), g @ w[ka:].t()
        gwa = _mm_tn(a, g) if ctx.needs_input_grad[1] else None
        gwb = _mm_tn(b, g) if ctx.needs_input_grad[3] else None
        gbias = ops.column_sum(g) if (ctx.has_bias and ctx.needs_input_grad[4]) else None
        return (ga if need_a else None), gwa, (gb_ if need_b else None), gwb, gbias


def matmul_pair(a: Tensor, w_a: Tensor, b: Tensor, w_b: Tensor, bias: Optional[Tensor] = None) -> Tensor:
    """a W_a + b W_b + bias for row-major [K, N] weights, one launch when the widths are on the kernel's grid."""
    if _pair_ok(a, w_a.size(1), a.size(1), b.size(1)) and b.dtype == torch.float32 and w_a.dtype == torch.float32:
        return _MatmulPair.apply(a, w_a, b, w_b, bias)
    y = _MM.apply(a, w_a) + _MM.apply(b, w_b)
    return y if bias is None else y + bias.to(y.dtype)


# ---------------------------------------------------------------------------------------------- segment / grouped matmul
def _mm(a: Tensor, b: Tensor) -> Tensor:
    """a [M, K] @ b [K, N] (b row-major, as it lies in memory) -- the 3xTF32 wgmma kernel where the shape allows."""
    k, n = b.shape
    if (_BACKEND == "tf32x3" and a.is_cuda and a.dtype == torch.float32 and b.dtype == torch.float32 and a.size(0) > 0
            and k % 32 == 0 and _width_ok(n) and a.size(0) < 2**31):
        w_hi, w_lo = split_tf32(b)
        return linear_grad_input(a.contiguous(), w_hi, w_lo)             # g[M,"N"=k] . w["N"=k, "K"=n]
    return a @ b.to(a.dtype)


def _mm_nt(a: Tensor, b: Tensor) -> Tensor:
    """a [M, N] @ b[K, N]^T."""
    k, n = b.shape
    if (_BACKEND == "tf32x3" and a.is_cuda and a.dtype == torch.float32 and b.dtype == torch.float32 and a.size(0) > 0
            and n % 32 == 0 and _width_ok(k) and a.size(0) < 2**31):
        w_hi, w_lo = split_tf32(b)
        return linear_forward(a.contiguous(), w_hi, w_lo)
    return a @ b.to(a.dtype).t()


def _mm_tn(a: Tensor, b: Tensor) -> Tensor:
    """a [M, K]^T @ b [M, N] -> [K, N] (deterministic split-K kernel where the shape allows)."""
    m, k = a.shape
    n = b.size(1)
    if (_BACKEND == "tf32x3" and a.is_cuda and a.dtype == torch.float32 and b.dtype == torch.float32 and m > 0
            and k % 128 == 0 and _width_ok(n) and m < 2**31):
        return linear_grad_weight(a.contiguous(), b.contiguous())       # g = a ["N" = k], x = b ["K" = n]
    return a.t() @ b


def _grouped(a: Tensor, ptr: Tensor, w_hi: Tensor, w_lo: Tensor, b_layout: int, n_out: int) -> Tensor:
    m, k = a.shape
    c = torch.empty((m, n_out), dtype=torch.float32, device=a.device)
    ops._timed("segment_matmul_tf32x3", 1, lib().b200mp_segment_matmul_tf32x3, a.data_ptr(), ptr.data_ptr(), ptr.numel() - 1,
               w_hi.data_ptr(), w_lo.data_ptr(), int(b_layout), c.data_ptr(), m, k, n_out, ops._stream())
    return c


def _grouped_ok(inputs: Tensor, other: Tensor) -> bool:
    R, k, n = other.shape
    return (_BACKEND == "tf32x3" and inputs.is_cuda and inputs.dtype == torch.float32 and other.dtype == torch.float32
            and inputs.size(0) > 0 and k % 32 == 0 and n % 128 == 0 and R <= 120 and inputs.size(0) < 2**31)


class _SegmentMatmul(torch.autograd.Function):
    """Forward and the input gradient are ONE persistent launch each of the grouped wgmma kernel (ptr stays on the
    device); the weight gradient (a reduction over each segment's rows) runs the split-K kernel per segment and reads
    the R + 1 segment bounds to the host once, in the backward only."""

    @staticmethod
    def forward(ctx, inputs: Tensor, ptr: Tensor, other: Tensor):
        inputs = inputs.contiguous()
        ptr64 = ptr.to(torch.int64).contiguous()
        w_hi, w_lo = split_tf32(other)
        ctx.save_for_backward(inputs, ptr64, w_hi, w_lo)
        return _grouped(inputs, ptr64, w_hi, w_lo, 1, other.size(2))

    @staticmethod
    def backward(ctx, g: Tensor):
        inputs, ptr64, w_hi, w_lo = ctx.saved_tensors
        g = g.contiguous()
        R, k, n = w_hi.shape
        gi = go = None
        if ctx.needs_input_grad[0]:
            if n % 32 == 0 and k % 128 == 0:
                gi = _grouped(g, ptr64, w_hi, w_lo, 0, k)                 # g[seg] . w[r]^T
            else:
                gi = torch.empty_like(inputs)
        bounds = None
        if ctx.needs_input_grad[2] or (gi is not None and not (n % 32 == 0 and k % 128 == 0)):
            bounds = ptr64.tolist()
        if ctx.needs_input_grad[0] and not (n % 32 == 0 and k % 128 == 0):
            w = w_hi + w_lo
            for r in range(R):
                s, e = bounds[r], bounds[r + 1]
                if e > s:
                    gi[s:e] = g[s:e] @ w[r].t()
        if ctx.needs_input_grad[2]:
            go = torch.zeros((R, k, n), dtype=torch.float32, device=g.device)
            for r in range(R):
                s, e = bounds[r], bounds[r + 1]
                if e > s:
                    go[r] = _mm_tn(inputs[s:e], g[s:e])
        return gi, None, go


class _SegmentMatmulLoop(torch.autograd.Function):
    """Shapes off the grouped kernel's grid: one product per segment (library GEMM or the single-segment kernels)."""

    @staticmethod
    def forward(ctx, inputs: Tensor, other: Tensor, bounds: tuple):
        out = torch.empty((inputs.size(0), other.size(2)), dtype=inputs.dtype, device=inputs.device)
        for r in range(other.size(0)):
            s, e = bounds[r], bounds[r + 1]
            if e > s:
                out[s:e] = _mm(inputs[s:e], other[r])
        ctx.bounds = bounds
        ctx.save_for_backward(inputs, other)
        return out

    @staticmethod
    def backward(ctx, g: Tensor):
        inputs, other = ctx.saved_tensors
        bounds = ctx.bounds
        g = g.contiguous()
        gi = torch.empty_like(inputs) if ctx.needs_input_grad[0] else None
        go = torch.zeros_like(other) if ctx.needs_input_grad[1] else None
        for r in range(other.size(0)):
            s, e = bounds[r], bounds[r + 1]
            if e <= s:
                continue
            if gi is not None:
                gi[s:e] = _mm_nt(g[s:e], other[r])
            if go is not None:
                go[r] = _mm_tn(inputs[s:e], g[s:e])
        return gi, go, None


def segment_matmul(inputs: Tensor, ptr: Tensor, other: Tensor) -> Tensor:
    """pyg_lib.ops.segment_matmul (nn/dense/linear.py:248-255, nn/conv/rgcn_conv.py:288):
    out[ptr[r]:ptr[r+1]] = inputs[ptr[r]:ptr[r+1]] @ other[r], other: [R, K, N] -- ONE persistent launch of the grouped
    3xTF32 wgmma kernel (fp32-accurate; `ptr` is never read on the host) when K % 32 == 0 and N % 128 == 0, else one
    product per segment."""
    if not inputs.is_cuda:
        raise RuntimeError("pytorch_geometric_b200 ops run on CUDA tensors only (no CPU fallback)")
    if other.dim() != 3 or inputs.dim() != 2 or inputs.size(1) != other.size(1) or ptr.numel() != other.size(0) + 1:
        raise ValueError("segment_matmul expects inputs [M, K], ptr [R + 1], other [R, K, N]")
    if _grouped_ok(inputs, other):
        return _SegmentMatmul.apply(inputs, ptr, other)
    bounds = tuple(int(v) for v in ptr.tolist())
    return _SegmentMatmulLoop.apply(inputs, other, bounds)


def grouped_matmul(inputs, others, biases=None):
    """pyg_lib.ops.grouped_matmul (nn/dense/linear.py:304-330, 437-446): [x_i @ w_i (+ b_i)] for lists of matrices."""
    outs = []
    for i, (x, w) in enumerate(zip(inputs, others)):
        y = _MM.apply(x, w)
        if biases is not None and biases[i] is not None:
            y = y + biases[i]
        outs.append(y)
    return outs


class _MM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a: Tensor, b: Tensor):
        ctx.save_for_backward(a, b)
        return _mm(a, b)

    @staticmethod
    def backward(ctx, g: Tensor):
        a, b = ctx.saved_tensors
        g = g.contiguous()
        ga = _mm_nt(g, b) if ctx.needs_input_grad[0] else None
        gb = _mm_tn(a, g) if ctx.needs_input_grad[1] else None
        return ga, gb
