"""LazyRows -- the hook behind `MessagePassing._collect / _lift / _index_select`
(nn/conv/message_passing.py:263-333, collect.jinja:118-139).

The reference materialises `x_j = x.index_select(node_dim, edge_index_j)` ([E, F]: 113 GB at the headline shape),
runs `message` on it and scatters the result.  With the plug-in installed, `_index_select` on a CUDA fp32 / bf16
feature matrix returns a `LazyRows`: a tensor subclass that only REMEMBERS (matrix, index[, per-edge scale]
[, per-edge rows to add, ReLU]).

  * `message` returning `x_j` or `edge_weight.view(-1, 1) * x_j` (GCNConv, SAGEConv, GINConv, GraphConv, ... --
    gcn_conv.py:270-271, graph_conv.py:100-101) keeps it lazy: the multiplication is folded into the scale;
  * `message` returning `(x_j + edge_attr).relu()` (GINEConv, gin_conv.py:195-204) keeps it lazy too, folded in this
    order only: first `lazy + t` / `t + lazy` / `torch.add(lazy, t)` (no alpha, no out) with `t` a plain dense
    tensor of shape [E, *x_j.shape[1:]], x_j's dtype and device, on a lazy without scale; then `relu` (Tensor.relu,
    torch.relu, F.relu without inplace);
  * `message` returning `act(k_i + q_j) * v_j` with the sigmoid (ResGatedGraphConv, res_gated_graph_conv.py:138-148)
    becomes a `GatedRows`, folded in this order only: `lazy_a + lazy_b` / `torch.add(lazy_a, lazy_b)` of two plain
    LazyRows (no scale, no add) of one shape, dtype and device; then `sigmoid` (Tensor.sigmoid, torch.sigmoid,
    F.sigmoid, nn.Sigmoid -- not `sigmoid_`, not `out=`); then `gate * lazy_v` / `lazy_v * gate` with `lazy_v` a plain
    LazyRows of the same shape, dtype and device;
  * `aggregate` -> `Aggregation.reduce` -> `scatter` / `segment` (nn/aggr/base.py:173-185) sees the LazyRows and runs
    ONE fused gather-reduce over a CSR (`b200mp_spmm_csr`, or `b200mp_edge_relu_csr` for the ReLU message and
    `b200mp_gated_csr` for the gated one, sum / mean) -- adopted from the sorted `Index`/`ptr` the layer collected, or
    built by one cached stable sort -- instead of index_select + atomics;
  * anything else a layer does with `x_j` (concatenation, an MLP, attention logits, `* w` after an add, `+ eps` after
    the ReLU, a min / max reduction, ...) materialises it through `__torch_function__` with the very ops the reference
    would have run -- index_select, then `+ t`, then relu; or index_select x2, `+`, sigmoid, `*` -- so behaviour,
    including type promotion, is unchanged.

explain mode and `decomposed_layers > 1` keep working: they call the same `_index_select` / `aggregate`.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from ._util import plain

_META = {"size", "dim", "numel", "stride", "is_floating_point", "is_complex", "is_contiguous", "element_size", "nelement",
         "ndimension", "type", "__len__", "is_cuda", "dtype", "device", "shape", "requires_grad", "ndim", "layout", "names",
         "is_sparse", "is_quantized", "is_meta", "grad_fn", "is_leaf", "data_ptr", "_version", "__get__", "__repr__",
         "__format__", "__class__", "__hash__", "__reduce_ex__", "untyped_storage", "storage_offset"}
_ADD = ("add", "__add__", "__radd__")
_MUL = ("mul", "__mul__", "__rmul__", "multiply")


class LazyRows(Tensor):
    """rows `index` of `src` along dim 0 (times `scale[e]` per row when set; plus `add[e]`, then ReLU'd when `relu`),
    not yet gathered."""

    @staticmethod
    def __new__(cls, src: Tensor, index: Tensor, scale: Optional[Tensor] = None, add: Optional[Tensor] = None,
                relu: bool = False):
        shape = (index.numel(), ) + tuple(src.shape[1:])
        r = Tensor._make_wrapper_subclass(cls, shape, dtype=src.dtype, device=src.device, requires_grad=False)
        r._src, r._index, r._scale, r._add, r._relu = src, index, scale, add, relu
        return r

    def __repr__(self):                                            # noqa: D105
        return (f"LazyRows(rows={self._index.numel()}, of={tuple(self._src.shape)}, scaled={self._scale is not None}, "
                f"added={self._add is not None}, relu={self._relu})")

    def materialise(self) -> Tensor:
        """What the reference computes: src.index_select(0, index) (* scale | + add (.relu()))."""
        with torch._C.DisableTorchFunctionSubclass():
            idx = plain(self._index)
            out = self._src.index_select(0, idx)
            if self._scale is not None:
                s = self._scale
                out = s.view((-1, ) + (1, ) * (out.dim() - 1)) * out
            if self._add is not None:
                out = out + self._add
                if self._relu:
                    out = out.relu()
        return out

    def _scaled_by(self, w: Tensor) -> Optional["LazyRows"]:
        """self * w for a per-edge weight w of shape [E] / [E, 1, ...]; None when w is anything else."""
        E = self._index.numel()
        if self._add is not None:
            return None
        if not isinstance(w, Tensor) or isinstance(w, LazyRows) or w.numel() != E or w.dim() == 0:
            return None
        if w.dim() > 1 and tuple(w.shape) != (E, ) + (1, ) * (w.dim() - 1):
            return None
        if not w.is_floating_point() or w.device != self.device:
            return None
        w1 = w.reshape(-1)
        return LazyRows(self._src, self._index, w1 if self._scale is None else self._scale * w1)

    def _plus(self, t) -> Optional["LazyRows"]:
        """self + t for per-edge rows t of exactly self's shape, dtype and device; None when t is anything else."""
        if self._scale is not None or self._add is not None:
            return None
        if type(t) is not Tensor or t.layout != torch.strided:
            return None
        if tuple(t.shape) != tuple(self.shape) or t.dtype != self.dtype or t.device != self.device:
            return None
        return LazyRows(self._src, self._index, add=t)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = getattr(func, "__name__", "")
        if name in _META:
            with torch._C.DisableTorchFunctionSubclass():
                return func(*args, **kwargs)
        if len(args) == 2 and not kwargs and (name in _ADD or name in _MUL):
            r = (GatedRows.gate_sum if name in _ADD else GatedRows.gated_message)(*args)
            if r is not None:
                return r
        if (name == "sigmoid" and len(args) == 1 and not kwargs and isinstance(args[0], GatedRows)
                and args[0]._stage == "sum"):
            return GatedRows(args[0]._a, args[0]._b, "gate")
        if name in _MUL and len(args) == 2 and not kwargs:
            a, b = args
            lazy, other = (a, b) if isinstance(a, LazyRows) else (b, a)
            if isinstance(lazy, LazyRows):
                r = lazy._scaled_by(other)
                if r is not None:
                    return r
        if name in _ADD and len(args) == 2 and not kwargs:
            a, b = args
            lazy, other = (a, b) if isinstance(a, LazyRows) else (b, a)
            if isinstance(lazy, LazyRows):
                r = lazy._plus(other)
                if r is not None:
                    return r
        if (name == "relu" and len(args) == 1 and isinstance(args[0], LazyRows)
                and (not kwargs or (func is F.relu and kwargs == {"inplace": False}))):
            lazy = args[0]
            if lazy._add is not None and not lazy._relu:
                return LazyRows(lazy._src, lazy._index, add=lazy._add, relu=True)
        # anything else: gather now (exactly the reference's ops) and carry on with a plain tensor

        def mat(v):
            if isinstance(v, LazyRows):
                return v.materialise()
            if isinstance(v, (list, tuple)):
                return type(v)(mat(u) for u in v)
            return v
        with torch._C.DisableTorchFunctionSubclass():
            return func(*mat(args), **{k: mat(v) for k, v in kwargs.items()})

    @classmethod
    def __torch_dispatch__(cls, func, types, args=(), kwargs=None):
        # reached only by operations that bypassed __torch_function__ (e.g. autograd internals): materialise
        def mat(v):
            if isinstance(v, LazyRows):
                return v.materialise()
            if isinstance(v, (list, tuple)):
                return type(v)(mat(u) for u in v)
            return v
        return func(*mat(args), **{k: mat(v) for k, v in (kwargs or {}).items()})


def _plain_lazy(t) -> bool:
    return type(t) is LazyRows and t._scale is None and t._add is None


class GatedRows(LazyRows):
    """ResGatedGraphConv's message, pending (res_gated_graph_conv.py:148): `a + b` of two plain LazyRows (stage
    "sum"), its sigmoid ("gate"), then the gate times a plain LazyRows `v` ("message"; `v_first` keeps the operand
    order).  Still a LazyRows, so every site that materialises a lazy message materialises this one too."""

    @staticmethod
    def __new__(cls, a: LazyRows, b: LazyRows, stage: str = "sum", v: Optional[LazyRows] = None, v_first: bool = False):
        r = Tensor._make_wrapper_subclass(cls, a.shape, dtype=a.dtype, device=a.device, requires_grad=False)
        r._a, r._b, r._stage, r._v, r._v_first = a, b, stage, v, v_first
        r._scale, r._add, r._relu = None, None, False
        return r

    def __repr__(self):                                            # noqa: D105
        return f"GatedRows(rows={self.shape[0]}, stage={self._stage})"

    def materialise(self) -> Tensor:
        """What the reference computes: a + b (.sigmoid() (* v))."""
        with torch._C.DisableTorchFunctionSubclass():
            out = self._a.materialise() + self._b.materialise()
            if self._stage == "sum":
                return out
            out = torch.sigmoid(out)
            if self._stage == "gate":
                return out
            v = self._v.materialise()
            return v * out if self._v_first else out * v

    def _scaled_by(self, w):
        return None

    def _plus(self, t):
        return None

    @staticmethod
    def gate_sum(a, b) -> Optional["GatedRows"]:
        """a + b for two plain LazyRows of one shape, dtype and device; None otherwise."""
        if not (_plain_lazy(a) and _plain_lazy(b)):
            return None
        if a.shape != b.shape or a.dtype != b.dtype or a.device != b.device:
            return None
        return GatedRows(a, b)

    @staticmethod
    def gated_message(a, b) -> Optional["GatedRows"]:
        """gate * v or v * gate for a sigmoid gate and a plain LazyRows v of its shape, dtype and device; None
        otherwise."""
        v_first = isinstance(b, GatedRows)
        gate, v = (b, a) if v_first else (a, b)
        if not isinstance(gate, GatedRows) or gate._stage != "gate" or not _plain_lazy(v):
            return None
        if v.shape != gate.shape or v.dtype != gate.dtype or v.device != gate.device:
            return None
        return GatedRows(gate._a, gate._b, "message", v, v_first)
