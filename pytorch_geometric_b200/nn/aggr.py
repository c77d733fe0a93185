"""Aggregation modules: mirrors of torch_geometric.nn.aggr.{Sum,Mean,Max,Min,Var,Std,Softmax,PowerMean}Aggregation
(nn/aggr/base.py:102-185, basic.py:12-50,83-139,142-297), {Quantile,Median}Aggregation (quantile.py:10-161),
FusedAggregation (fused.py:20-336) and MultiAggregation (multi.py:14-200) on the sm_90a kernels.

`__call__(x, index=None, ptr=None, dim_size=None, dim=-2)` has the reference's meaning and error
behaviour.  Unlike the reference (base.py:177-180 only uses `ptr` in deterministic mode), the CSR
kernel is used whenever `ptr` is given: the result is the same (test/nn/aggr/test_basic.py:63)
and it is the deterministic, atomics-free path.  Without `ptr` the index is treated as unsorted
(atomic COO kernel) unless `index_sorted=True` is passed.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from .. import _debug
from .. import functional as Fn
from .. import ops
from .. import utils as U


class Aggregation(torch.nn.Module):
    reduce_op = "sum"

    def __call__(self, x: Tensor, index: Optional[Tensor] = None, ptr: Optional[Tensor] = None,
                 dim_size: Optional[int] = None, dim: int = -2, index_sorted: bool = False, **kwargs) -> Tensor:
        if dim >= x.dim() or dim < -x.dim():
            raise ValueError(f"Encountered invalid dimension '{dim}' of source tensor with {x.dim()} dimensions")
        if index is None and ptr is None:
            index = x.new_zeros(x.size(dim), dtype=torch.long)
        if ptr is not None:
            if dim_size is None:
                dim_size = ptr.numel() - 1
            elif dim_size != ptr.numel() - 1:
                raise ValueError(f"Encountered invalid 'dim_size' (got '{dim_size}' but expected "
                                 f"'{ptr.numel() - 1}')")
        if index is not None and dim_size is None:
            # the reference pays the same device->host read here (aggr/base.py:128: int(index.max()) + 1)
            dim_size = (ops.index_stats(index)[1] + 1) if index.numel() > 0 else 0
        elif index is not None and index.numel() > 0 and ptr is None and _debug.enabled():
            # The reference finds a too-small dim_size by catching the backend's error and re-checking
            # index.max() (aggr/base.py:130-139).  A CUDA kernel cannot raise, and reading index.max() on every
            # call would add a device->host sync the reference does not have: the engine's kernels drop
            # out-of-range rows instead, and this check runs only in debug mode (pytorch_geometric_b200.debug()).
            mx = ops.index_stats(index)[1]
            if mx >= dim_size:
                raise ValueError(f"Encountered invalid 'dim_size' (got '{dim_size}' but expected >= '{mx + 1}')")
        return super().__call__(x, index=index, ptr=ptr, dim_size=dim_size, dim=dim, index_sorted=index_sorted,
                                **kwargs)

    def reduce(self, x: Tensor, index: Optional[Tensor], ptr: Optional[Tensor], dim_size: Optional[int], dim: int,
               reduce: str, index_sorted: bool = False) -> Tensor:
        d = dim + x.dim() if dim < 0 else dim
        if ptr is not None:
            xm = x if d == 0 else x.movedim(d, 0).contiguous()
            out = Fn.segment(xm, ptr, reduce)
            return out if d == 0 else out.movedim(0, d)
        return U.scatter(x, index, d, dim_size, reduce, sorted=index_sorted)

    def forward(self, x, index=None, ptr=None, dim_size=None, dim=-2, index_sorted=False):
        return self.reduce(x, index, ptr, dim_size, dim, self.reduce_op, index_sorted)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}()"


class SumAggregation(Aggregation):
    reduce_op = "sum"


class MeanAggregation(Aggregation):
    reduce_op = "mean"


class MaxAggregation(Aggregation):
    reduce_op = "max"


class MinAggregation(Aggregation):
    reduce_op = "min"


class SoftmaxAggregation(Aggregation):
    """alpha = softmax(t * x) per group; out = sum(alpha * x)   (nn/aggr/basic.py:142-218), as one online-softmax
    sweep over the messages (functional.softmax_aggregate): no [E, F] intermediate is stored, and a learnable t is
    read on the device."""

    def __init__(self, t: float = 1.0, learn: bool = False, semi_grad: bool = False, channels: int = 1):
        super().__init__()
        if learn and semi_grad:
            raise ValueError(f"Cannot enable 'semi_grad' in '{self.__class__.__name__}' in case the temperature term "
                             f"'t' is learnable")
        if not learn and channels != 1:
            raise ValueError(f"Cannot set 'channels' greater than '1' in case '{self.__class__.__name__}' is not "
                             f"trainable")
        self._init_t = t
        self.learn, self.semi_grad, self.channels = learn, semi_grad, channels
        self.t = torch.nn.Parameter(torch.empty(channels)) if learn else t
        self.reset_parameters()

    def reset_parameters(self):
        if isinstance(self.t, Tensor):
            self.t.data.fill_(self._init_t)

    def forward(self, x, index=None, ptr=None, dim_size=None, dim=-2, index_sorted=False):
        d = dim + x.dim() if dim < 0 else dim
        if self.channels != 1:                                           # base.py:162-169
            if x.dim() != 2:
                raise ValueError(f"Aggregation requires two-dimensional inputs (got '{x.dim()}')")
            if dim not in (-2, 0):
                raise ValueError(f"Aggregation needs to perform aggregation in first dimension (got '{dim}')")
        if not _softmax_fusable(x, self.t):
            return self._composed(x, index, ptr, dim_size, d, index_sorted)
        # the aggregated dimension first, every other one folded into the feature width (t broadcasts over the last)
        xm = x.movedim(d, 0)
        rest = xm.shape[1:]
        x2 = xm.reshape(xm.size(0), -1)
        out = _softmax_forward(x2, self.t, self.semi_grad and not self.learn, index, ptr, dim_size, index_sorted)
        return out.view(out.size(0), *rest).movedim(0, d)

    def _composed(self, x, index, ptr, dim_size, d, index_sorted):
        """The reference's op sequence (basic.py:196-215) on the engine's softmax and scatter, which compute in fp32:
        for messages the fused sweep does not take (fp16, fp64), and for a t whose dtype differs from the messages',
        where x * t promotes and the result takes the promoted dtype."""
        t = self.t
        if self.channels != 1:
            t = t.view(-1, self.channels)
        alpha = x
        if not isinstance(t, (int, float)) or t != 1:
            alpha = x * t
        if not self.learn and self.semi_grad:
            with torch.no_grad():
                alpha = U.softmax(alpha, index, ptr, dim_size, d)
        else:
            alpha = U.softmax(alpha, index, ptr, dim_size, d)
        return self.reduce(x * alpha, index, ptr, dim_size, d, "sum", index_sorted)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(learn={self.learn})"


def _softmax_fusable(x: Tensor, t) -> bool:
    """The fused sweep takes CUDA float32 / bfloat16 messages, with a Python-number t or a t of the messages' dtype."""
    return x.is_cuda and x.dtype in (torch.float32, torch.bfloat16) and (not isinstance(t, Tensor) or t.dtype == x.dtype)


def _softmax_forward(x, t, semi_grad, index, ptr, dim_size, index_sorted):
    """softmax_aggregate over a [E, F] message matrix, grouped by ptr or index (as _fused_forward groups them)."""
    if ptr is None and index is None:
        raise NotImplementedError("Aggregation requires 'index' to be specified")
    if x.size(0) == 0:
        n = dim_size if dim_size is not None else (ptr.numel() - 1 if ptr is not None else 0)
        return x.new_zeros(n, x.size(1))
    if ptr is None and index_sorted:
        ptr = ops.index2ptr(index, dim_size)
    if ptr is not None:
        return Fn.softmax_aggregate((ptr, ops.segment_plan(ptr, x.size(0))), None, x, t, semi_grad=semi_grad)
    # unsorted index: a CSR over the messages themselves; the sweep reads message perm[e] of CSR slot e in place
    from ..graph import CSRGraph
    e = torch.arange(index.numel(), device=index.device, dtype=index.dtype)
    return Fn.softmax_aggregate(CSRGraph(e, index, index.numel(), dim_size), None, x, t, semi_grad=semi_grad)


class PowerMeanAggregation(Aggregation):
    """out = clamp(mean(clamp(x)^p))^(1/p) per group   (nn/aggr/basic.py:221-297), as one sweep over the messages
    (functional.power_mean_aggregate): no [E, F] intermediate is stored, and a learnable p is read on the device."""

    def __init__(self, p: float = 1.0, learn: bool = False, channels: int = 1, clamp_min: Optional[float] = 1e-4,
                 clamp_max: Optional[float] = 100.):
        super().__init__()
        if not learn and channels != 1:
            raise ValueError(f"Cannot set 'channels' greater than '1' in case '{self.__class__.__name__}' is not "
                             f"trainable")
        self._init_p = p
        self.learn, self.channels = learn, channels
        self.p = torch.nn.Parameter(torch.empty(channels)) if learn else p
        self.reset_parameters()
        self.min_value, self.max_value = clamp_min, clamp_max

    def reset_parameters(self):
        if isinstance(self.p, Tensor):
            self.p.data.fill_(self._init_p)

    def forward(self, x, index=None, ptr=None, dim_size=None, dim=-2, index_sorted=False):
        d = dim + x.dim() if dim < 0 else dim
        if self.channels != 1:                                           # base.py:162-169
            if x.dim() != 2:
                raise ValueError(f"Aggregation requires two-dimensional inputs (got '{x.dim()}')")
            if dim not in (-2, 0):
                raise ValueError(f"Aggregation needs to perform aggregation in first dimension (got '{dim}')")
        if not power_mean_fusable(x, self.p, self.min_value, self.max_value):
            return self._composed(x, index, ptr, dim_size, d, index_sorted)
        xm = x.movedim(d, 0)
        rest = xm.shape[1:]
        x2 = xm.reshape(xm.size(0), -1)
        out = _group_forward(Fn.power_mean_aggregate, x2, index, ptr, dim_size, index_sorted, p=self.p,
                             clamp_min=self.min_value, clamp_max=self.max_value)
        return out.view(out.size(0), *rest).movedim(0, d)

    def _composed(self, x, index, ptr, dim_size, d, index_sorted):
        """The reference's op sequence (basic.py:279-293) on the engine's mean: for messages the fused sweep does not
        take (fp16, fp64), a p whose dtype differs from the messages' (x.pow(p) promotes, and the result takes the
        promoted dtype), and clamp bounds off the fused path."""
        p = self.p
        if self.channels != 1:
            p = p.view(-1, self.channels)
        pow_ = not isinstance(p, (int, float)) or p != 1
        if pow_:
            x = x.clamp(min=self.min_value, max=self.max_value).pow(p)
        out = self.reduce(x, index, ptr, dim_size, d, "mean", index_sorted)
        if pow_:
            out = out.clamp(min=self.min_value, max=self.max_value).pow(1. / p)
        return out

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(learn={self.learn})"


def power_mean_fusable(x: Tensor, p, clamp_min, clamp_max) -> bool:
    """The fused sweep takes CUDA float32 / bfloat16 messages with a Python-number p or a p of the messages' dtype, and,
    unless p is the number 1, a positive clamp_min with clamp_max None or >= clamp_min."""
    if not (x.is_cuda and x.dtype in (torch.float32, torch.bfloat16)):
        return False
    if not isinstance(p, Tensor):
        if float(p) == 1.0:
            return True
    elif p.dtype != x.dtype:
        return False
    return (isinstance(clamp_min, (int, float)) and clamp_min > 0 and
            (clamp_max is None or (isinstance(clamp_max, (int, float)) and clamp_max >= clamp_min)))


def _group_forward(fn, x, index, ptr, dim_size, index_sorted, **kw):
    """fn(graph, None, x, **kw) over a [E, F] message matrix grouped by ptr or index (as _fused_forward groups them)."""
    if ptr is None and index is None:
        raise NotImplementedError("Aggregation requires 'index' to be specified")
    if ptr is None and index_sorted:
        ptr = ops.index2ptr(index, dim_size)
    if ptr is not None:
        return fn((ptr, ops.segment_plan(ptr, x.size(0))), None, x, **kw)
    # unsorted index: a CSR over the messages themselves; the sweep reads message perm[e] of CSR slot e in place
    from ..graph import CSRGraph
    e = torch.arange(index.numel(), device=index.device, dtype=index.dtype)
    return fn(CSRGraph(e, index, index.numel(), dim_size), None, x, **kw)


class QuantileAggregation(Aggregation):
    """The feature-wise q-quantile(s) of each group (nn/aggr/quantile.py:10-134), as one selection sweep over the
    messages (functional.quantile_aggregate) instead of two sorts of the [E, F] matrix.  q is the reference's float32
    buffer of shape [Q, 1], read on the device.  Ranks past 2^24 messages are exact, ties go to the earlier message and
    an empty first group gives fill_value (the reference raises IndexError there): csrc/quantile.cu states the
    contract.  Takes CUDA float32 / bfloat16 messages; other dtypes raise TypeError."""
    interpolations = {"linear", "lower", "higher", "nearest", "midpoint"}

    def __init__(self, q, interpolation: str = "linear", fill_value: float = 0.0):
        super().__init__()
        qs = [q] if not isinstance(q, (list, tuple)) else q
        if len(qs) == 0:
            raise ValueError("Provide at least one quantile value for `q`.")
        if not all(0. <= quantile <= 1. for quantile in qs):
            raise ValueError("`q` must be in the range [0, 1].")
        if interpolation not in self.interpolations:
            raise ValueError(f"Invalid interpolation method got ('{interpolation}')")
        self._q = q
        self.register_buffer("q", torch.tensor(qs).view(-1, 1))
        self.interpolation = interpolation
        self.fill_value = fill_value

    def forward(self, x, index=None, ptr=None, dim_size=None, dim=-2, index_sorted=False):
        d = dim + x.dim() if dim < 0 else dim
        if index is None:
            raise NotImplementedError("Aggregation requires 'index' to be specified")
        if x.dtype not in (torch.float32, torch.bfloat16):
            raise TypeError(f"QuantileAggregation takes float32 or bfloat16 messages, got {x.dtype}")
        if self.q.dtype != torch.float32:
            raise TypeError(f"QuantileAggregation needs a float32 q buffer, got {self.q.dtype}")
        if dim_size is None:
            dim_size = ptr.numel() - 1 if ptr is not None else (
                ops.index_stats(index)[1] + 1 if index.numel() > 0 else 0)
        xm = x.movedim(d, 0)
        x2 = xm.reshape(xm.size(0), -1)
        if x2.size(0) == 0:
            out = torch.full((dim_size, self.q.numel() * x2.size(1)), self.fill_value, device=x.device,
                             dtype=ops.quantile_out_dtype(x.dtype, self.interpolation))
        else:
            out = _group_forward(Fn.quantile_aggregate, x2, index, ptr, dim_size, index_sorted, q=self.q,
                                 interpolation=self.interpolation, fill_value=self.fill_value)
        return quantile_layout(out, self.q.numel(), x.shape, d)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(q={self._q})"


class MedianAggregation(QuantileAggregation):
    """The feature-wise lower median of each group (nn/aggr/quantile.py:137-161): QuantileAggregation(0.5, 'lower')."""

    def __init__(self, fill_value: float = 0.0):
        super().__init__(0.5, "lower", fill_value)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}()"


def quantile_layout(out: Tensor, n_q: int, shape, d: int) -> Tensor:
    """The reference's layout (quantile.py:125-129) of a [N, Q * W] sweep result over x of `shape` aggregated along d
    (W: every other dimension, in order): [..., N, Q * shape[d + 1], ...], [..., N, Q] when d is the last dimension,
    and x's own shape with N at d for one q."""
    rest = list(shape[:d]) + list(shape[d + 1:])
    n = out.size(0)
    out = out.view(n, n_q, *rest).movedim((0, 1), (d, d + 1))
    if n_q == 1:
        return out.reshape(*shape[:d], n, *shape[d + 1:])
    if d + 1 < len(shape):
        return out.reshape(*shape[:d], n, n_q * shape[d + 1], *shape[d + 2:])
    return out.reshape(*shape[:d], n, n_q)


class VarAggregation(Aggregation):
    """var = mean(x^2) - mean(x)^2 per group (nn/aggr/basic.py:83-111), one fused sweep."""
    fused_name = "var"

    def __init__(self, semi_grad: bool = False):
        super().__init__()
        self.semi_grad = semi_grad

    def forward(self, x, index=None, ptr=None, dim_size=None, dim=-2, index_sorted=False):
        return _fused_forward([self.fused_name], self.semi_grad, x, index, ptr, dim_size, dim, index_sorted)[0]


class StdAggregation(VarAggregation):
    """std = sqrt(clamp(var, 1e-5)), 0 where that is <= sqrt(1e-5) (nn/aggr/basic.py:114-139)."""
    fused_name = "std"


def _fused_forward(names, semi_grad, x, index, ptr, dim_size, dim, index_sorted):
    d = dim + x.dim() if dim < 0 else dim
    if x.dim() != 2 or d != 0:
        raise ValueError("Aggregation requires two-dimensional inputs (got '{}') aggregated along dim 0".format(x.dim()))
    if ptr is None and index is None:
        raise NotImplementedError("Aggregation requires 'index' to be specified")
    if x.size(0) == 0:                       # no messages: zeros (test/nn/aggr/test_fused.py:46-55)
        n = dim_size if dim_size is not None else (ptr.numel() - 1 if ptr is not None else 0)
        return [x.new_zeros(n, x.size(1)) for _ in names]
    if ptr is None and index_sorted:
        ptr = ops.index2ptr(index, dim_size)
    if ptr is not None:
        if index is None:
            index = ops.ptr2index(ptr, x.size(0))
        return Fn.multi_aggregate((ptr, index, ops.segment_plan(ptr, x.size(0))), x, names, semi_grad)
    # unsorted index: a CSR over the messages themselves (source e -> destination index[e]); the kernel
    # gathers x[perm[.]] row by row, so the permuted [E, F] matrix is never materialised
    from ..graph import CSRGraph
    e = torch.arange(index.numel(), device=index.device, dtype=index.dtype)
    return Fn.multi_aggregate(CSRGraph(e, index, index.numel(), dim_size), x, names, semi_grad)


class FusedAggregation(Aggregation):
    """Mirror of torch_geometric.nn.aggr.fused.FusedAggregation (fused.py:20-336): a list of outputs, one
    per aggregation in `aggrs`, all taken from ONE sweep over the messages (the reference shares the count
    and the sum but still runs one scatter per base reduction).  'mul' is not fusable here."""
    FUSABLE = ("SumAggregation", "MeanAggregation", "MinAggregation", "MaxAggregation", "VarAggregation",
               "StdAggregation")
    NAME = {"SumAggregation": "sum", "MeanAggregation": "mean", "MinAggregation": "min", "MaxAggregation": "max",
            "VarAggregation": "var", "StdAggregation": "std"}

    def __init__(self, aggrs):
        super().__init__()
        if not isinstance(aggrs, (list, tuple)):
            raise ValueError(f"'aggrs' of '{self.__class__.__name__}' should be a list or tuple (got '{type(aggrs)}').")
        if len(aggrs) == 0:
            raise ValueError(f"'aggrs' of '{self.__class__.__name__}' should not be empty.")
        aggrs = [aggregation_resolver(a) if isinstance(a, str) else a for a in aggrs]
        self.aggr_names = [a.__class__.__name__ for a in aggrs]
        for name in self.aggr_names:
            if name not in self.FUSABLE:
                raise ValueError(f"Received aggregation '{name}' in '{self.__class__.__name__}' which is not fusable")
        self.semi_grad = any(getattr(a, "semi_grad", False) for a in aggrs)
        self.names = [self.NAME[n] for n in self.aggr_names]

    def forward(self, x, index=None, ptr=None, dim_size=None, dim=-2, index_sorted=False):
        # an aggregation listed twice is computed once and returned twice
        uniq = list(dict.fromkeys(self.names))
        outs = dict(zip(uniq, _fused_forward(uniq, self.semi_grad, x, index, ptr, dim_size, dim, index_sorted)))
        return [outs[n] for n in self.names]


class MultiAggregation(Aggregation):
    """Mirror of torch_geometric.nn.aggr.multi.MultiAggregation (multi.py:14-200) for the combine modes
    cat / proj / sum / mean / max / min / logsumexp / std / var; fusable members share one sweep."""

    def __init__(self, aggrs, aggrs_kwargs=None, mode: Optional[str] = "cat", mode_kwargs=None):
        super().__init__()
        if not isinstance(aggrs, (list, tuple)):
            raise ValueError(f"'aggrs' of '{self.__class__.__name__}' should be a list or tuple (got '{type(aggrs)}').")
        if len(aggrs) == 0:
            raise ValueError(f"'aggrs' of '{self.__class__.__name__}' should not be empty.")
        if aggrs_kwargs is None:
            aggrs_kwargs = [{}] * len(aggrs)
        elif len(aggrs) != len(aggrs_kwargs):
            raise ValueError(f"'aggrs_kwargs' with invalid length passed to '{self.__class__.__name__}' (got "
                             f"'{len(aggrs_kwargs)}', expected '{len(aggrs)}'). Ensure that both 'aggrs' and "
                             f"'aggrs_kwargs' are consistent.")
        self.aggrs = torch.nn.ModuleList([aggregation_resolver(a, **kw) if isinstance(a, str) else a
                                          for a, kw in zip(aggrs, aggrs_kwargs)])
        self.is_fused = [a.__class__.__name__ in FusedAggregation.FUSABLE for a in self.aggrs]
        fused = [a for a, f in zip(self.aggrs, self.is_fused) if f]
        self.fused_aggr = FusedAggregation(fused) if fused else None
        self.mode = mode
        mode_kwargs = dict(mode_kwargs or {})
        self.in_channels = mode_kwargs.pop("in_channels", None)
        self.out_channels = mode_kwargs.pop("out_channels", None)
        if mode == "attn":
            raise NotImplementedError("combine mode 'attn' is outside the aggregation path")
        if mode == "proj":
            if len(aggrs) == 1:
                raise ValueError("Multiple aggregations are required for 'proj' or 'attn' combine mode.")
            if (self.in_channels and self.out_channels) is None:
                raise ValueError(f"Combine mode '{mode}' must have `in_channels` and `out_channels` specified.")
            if isinstance(self.in_channels, int):
                self.in_channels = [self.in_channels] * len(aggrs)
            self.lin = torch.nn.Linear(sum(self.in_channels), self.out_channels, **mode_kwargs)
        if mode in ("sum", "mean", "max", "min", "logsumexp", "std", "var"):
            self.dense_combine = getattr(torch, mode)

    def get_out_channels(self, in_channels: int) -> int:
        if self.out_channels is not None:
            return self.out_channels
        return in_channels * len(self.aggrs) if self.mode == "cat" else in_channels

    def forward(self, x, index=None, ptr=None, dim_size=None, dim=-2, index_sorted=False):
        d = dim + x.dim() if dim < 0 else dim
        outs = [None] * len(self.aggrs)
        if self.fused_aggr is not None and x.dim() == 2 and d == 0:
            it = iter(self.fused_aggr(x, index, ptr, dim_size, dim, index_sorted=index_sorted))
            for i, f in enumerate(self.is_fused):
                if f:
                    outs[i] = next(it)
        for i, a in enumerate(self.aggrs):
            if outs[i] is None:
                outs[i] = a(x, index, ptr, dim_size, dim, index_sorted=index_sorted)
        return self.combine(outs)

    def combine(self, inputs):
        if len(inputs) == 1:
            return inputs[0]
        if self.mode == "cat":
            return torch.cat(inputs, dim=-1)
        if hasattr(self, "lin"):
            return self.lin(torch.cat(inputs, dim=-1))
        out = self.dense_combine(torch.stack(inputs, dim=0), dim=0)
        return out if isinstance(out, Tensor) else out[0]


def aggregation_resolver(name: str, **kwargs) -> Aggregation:
    table = {"sum": SumAggregation, "add": SumAggregation, "mean": MeanAggregation, "max": MaxAggregation,
             "min": MinAggregation, "var": VarAggregation, "std": StdAggregation, "softmax": SoftmaxAggregation,
             "powermean": PowerMeanAggregation, "median": MedianAggregation, "quantile": QuantileAggregation}
    if name not in table:
        raise ValueError(f"Could not resolve '{name}' among the aggregations on the hot path {sorted(table)}")
    return table[name](**kwargs)
