"""The reference-side binding: plugs the engine into an installed `torch_geometric` (SURVEY.md section 8(b)).

The reference has no FFI; it late-binds Python callables and a handful of optional-extension operator signatures.
`install()` rebinds exactly those seams, `uninstall()` restores every one of them:

  (1) functions     torch_geometric.utils.{scatter, segment, softmax, spmm} and every module that imported them by
                    name (64 modules), `edge_index._spmm` (EdgeIndex.matmul / `@`), `Aggregation.reduce`,
                    `FusedAggregation.forward`, `QuantileAggregation.forward`               -> routing.py
  (2) the gather    `MessagePassing._index_select` (what `_collect` / `_lift` call) returns a lazy row view, so a
                    layer whose message is `x_j` or `w * x_j` runs ONE fused CSR gather-reduce            -> lazy.py
  (3) extensions    the exact `torch_scatter` / `pyg_lib.ops` / `torch.ops.torch_sparse` operator signatures the
                    reference calls, bound into `torch_geometric.typing` and its consumers; with `flip_flags=True`
                    the `WITH_*` switches are turned on so the reference's own extension branches run them  -> shims.py
  (4) layers        subclasses of the reference's layer classes with fully fused `forward` / `message_and_aggregate`
                    (`pytorch_geometric_b200.plugin.conv`); `layers=True` rebinds `torch_geometric.nn.<Layer>`      -> conv.py
                    and `torch_geometric.nn.Node2Vec` to a subclass whose graph moves to the GPU with it      -> models.py

CPU tensors, unsupported dtypes and `torch.compile` tracing (`is_compiling()`, as the reference gates its own
extension calls: utils/_scatter.py:85,120) fall through to the untouched reference code.
"""
from __future__ import annotations

import sys
from typing import Dict, List, Tuple

_PATCHED: List[Tuple[object, str, object, bool]] = []      # (holder, attribute, original, existed)
_MISSING = object()


def _set(holder, name: str, value) -> None:
    orig = holder.__dict__.get(name, _MISSING) if isinstance(holder, type) else getattr(holder, name, _MISSING)
    _PATCHED.append((holder, name, orig, orig is not _MISSING))
    setattr(holder, name, value)


def _tg_modules():
    return [m for m in list(sys.modules.values())
            if m is not None and getattr(m, "__name__", "").startswith("torch_geometric")]


def _rebind_everywhere(name: str, theirs, ours) -> int:
    n = 0
    for mod in _tg_modules():
        if mod.__dict__.get(name, None) is theirs:
            _set(mod, name, ours)
            n += 1
    return n


def installed() -> bool:
    return bool(_PATCHED)


def install(layers: bool = False, extensions: bool = True, flip_flags: bool = False, lazy_gather: bool = True) -> Dict[str, int]:
    """Rebinds the reference's seams to the engine.  Returns {seam: number of rebinds}."""
    import torch_geometric  # noqa: F401  (must be importable: this is the reference-side binding)
    import torch_geometric.edge_index as tg_edge_index
    import torch_geometric.typing as tg_typing
    from torch_geometric.nn.aggr.base import Aggregation
    from torch_geometric.nn.aggr.fused import FusedAggregation as TheirFused
    from torch_geometric.nn.conv.message_passing import MessagePassing
    from torch_geometric.utils import _scatter, _segment, _softmax, _spmm

    from . import routing, shims

    if _PATCHED:
        return {}
    counts: Dict[str, int] = {}
    for name, home, make in (("scatter", _scatter, routing.make_scatter), ("segment", _segment, routing.make_segment),
                             ("softmax", _softmax, routing.make_softmax), ("spmm", _spmm, routing.make_spmm)):
        theirs = getattr(home, name)
        counts[name] = _rebind_everywhere(name, theirs, make(theirs))

    _set(tg_edge_index, "_spmm", routing.make_edge_index_spmm(tg_edge_index._spmm))
    counts["edge_index._spmm"] = 1
    _set(Aggregation, "reduce", routing.make_aggr_reduce(Aggregation.reduce))
    counts["Aggregation.reduce"] = 1
    if lazy_gather:
        _set(MessagePassing, "_index_select", routing.make_index_select(MessagePassing._index_select))
        counts["MessagePassing._index_select"] = 1

    # FusedAggregation.forward (nn/aggr/fused.py:191): every fusable list except those containing 'mul'
    from ..nn import aggr as our_aggr
    theirs_fwd = TheirFused.forward

    def fused_forward(self, x, index=None, ptr=None, dim_size=None, dim=-2):
        from .lazy import LazyRows
        if isinstance(x, LazyRows):
            x = x.materialise()
        names = [our_aggr.FusedAggregation.NAME.get(n) for n in self.aggr_names]
        if not routing.engine_ok(x) or None in names or x.dim() != 2 or index is None or routing._compiling():
            return theirs_fwd(self, x, index, ptr, dim_size, dim)
        if dim_size is None:
            dim_size = ptr.numel() - 1 if ptr is not None else (int(index.max()) + 1 if index.numel() > 0 else 0)
        if ptr is None:
            ptr = routing._sorted_ptr(index, dim_size)
        uniq = list(dict.fromkeys(names))
        # the reference ignores `ptr` here and scatters by `index`; a given ptr means the index is sorted
        outs = dict(zip(uniq, our_aggr._fused_forward(uniq, self.semi_grad, x, routing._plain(index), ptr, dim_size, dim, False)))
        return [outs[n] for n in names]

    _set(TheirFused, "forward", fused_forward)
    counts["fused_aggregation"] = 1

    # QuantileAggregation.forward (nn/aggr/quantile.py:71-131), which MedianAggregation inherits
    from torch_geometric.nn.aggr.quantile import QuantileAggregation as TheirQuantile
    _set(TheirQuantile, "forward", routing.make_quantile_forward(TheirQuantile.forward))
    counts["quantile_aggregation"] = 1

    if extensions:
        from . import library
        counts["b200mp_ops"] = int(library.register())
        ts, pl = shims.torch_scatter_module(), shims.pyg_lib_module()
        counts["torch_sparse_ops"] = int(shims.register_torch_sparse_ops())
        n = 0
        for mod in _tg_modules():
            for attr, shim in (("torch_scatter", ts), ("pyg_lib", pl)):
                if attr in mod.__dict__ and mod.__dict__[attr] is object:       # the placeholder of typing.py:95,147
                    _set(mod, attr, shim)
                    n += 1
        counts["extension_modules"] = n
        # SplineConv imports spline_basis / spline_weighting by name and leaves them None without pyg-lib
        # (nn/conv/spline_conv.py:15-18); its constructor raises ImportError until they are bound
        import torch_geometric.nn.conv.spline_conv as tg_spline
        k = 0
        for name in ("spline_basis", "spline_weighting"):
            if getattr(tg_spline, name, None) is None:
                _set(tg_spline, name, getattr(pl.ops, name))
                k += 1
        counts["spline_ops"] = k
        # the point-cloud functions and DynamicEdgeConv / GravNetConv / XConv call torch.ops.pyg.* directly
        counts["point_ops"] = shims.register_point_ops()
        # graclus and voxel_grid call torch.ops.pyg.graclus_cluster / grid_cluster directly
        counts["cluster_ops"] = shims.register_cluster_ops()
        # Node2Vec, dropout_path and RootedRWSubgraph call torch.ops.pyg.random_walk directly
        counts["walk_ops"] = shims.register_walk_ops()
        if flip_flags:
            for flag in ("WITH_TORCH_SCATTER", "WITH_SOFTMAX", "WITH_INDEX_SORT", "WITH_SEGMM", "WITH_GMM"):
                _set(tg_typing, flag, True)
            counts["flags"] = 5
            _set(tg_typing, "WITH_SPLINE", True)
            counts["spline_flag"] = 1
            for flag in ("WITH_KNN", "WITH_RADIUS", "WITH_FPS", "WITH_NEAREST"):
                _set(tg_typing, flag, True)
            counts["point_flags"] = 4
            for flag in ("WITH_GRACLUS", "WITH_GRID_CLUSTER"):
                _set(tg_typing, flag, True)
            counts["cluster_flags"] = 2
            # Node2Vec and dropout_path gate on WITH_PYG_LIB, which NeighborLoader and to_hetero read too: the global
            # stays off (the engine has no neighbour sampler); node2vec's own binding of it is set, and dropout_path
            # is wrapped to switch it on for its own call only
            import torch_geometric.nn.models.node2vec as tg_node2vec
            from torch_geometric.utils import dropout as tg_dropout
            _set(tg_node2vec, "WITH_PYG_LIB", True)
            theirs = tg_dropout.dropout_path
            counts["walk_flags"] = 1 + _rebind_everywhere("dropout_path", theirs, shims.make_dropout_path(theirs))

    if layers:
        import torch_geometric.nn as tgnn
        import torch_geometric.nn.conv as tgconv

        from . import conv as ours_conv
        k = 0
        for cls, sub in ours_conv.LAYERS.items():
            for mod in (tgnn, tgconv):
                if hasattr(mod, cls):
                    _set(mod, cls, getattr(ours_conv, sub))
                    k += 1
        counts["layers"] = k
        # Node2Vec keeps its graph in buffers that follow the module to the GPU (models.py)
        import torch_geometric.nn.models as tgmodels

        from .models import B200Node2Vec
        k = 0
        for mod in (tgnn, tgmodels):
            if hasattr(mod, "Node2Vec"):
                _set(mod, "Node2Vec", B200Node2Vec)
                k += 1
        counts["models"] = k
    return counts


def uninstall() -> None:
    while _PATCHED:
        holder, name, orig, existed = _PATCHED.pop()
        if existed:
            setattr(holder, name, orig)
        else:
            try:
                delattr(holder, name)
            except AttributeError:
                pass
    from . import graphs
    graphs.clear_cache()
