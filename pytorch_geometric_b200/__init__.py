"""pytorch_geometric_b200 -- an H100-native (sm_90a) message-passing aggregation engine that drops
in behind PyG's scatter / segment / softmax / spmm / MessagePassing.propagate path.

Layout: csrc/ (CUDA kernels + the C ABI of include/b200mp.h), _lib.py/ops.py (ctypes binding),
graph.py (cached CSR/CSC structure), functional.py (autograd), utils.py / nn/ (host-side mirror of
the reference's interface for this path), dist.py (node-range sharding + halo exchange),
install.py (plugs the engine into an installed torch_geometric).
"""
from . import minibatch, ops, utils  # noqa: F401
from .functional import aggregate, scatter_coo, segment, softmax_csr  # noqa: F401
from .graph import CSRGraph  # noqa: F401
from ._lib import B200MPError, header_symbols, lib  # noqa: F401
from ._debug import debug, set_debug  # noqa: F401

__version__ = "0.1.0"
