"""b200mp_spmm_csr_self_colsum checks its arguments before it launches anything: the transposed CSR's long-row plan
(n_long_rows_t >= 0 and n_chunks_t >= 0; with long rows the row list, the chunk offsets, a positive chunk and the fp32
partials), the required edge weights, and the column-sum workspace."""
import numpy as np
import pytest
import torch

import pytorch_geometric_b200 as pgb

# The calls pass host addresses where the library expects device buffers.  Without a device a call that gets past its
# checks fails at the launch (B200MP_ERR_CUDA); on a GPU it would launch a kernel on those addresses.
pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="passes host buffers as device pointers")

INVALID_ARG = -1
_RAW = np.zeros(1 << 16, dtype=np.uint8)
BUF = _RAW.ctypes.data + (-_RAW.ctypes.data) % 16


def _call(**override):
    # 4 rows of 8 fp32 features, int64 indices, no long rows, a workspace of 4 partial rows
    args = dict(rowptr_t=BUF, col_t=BUF, val_t=BUF, x=BUF, out=BUF, colsum_out=BUF, n_rows=4, feat=8, long_rows_t=BUF,
                chunk_ptr_t=BUF, n_long_rows_t=0, n_chunks_t=0, chunk=4, partials_t=BUF, colsum_parts=BUF, n_parts=4,
                idx_dtype=1, val_dtype=0, stream=None)
    args.update(override)
    return pgb.lib().b200mp_spmm_csr_self_colsum(*args.values())


@pytest.mark.parametrize("long_rows", [False, True], ids=["no_long_rows", "long_rows"])
def test_valid_arguments_pass_the_checks(long_rows):
    override = dict(n_long_rows_t=1, n_chunks_t=1) if long_rows else {}
    assert _call(**override) != INVALID_ARG, pgb.lib().b200mp_last_error()


@pytest.mark.parametrize("override", [
    dict(n_long_rows_t=-1),
    dict(n_long_rows_t=1, n_chunks_t=-1),
    dict(n_long_rows_t=1, n_chunks_t=1, chunk=0),
    dict(n_long_rows_t=1, n_chunks_t=1, chunk_ptr_t=None),
    dict(n_long_rows_t=1, n_chunks_t=1, partials_t=None),
    dict(val_t=None),
    dict(colsum_out=None),
    dict(colsum_parts=None),
    dict(n_parts=0),
    dict(n_rows=-1),
], ids=["negative_long_rows", "negative_chunks", "zero_chunk", "no_chunk_offsets", "no_partials", "no_weights",
        "no_colsum_out", "no_colsum_parts", "no_parts", "negative_rows"])
def test_malformed_arguments_are_rejected(override):
    assert _call(**override) == INVALID_ARG, pgb.lib().b200mp_last_error()
