"""Numpy restatement of the long-row chunk plan ``b200_spmm_csr`` takes (csrc/spmm.cu): rows with more
than ``threshold`` non-zeros are cut into ``ceil(nnz / chunk)`` chunks of ``chunk`` non-zeros.

* ``long_rows[i]``: the i-th long row, ascending;
* ``long_chunk_ptr[i] .. long_chunk_ptr[i + 1]``: its chunks;
* ``chunk_row[c]`` / ``chunk_k[c]``: the row of chunk c and its index inside that row, so that the chunk
  covers non-zeros ``indptr[row] + k * chunk`` up to the row's end."""
import numpy as np


def long_row_plan(indptr, threshold, chunk):
    deg = np.diff(np.asarray(indptr, dtype=np.int64))
    long_rows = np.flatnonzero(deg > threshold)
    nch = (deg[long_rows] + chunk - 1) // chunk
    long_chunk_ptr = np.zeros(len(long_rows) + 1, dtype=np.int64)
    long_chunk_ptr[1:] = np.cumsum(nch)
    chunk_row = np.repeat(long_rows, nch).astype(np.int32)
    chunk_k = (np.arange(int(long_chunk_ptr[-1])) - np.repeat(long_chunk_ptr[:-1], nch)).astype(np.int32)
    return dict(long_rows=long_rows.astype(np.int32), long_chunk_ptr=long_chunk_ptr, chunk_row=chunk_row,
                chunk_k=chunk_k, n_long=len(long_rows), n_chunks=int(long_chunk_ptr[-1]))
