"""Host-side mirror of the reference's operator API for the block-multiply path.

``MatfastSession`` replaces ``MatfastSession.builder().getOrCreate()`` (M/MatfastSession.scala:177-234)
and ``Dataset`` keeps the method names and argument order of M/Dataset.scala:57-152
(``matrixMultiply``, ``transpose``/``t``, ``addElement``, ``multiplyElement``, ``divideElement``,
``addScalar``, ``multiplyScalar``, ``power``, ``matrixRankOneUpdate``), each forwarding to the C ABI
(include/matrel.h) which launches the sm_90a kernels.  Execution is eager and asynchronous on the
session's CUDA stream instead of lazy through Catalyst; results are observationally the same
because operators are pure.

M/ = <reference>/src/main/scala/org/apache/spark/sql/matfast/
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Optional, Sequence

import numpy as np

from . import _native as N
from .matrix import DenseMatrix, MatrixBlock, MLMatrix, SparseMatrix


def _i32p(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _f64p(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class MatfastSession:
    """One engine context per process per GPU (``mr_init`` / ``mr_shutdown``)."""

    def __init__(self, device: int = -1, compat_bugs: bool = True, stream: Optional[int] = None,
                 gemm_algo: int = 0, ozaki_slices: int = 0):
        opts = N.mr_options(int(device), int(bool(compat_bugs)), int(gemm_algo), int(ozaki_slices),
                            C.c_void_p(stream) if stream else None)
        self._ctx = C.c_void_p()
        N.check(N.lib.mr_init(C.byref(opts), C.byref(self._ctx)))
        self._device = int(device)

    # -- lifetime ---------------------------------------------------------------------------
    def stop(self) -> None:
        if self._ctx:
            N.check(N.lib.mr_shutdown(self._ctx))
            self._ctx = C.c_void_p()

    close = stop

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.stop()

    def __del__(self):
        try:
            self.stop()
        except Exception:
            pass

    def sync(self) -> None:
        N.check(N.lib.mr_sync(self._ctx))

    def wait_ingest(self) -> None:
        """Device-side: the session stream waits for every host->device block copy submitted so far."""
        N.check(N.lib.mr_wait_ingest(self._ctx))

    def wait_ingest_on(self, cuda_stream: int) -> None:
        """Device-side: the given CUDA stream waits for every host->device block copy submitted so far."""
        N.check(N.lib.mr_wait_ingest_on(self._ctx, C.c_void_p(cuda_stream)))

    def set_stream(self, cuda_stream: Optional[int]) -> None:
        N.check(N.lib.mr_set_stream(self._ctx, C.c_void_p(cuda_stream) if cuda_stream else None))

    def set_option(self, key: str, value: int) -> None:
        N.check(N.lib.mr_set_option(self._ctx, key.encode(), int(value)))

    def stats(self) -> dict:
        s = N.mr_stats()
        N.check(N.lib.mr_get_stats(self._ctx, C.byref(s)))
        return {k: getattr(s, k) for k, _ in N.mr_stats._fields_}

    def reset_stats(self) -> None:
        N.check(N.lib.mr_reset_stats(self._ctx))

    # -- dataset construction ---------------------------------------------------------------
    def createDataset(self, blocks: Iterable[MatrixBlock]) -> "Dataset":
        """``Seq(MatrixBlock(...)).toDS()`` (M/example/BasicMatrixOps.scala:115-116)."""
        ds = Dataset._new(self)
        ds.put_blocks(blocks)
        return ds

    toDS = createDataset

    def createHostDataset(self, blocks: Iterable[MatrixBlock] = ()) -> "Dataset":
        """A host-resident dataset: the blocks are copied into page-locked host memory owned by the engine (the arrays passed in
        are free again at once).  ``matrixMultiply`` streams such operands through the device tile by tile, so products larger
        than device memory run; every other operator needs :meth:`Dataset.toDevice` first."""
        h = C.c_void_p()
        N.check(N.lib.mr_matrix_create_host(self._ctx, C.byref(h)))
        ds = Dataset(self, h)
        ds.put_blocks(blocks)
        return ds

    def emptyDataset(self) -> "Dataset":
        return Dataset._new(self)

    def _cuda_device(self) -> int:
        if self._device >= 0:
            return self._device
        import torch
        return torch.cuda.current_device()

    def fromDense(self, a, blkSize: int, host: bool = False) -> "Dataset":
        """A whole 2-D float64 matrix as a dataset of ``blkSize`` blocks, every block present (``mr_matrix_from_dense``).  ``a`` is a
        numpy array or a torch tensor with one unit-stride dimension (C order, F order, or a slice of either); blocks of a row-major
        ``a`` are stored row-major (``isTransposed``), so nothing is transposed on the way in.  A CUDA tensor must be on the session's
        device; its copy is ordered after ``torch.cuda.current_stream()``.  ``host``: a host-resident dataset.  A CUDA tensor or a
        page-locked CPU tensor is read asynchronously: the dataset keeps a reference to it, and it must not be modified before
        :meth:`Dataset.wait_ingest` (or :meth:`sync`)."""
        keep, stream = None, None
        if not isinstance(a, np.ndarray):
            import torch
            if not isinstance(a, torch.Tensor):
                raise TypeError(f"fromDense takes a numpy array or a torch tensor, got {type(a).__name__}")
            if a.dtype != torch.float64:
                raise TypeError(f"fromDense needs float64 data, got a tensor of {a.dtype}")
            if a.device.type == "cuda":
                if a.device.index != self._cuda_device():
                    raise ValueError(f"fromDense: the tensor is on {a.device}, the session runs on cuda:{self._cuda_device()}")
                keep, stream = a, _torch_stream(a.device)
                ptr, shape, strides = a.data_ptr(), tuple(a.shape), tuple(a.stride())
            elif a.device.type == "cpu":
                if a.is_pinned():
                    keep = a
                a = a.detach().numpy()
            else:
                raise ValueError(f"fromDense: a tensor on device {a.device} (CPU and CUDA tensors only)")
        if isinstance(a, np.ndarray):
            if a.dtype != np.float64:
                raise TypeError(f"fromDense needs float64 data, got an array of {a.dtype}")
            ptr, shape, strides = a.ctypes.data, a.shape, tuple(s // a.itemsize if s % a.itemsize == 0 else 0 for s in a.strides)
        if len(shape) != 2:
            raise ValueError(f"fromDense needs a 2-D matrix, got shape {shape}")
        rowMajor, ld = _dense_layout(shape, strides)
        h = C.c_void_p()
        N.check(N.lib.mr_matrix_from_dense(self._ctx, C.c_void_p(ptr), shape[0], shape[1], ld, rowMajor, int(blkSize),
                                           1 if host else 0, C.c_void_p(stream) if stream else None, C.byref(h)))
        ds = Dataset(self, h)
        ds._source = keep
        return ds

    def rand(self, nrows: int, ncols: int, blkSize: int, seed0: int) -> "Dataset":
        """Every block ``DenseMatrix.rand(r, c, new java.util.Random(seed0 + rid*nbc + cid))``
        (M/matrix/MLMatrix.scala:453-457), generated on the device."""
        h = C.c_void_p()
        N.check(N.lib.mr_matrix_rand(self._ctx, nrows, ncols, blkSize, seed0, C.byref(h)))
        return Dataset(self, h)


def _torch_stream(device) -> int:
    """torch's current stream on `device` as a cudaStream_t; its default stream is the legacy one (handle 0), passed as
    cudaStreamLegacy (0x1) because NULL means "no stream" to mr_matrix_from_dense / mr_matrix_to_dense."""
    import torch
    return torch.cuda.current_stream(device).cuda_stream or 1


def _dense_layout(shape, strides):
    """(rowMajor, ld) of a 2-D matrix with element strides `strides`; the stride of a dimension of extent 1 does not matter."""
    (r, c), (s0, s1) = shape, strides
    if s1 == 1 and (r == 1 or s0 >= c):
        return 1, (s0 if r > 1 else c)
    if s0 == 1 and (c == 1 or s1 >= r):
        return 0, (s1 if c > 1 else r)
    raise ValueError(f"fromDense needs one unit-stride dimension (C order, F order or a slice of either); "
                     f"got shape {tuple(shape)} with element strides {tuple(strides)}")


def sprand(session: "MatfastSession", nrows: int, ncols: int, blkSize: int, density: float, seed0: int, csr: bool = True) -> "Dataset":
    """Every block ``SparseMatrix.sprand(..., new java.util.Random(seed0 + rid*nbc + cid))`` (M/matrix/MLMatrix.scala:791-856),
    generated on the device; ``csr`` presents each block in CSR form (the transpose of a sprand block)."""
    h = C.c_void_p()
    N.check(N.lib.mr_matrix_sprand(session._ctx, int(nrows), int(ncols), int(blkSize), float(density), int(seed0), 1 if csr else 0, C.byref(h)))
    return Dataset(session, h)


def rand_partition(session: "MatfastSession", nrows: int, ncols: int, blkSize: int, seed0: int, pr: int, pc: int,
                   r: int, c: int, slab_ptr: int, slot_elems: int) -> "Dataset":
    """The blocks rank (r, c) of a pr x pc grid owns, generated into a caller-owned device slab."""
    h = C.c_void_p()
    N.check(N.lib.mr_matrix_rand_partition(session._ctx, nrows, ncols, blkSize, seed0, pr, pc, r, c,
                                           C.c_void_p(slab_ptr), slot_elems, C.byref(h)))
    return Dataset(session, h)


def _layout(nrows, ncols, blkSize, pr, pc, r, c):
    return N.mr_grid_layout(int(nrows), int(ncols), int(blkSize), int(pr), int(pc), int(r), int(c))


def create_sharded(session: "MatfastSession", nrows: int, ncols: int, blkSize: int, pr: int, pc: int, r: int, c: int) -> "Dataset":
    """A zero-filled dataset sharded over a pr x pc process grid: this rank's blocks in one IPC-exportable slab."""
    h = C.c_void_p()
    lay = _layout(nrows, ncols, blkSize, pr, pc, r, c)
    N.check(N.lib.mr_matrix_create_sharded(session._ctx, C.byref(lay), C.byref(h)))
    return Dataset(session, h)


def adopt_sharded(session: "MatfastSession", nrows: int, ncols: int, blkSize: int, pr: int, pc: int, r: int, c: int,
                  slab_ptr: int, isTransposed: bool = False) -> "Dataset":
    """The same over a caller-owned device slab (e.g. a torch tensor)."""
    h = C.c_void_p()
    lay = _layout(nrows, ncols, blkSize, pr, pc, r, c)
    N.check(N.lib.mr_matrix_adopt_sharded(session._ctx, C.byref(lay), C.c_void_p(slab_ptr), 1 if isTransposed else 0, C.byref(h)))
    return Dataset(session, h)


def ipc_export(device_ptr: int):
    """(64-byte CUDA IPC handle, offset) of the allocation that contains device_ptr."""
    buf = C.create_string_buffer(64)
    off = C.c_int64()
    N.check(N.lib.mr_ipc_export(C.c_void_p(device_ptr), buf, C.byref(off)))
    return bytes(buf.raw), int(off.value)


def ipc_open(session: "MatfastSession", handle: bytes, offset: int) -> int:
    p = C.c_void_p()
    N.check(N.lib.mr_ipc_open(session._ctx, C.create_string_buffer(handle, 64), int(offset), C.byref(p)))
    return p.value or 0


def memcpy_d2h(session: "MatfastSession", device_ptr: int, out: np.ndarray) -> np.ndarray:
    N.check(N.lib.mr_memcpy_d2h(session._ctx, C.c_void_p(device_ptr), out.ctypes.data_as(C.c_void_p), out.nbytes))
    return out


def grid_multiply(session: "MatfastSession", A: "Dataset", B: "Dataset", slabsA_row: Sequence[int], slabsB_col: Sequence[int],
                  nchunks: int = 4, gates: Optional[Sequence[Optional[int]]] = None) -> "Dataset":
    """``mr_grid_multiply``: this rank's share of C = A B; the slab pointers are valid in this process (IPC-opened peers).
    ``gates`` (optional, 2 * nchunks raw cudaEvent_t handles or None): gates[2 ch] guards the pull of piece ch of A (block rows),
    gates[2 ch + 1] the pull of piece ch of B (block columns) (``mr_grid_multiply_gated``)."""
    pa = (C.c_void_p * len(slabsA_row))(*[int(x) for x in slabsA_row])
    pb = (C.c_void_p * len(slabsB_col))(*[int(x) for x in slabsB_col])
    h = C.c_void_p()
    if gates is None:
        N.check(N.lib.mr_grid_multiply(A._h, B._h, pa, pb, int(nchunks), C.byref(h)))
    else:
        assert len(gates) == 2 * nchunks
        pg = (C.c_void_p * len(gates))(*[int(g) if g else None for g in gates])
        N.check(N.lib.mr_grid_multiply_gated(A._h, B._h, pa, pb, int(nchunks), pg, C.byref(h)))
    return Dataset(session, h)


def grid_multiply_rows(session: "MatfastSession", A_rows: "Dataset", leftRowNum: int, leftColNum: int, B: "Dataset",
                       slabsB_col: Sequence[int]) -> "Dataset":
    """``mr_grid_multiply_rows``: the left operand holds the complete block rows this rank owns (sparse or dense, replicated by
    the caller), only the sharded dense right operand is pulled from the grid column."""
    pb = (C.c_void_p * len(slabsB_col))(*[int(x) for x in slabsB_col])
    h = C.c_void_p()
    N.check(N.lib.mr_grid_multiply_rows(A_rows._h, int(leftRowNum), int(leftColNum), B._h, pb, C.byref(h)))
    return Dataset(session, h)


class Dataset:
    """A bag of ``(rid, cid, block)`` rows resident in HBM, or in page-locked host memory (``isHost``) (an ``mr_matrix`` handle)."""

    def __init__(self, session: MatfastSession, handle: C.c_void_p):
        self.matfastSession = session
        self._h = handle

    @staticmethod
    def _new(session: MatfastSession) -> "Dataset":
        h = C.c_void_p()
        N.check(N.lib.mr_matrix_create(session._ctx, C.byref(h)))
        return Dataset(session, h)

    def __del__(self):
        try:
            if self._h and self.matfastSession._ctx:
                N.lib.mr_matrix_free(self._h)
            self._h = C.c_void_p()
        except Exception:
            pass

    # -- block ingest / egress (MLMatrixSerializer.deserialize / serialize) -------------------
    def _put(self, rid: int, cid: int, m: MLMatrix) -> None:
        d = N.mr_block_desc()
        d.numRows, d.numCols = m.numRows, m.numCols
        d.isTransposed = 1 if m.isTransposed else 0
        d.values = _f64p(m.values)
        d.valuesLen = m.values.size
        if isinstance(m, SparseMatrix):
            d.type = 0
            d.colPtrs, d.colPtrsLen = _i32p(m.colPtrs), m.colPtrs.size
            d.rowIndices, d.rowIndicesLen = _i32p(m.rowIndices), m.rowIndices.size
        else:
            d.type = 1
        N.check(N.lib.mr_matrix_put_block(self._h, rid, cid, C.byref(d)))

    def put_block(self, rid: int, cid: int, m: MLMatrix) -> None:
        self._put(rid, cid, m)

    def put_blocks(self, blocks) -> None:
        """A whole Seq[MatrixBlock] in ONE ABI call (the per-block Python / ctypes overhead would otherwise delay the
        launch of a multiply that is pipelined against these very copies)."""
        blocks = list(blocks)
        n = len(blocks)
        if n == 0:
            return
        descs = (N.mr_block_desc * n)()
        rids = np.empty(n, dtype=np.int32)
        cids = np.empty(n, dtype=np.int32)
        for i, b in enumerate(blocks):
            m, d = b.matrix, descs[i]
            rids[i], cids[i] = b.rid, b.cid
            d.numRows, d.numCols = m.numRows, m.numCols
            d.isTransposed = 1 if m.isTransposed else 0
            d.values = _f64p(m.values)
            d.valuesLen = m.values.size
            if isinstance(m, SparseMatrix):
                d.type = 0
                d.colPtrs, d.colPtrsLen = _i32p(m.colPtrs), m.colPtrs.size
                d.rowIndices, d.rowIndicesLen = _i32p(m.rowIndices), m.rowIndices.size
            else:
                d.type = 1
        N.check(N.lib.mr_matrix_put_blocks(self._h, n, _i32p(rids), _i32p(cids), descs))

    def wait_ingest(self) -> None:
        """Host-blocking: every host->device copy of this dataset's blocks has completed (pinned sources may be reused)."""
        N.check(N.lib.mr_matrix_wait_ingest(self._h))

    def put_block_device(self, rid: int, cid: int, numRows: int, numCols: int, device_ptr: int,
                         isTransposed: bool = False) -> None:
        """Adopt a dense block that already lives in device memory (not freed by the engine)."""
        N.check(N.lib.mr_matrix_put_block_device(self._h, rid, cid, numRows, numCols,
                                                 C.c_void_p(device_ptr), 1 if isTransposed else 0))

    def put_blocks_device(self, rids, cids, numRows, numCols, device_ptrs, isTransposed=None) -> None:
        """Batched :meth:`put_block_device` (one ABI call for a whole gathered panel)."""
        n = len(rids)
        rids = np.ascontiguousarray(rids, dtype=np.int32)
        cids = np.ascontiguousarray(cids, dtype=np.int32)
        nr = np.ascontiguousarray(numRows, dtype=np.int32)
        nc = np.ascontiguousarray(numCols, dtype=np.int32)
        ptrs = (C.c_void_p * n)(*[int(p) for p in device_ptrs])
        flags = None
        if isTransposed is not None:
            flags = np.ascontiguousarray(isTransposed, dtype=np.uint8).ctypes.data_as(C.POINTER(C.c_uint8))
        N.check(N.lib.mr_matrix_put_blocks_device(self._h, n, _i32p(rids), _i32p(cids), _i32p(nr), _i32p(nc), ptrs, flags))

    def filter_blocks(self, row_mod: int = 1, row_rem: int = 0, col_mod: int = 1, col_rem: int = 0) -> "Dataset":
        """The blocks with rid % row_mod == row_rem and cid % col_mod == col_rem (a partition's share; no copy)."""
        h = C.c_void_p()
        N.check(N.lib.mr_matrix_filter_blocks(self._h, int(row_mod), int(row_rem), int(col_mod), int(col_rem), C.byref(h)))
        return Dataset(self.matfastSession, h)

    def has_block(self, rid: int, cid: int) -> bool:
        out = C.c_int32()
        N.check(N.lib.mr_matrix_has_block(self._h, int(rid), int(cid), C.byref(out)))
        return bool(out.value)

    def block_ids(self) -> List[tuple]:
        n = C.c_int64()
        N.check(N.lib.mr_matrix_num_blocks(self._h, C.byref(n)))
        rids = np.empty(n.value, dtype=np.int32)
        cids = np.empty(n.value, dtype=np.int32)
        if n.value:
            N.check(N.lib.mr_matrix_block_ids(self._h, _i32p(rids), _i32p(cids), n.value))
        return list(zip(rids.tolist(), cids.tolist()))

    def get_block(self, rid: int, cid: int, out: Optional[np.ndarray] = None) -> MLMatrix:
        d = N.mr_block_desc()
        N.check(N.lib.mr_matrix_get_block(self._h, rid, cid, C.byref(d)))  # sizes only
        values = out if out is not None else np.empty(d.valuesLen, dtype=np.float64)
        assert values.size >= d.valuesLen and values.dtype == np.float64
        d.values = _f64p(values)
        if d.type == 0:
            colPtrs = np.empty(d.colPtrsLen, dtype=np.int32)
            rowIndices = np.empty(d.rowIndicesLen, dtype=np.int32)
            d.colPtrs, d.rowIndices = _i32p(colPtrs), _i32p(rowIndices)
        N.check(N.lib.mr_matrix_get_block(self._h, rid, cid, C.byref(d)))
        if d.type == 0:
            return SparseMatrix(d.numRows, d.numCols, colPtrs, rowIndices, values[:d.valuesLen],
                                bool(d.isTransposed))
        return DenseMatrix(d.numRows, d.numCols, values[:d.valuesLen], bool(d.isTransposed))

    def block_device_ptr(self, rid: int, cid: int) -> int:
        p = C.c_void_p()
        N.check(N.lib.mr_matrix_block_device_ptr(self._h, rid, cid, C.byref(p)))
        return p.value or 0

    def collect(self) -> List[MatrixBlock]:
        """``.collect()`` / ``.rdd.foreach``: every row back on the host, ordered by (rid, cid)."""
        return [MatrixBlock(r, c, self.get_block(r, c)) for r, c in self.block_ids()]

    def toNumpy(self, nrows: int, ncols: int, blkSize: int, order: str = "C") -> np.ndarray:
        """The dataset as one ``nrows x ncols`` array (``mr_matrix_to_dense``): absent blocks are zeros, sparse blocks scattered,
        ``isTransposed`` honoured; assembled on the device, panel by panel."""
        if order not in ("C", "F"):
            raise ValueError(f"order must be 'C' or 'F', got {order!r}")
        out = np.empty((int(nrows), int(ncols)), dtype=np.float64, order=order)
        rowMajor = 1 if order == "C" else 0
        N.check(N.lib.mr_matrix_to_dense(self._h, int(nrows), int(ncols), int(blkSize), C.c_void_p(out.ctypes.data),
                                         int(ncols) if rowMajor else int(nrows), rowMajor, None))
        return out

    def toTorch(self, nrows: int, ncols: int, blkSize: int):
        """The same as a contiguous float64 CUDA tensor on the session's device; ``torch.cuda.current_stream()`` is ordered behind
        the assembly (no host wait)."""
        import torch
        dev = torch.device("cuda", self.matfastSession._cuda_device())
        out = torch.empty((int(nrows), int(ncols)), dtype=torch.float64, device=dev)
        N.check(N.lib.mr_matrix_to_dense(self._h, int(nrows), int(ncols), int(blkSize), C.c_void_p(out.data_ptr()), int(ncols), 1,
                                         C.c_void_p(_torch_stream(dev))))
        return out

    # -- residence ------------------------------------------------------------------------------
    @property
    def isHost(self) -> bool:
        """True when the blocks live in page-locked host memory (``createHostDataset`` / ``toHost``)."""
        out = C.c_int32()
        N.check(N.lib.mr_matrix_is_host(self._h, C.byref(out)))
        return bool(out.value)

    def toHost(self) -> "Dataset":
        """A host-resident copy (ids, shapes, formats and isTransposed flags kept)."""
        return self._unary(N.lib.mr_matrix_to_host)

    def toDevice(self) -> "Dataset":
        """A device-resident copy; the copy runs on the ingest stream and a multiply may start before it has finished."""
        return self._unary(N.lib.mr_matrix_to_device)

    # -- operators: signatures of M/Dataset.scala:57-152 ----------------------------------------
    def _binary(self, fn, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize) -> "Dataset":
        h = C.c_void_p()
        N.check(fn(self._h, int(leftRowNum), int(leftColNum), right._h, int(rightRowNum), int(rightColNum),
                   int(blkSize), C.byref(h)))
        return Dataset(self.matfastSession, h)

    def matrixMultiply(self, leftRowNum, leftColNum, right: "Dataset", rightRowNum, rightColNum, blkSize) -> "Dataset":
        """M/Dataset.scala:134-142."""
        return self._binary(N.lib.mr_matrix_multiply, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize)

    def addElement(self, leftRowNum, leftColNum, right: "Dataset", rightRowNum, rightColNum, blkSize) -> "Dataset":
        """M/Dataset.scala:105-112."""
        return self._binary(N.lib.mr_add_element, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize)

    def multiplyElement(self, leftRowNum, leftColNum, right: "Dataset", rightRowNum, rightColNum, blkSize) -> "Dataset":
        """M/Dataset.scala:114-122."""
        return self._binary(N.lib.mr_multiply_element, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize)

    def divideElement(self, leftRowNum, leftColNum, right: "Dataset", rightRowNum, rightColNum, blkSize) -> "Dataset":
        """M/Dataset.scala:124-132."""
        return self._binary(N.lib.mr_divide_element, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize)

    def matrixRankOneUpdate(self, leftRowNum, leftColNum, right: "Dataset", rightRowNum, rightColNum, blkSize) -> "Dataset":
        """M/Dataset.scala:144-152."""
        return self._binary(N.lib.mr_rank_one_update, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize)

    def _unary(self, fn, *args) -> "Dataset":
        h = C.c_void_p()
        N.check(fn(self._h, *args, C.byref(h)))
        return Dataset(self.matfastSession, h)

    def transpose(self) -> "Dataset":
        """M/Dataset.scala:59-61."""
        return self._unary(N.lib.mr_transpose)

    def t(self) -> "Dataset":
        """M/Dataset.scala:57."""
        return self.transpose()

    def addScalar(self, alpha: float) -> "Dataset":
        """M/Dataset.scala:89-91."""
        return self._unary(N.lib.mr_add_scalar, float(alpha))

    def multiplyScalar(self, alpha: float) -> "Dataset":
        """M/Dataset.scala:93-97."""
        return self._unary(N.lib.mr_multiply_scalar, float(alpha))

    def power(self, alpha: float) -> "Dataset":
        """M/Dataset.scala:99-103."""
        return self._unary(N.lib.mr_power, float(alpha))

    def vec(self, nrows, ncols, blkSize) -> "Dataset":
        """M/Dataset.scala:84-87."""
        return self._unary(N.lib.mr_vec, int(nrows), int(ncols), int(blkSize))

    def project(self, nrows, ncols, blkSize, rowOrCol: bool, index) -> "Dataset":
        """M/Dataset.scala:38-47."""
        return self._unary(N.lib.mr_project, int(nrows), int(ncols), int(blkSize), 1 if rowOrCol else 0, int(index))

    def selection(self, nrows, ncols, blkSize, rowIdx, colIdx) -> "Dataset":
        """M/Dataset.scala:49-55."""
        return self._unary(N.lib.mr_selection, int(nrows), int(ncols), int(blkSize), int(rowIdx), int(colIdx))

    def rowSum(self, nrows, ncols) -> "Dataset":
        """M/Dataset.scala:63-66."""
        return self._unary(N.lib.mr_row_sum, int(nrows), int(ncols))

    def colSum(self, nrows, ncols) -> "Dataset":
        """M/Dataset.scala:68-71."""
        return self._unary(N.lib.mr_col_sum, int(nrows), int(ncols))

    def sum(self, nrows, ncols) -> "Dataset":
        """M/Dataset.scala:73-76."""
        return self._unary(N.lib.mr_sum, int(nrows), int(ncols))

    def trace(self, nrows, ncols) -> "Dataset":
        """M/Dataset.scala:78-82."""
        return self._unary(N.lib.mr_trace, int(nrows), int(ncols))

    def materialize(self) -> "Dataset":
        """Every dense block rewritten column-major (``toArray``, M/matrix/MLMatrix.scala:55-61)."""
        return self._unary(N.lib.mr_materialize)
