"""matrel_b200 -- H100-native block-matrix engine behind the MatRel/MatFast Dataset operator API.

Layout (only what the block-multiply hot path needs):
  csrc/            sm_90a CUDA kernels + the C-ABI host layer (include/matrel.h)
  _native.py       ctypes binding of the C ABI (fails loudly when the .so is missing)
  matrix.py        DenseMatrix / SparseMatrix / MatrixBlock containers (reference data model)
  dataset.py       MatfastSession + Dataset: the reference's operator names and argument order
  partitioner.py   Row / Column / Index / BlockCyclic partitioners (bit-exact ids)
  plan.py          lazy logical nodes + the planner's algebraic rewrites (MatfastPlanner.scala)
  distributed.py   one process per GPU: sharded multiply, transpose, element-wise ops and aggregates over torch.distributed (NCCL)
"""
from .matrix import DenseMatrix, MatrixBlock, SparseMatrix  # noqa: F401
from .dataset import Dataset, MatfastSession  # noqa: F401
from .partitioner import (BlockCyclicPartitioner, ColumnPartitioner, IndexPartitioner,  # noqa: F401
                          RowPartitioner, genBlockCyclicPartitioner, partition_id)
from ._native import (CudaError, IllegalArgumentException, MatrelError,  # noqa: F401
                      UnsupportedOperation)

__version__ = "0.1.0"
