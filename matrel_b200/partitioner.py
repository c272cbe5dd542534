"""Block -> partition maps, bit-exact with M/partitioner/*.scala, evaluated by the C ABI.

M/ = <reference>/src/main/scala/org/apache/spark/sql/matfast/
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

from . import _native as N


class RowPartitioner:
    """M/partitioner/RowPartitioner.scala:26-48."""

    def __init__(self, partitions: int):
        self.numPartitions = int(partitions)

    def getPartition(self, key: Tuple[int, ...]) -> int:
        _check_key(key)
        out = C.c_int32()
        N.check(N.lib.mr_row_partition(key[0], key[1], self.numPartitions, C.byref(out)))
        return out.value


class ColumnPartitioner:
    """M/partitioner/ColumnPartitioner.scala:26-48."""

    def __init__(self, partitions: int):
        self.numPartitions = int(partitions)

    def getPartition(self, key: Tuple[int, ...]) -> int:
        _check_key(key)
        out = C.c_int32()
        N.check(N.lib.mr_column_partition(key[0], key[1], self.numPartitions, C.byref(out)))
        return out.value


class IndexPartitioner:
    """M/partitioner/IndexPartitioner.scala:23-45."""

    def __init__(self, partitions: int):
        self.numPartitions = int(partitions)

    def getPartition(self, key: int) -> int:
        if not isinstance(key, int):
            raise ValueError(f"Unrecognized key: {key}")
        out = C.c_int32()
        N.check(N.lib.mr_index_partition(key, self.numPartitions, C.byref(out)))
        return out.value


class BlockCyclicPartitioner:
    """M/partitioner/BlockCyclicPartitioner.scala:31-62 (ids reproduced bit-exactly, incl. defect B2)."""

    def __init__(self, ROW_BLKS: int, COL_BLKS: int, ROW_BLKS_PER_PARTITION: int, COL_BLKS_PER_PARTITION: int):
        self.params = (C.c_int32 * 4)(ROW_BLKS, COL_BLKS, ROW_BLKS_PER_PARTITION, COL_BLKS_PER_PARTITION)
        out = C.c_int32()
        N.check(N.lib.mr_block_cyclic_num_partitions(self.params, C.byref(out)))
        self.numPartitions = out.value

    def getPartition(self, key: Tuple[int, ...]) -> int:
        _check_key(key)
        out = C.c_int32()
        N.check(N.lib.mr_block_cyclic_partition(self.params, key[0], key[1], C.byref(out)))
        return out.value


def genBlockCyclicPartitioner(nrows: int, ncols: int, blkSize: int) -> Tuple[int, int, int, int]:
    """M/execution/MatfastExecutionHelper.scala:46-62."""
    out = (C.c_int32 * 4)()
    N.check(N.lib.mr_gen_block_cyclic(nrows, ncols, blkSize, out))
    return tuple(out)


PART_ROW, PART_COLUMN, PART_INDEX, PART_BLOCK_CYCLIC = 0, 1, 2, 3


def partition_id(scheme: int, params, rid: int, cid: int) -> int:
    """`mr_partition_id`: one entry point over the four schemes (params = (partitions,) or the block-cyclic 4-tuple)."""
    p = (C.c_int32 * 4)(*(list(params) + [0, 0, 0, 0])[:4])
    out = C.c_int32()
    N.check(N.lib.mr_partition_id(int(scheme), p, int(rid), int(cid), C.byref(out)))
    return out.value


def _check_key(key) -> None:
    if not (isinstance(key, tuple) and len(key) in (2, 3) and all(isinstance(k, int) for k in key)):
        raise ValueError(f"Unrecognized key: {key}")  # IllegalArgumentException(s"Unrecognized key: $key")
