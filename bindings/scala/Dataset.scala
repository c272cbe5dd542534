/*
 * Scala facade a MatRel maintainer adds next to
 * src/main/scala/org/apache/spark/sql/matfast/Dataset.scala to route the block-multiply path to the
 * H100 engine.  Same method names / argument order as the reference's Dataset (Dataset.scala:38-152);
 * each call forwards to the C ABI (include/matrel.h) through the JNI shim (bindings/jni/matrel_jni.cpp).
 * NOT compiled in this image (no scalac / JDK).
 */
package org.apache.spark.sql.matfast.b200

import org.apache.spark.sql.matfast.matrix.{DenseMatrix, MLMatrix, MatrixBlock, SparseMatrix}

private[b200] object Native {
  System.loadLibrary("matrel_jni") // links libmatrel_b200.so
  @native def init(device: Int, compatBugs: Boolean, gemmAlgo: Int): Long
  @native def shutdown(ctx: Long): Unit
  @native def sync(ctx: Long): Unit
  @native def matrixCreate(ctx: Long): Long
  @native def matrixFree(m: Long): Unit
  @native def matrixCreateHost(ctx: Long): Long
  @native def isHost(m: Long): Boolean
  @native def toHost(m: Long): Long
  @native def toDevice(m: Long): Long
  @native def putBlock(m: Long, rid: Int, cid: Int, tpe: Byte, numRows: Int, numCols: Int,
                       colPtrs: Array[Int], rowIndices: Array[Int], values: Array[Double],
                       isTransposed: Boolean): Unit
  @native def matrixFromArray(ctx: Long, values: Array[Double], nrows: Long, ncols: Long, blk: Int): Long
  @native def matrixToArray(m: Long, nrows: Long, ncols: Long, blk: Int, out: Array[Double]): Unit
  @native def numBlocks(m: Long): Long
  @native def hasBlock(m: Long, rid: Int, cid: Int): Boolean
  @native def blockIds(m: Long): Array[Int] // (rid, cid) pairs, ascending
  /** {type, numRows, numCols, isTransposed, valuesLen, colPtrsLen, rowIndicesLen} */
  @native def blockMeta(m: Long, rid: Int, cid: Int): Array[Long]
  @native def blockArrays(m: Long, rid: Int, cid: Int, colPtrs: Array[Int], rowIndices: Array[Int], values: Array[Double]): Unit
  @native def matrixMultiply(l: Long, lr: Long, lc: Long, r: Long, rr: Long, rc: Long, blk: Int): Long
  @native def addElement(l: Long, lr: Long, lc: Long, r: Long, rr: Long, rc: Long, blk: Int): Long
  @native def multiplyElement(l: Long, lr: Long, lc: Long, r: Long, rr: Long, rc: Long, blk: Int): Long
  @native def divideElement(l: Long, lr: Long, lc: Long, r: Long, rr: Long, rc: Long, blk: Int): Long
  @native def matrixRankOneUpdate(l: Long, lr: Long, lc: Long, r: Long, rr: Long, rc: Long, blk: Int): Long
  @native def transpose(a: Long): Long
  @native def addScalar(a: Long, alpha: Double): Long
  @native def multiplyScalar(a: Long, alpha: Double): Long
  @native def power(a: Long, alpha: Double): Long
  @native def rowSum(a: Long, nrows: Long, ncols: Long): Long
  @native def colSum(a: Long, nrows: Long, ncols: Long): Long
  @native def sum(a: Long, nrows: Long, ncols: Long): Long
  @native def trace(a: Long, nrows: Long, ncols: Long): Long
  @native def project(a: Long, nrows: Long, ncols: Long, blk: Int, rowOrCol: Boolean, index: Long): Long
  @native def selection(a: Long, nrows: Long, ncols: Long, blk: Int, rowIdx: Long, colIdx: Long): Long
  @native def vec(a: Long, nrows: Long, ncols: Long, blk: Int): Long
  @native def partitionId(scheme: Int, p0: Int, p1: Int, p2: Int, p3: Int, rid: Int, cid: Int): Int
  @native def genBlockCyclic(nrows: Long, ncols: Long, blk: Int): Array[Int]
  // one JVM, all GPUs
  @native def gridInit(ngpus: Int, compatBugs: Boolean, gemmAlgo: Int): Long
  @native def gridShutdown(g: Long): Unit
  @native def dmatrixCreate(g: Long, nrows: Long, ncols: Long, blk: Int): Long
  @native def dmatrixFree(m: Long): Unit
  @native def dmatrixPutBlock(m: Long, rid: Int, cid: Int, tpe: Byte, numRows: Int, numCols: Int,
                              colPtrs: Array[Int], rowIndices: Array[Int], values: Array[Double],
                              isTransposed: Boolean): Unit
  @native def dmatrixHasBlock(m: Long, rid: Int, cid: Int): Boolean
  @native def dmatrixBlockMeta(m: Long, rid: Int, cid: Int): Array[Long]
  @native def dmatrixBlockArrays(m: Long, rid: Int, cid: Int, colPtrs: Array[Int], rowIndices: Array[Int], values: Array[Double]): Unit
  @native def dmatrixOwner(m: Long, rid: Int, cid: Int): Int
  @native def dmatrixMultiply(a: Long, b: Long): Long
  @native def dmatrixMultiplySplitK(a: Long, b: Long): Long
  @native def dmatrixElementwise(op: Int, a: Long, b: Long): Long
  @native def dmatrixReduceScalar(a: Long, what: Int): Double
  @native def dmatrixRepartition(a: Long, newPr: Int, newPc: Int): Long
  @native def dmatrixTranspose(a: Long): Long
  @native def dmatrixScalar(op: Int, a: Long, alpha: Double): Long
  @native def dmatrixAxisSum(a: Long, axis: Int): Long
  @native def dmatrixProject(a: Long, rowOrCol: Boolean, index: Long): Long
  @native def dmatrixSelection(a: Long, rowIdx: Long, colIdx: Long): Long

  /** MLMatrixSerializer.deserialize (util/MLMatrixSerializer.scala:50-69) from the two-call protocol. */
  def readBlock(meta: Array[Long], fill: (Array[Int], Array[Int], Array[Double]) => Unit): MLMatrix = {
    val (tpe, numRows, numCols, isT) = (meta(0), meta(1).toInt, meta(2).toInt, meta(3) != 0)
    val values = new Array[Double](meta(4).toInt)
    if (tpe == 1) {
      fill(null, null, values)
      new DenseMatrix(numRows, numCols, values, isT)
    } else {
      val colPtrs = new Array[Int](meta(5).toInt)
      val rowIndices = new Array[Int](meta(6).toInt)
      fill(colPtrs, rowIndices, values)
      new SparseMatrix(numRows, numCols, colPtrs, rowIndices, values, isT)
    }
  }

  def put(h: Long, b: MatrixBlock, f: (Long, Int, Int, Byte, Int, Int, Array[Int], Array[Int], Array[Double], Boolean) => Unit): Unit =
    b.matrix match { // the 7 fields of MLMatrixSerializer.serialize (util/MLMatrixSerializer.scala:26-48)
      case d: DenseMatrix => f(h, b.rid, b.cid, 1, d.numRows, d.numCols, null, null, d.values, d.isTransposed)
      case s: SparseMatrix => f(h, b.rid, b.cid, 0, s.numRows, s.numCols, s.colPtrs, s.rowIndices, s.values, s.isTransposed)
    }
}

/** gemmAlgo: 0 = auto (wgmma Ozaki-II with the device-side guard, DMMA otherwise), 1 = DMMA fp64 (see matrel.h). */
class B200Session(device: Int = -1, compatBugs: Boolean = true, gemmAlgo: Int = 0) {
  private[b200] val ctx: Long = Native.init(device, compatBugs, gemmAlgo)
  def stop(): Unit = Native.shutdown(ctx)
  def sync(): Unit = Native.sync(ctx)

  /** Seq(MatrixBlock(...)).toDS() (example/BasicMatrixOps.scala:115-116) */
  def toDS(blocks: Seq[MatrixBlock]): B200Dataset = {
    val h = Native.matrixCreate(ctx)
    blocks.foreach(b => Native.put(h, b, Native.putBlock))
    new B200Dataset(this, h)
  }

  /** The same, host-resident: the blocks live in page-locked host memory owned by the engine (datasets larger than the GPU);
   *  matrixMultiply streams them through the device, every other operator needs toDevice() first */
  def toHostDS(blocks: Seq[MatrixBlock]): B200Dataset = {
    val h = Native.matrixCreateHost(ctx)
    blocks.foreach(b => Native.put(h, b, Native.putBlock))
    new B200Dataset(this, h)
  }

  /** A whole nrows x ncols matrix (values column-major, as DenseMatrix.values) as a dataset of blkSize x blkSize DenseMatrix
   *  blocks, every block present; cut on the device */
  def fromArray(values: Array[Double], nrows: Long, ncols: Long, blkSize: Int): B200Dataset =
    new B200Dataset(this, Native.matrixFromArray(ctx, values, nrows, ncols, blkSize))
}

class B200Dataset private[b200](val session: B200Session, private[b200] val h: Long) {
  private def wrap(x: Long) = new B200Dataset(session, x)

  // ---- egress: what .collect() / .rdd.foreach return in the reference (rows (rid, cid, matrix))
  def blockIds: Seq[(Int, Int)] = Native.blockIds(h).grouped(2).map(p => (p(0), p(1))).toSeq
  def hasBlock(rid: Int, cid: Int): Boolean = Native.hasBlock(h, rid, cid)
  def getBlock(rid: Int, cid: Int): MLMatrix =
    Native.readBlock(Native.blockMeta(h, rid, cid), (cp, ri, v) => Native.blockArrays(h, rid, cid, cp, ri, v))
  def collect(): Seq[MatrixBlock] = blockIds.map { case (i, j) => MatrixBlock(i, j, getBlock(i, j)) }
  /** DenseMatrix.toArray (matrix/MLMatrix.scala:55-61) for the whole dataset: column-major, absent blocks are zeros */
  def toArray(nrows: Long, ncols: Long, blkSize: Int): Array[Double] = {
    require(nrows * ncols <= Int.MaxValue, s"a $nrows x $ncols matrix does not fit one JVM array")
    val out = new Array[Double]((nrows * ncols).toInt)
    Native.matrixToArray(h, nrows, ncols, blkSize, out)
    out
  }

  // ---- residence
  def isHost: Boolean = Native.isHost(h)
  def toHost(): B200Dataset = wrap(Native.toHost(h))
  def toDevice(): B200Dataset = wrap(Native.toDevice(h))

  // ---- operators: Dataset.scala:38-152
  def project(nrows: Long, ncols: Long, blkSize: Int, rowOrCol: Boolean, index: Long): B200Dataset =
    wrap(Native.project(h, nrows, ncols, blkSize, rowOrCol, index))
  def selection(nrows: Long, ncols: Long, blkSize: Int, rowIdx: Long, colIdx: Long): B200Dataset =
    wrap(Native.selection(h, nrows, ncols, blkSize, rowIdx, colIdx))
  def t(): B200Dataset = transpose()
  def transpose(): B200Dataset = wrap(Native.transpose(h))
  def rowSum(nrows: Long, ncols: Long): B200Dataset = wrap(Native.rowSum(h, nrows, ncols))
  def colSum(nrows: Long, ncols: Long): B200Dataset = wrap(Native.colSum(h, nrows, ncols))
  def sum(nrows: Long, ncols: Long): B200Dataset = wrap(Native.sum(h, nrows, ncols))
  def trace(nrows: Long, ncols: Long): B200Dataset = wrap(Native.trace(h, nrows, ncols))
  def vec(nrows: Long, ncols: Long, blkSize: Int): B200Dataset = wrap(Native.vec(h, nrows, ncols, blkSize))
  def addScalar(alpha: Double): B200Dataset = wrap(Native.addScalar(h, alpha))
  def multiplyScalar(alpha: Double): B200Dataset = wrap(Native.multiplyScalar(h, alpha))
  def power(alpha: Double): B200Dataset = wrap(Native.power(h, alpha))
  def addElement(leftRowNum: Long, leftColNum: Long, right: B200Dataset,
                 rightRowNum: Long, rightColNum: Long, blkSize: Int): B200Dataset =
    wrap(Native.addElement(h, leftRowNum, leftColNum, right.h, rightRowNum, rightColNum, blkSize))
  def multiplyElement(leftRowNum: Long, leftColNum: Long, right: B200Dataset,
                      rightRowNum: Long, rightColNum: Long, blkSize: Int): B200Dataset =
    wrap(Native.multiplyElement(h, leftRowNum, leftColNum, right.h, rightRowNum, rightColNum, blkSize))
  def divideElement(leftRowNum: Long, leftColNum: Long, right: B200Dataset,
                    rightRowNum: Long, rightColNum: Long, blkSize: Int): B200Dataset =
    wrap(Native.divideElement(h, leftRowNum, leftColNum, right.h, rightRowNum, rightColNum, blkSize))
  def matrixMultiply(leftRowNum: Long, leftColNum: Long, right: B200Dataset,
                     rightRowNum: Long, rightColNum: Long, blkSize: Int): B200Dataset =
    wrap(Native.matrixMultiply(h, leftRowNum, leftColNum, right.h, rightRowNum, rightColNum, blkSize))
  def matrixRankOneUpdate(leftRowNum: Long, leftColNum: Long, right: B200Dataset,
                          rightRowNum: Long, rightColNum: Long, blkSize: Int): B200Dataset =
    wrap(Native.matrixRankOneUpdate(h, leftRowNum, leftColNum, right.h, rightRowNum, rightColNum, blkSize))
  override def finalize(): Unit = Native.matrixFree(h)
}

/** Bit-exact restatement of M/partitioner/{Row,Column,Index,BlockCyclic}Partitioner.getPartition. */
object B200Partitioner {
  val Row = 0; val Column = 1; val Index = 2; val BlockCyclic = 3
  def partitionId(scheme: Int, params: Array[Int], rid: Int, cid: Int): Int = {
    val p = params.padTo(4, 0)
    Native.partitionId(scheme, p(0), p(1), p(2), p(3), rid, cid)
  }
  /** MatfastExecutionHelper.genBlockCyclicPartitioner (:46-62) */
  def genBlockCyclic(nrows: Long, ncols: Long, blkSize: Int): Array[Int] = Native.genBlockCyclic(nrows, ncols, blkSize)
}

/**
 * One JVM drives all GPUs of the box (mr_init_grid): block partitions are sharded over a pr x pc grid by the reference's
 * RowPartitioner x ColumnPartitioner arithmetic; the co-partition shuffle of matrixMultiplyGeneral becomes copy-engine pulls
 * over NVLink, overlapped with the multiply; reductions and re-partitioning go through NCCL.  No Spark executors.
 */
class B200GridSession(ngpus: Int, compatBugs: Boolean = true, gemmAlgo: Int = 0) {
  private[b200] val g: Long = Native.gridInit(ngpus, compatBugs, gemmAlgo)
  def stop(): Unit = Native.gridShutdown(g)
  def toDS(nrows: Long, ncols: Long, blkSize: Int, blocks: Seq[MatrixBlock]): B200GridDataset = {
    val h = Native.dmatrixCreate(g, nrows, ncols, blkSize)
    blocks.foreach(b => Native.put(h, b, Native.dmatrixPutBlock)) // each block goes to the GPU that owns it
    new B200GridDataset(this, h, nrows, ncols, blkSize)
  }
}

class B200GridDataset private[b200](val session: B200GridSession, private[b200] val h: Long,
                                    val nrows: Long, val ncols: Long, val blkSize: Int) {
  private def wrap(x: Long, r: Long, c: Long) = new B200GridDataset(session, x, r, c, blkSize)
  def owner(rid: Int, cid: Int): Int = Native.dmatrixOwner(h, rid, cid)
  def getBlock(rid: Int, cid: Int): MLMatrix =
    Native.readBlock(Native.dmatrixBlockMeta(h, rid, cid), (cp, ri, v) => Native.dmatrixBlockArrays(h, rid, cid, cp, ri, v))
  def collect(): Seq[MatrixBlock] = {
    val nbr = ((nrows + blkSize - 1) / blkSize).toInt
    val nbc = ((ncols + blkSize - 1) / blkSize).toInt
    for (i <- 0 until nbr; j <- 0 until nbc if Native.dmatrixHasBlock(h, i, j)) yield MatrixBlock(i, j, getBlock(i, j))
  }
  /** Dataset.matrixMultiply (:134-142); the dimensions travel with the handles */
  def matrixMultiply(right: B200GridDataset): B200GridDataset = wrap(Native.dmatrixMultiply(h, right.h), nrows, right.ncols)
  /** The same product split over K (matrixMultiplyGeneral's join + reduceByKey(add), MatfastExecutionHelper.scala:235-263): for
   *  products with few output blocks (Gram matrices, low-rank factors); the partials are summed in GPU order, bit-reproducibly */
  def matrixMultiplySplitK(right: B200GridDataset): B200GridDataset =
    wrap(Native.dmatrixMultiplySplitK(h, right.h), nrows, right.ncols)
  def addElement(right: B200GridDataset): B200GridDataset = wrap(Native.dmatrixElementwise(0, h, right.h), nrows, ncols)
  def multiplyElement(right: B200GridDataset): B200GridDataset = wrap(Native.dmatrixElementwise(1, h, right.h), nrows, ncols)
  def divideElement(right: B200GridDataset): B200GridDataset = wrap(Native.dmatrixElementwise(2, h, right.h), nrows, ncols)
  def sum(): Double = Native.dmatrixReduceScalar(h, 0)
  def trace(): Double = Native.dmatrixReduceScalar(h, 1)
  /** repartitionWithTargetPartitioner (MatfastExecutionHelper.scala:34-44): (P, 1) = RowPartitioner, (1, P) = ColumnPartitioner */
  def repartition(newPr: Int, newPc: Int): B200GridDataset = wrap(Native.dmatrixRepartition(h, newPr, newPc), nrows, ncols)
  /** Dataset.t / transpose (:57-61): blocks swap ids and move to their new owners; payloads untouched, isTransposed flipped */
  def t(): B200GridDataset = transpose()
  def transpose(): B200GridDataset = wrap(Native.dmatrixTranspose(h), ncols, nrows)
  /** Dataset.addScalar / multiplyScalar / power (:89-103): a map over the blocks each GPU owns */
  def addScalar(alpha: Double): B200GridDataset = wrap(Native.dmatrixScalar(0, h, alpha), nrows, ncols)
  def multiplyScalar(alpha: Double): B200GridDataset = wrap(Native.dmatrixScalar(1, h, alpha), nrows, ncols)
  def power(alpha: Double): B200GridDataset = wrap(Native.dmatrixScalar(2, h, alpha), nrows, ncols)
  /** Dataset.rowSum / colSum (:63-72): local line sums + one ncclAllReduce; the result is nrows x 1 / 1 x ncols */
  def rowSum(): B200GridDataset = wrap(Native.dmatrixAxisSum(h, 0), nrows, 1L)
  def colSum(): B200GridDataset = wrap(Native.dmatrixAxisSum(h, 1), 1L, ncols)
  /** Dataset.project (:38-47) / selection (:49-55); dimensions and block size travel with the handle */
  def project(rowOrCol: Boolean, index: Long): B200GridDataset =
    if (rowOrCol) wrap(Native.dmatrixProject(h, true, index), 1L, ncols) else wrap(Native.dmatrixProject(h, false, index), nrows, 1L)
  def selection(rowIdx: Long, colIdx: Long): B200GridDataset = wrap(Native.dmatrixSelection(h, rowIdx, colIdx), 1L, 1L)
  override def finalize(): Unit = Native.dmatrixFree(h)
}
