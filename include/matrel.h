/*
 * matrel.h -- C ABI of the H100-native block-matrix engine (drop-in for the MatRel/MatFast
 * block-multiply hot path).  Plain C: opaque handles, pointers and sizes; no C++/torch types.
 *
 * Every entry point names the reference interface it replaces.  Paths are relative to
 * <reference>/src/main/scala/org/apache/spark/sql/matfast/ ("M/").
 *
 * Conventions
 *   - every function returns mr_status; on failure mr_last_error() (thread-local) holds the
 *     message, reproducing the reference's `require` text ("requirement failed: ...") so a JNI
 *     shim can ThrowNew(IllegalArgumentException, msg).  Nothing throws or aborts across the ABI.
 *   - a "dataset" (mr_matrix) is a bag of (rid, cid, block) rows exactly like the reference's
 *     Dataset rows (rid Int, cid Int, struct7); absent blocks are implicit zeros.  Matrix
 *     dimensions are passed per operator call, as in M/Dataset.scala.
 *   - blocks live in device memory (HBM) behind the handle; operators enqueue CUDA kernels on the
 *     context stream and return new handles (operators are pure).  There is NO CPU fallback:
 *     without a usable CUDA device mr_init fails with MR_ECUDA.
 */
#ifndef MATREL_H_
#define MATREL_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MR_API __attribute__((visibility("default")))

typedef int32_t mr_status;
enum {
  MR_OK = 0,
  MR_EINVAL = 1,  /* IllegalArgumentException("requirement failed: ...") */
  MR_EDIM = 2,    /* dimension `require` of an operator failed (also IllegalArgumentException) */
  MR_ENOMEM = 3,
  MR_ECUDA = 4,
  MR_ENOTSUP = 5, /* SparkException("Unsupported matrix type ...") / out-of-scope dispatch row */
  MR_ENOTFOUND = 6,
  MR_ENCCL = 7    /* a collective of the multi-GPU layer failed, or NCCL could not be loaded */
};

typedef struct mr_context mr_context; /* one per process per GPU (replaces MatfastSession) */
typedef struct mr_matrix mr_matrix;   /* a Dataset of MatrixBlock rows, device resident */
typedef struct mr_grid mr_grid;       /* one process driving several GPUs: a pr x pc grid of contexts (mr_init_grid) */
typedef struct mr_dmatrix mr_dmatrix; /* a Dataset sharded over the GPUs of an mr_grid */

/* The 7-field block struct of MatrixUDT / MLMatrixSerializer
 * (M/matrix/MLMatrix.scala:176-184, M/util/MLMatrixSerializer.scala:26-48). */
typedef struct mr_block_desc {
  uint8_t type;          /* [0] 0 = sparse, 1 = dense */
  int32_t numRows;       /* [1] */
  int32_t numCols;       /* [2] */
  int32_t* colPtrs;      /* [3] NULL for dense; length (isTransposed ? numRows : numCols) + 1 */
  int32_t* rowIndices;   /* [4] NULL for dense; length nnz */
  double* values;        /* [5] dense: numRows*numCols, column-major (row-major if isTransposed) */
  uint8_t isTransposed;  /* [6] */
  int64_t colPtrsLen;    /* array lengths (JVM arrays carry theirs; C needs them spelled out) */
  int64_t rowIndicesLen;
  int64_t valuesLen;
} mr_block_desc;

typedef struct mr_options {
  int32_t device;       /* CUDA device ordinal; -1 = current device */
  int32_t compat_bugs;  /* 1 = reproduce reference defects B3/B4 (SURVEY.md 2.3); 0 = intended math */
  int32_t gemm_algo;    /* 0 = auto: large regular dense products run on the int8 tensor cores (Ozaki-II: int8 residue GEMMs +
                           CRT, fp64-exact to 1e-14 on data of ordinary range), guarded on the device: isolated elements more than
                           alpha - 18 binary orders (29 at K = 16384) below the maximum of their row of A / column of B are left out
                           of the residues and their products added exactly in fp64; Inf / NaN operands, more than 64 such elements
                           in one block row / block column, K >= 2^17, irregular block grids and small products take the exact DMMA
                           kernel instead;
                           1 = DMMA fp64 tensor-core kernel (mma.sync m8n8k4 f64), always;
                           2 = Ozaki-I int8 wgmma kernel (digit slices); 3 = 3xTF32 wgmma kernel (fp32 results);
                           4 = Ozaki-II without the range guard.  mr_set_option "crt_moduli": 6..16 residue moduli, 0 (default) = chosen
                              from K so that the operand truncation stays below half the fp64 dot-product bound K 2^-53 (14) */
  int32_t ozaki_slices; /* number of int8 slices for gemm_algo 2 (0 = default) */
  void* stream;         /* cudaStream_t to run on; NULL = a stream owned by the context */
} mr_options;

/* ---- lifetime: replaces MatfastSession.builder().getOrCreate() (M/MatfastSession.scala:177-234).
 * Destruction order: every mr_matrix / mr_dmatrix of a context must be freed BEFORE mr_shutdown (mr_grid_shutdown) of that
 * context; handles are dangling afterwards.  mr_shutdown waits for all enqueued work, returns the memory the context's
 * operators cached in the device's stream-ordered pool to the driver and restores the pool's release threshold. */
MR_API mr_status mr_init(const mr_options* opts, mr_context** out);
MR_API mr_status mr_shutdown(mr_context* ctx);
MR_API mr_status mr_set_stream(mr_context* ctx, void* cuda_stream);
/* keys: "compat_bugs", "gemm_algo", "ozaki_slices", "crt_moduli", "ozaki_scratch_mb", "spmm_algo", "pipeline", "time_kernels", "gemm_variant",
 *       "stream_budget_mb" (device memory a streamed multiply may use, in MiB; 0 = free device memory at the call minus 1 GiB),
 *       "oz2_ksplit" (the CTA-pair wgmma GEMM walks (modulus, K half, tile pair) work items -- half the L2 footprint of the
 *       residue panels in flight, bit-identical results: 1 = for long tile lists and K >= 8192 only, 2 = whenever possible; default 0,
 *       or the environment variable MATREL_OZ2_KSPLIT at mr_init),
 *       "oz2_strassen" (1, the default: a resident Ozaki-II multiply of an even, full block grid with M, N, K >= 16384 runs one
 *       level of Strassen per modulus -- seven half-size int8 residue products instead of eight, bit-identical results; 2 = at every
 *       eligible size; 0 = off) */
MR_API mr_status mr_set_option(mr_context* ctx, const char* key, int64_t value);
MR_API mr_status mr_sync(mr_context* ctx);
/* Orders the context stream (device side, no host wait) after every host->device block copy submitted so far. */
MR_API mr_status mr_wait_ingest(mr_context* ctx);
MR_API mr_status mr_wait_ingest_on(mr_context* ctx, void* cuda_stream);   /* the same for a caller-owned stream */
MR_API const char* mr_last_error(void);
MR_API const char* mr_version(void);

/* ---- datasets: replaces Seq(MatrixBlock(...)).toDS() (M/example/BasicMatrixOps.scala:115-116)
 *      and .collect() / .rdd.foreach on the result. */
MR_API mr_status mr_matrix_create(mr_context* ctx, mr_matrix** out);
MR_API mr_status mr_matrix_free(mr_matrix* m);
/* Copies the block to the device (MLMatrixSerializer.deserialize, :50-69, incl. the ctor
 * `require`s of DenseMatrix :240 and SparseMatrix :533-542).  Host arrays stay caller-owned.
 * WHEN the host arrays may be reused: the copy is enqueued on the context's ingest stream.  From PAGEABLE memory (malloc, JVM
 * heap staging, numpy) CUDA has staged the data when the call returns: the arrays are free at once.  From PAGE-LOCKED memory
 * (cudaHostAlloc / cudaHostRegister) the copy engine reads the arrays asynchronously -- that is what lets a multiply overlap
 * its own ingest -- so they must stay valid and unmodified until mr_matrix_wait_ingest(m) or mr_sync(ctx) has returned (or a
 * mr_matrix_get_block of a result computed from this block has). */
MR_API mr_status mr_matrix_put_block(mr_matrix* m, int32_t rid, int32_t cid, const mr_block_desc* blk);
/* Batched mr_matrix_put_block: `count` blocks in one call (one ABI crossing per Seq[MatrixBlock], not per row). */
MR_API mr_status mr_matrix_put_blocks(mr_matrix* m, int64_t count, const int32_t* rids, const int32_t* cids,
                                      const mr_block_desc* blks);
/* Blocks the calling thread until every host->device copy of this dataset's blocks has completed (see mr_matrix_put_block). */
MR_API mr_status mr_matrix_wait_ingest(mr_matrix* m);
/* Adopts (borrows) a dense block already resident in device memory; not freed by the library. */
MR_API mr_status mr_matrix_put_block_device(mr_matrix* m, int32_t rid, int32_t cid, int32_t numRows,
                                            int32_t numCols, const double* dvalues, uint8_t isTransposed);
/* Batched form of mr_matrix_put_block_device (count blocks; arrays of length count). */
MR_API mr_status mr_matrix_put_blocks_device(mr_matrix* m, int64_t count, const int32_t* rids, const int32_t* cids,
                                             const int32_t* numRows, const int32_t* numCols,
                                             const double* const* dvalues, const uint8_t* isTransposed);
MR_API mr_status mr_matrix_num_blocks(const mr_matrix* m, int64_t* out);
/* *out = 1 iff block (rid, cid) is present (absent blocks are implicit zeros: the join semantics of
 * MatfastExecutionHelper.scala:64-263 depend on presence, not on values) */
MR_API mr_status mr_matrix_has_block(const mr_matrix* m, int32_t rid, int32_t cid, int32_t* out);
/* Fills rids/cids (capacity cap) in ascending (rid, cid) order. */
MR_API mr_status mr_matrix_block_ids(const mr_matrix* m, int32_t* rids, int32_t* cids, int64_t cap);
/* Two-call protocol (MLMatrixSerializer.serialize, :26-48): with NULL array pointers only the
 * scalar fields and *Len fields are filled; with non-NULL pointers the arrays are copied out
 * (capacity given by the *Len fields on entry). */
MR_API mr_status mr_matrix_get_block(mr_matrix* m, int32_t rid, int32_t cid, mr_block_desc* inout);
/* Device pointer of a dense block's values (for zero-copy consumers such as NCCL). */
MR_API mr_status mr_matrix_block_device_ptr(mr_matrix* m, int32_t rid, int32_t cid, double** dptr);
/* DenseMatrix.rand(numRows, numCols, new java.util.Random(seed)) generated on the device for
 * every block of an nrows x ncols matrix (M/matrix/MLMatrix.scala:453-457); per-block seed =
 * seed0 + rid*ceil(ncols/blk) + cid.  Used for synthetic benchmark inputs. */
MR_API mr_status mr_matrix_rand(mr_context* ctx, int64_t nrows, int64_t ncols, int32_t blkSize,
                                int64_t seed0, mr_matrix** out);

/* SparseMatrix.sprand(r, c, density, new java.util.Random(seed0 + rid * ceil(ncols / blk) + cid)) for every block
 * (M/matrix/MLMatrix.scala:791-856: nnz = ceil(r * c * density) distinct coordinates drawn one by one, column-major order, values
 * U(0,1) in storage order), generated on the device bit-identically to the JVM.  csr != 0: block (rid, cid) is the transpose of
 * sprand(c, r, ...), i.e. CSR storage (isTransposed = true).  Power-of-two block dimensions, 0 < density < 0.34 (MR_ENOTSUP else). */
MR_API mr_status mr_matrix_sprand(mr_context* ctx, int64_t nrows, int64_t ncols, int32_t blkSize, double density, int64_t seed0,
                                  uint8_t csr, mr_matrix** out);

/* Same generator restricted to the blocks a rank of a pr x pc process grid owns
 * (rid % pr == r, RowPartitioner.scala:34; cid % pc == c, ColumnPartitioner.scala:34), written into a
 * caller-provided device slab: block (rid, cid) starts at dslab + ((rid / pr) * ceil(nbc / pc) + cid / pc) * slotElems.
 * The returned dataset borrows the slab. */
MR_API mr_status mr_matrix_rand_partition(mr_context* ctx, int64_t nrows, int64_t ncols, int32_t blkSize, int64_t seed0,
                                          int32_t pr, int32_t pc, int32_t r, int32_t c, double* dslab,
                                          int64_t slotElems, mr_matrix** out);

/* ---- host-resident datasets: for products larger than device memory.  The blocks live in page-locked host memory owned by
 *      the library (allocated in chunks of up to 1 GiB, kept for reuse until mr_shutdown).  mr_matrix_put_block copies the caller's
 *      arrays into it (they are free again when the call returns) with the same checks as a device dataset; get_block, has_block,
 *      block_ids, num_blocks and free behave as for a device dataset.  mr_matrix_multiply streams a host-resident operand through
 *      the device tile by tile and returns a host-resident C, bit-identical to the resident product under gemm_algo 0, 1 and 4 (DESIGN.md
 *      section 4.6; gemm_algo 2 / 3 derive their scaling from the operand extent they are given, so each tile gets its own); its
 *      device budget is the option "stream_budget_mb" (0 = free device memory at the call minus 1 GiB).  Every other operator
 *      fails with MR_ENOTSUP on a host-resident operand: call mr_matrix_to_device first.  Sharded datasets stay device-only. */
MR_API mr_status mr_matrix_create_host(mr_context* ctx, mr_matrix** out);
/* *out = 1 iff m is host-resident */
MR_API mr_status mr_matrix_is_host(const mr_matrix* m, int32_t* out);
/* Copies between the residences; ids, shapes, formats and isTransposed flags are kept.  to_host copies on the egress stream after
 * each block's producer; to_device copies on the ingest stream with an event and an ingest number per block (as put_block), so a
 * multiply can start while the copy runs.  A dataset already in the target residence gives a new handle sharing its blocks. */
/* to_host reads the device arrays asynchronously; arrays the library owns are released only after those reads, arrays a caller lent
 * (mr_matrix_put_block_device) must stay valid until mr_sync. */
MR_API mr_status mr_matrix_to_host(mr_matrix* m, mr_matrix** out);
MR_API mr_status mr_matrix_to_device(mr_matrix* m, mr_matrix** out);

/* ---- whole dense matrices: Seq(MatrixBlock) of DenseMatrix blocks cut from one array, and DenseMatrix.toArray (M/matrix/MLMatrix.scala:55-61)
 *      for a whole dataset.  Element (i, j) of a column-major matrix (rowMajor = 0) is at p[i + ld*j], of a row-major one
 *      (rowMajor = 1) at p[i*ld + j]; ld must be at least the contiguous dimension (nrows, or ncols when row-major).  nrows, ncols,
 *      blkSize > 0, and the block grid must fit Int ids (MR_EINVAL otherwise).  The host only copies; layout changes run on the GPU. */
/* The nrows x ncols matrix at src as a dataset of blkSize x blkSize blocks (ragged at the bottom / right edge), EVERY block present.
 * Blocks of a row-major src are stored row-major, isTransposed = 1: a row-major sub-block IS the reference's transposed dense block
 * (M/matrix/MLMatrix.scala:285-289), so no element is transposed on the way in.  src may be host memory (pageable or page-locked)
 * or device memory of this context's GPU (MR_EINVAL for another GPU's).  host_resident != 0: a host-resident dataset (see above).
 * stream (cudaStream_t): the copies first wait for the work enqueued on it so far (the producer of a device src; NULL = none).
 * Device-resident result: the copies run on the ingest stream, each block with its own event and ingest number for a host src (one
 * gather kernel and one event for a device src), so a multiply issued right after the call starts on the blocks that have landed.
 * WHEN src may be reused: as mr_matrix_put_block -- PAGEABLE host memory is free when the call returns; PAGE-LOCKED host memory and
 * DEVICE memory are read asynchronously and must stay valid and unmodified until mr_matrix_wait_ingest(*out) or mr_sync(ctx) has
 * returned.  A host-resident result from host memory is copied before the call returns. */
MR_API mr_status mr_matrix_from_dense(mr_context* ctx, const double* src, int64_t nrows, int64_t ncols, int64_t ld, int32_t rowMajor,
                                      int32_t blkSize, int32_t host_resident, void* stream, mr_matrix** out);
/* The dataset as one dense nrows x ncols matrix at dst (host or device memory of this context's GPU): block (rid, cid) covers rows
 * rid*blkSize .. and columns cid*blkSize ..; absent blocks and the part of a cell a smaller block leaves are zeros, sparse blocks (CSC
 * or CSR) are scattered, every block's isTransposed flag is honoured.  Any residence, sharded datasets included (blocks a rank does
 * not hold are absent).  A block outside the matrix (numRows > blkSize, rid*blkSize + numRows > nrows, or the same for columns)
 * fails with MR_EDIM.  A host dst is filled panel by panel (block rows of a row-major dst, block columns of a column-major one)
 * through two device buffers; their memory, and the staging of host-resident blocks, follow the option "stream_budget_mb"
 * (MR_ENOMEM when one panel does not fit).  stream (cudaStream_t): the assembly first waits for the work enqueued on it so far, and
 * it then waits for the assembly (the consumer of dst) -- no host wait; NULL = the call returns once dst is written. */
MR_API mr_status mr_matrix_to_dense(mr_matrix* m, int64_t nrows, int64_t ncols, int32_t blkSize, double* dst, int64_t ld,
                                    int32_t rowMajor, void* stream);

/* ---- operators: argument-for-argument with M/Dataset.scala:57-152 and the physical operators
 *      of M/execution/MatfastExecution.scala. */
/* Dataset.matrixMultiply :134-142 -> MatrixMatrixMultiplicationExecution :688-726 ->
 * MatfastExecutionHelper.matrixMultiplyGeneral :235-263 / multiplyOuterProductDuplicate* :175-221 */
MR_API mr_status mr_matrix_multiply(mr_matrix* left, int64_t leftRowNum, int64_t leftColNum,
                                    mr_matrix* right, int64_t rightRowNum, int64_t rightColNum,
                                    int32_t blkSize, mr_matrix** out);
/* Dataset.transpose / t :57-61 -> MatrixTransposeExecution :215-236 (flag flip + index swap) */
MR_API mr_status mr_transpose(mr_matrix* a, mr_matrix** out);
/* Dataset.addElement :105-112 -> MatrixElementAddExecution :571-607 (outer join) */
MR_API mr_status mr_add_element(mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right,
                                int64_t rightRowNum, int64_t rightColNum, int32_t blkSize, mr_matrix** out);
/* Dataset.multiplyElement :114-122 -> MatrixElementMultiplyExecution :609-644 (inner join) */
MR_API mr_status mr_multiply_element(mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right,
                                     int64_t rightRowNum, int64_t rightColNum, int32_t blkSize, mr_matrix** out);
/* Dataset.divideElement :124-132 -> MatrixElementDivideExecution :646-686 (inner join) */
MR_API mr_status mr_divide_element(mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right,
                                   int64_t rightRowNum, int64_t rightColNum, int32_t blkSize, mr_matrix** out);
/* Dataset.addScalar :89-91 -> MatrixScalarAddExecution :465-486 -> LocalMatrix.addScalar */
MR_API mr_status mr_add_scalar(mr_matrix* a, double alpha, mr_matrix** out);
/* Dataset.multiplyScalar :93-97 -> MatrixScalarMultiplyExecution :488-509 */
MR_API mr_status mr_multiply_scalar(mr_matrix* a, double alpha, mr_matrix** out);
/* Dataset.power :99-103 -> MatrixPowerExecution :511-532 */
MR_API mr_status mr_power(mr_matrix* a, double alpha, mr_matrix** out);
/* Dataset.matrixRankOneUpdate :144-152 -> RankOneUpdateExecution :728-747 */
MR_API mr_status mr_rank_one_update(mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right,
                                    int64_t rightRowNum, int64_t rightColNum, int32_t blkSize, mr_matrix** out);
/* ---- aggregates (SURVEY.md section 8f-2).  The mathematically intended reductions; the reference's index defects
 *      for non-square transposed / sparse blocks (MatfastExecution.scala:262-287, 338-357 = defect B5) are not reproduced. */
/* Dataset.rowSum :63-66 -> RowSumDirectExecution :239-300: blocks (rid, 0) of shape rows x 1 */
MR_API mr_status mr_row_sum(mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out);
/* Dataset.colSum :68-71 -> ColumnSumDirectExecution :303-366: blocks (0, cid) of shape 1 x cols */
MR_API mr_status mr_col_sum(mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out);
/* Dataset.sum :73-76 -> SumDirectExecution :369-398: one 1 x 1 block (0, 0) */
MR_API mr_status mr_sum(mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out);
/* Dataset.trace :78-82 -> TraceDirectExecution :401-463: one 1 x 1 block (0, 0) from the diagonal blocks */
MR_API mr_status mr_trace(mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out);
/* ---- slicing (SURVEY.md section 8f-4); intended semantics (the reference's transposed / sparse index defects are not reproduced) */
/* Dataset.project :38-47 -> Project{Row,Column}DirectExecution :31-150: rowOrCol != 0 -> row `index` as blocks (0, cid) of
 * shape 1 x cols; rowOrCol == 0 -> column `index` as blocks (rid, 0) of shape rows x 1 */
MR_API mr_status mr_project(mr_matrix* a, int64_t nrows, int64_t ncols, int32_t blkSize, int32_t rowOrCol, int64_t index,
                            mr_matrix** out);
/* Dataset.selection :49-55 -> SelectDirectExecution :152-213: the element (rowIdx, colIdx) as one 1 x 1 block (0, 0) */
MR_API mr_status mr_selection(mr_matrix* a, int64_t nrows, int64_t ncols, int32_t blkSize, int64_t rowIdx, int64_t colIdx,
                              mr_matrix** out);
/* Dataset.vec :84-87 -> VectorizeExecution :534-569: column t of block (i, j) becomes the rows x 1 block
 * ((j * blkSize + t) * ceil(nrows / blkSize) + i, 0).  Intended semantics (defect B6 -- the reference strides by numLocalCols --
 * is not reproduced); the output blocks are zero-copy views of the (column-major) input columns. */
MR_API mr_status mr_vec(mr_matrix* a, int64_t nrows, int64_t ncols, int32_t blkSize, mr_matrix** out);
/* Materialise every dense block as column-major, isTransposed = false (DenseMatrix.toArray,
 * M/matrix/MLMatrix.scala:55-61, as a device transpose kernel). */
MR_API mr_status mr_materialize(mr_matrix* a, mr_matrix** out);

/* ---- placement: bit-exact restatement of M/partitioner/{Row,Column,Index,BlockCyclic}Partitioner.scala (pure integer, host side) */
/* RowPartitioner.getPartition (RowPartitioner.scala:32-38) */
MR_API mr_status mr_row_partition(int32_t rid, int32_t cid, int32_t partitions, int32_t* out);
/* ColumnPartitioner.getPartition (ColumnPartitioner.scala:32-38) */
MR_API mr_status mr_column_partition(int32_t rid, int32_t cid, int32_t partitions, int32_t* out);
/* IndexPartitioner.getPartition (IndexPartitioner.scala:29-34) */
MR_API mr_status mr_index_partition(int32_t key, int32_t partitions, int32_t* out);
/* MatfastExecutionHelper.genBlockCyclicPartitioner (MatfastExecutionHelper.scala:46-62):
 * out = {ROW_BLK_NUM, COL_BLK_NUM, ROW_BLKS_PER_PARTITION, COL_BLKS_PER_PARTITION} */
MR_API mr_status mr_gen_block_cyclic(int64_t nrows, int64_t ncols, int32_t blkSize, int32_t out[4]);
/* BlockCyclicPartitioner.getPartition / numPartitions (BlockCyclicPartitioner.scala:31-62) */
MR_API mr_status mr_block_cyclic_partition(const int32_t params[4], int32_t rid, int32_t cid, int32_t* out);
MR_API mr_status mr_block_cyclic_num_partitions(const int32_t params[4], int32_t* out);
/* One entry point over the four schemes (Partitioner.getPartition of the four M/partitioner classes): params[0] = partitions for
 * MR_PART_ROW / MR_PART_COLUMN / MR_PART_INDEX (INDEX keys on rid), params[0..3] = the mr_gen_block_cyclic tuple for
 * MR_PART_BLOCK_CYCLIC. */
typedef enum mr_partition_scheme { MR_PART_ROW = 0, MR_PART_COLUMN = 1, MR_PART_INDEX = 2, MR_PART_BLOCK_CYCLIC = 3 } mr_partition_scheme;
MR_API mr_status mr_partition_id(int32_t scheme, const int32_t params[4], int32_t rid, int32_t cid, int32_t* out);


/* ======================================================================================================================
 * Multi-GPU: block partitions sharded across the GPUs of one box (SURVEY.md 8e).
 *
 * Placement is the reference's RowPartitioner x ColumnPartitioner arithmetic on a pr x pc process grid
 * (M/partitioner/RowPartitioner.scala:34, ColumnPartitioner.scala:34): rank (r, c) owns the blocks with rid % pr == r and
 * cid % pc == c.  A SHARDED dataset keeps the blocks a rank owns in ONE device slab: block (rid, cid) is the blkSize^2-double slot
 * (rid / pr) * ceil(nbc / pc) + cid / pc, column-major, leading dimension = the block's own row count.  A sharded dataset is
 * dense over its block grid (slots never written read as zeros) and all of its blocks share one isTransposed flag.
 *
 * Two ways to drive the GPUs:
 *   (1) one process per GPU (torch.distributed / MPI launch): each process creates its shard with mr_matrix_create_sharded,
 *       exports the slab with mr_ipc_export, opens its peers' slabs with mr_ipc_open and calls mr_grid_multiply;
 *   (2) one process for all GPUs: mr_init_grid + the mr_dmatrix_* entry points below (no Spark executors, no MPI).
 * Either way the groupByKey + join shuffles of matrixMultiplyGeneral (M/execution/MatfastExecutionHelper.scala:236-249) become
 * copy-engine pulls of the peers' slabs over NVLink, chunked so that the multiply overlaps them; reduceByKey (:255) disappears
 * (C-stationary); reductions and re-partitioning go through NCCL (ncclCommInitAll; failures are reported as MR_ENCCL).
 * ====================================================================================================================== */
typedef struct mr_grid_layout {
  int64_t nrows, ncols;   /* matrix dimensions */
  int32_t blkSize;
  int32_t pr, pc;         /* process grid */
  int32_t r, c;           /* this rank's coordinates */
} mr_grid_layout;

/* A zero-filled sharded dataset of this rank (cudaMalloc-backed, exportable through CUDA IPC). */
MR_API mr_status mr_matrix_create_sharded(mr_context* ctx, const mr_grid_layout* layout, mr_matrix** out);
/* The same over a caller-owned device slab (e.g. a torch tensor); not freed by the library. */
MR_API mr_status mr_matrix_adopt_sharded(mr_context* ctx, const mr_grid_layout* layout, double* dslab, uint8_t isTransposed,
                                         mr_matrix** out);
MR_API mr_status mr_matrix_layout(const mr_matrix* m, mr_grid_layout* out);
MR_API mr_status mr_matrix_slab(mr_matrix* m, double** dslab, int64_t* bytes);
/* CUDA IPC plumbing for (1): handle64 = the 64-byte cudaIpcMemHandle_t of the allocation containing dptr, *offset = dptr's
 * offset inside it.  mr_ipc_open maps a peer's allocation (once per handle) and returns the pointer at that offset. */
MR_API mr_status mr_ipc_export(const void* dptr, void* handle64, int64_t* offset);
MR_API mr_status mr_ipc_open(mr_context* ctx, const void* handle64, int64_t offset, void** dptr);
MR_API mr_status mr_ipc_close_all(mr_context* ctx);
/* Synchronous read of device memory valid in this process (own, peer-mapped or mr_ipc_open'ed) into a host buffer. */
MR_API mr_status mr_memcpy_d2h(mr_context* ctx, const void* dptr, void* host, int64_t bytes);
/* This rank's share of C = A B (Dataset.matrixMultiply, M/Dataset.scala:134-142, on the grid).  A, B: this rank's sharded operands;
 * slabsA_row[c'] (c' = 0 .. pc-1) / slabsB_col[r'] (r' = 0 .. pr-1): slab base pointers of the ranks of this rank's grid row / grid
 * column, valid in this process (own slab, peer-mapped, or mr_ipc_open'ed).  The caller makes sure the peers' slabs are complete
 * before the call and stay untouched until every rank's call has run on the device (a stream barrier before and after; mr_dmatrix
 * does it with events).  nchunks >= 1 (<= 64): the pull is cut into nchunks pieces of A's block rows and nchunks pieces of B's block
 * columns, fetched alternately (A0, B0, A1, B1, ...); the multiply starts on the corner of C the first pair unlocks and grows it
 * piece by piece.  *out is sharded. */
MR_API mr_status mr_grid_multiply(mr_matrix* A, mr_matrix* B, const double* const* slabsA_row, const double* const* slabsB_col,
                                  int32_t nchunks, mr_matrix** out);
/* mr_grid_multiply with one CUDA event (cudaEvent_t) per piece of the pull, 2 * nchunks of them: gates[2 ch] guards piece ch of A
 * (this rank's block rows [rows ch / nchunks, rows (ch + 1) / nchunks)), gates[2 ch + 1] piece ch of B (its block columns, cut the
 * same way); NULL = in place.  Lets every rank overlap its peers' host->device ingest with its own multiply. */
MR_API mr_status mr_grid_multiply_gated(mr_matrix* A, mr_matrix* B, const double* const* slabsA_row, const double* const* slabsB_col,
                                        int32_t nchunks, const void* const* gates, mr_matrix** out);
/* The blocks a partition owns (rid % row_mod == row_rem, cid % col_mod == col_rem); shares the device arrays with `a`. */
MR_API mr_status mr_matrix_filter_blocks(mr_matrix* a, int32_t row_mod, int32_t row_rem, int32_t col_mod, int32_t col_rem,
                                         mr_matrix** out);
/* The same with a left operand that is NOT sharded: A_rows holds every block A(i, k) -- sparse or dense -- of the block rows this
 * rank owns (the thin / sparse operand is replicated where it is needed, the reference's duplicateCrossPartitions,
 * MatfastExecutionHelper.scala:224-233); only the dense B is pulled from the grid column.  BASELINE configs[4]. */
MR_API mr_status mr_grid_multiply_rows(mr_matrix* A_rows, int64_t leftRowNum, int64_t leftColNum, mr_matrix* B,
                                       const double* const* slabsB_col, mr_matrix** out);

/* ---- (2) one process, all GPUs.  Replaces MatfastSession + the executors (M/MatfastSession.scala:177-234). */
MR_API mr_status mr_init_grid(const mr_options* opts, int32_t ngpus, mr_grid** out);  /* devices 0 .. ngpus-1, grid 1x1 / 1x2 / 2x2 / 2x4 */
MR_API mr_status mr_grid_shutdown(mr_grid* g);
MR_API mr_status mr_grid_info(const mr_grid* g, int32_t* ngpus, int32_t* pr, int32_t* pc, int32_t* has_nccl);
MR_API mr_status mr_grid_context(mr_grid* g, int32_t rank, mr_context** ctx);          /* rank = r * pc + c, on device `rank` */
MR_API mr_status mr_grid_sync(mr_grid* g);
/* mr_matrix_create(nrows, ncols, blk, ...) of SURVEY.md 8b: the dimensions live in the handle. */
MR_API mr_status mr_dmatrix_create(mr_grid* g, int64_t nrows, int64_t ncols, int32_t blkSize, mr_dmatrix** out);
MR_API mr_status mr_dmatrix_rand(mr_grid* g, int64_t nrows, int64_t ncols, int32_t blkSize, int64_t seed0, mr_dmatrix** out);
MR_API mr_status mr_dmatrix_free(mr_dmatrix* m);
MR_API mr_status mr_dmatrix_dims(const mr_dmatrix* m, int64_t* nrows, int64_t* ncols, int32_t* blkSize);
MR_API mr_status mr_dmatrix_owner(const mr_dmatrix* m, int32_t rid, int32_t cid, int32_t* rank);
MR_API mr_status mr_dmatrix_part(mr_dmatrix* m, int32_t rank, mr_matrix** out);         /* borrowed: the blocks that rank owns */
MR_API mr_status mr_dmatrix_put_block(mr_dmatrix* m, int32_t rid, int32_t cid, const mr_block_desc* blk);  /* routed to the owner */
MR_API mr_status mr_dmatrix_get_block(mr_dmatrix* m, int32_t rid, int32_t cid, mr_block_desc* inout);
MR_API mr_status mr_dmatrix_has_block(const mr_dmatrix* m, int32_t rid, int32_t cid, int32_t* out);
MR_API mr_status mr_dmatrix_num_blocks(const mr_dmatrix* m, int64_t* out);
/* Dataset.matrixMultiply :134-142 */
MR_API mr_status mr_dmatrix_multiply(mr_dmatrix* A, mr_dmatrix* B, mr_dmatrix** out);
/* The same product split over K, the reference's own algorithm (matrixMultiplyGeneral, MatfastExecutionHelper.scala:235-263: join
 * A(:, k) with B(k, :), reduceByKey(add) of the partial blocks at :255), for products whose C has fewer block rows than pr or block
 * columns than pc (Gram matrices A^T A, factors of low rank).  With n GPUs and nbk = ceil(K / blk), GPU g multiplies the k-blocks
 * [floor(g nbk / n), floor((g + 1) nbk / n)), pulling the blocks it lacks from their owners under the operands' own placement;
 * every owner then sums its C blocks' partials over NVLink in ascending GPU order, starting from GPU 0's partial, so the result is
 * bit-reproducible.  Errors as mr_dmatrix_multiply; the result is laid out exactly like its result (ids, shapes, owners, dense
 * column-major blocks).  On a 1-GPU grid this is mr_dmatrix_multiply. */
MR_API mr_status mr_dmatrix_multiply_ksplit(mr_dmatrix* A, mr_dmatrix* B, mr_dmatrix** out);
/* Dataset.addElement / multiplyElement / divideElement :105-132 on co-partitioned operands (op 0 / 1 / 2): no block moves */
MR_API mr_status mr_dmatrix_elementwise(int32_t op, mr_dmatrix* A, mr_dmatrix* B, mr_dmatrix** out);
/* Dataset.sum / trace :73-82 (what = 0 / 1): local reduction kernels + one ncclAllReduce */
MR_API mr_status mr_dmatrix_reduce_scalar(mr_dmatrix* A, int32_t what, double* value);
/* repartitionWithTargetPartitioner (MatfastExecutionHelper.scala:34-44): the blocks move to their owners under a new_pr x new_pc
 * grid of the same GPUs ((P, 1) = RowPartitioner, (1, P) = ColumnPartitioner) as grouped ncclSend / ncclRecv between the slabs. */
MR_API mr_status mr_dmatrix_repartition(mr_dmatrix* A, int32_t new_pr, int32_t new_pc, mr_dmatrix** out);
/* Dataset.t / transpose :57-61 (MatrixTransposeExecution, MatfastExecution.scala:215-236): block (i, j) becomes block (j, i) on
 * the same placement function and moves to its new owner (grouped ncclSend / ncclRecv); payloads are untouched, the result's
 * blocks carry isTransposed = 1, exactly as the reference's flag flip (MLMatrix.scala:312). */
MR_API mr_status mr_dmatrix_transpose(mr_dmatrix* A, mr_dmatrix** out);
/* Dataset.addScalar / multiplyScalar / power :89-103 (op 0 / 1 / 2): every GPU maps the blocks it owns, no block moves */
MR_API mr_status mr_dmatrix_scalar(int32_t op, mr_dmatrix* A, double alpha, mr_dmatrix** out);
/* Dataset.rowSum / colSum :63-72 (axis 0 / 1; RowSum / ColumnSumDirectExecution + reduceByKey(add), MatfastExecution.scala:239-370):
 * local line-sum kernels, ONE ncclAllReduce of a vector covering the axis, result blocks (i, 0) / (0, j) registered at their owners */
MR_API mr_status mr_dmatrix_axis_sum(mr_dmatrix* A, int32_t axis, mr_dmatrix** out);
/* Dataset.project :38-47 (rowOrCol != 0: row `index` as 1 x ncols, else column `index` as nrows x 1) and Dataset.selection :49-55
 * (entry (rowIdx, colIdx) as a 1 x 1 dataset): the owners extract their pieces, the same vector all-reduce re-keys and places them */
MR_API mr_status mr_dmatrix_project(mr_dmatrix* A, int32_t rowOrCol, int64_t index, mr_dmatrix** out);
MR_API mr_status mr_dmatrix_selection(mr_dmatrix* A, int64_t rowIdx, int64_t colIdx, mr_dmatrix** out);

/* ---- introspection used by bench/tests (not part of the reference surface) */
typedef struct mr_stats {
  int64_t kernel_launches;  /* CUDA kernels launched by this library since mr_init / reset */
  int64_t gemm_launches;
  int64_t h2d_bytes;
  int64_t d2h_bytes;
  double last_gemm_ms;      /* CUDA-event duration of the most recent GEMM kernel launch(es) */
  double gemm_ms_total;     /* sum of CUDA-event GEMM durations since reset (timing enabled only) */
  int64_t last_gemm_flops;
  double tc_gemm_ms_total;  /* CUDA-event time of the wgmma int8 GEMM launches since reset (timing enabled only) */
  int64_t tc_gemm_launches; /* multiplies that ran on the tensor-core path since reset */
  int64_t tc_int8_ops;      /* int8 multiply-add operations (x 2) of the most recent tensor-core multiply */
  int64_t p2p_bytes;        /* bytes pulled from peer GPUs over NVLink by this context (grid multiply) */
  int64_t tc_moduli;        /* residue moduli of the most recent tensor-core (Ozaki-II) multiply */
  int64_t stream_tiles;     /* C tiles of the most recent streamed multiply (a host-resident operand; mr_matrix_create_host) */
  int64_t stream_h2d_bytes; /* operand panels that multiply moved host -> device (h2d_bytes also counts its descriptor tables) */
  int64_t stream_d2h_bytes; /* result blocks that multiply moved device -> host */
  int64_t spgemm_pairs;     /* block pairs of the most recent mr_matrix_multiply computed by the sparse x sparse kernel (output blocks
                               whose partials are all low-density sparse x sparse; summed over the tiles of a streamed multiply) */
  int64_t spgemm_products;  /* scalar products that kernel performed: sum over its pairs and k of nnz(A(:,k)) * nnz(B(k,:)) */
  int64_t dspmm_pairs;      /* block pairs of the most recent mr_matrix_multiply computed by the dense x low-density sparse kernel
                               (summed over the tiles of a streamed multiply) */
  int64_t dspmm_products;   /* sum over those pairs of stored entries of the sparse block x rows of the dense block */
  int64_t ew_sparse_pairs;  /* block pairs of the most recent element-wise join (add / multiply / divide element) with a sparse side */
  int64_t ew_sparse_entries; /* stored entries of the sparse blocks those pairs read */
  int64_t agg_sparse_blocks; /* sparse blocks the most recent rowSum / colSum / trace / project / selection read on their stored entries */
  int64_t agg_sparse_entries; /* stored entries of those blocks */
  int64_t mv_pairs;         /* block pairs of the most recent mr_matrix_multiply computed by the matrix x vector / thin-matrix route
                               (thin side of 1 to 8 dense columns or rows; a pair is a matrix block and a thin-side block, whatever
                               its width; summed over the tiles of a streamed multiply) */
  int64_t mv_sparse_entries; /* stored entries of the sparse blocks among those pairs */
  int64_t gram_blocks;      /* output blocks computed for the most recent mr_matrix_multiply when it was a Gram product (A^T A or
                               A A^T over shared arrays): by the dense engines, the blocks on and above the diagonal; by the sparse
                               x sparse chains, those and the non-square blocks below it; 0 otherwise */
  int64_t gram_mirrored_blocks; /* blocks below the diagonal of that product written from their transposes (dense: the mirror pass;
                               sparse: square blocks, mirrored, sharing their transposes' arrays or converted from them) */
  int64_t tc_strassen_jobs; /* Ozaki-II jobs of the most recent mr_matrix_multiply that ran one Strassen level (seven half-size
                               residue products per modulus instead of eight; option "oz2_strassen") */
} mr_stats;
MR_API mr_status mr_get_stats(mr_context* ctx, mr_stats* out);
MR_API mr_status mr_reset_stats(mr_context* ctx);

#ifdef __cplusplus
}
#endif
#endif /* MATREL_H_ */
