// Internal interface between the C-ABI host layer (abi_*.cpp, host.h) and the sm_90a kernels.
// Not part of the public ABI (see include/matrel.h).
#pragma once
#include <cuda_runtime.h>

#include <mutex>
#include <stdint.h>

namespace matrel {

// Kernel function attributes and __constant__ tables are per DEVICE: "configure once" must be keyed by the current device
// (one process may drive several GPUs) and be safe against concurrent first calls from different contexts.
class PerDeviceOnce {
 public:
  template <class F>
  cudaError_t run(F&& f) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> g(mu_);
    if (dev < 0 || dev >= kMaxDevices) return f();
    if (done_[dev]) return cudaSuccess;
    e = f();
    if (e == cudaSuccess) done_[dev] = true;
    return e;
  }

 private:
  static constexpr int kMaxDevices = 64;
  std::mutex mu_;
  bool done_[kMaxDevices] = {};
};


// ---- block GEMM ----------------------------------------------------------------------------------
// One k-block contribution A(i,k) * B(k,j) to an output block; the block-GEMM kernel walks the
// pair list of an output block inside its K loop, which fuses the reference's
// reduceByKey(LocalMatrix.add) (MatfastExecutionHelper.scala:255) into the accumulators.
struct GemmPair {
  const double* A;  // values of A(i,k): m x kdim, column-major (lda = m) or row-major if aT (lda = kdim)
  const double* B;  // values of B(k,j): kdim x n, column-major (ldb = kdim) or row-major if bT (ldb = n)
  int32_t lda, ldb;
  int32_t kdim;
  int32_t tmA, tmB; // index of the operand's K-contiguous CUtensorMap in the launch's table, -1 = none
  uint8_t aT, bT;   // isTransposed flags (BLAS.gemmddd's "T"/"N", BLAS.scala:333-336)
  uint8_t pad[2];
};

struct GemmOut {
  double* C;        // m x n, column-major, ldc = m (DenseMatrix.zeros(m, n), MLMatrix.scala:101)
  int32_t m, n;
  int32_t pair_begin, pair_count;
};

struct GemmTile {
  int32_t out;      // index into GemmOut[]
  int32_t tm, tn;   // tile coordinates inside the output block
  int32_t pad;
};

enum GemmVariant { GEMM_128x128 = 0, GEMM_64x64 = 1 };
int gemm_tile_m(int variant);
int gemm_tile_n(int variant);

// Encodes the 128-byte CUtensorMap of a K-contiguous operand block (rows x kdim, line stride ld doubles,
// box {16, tile_rows}, SWIZZLE_128B).  Returns false when TMA cannot address it (odd ld / unaligned base).
bool encode_kcontig_tmap(void* out128, const double* base, int64_t kdim, int64_t rows, int64_t ld, int tile_rows);

// run_if (optional, device): the launch is a no-op unless *run_if != 0 (the fallback behind an Ozaki-II job)
cudaError_t launch_gemm_f64(const GemmOut* d_outs, const GemmPair* d_pairs, const GemmTile* d_tiles,
                            int ntiles, const void* d_tmaps, int variant, cudaStream_t stream, const int* run_if = nullptr);

// ---- fp64 block GEMM on wgmma (s8) through Ozaki splitting (gemm_ozaki.cu) --------------------------------
struct OzakiOperand {
  const double* v;     // dense block values (column-major, row-major if isT)
  int32_t rows, cols;  // logical block dims
  int32_t row0, col0;  // global offset of the block inside its operand matrix
  uint8_t isT;
  uint8_t pad[7];
};
// C(blocks in h_ctab, nbr x nbc grid of blk-sized column-major blocks) (+)= A(M x K) * B(K x N); absent blocks are zeros.
// *nonfinite = 1 (and nothing written) when an operand holds Inf/NaN: the caller must use the exact kernel instead.
cudaError_t ozaki_gemm_f64(const OzakiOperand* a_blocks, int na, const OzakiOperand* b_blocks, int nb, int64_t M, int64_t K,
                           int64_t N, int slices, double* const* h_ctab, int blk, int nbr, int nbc, bool accumulate,
                           int* launches, int* nonfinite, cudaStream_t stream);

// Ozaki scheme II (gemm_algo 4 and the auto selection): residues modulo `moduli` pairwise-coprime p_t <= 256, one int8 tensor-core
// GEMM per modulus, Chinese-remainder reconstruction -- as a job engine over slot-organised residue buffers (gemm_ozaki.cu).
// All table arguments are DEVICE pointers (the caller uploads them through its own staging path); nothing synchronises with the
// host.  *oz2_flag() != 0 on the device means "operands not representable (Inf / NaN, or too wide a range in auto mode)": the
// engine's remaining kernels are no-ops then and the caller's gated DMMA launch produces the blocks instead.
struct Oz2Engine;
size_t oz2_scratch_bytes(int blk, int64_t K, int moduli, int cap_r, int cap_c, int max_tiles);
int oz2_tiles_per_block(int blk);
cudaError_t oz2_create(Oz2Engine** out, int blk, int64_t K, int moduli, int cap_r, int cap_c, int max_tiles, int guard_range,
                       cudaStream_t stream);
void oz2_destroy(Oz2Engine* e, cudaStream_t stream);
const void* oz2_host_maps(const Oz2Engine* e, size_t* bytes);   // 2 * moduli CUtensorMaps to be uploaded by the caller ...
void oz2_set_device_maps(Oz2Engine* e, const void* d_maps);     // ... and handed back as a device pointer
const int* oz2_flag(const Oz2Engine* e);
// Operand blocks of an output block, for the exact fp64 products of elements the residue scheme leaves out (oz2_fixup)
struct Oz2FixSrc {
  const double* A;      // a_rows x kdim, column-major, row-major if aT
  const double* B;      // kdim x b_cols, column-major, row-major if bT
  int32_t k0, kdim;     // inner-index range [k0, k0 + kdim) this pair covers
  int32_t a_rows, b_cols;
  uint8_t aT, bT;
  uint8_t pad[6];
};
struct Oz2FixOut {
  double* C;            // m x n, column-major
  int32_t m, n;
  int32_t rslot, cslot; // the engine slots its block row of A / block column of B were prepared into
  int32_t src_begin, src_count;
};
cudaError_t oz2_fixup(Oz2Engine* e, const Oz2FixOut* d_outs, int nouts, const Oz2FixSrc* d_srcs, cudaStream_t stream);
int oz2_alpha(const Oz2Engine* e);
int oz2_moduli(const Oz2Engine* e);
int oz2_moduli_for(int64_t K, int requested);  // requested <= 0: chosen from K (see gemm_ozaki.cu)
int oz2_slot_stride(const Oz2Engine* e);
void oz2_set_paired(Oz2Engine* e, bool paired);                  // tile lists come as (2a, b), (2a + 1, b) pairs: use the CTA-pair kernel
bool oz2_paired(const Oz2Engine* e);
void oz2_set_ksplit(Oz2Engine* e, int level);                    // CTA-pair kernel: (modulus, K half, tile pair) work items (see Oz2Items); 1 = large jobs, 2 = always
int oz2_launches(Oz2Engine* e);                                  // kernels launched since the last call
cudaError_t oz2_prepare(Oz2Engine* e, bool is_a, const OzakiOperand* d_blocks, int nblocks, int max_rows, int max_cols, int slot0,
                        int nslots, const int32_t* d_dims, bool need_zero, cudaStream_t stream);
cudaError_t oz2_multiply(Oz2Engine* e, const int2* d_tiles, int ntiles, double* const* d_ctab, cudaStream_t stream, double* ms_gemm,
                         cudaEvent_t ev0, cudaEvent_t ev1);
constexpr int kOz2TileM = 128, kOz2TileN = 256;
// fp32 multiply on wgmma tf32 (3xTF32 split, fp32 accumulation); same operand / output conventions.
cudaError_t tf32x3_gemm(const OzakiOperand* a_blocks, int na, const OzakiOperand* b_blocks, int nb, int64_t M, int64_t K, int64_t N,
                        double* const* h_ctab, int blk, int nbr, int nbc, int* launches, cudaStream_t stream);

// ---- element-wise / layout kernels (HBM-bound), batched over blocks ---------------------------------
enum EwOp { EW_ADD = 0, EW_MUL = 1, EW_DIV = 2, EW_RANK1 = 3, EW_RANK1_COMPAT = 4, EW_COPY = 5 };

// C (column-major rows x cols) = f(A(r,c), B(r,c)); A, B dense with their own isTransposed flag.
//   EW_ADD/MUL/DIV : LocalMatrix.addDense / elementWiseOpDenseDense (LocalMatrix.scala:56-63,493-505)
//   EW_COPY        : C = A  (DenseMatrix.toArray, MLMatrix.scala:55-61)            (B unused)
//   EW_RANK1       : C = A + x y^T with x = B (rows), y = Y (cols)                 (intended rankOneAdd)
//   EW_RANK1_COMPAT: flat C[k(r,c)] = x_r y_c, k = A's storage index (defect B3 restated, LocalMatrix.scala:1075-1093)
struct EwDesc {
  const double* A;
  const double* B;
  const double* Y;
  double* C;
  int32_t rows, cols;
  uint8_t aT, bT;
  uint8_t pad[6];
};
cudaError_t launch_ew_batched(int op, const EwDesc* d_descs, int nblocks, int max_rows, int max_cols,
                              bool any_transposed, cudaStream_t stream);

enum MapOp { MAP_ADD_SCALAR = 0, MAP_MUL_SCALAR = 1, MAP_POW = 2 };
struct MapDesc {
  const double* in;
  double* out;
  int64_t n;
};
// out[i] = f(in[i], alpha) over flat value arrays (layout preserving; LocalMatrix.scala:411-426,931-980)
cudaError_t launch_map_batched(int op, const MapDesc* d_descs, int nblocks, int64_t max_n, double alpha,
                               cudaStream_t stream);

// dense col-major rows x cols from CSC / CSR (SparseMatrix.toArray, MLMatrix.scala:55-61,637-663); out pre-zeroed
cudaError_t launch_sparse_to_dense(const int32_t* ptrs, const int32_t* idx, const double* vals, bool isT,
                                   double* out, int rows, int cols, cudaStream_t stream);
// C (col-major m x n) (+)= S (CSR if sT else CSC, m x k) * B (k x n dense, bT flag) ; BLAS.gemmsdd (BLAS.scala:352-458)
cudaError_t launch_spmm(const int32_t* ptrs, const int32_t* idx, const double* vals, bool sT,
                        const double* B, bool bT, double* C, int m, int k, int n, bool accumulate,
                        cudaStream_t stream);
// DenseMatrix.toSparse (MLMatrix.scala:353-374) on the device, batched: (1) per-column count of v != 0.0 (NaN counts,
// as in the reference's `arr(i) != 0`), (2) ordered per-column compaction into CSC given the column pointers.
struct CscDesc {
  const double* dense;   // column-major rows x cols
  int32_t rows, cols;
  int32_t* counts;       // [cols] out (pass 1)
  const int32_t* colPtrs;  // [cols + 1] in (pass 2)
  int32_t* rowIndices;   // out (pass 2)
  double* values;        // out (pass 2)
};
cudaError_t launch_csc_count(const CscDesc* d_descs, int nblocks, int max_cols, cudaStream_t stream);
cudaError_t launch_csc_fill(const CscDesc* d_descs, int nblocks, int max_cols, cudaStream_t stream);

// Fused block-row SpMM: for every output block, C (col-major m x n) (+)= sum over its (CSR sparse A(i,k), dense B(k,j)) pairs.
// One CTA = 8 output columns of one output block: the B column chunk and the C chunk live in shared memory, the K loop
// over the block pairs is fused (no partial blocks, no adds).  BLAS.gemmsdd CSR branches (BLAS.scala:375-413).
struct SpmmPair {
  const int32_t* ptrs;   // CSR row pointers (m + 1)
  const int32_t* idx;    // column indices
  const double* vals;
  const double* B;       // dense kdim x n (column-major, row-major if bT)
  int32_t kdim;
  uint8_t bT;
  uint8_t pad[3];
};
struct SpmmOut {
  double* C;
  int32_t m, n;
  int32_t pair_begin, pair_count;
  int32_t accumulate;    // 1: C already holds the dense-pair sum
  int32_t pad;
};
constexpr int kSpmmMaxDim = 1024;   // m and kdim limit of the shared-memory kernel
cudaError_t launch_spmm_fused(const SpmmOut* d_outs, int nouts, const SpmmPair* d_pairs, int max_n, cudaStream_t stream);

// ---- the pipelined CSR x dense kernel (spmm.cu): 256-row x 64-column tiles, row-major B staged by TMA, packed CSR segments.
constexpr int kSpmm2StripRows = 256, kSpmm2TileCols = 64, kSpmm2ChunkK = 128;
struct Spmm2Prep {        // one sparse (CSR) block to re-pack
  const int32_t* ptrs;    // CSR row pointers (m + 1)
  const int32_t* idx;     // column indices
  const double* vals;
  int32_t m, kdim;
  unsigned char* ent;     // out: packed entries (16 bytes each: value, byte offset of its B row inside the staged chunk), segment after segment
  int32_t* rp;            // out: [strips * chunks][TM + 4] row pointers relative to the segment (+ its length at [TM ..])
  int32_t* segoff;        // out: [strips * chunks + 1] first entry of every (strip, chunk) segment
};
struct Spmm2Pair {        // A(i,k) (prepared) x B(k,j) (row-major, through its tensor map)
  const unsigned char* ent;
  const int32_t* rp;
  const int32_t* segoff;
  int32_t kdim;
  int32_t tmB;            // index of B(k,j)'s CUtensorMap in the launch's table
};
struct Spmm2Out {
  double* C;              // column-major m x n
  int32_t m, n;
  int32_t pair_begin, pair_count;
  int32_t accumulate;     // 1: C already holds the dense-pair sum
  int32_t pad;
};
struct Spmm2Item {        // one CTA: 256 rows x 64 columns of one output block, all of its k-blocks
  int32_t out, strip, ctile, pad;
};
// SparseMatrix.sprand(rows, cols, density, new java.util.Random(seed)) on the device (power-of-two dims, draw-by-draw branch)
struct SprandDesc {
  int32_t rows, cols, nnz, draws;
  int64_t seed;
  int32_t* colPtrs;     // [cols + 1] out
  int32_t* rowIndices;  // [nnz] out
  double* values;       // [nnz] out
  int* status;          // set to 1 when the draws did not yield nnz distinct coordinates
};
int sprand_draws(int64_t nnz);
cudaError_t launch_sprand(const SprandDesc* d_descs, int nblocks, int max_cols, cudaStream_t stream);
size_t spmm2_aux_bytes(int m, int kdim, int64_t nnz, size_t* ent_off, size_t* rp_off, size_t* seg_off);
bool spmm2_encode_b_tmap(void* out128, const double* base, int64_t kdim, int64_t n, int64_t ld);
cudaError_t launch_spmm2_prep(const Spmm2Prep* d_preps, int nblocks, int max_m, int max_kdim, cudaStream_t stream);
cudaError_t launch_spmm2(const Spmm2Item* d_items, int nitems, const Spmm2Out* d_outs, const Spmm2Pair* d_pairs, const void* d_tmaps,
                         cudaStream_t stream);

// Aggregates (RowSum / ColumnSum / Sum / TraceDirectExecution, MatfastExecution.scala:239-463), batched over blocks;
// the cross-block reduceByKey(LocalMatrix.add) is fused in: every block adds straight into its output vector / scalar
// (fp64 atomics; the reference's reduce order is arbitrary as well).  Outputs must be zeroed before the launch.
struct AggDesc {
  const double* v;        // dense values (sparse blocks are densified by the caller)
  int32_t rows, cols;     // logical dims
  uint8_t isT;
  uint8_t pad[7];
  double* out;            // row sums [rows] / column sums [cols] / scalar
};
enum AggOp { AGG_ROW_SUM = 0, AGG_COL_SUM = 1, AGG_SUM = 2, AGG_TRACE = 3 };
cudaError_t launch_aggregate(int op, const AggDesc* d_descs, int nblocks, int max_rows, int max_cols, cudaStream_t stream);

// Project{Row,Column}DirectExecution / SelectDirectExecution (MatfastExecution.scala:31-213): one row or column of a dense
// block copied into a 1 x cols / rows x 1 block (a single element for selection), batched over blocks.
struct LineDesc {
  const double* v;
  int32_t rows, cols;
  int32_t offset;       // row (take_row) or column index inside the block
  int32_t len;          // elements to copy (cols / rows; 1 for selection with offset2)
  int32_t offset2;      // selection: the other index (-1 = whole line)
  uint8_t isT, take_row;
  uint8_t pad[2];
  double* out;
};
cudaError_t launch_extract_lines(const LineDesc* d_descs, int nblocks, int max_len, cudaStream_t stream);

// Small table upload that does NOT go through the copy engines: an SM-driven copy from mapped pinned host memory.  The
// descriptor tables of an operator must not queue behind gigabytes of block ingest on the H2D engine.
cudaError_t launch_copy_words(void* dst, const void* src_mapped, size_t bytes, cudaStream_t stream);

// java.util.Random-compatible U(0,1) fill: out[i] = i-th nextDouble() of new Random(seed), batched over blocks
struct RandDesc {
  double* out;
  int64_t n;
  int64_t seed;
};
cudaError_t launch_java_rand_batched(const RandDesc* d_descs, int nblocks, int64_t max_n, cudaStream_t stream);

}  // namespace matrel
