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
// C(blocks in h_ctab, nbr x nbc grid of blk-sized column-major blocks) = A(M x K) * B(K x N); absent blocks are zeros.
// *nonfinite = 1 (and nothing written) when an operand holds Inf/NaN: the caller must use the exact kernel instead.
cudaError_t ozaki_gemm_f64(const OzakiOperand* a_blocks, int na, const OzakiOperand* b_blocks, int nb, int64_t M, int64_t K,
                           int64_t N, int slices, double* const* h_ctab, int blk, int nbr, int nbc, int* launches,
                           int* nonfinite, cudaStream_t stream);

// Ozaki scheme II (gemm_algo 4 and the auto selection): residues modulo `moduli` pairwise-coprime p_t <= 256, one int8 tensor-core
// GEMM per modulus, Chinese-remainder reconstruction -- as a job engine over slot-organised residue buffers (gemm_ozaki.cu).
// All table arguments are DEVICE pointers (the caller uploads them through its own staging path); nothing synchronises with the
// host.  *oz2_flag() != 0 on the device means "operands not representable (Inf / NaN, or too wide a range in auto mode)": the
// engine's remaining kernels are no-ops then and the caller's gated DMMA launch produces the blocks instead.
struct Oz2Engine;
// share_ab: a Gram product (left = right^T, cap_r == cap_c): the A side of slot s is the B side of slot s, so only the B' residues
// are held (one operand's scratch) and preparing a B slot also makes its A slot.
// strassen: one Strassen level (DESIGN section 4.1.3).  Every slot is prepared at once, from whole blocks given in quads (quadrants
// (0,0), (0,1), (1,0), (1,1) of (line half, k half)); a tile list is cut into pieces of max_tiles = 7 x positions, each holding the
// 7 sub-products product-major: sub-product i of position (lm, ln) (a tile of a quadrant of C) is the buffer tile
// (i Mpad / 256 + lm, i Npad / 512 + ln).  The residue scratch is 7/4 of the plain one.
size_t oz2_scratch_bytes(int blk, int64_t K, int moduli, int cap_r, int cap_c, int max_tiles, bool share_ab = false, bool strassen = false);
int oz2_tiles_per_block(int blk);
cudaError_t oz2_create(Oz2Engine** out, int blk, int64_t K, int moduli, int cap_r, int cap_c, int max_tiles, int guard_range,
                       bool share_ab, bool strassen, cudaStream_t stream);
bool oz2_strassen(const Oz2Engine* e);
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
  int32_t upper;        // 1: a diagonal block of a Gram product, only the elements on and above its diagonal are fixed
  int32_t pad;
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
// Gram products C = A^T A or A A^T (gram.cu, DESIGN section 4.1.2): the engines compute the blocks on and above the diagonal;
// ONE launch then writes dst(p, q) = src(q, p) for every strictly-lower element.  dst is m x n, src n x m, both column-major.  A
// strictly-lower block C(i, j) has src = C(j, i); a diagonal block (diag = 1, src == dst, m == n) has only its elements below the
// diagonal written, from the ones above it.
struct GramMirror {
  const double* src;
  double* dst;
  int32_t m, n;
  int32_t diag, pad;
};
cudaError_t launch_gram_mirror(const GramMirror* d_items, int nitems, int max_m, int max_n, cudaStream_t stream);

// A symmetric n x n CSC block from its upper triangle U (CSC, rows <= column, ascending) and U^T (CSC, ascending): column c is
// U(:, c) followed by the entries of U^T(:, c) below the diagonal.  fill = false: cnt[c] = the column's entries (then
// launch_exclusive_scan makes optr); fill = true: writes oidx / oval at optr.
struct GramSym {
  const int32_t* up;
  const int32_t* ui;
  const double* uv;
  const int32_t* tp;
  const int32_t* ti;
  const double* tv;
  int32_t* cnt;
  const int32_t* optr;
  int32_t* oidx;
  double* oval;
  int32_t n;
  int32_t pad;
};
cudaError_t launch_gram_sym(bool fill, const GramSym* d_items, int nitems, int max_n, cudaStream_t stream);
// fp32 multiply on wgmma tf32 (3xTF32 split, fp32 accumulation); same operand / output conventions.
// *nonfinite = 1 (and nothing written) when an operand holds Inf/NaN: the caller must use the exact kernel instead.
cudaError_t tf32x3_gemm(const OzakiOperand* a_blocks, int na, const OzakiOperand* b_blocks, int nb, int64_t M, int64_t K, int64_t N,
                        double* const* h_ctab, int blk, int nbr, int nbc, int* launches, int* nonfinite, cudaStream_t stream);

// ---- element-wise / layout kernels (HBM-bound), batched over blocks ---------------------------------
enum EwOp { EW_ADD = 0, EW_MUL = 1, EW_DIV = 2, EW_RANK1 = 3, EW_RANK1_COMPAT = 4, EW_COPY = 5 };

// C (column-major rows x cols) = f(A(r,c), B(r,c)); A, B dense with their own isTransposed flag.  For EW_ADD/MUL/DIV a null A or
// B is an absent operand: 0.0 everywhere (the unstored positions of a sparse operand, see launch_sparse_ew_scatter).
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
// ---- element-wise joins with a sparse side, on the stored entries (sparse_ew.cu, DESIGN section 4.5.3) ----------------------
// sparse (+) sparse: one pair per output block, in a CSC frame (a CSR operand as its launch_sptrans CSC arrays).  How an operand's
// stored entries of one position make its value:
enum SpEwMode {
  SPEW_SUM = 0,    // 0.0 + v1 + v2 + ... in storage order (both operands CSC: addSparseSparseNative / elementWiseOpSparseSparseNative)
  SPEW_LAST = 1,   // the last stored v (toArray of a CSC operand when the other one is CSR)
  SPEW_FIRST = 2,  // the first v of an ascending line with repeats adjacent (toArray of a CSR operand, repeats reversed by sptrans)
};
struct SpEwPair {
  const int32_t* ap;      // A: column pointers (cols + 1), row indices, values
  const int32_t* ai;
  const double* av;
  const int32_t* bp;      // B: the same
  const int32_t* bi;
  const double* bv;
  int32_t rows, cols;
  uint8_t amode, bmode;   // SpEwMode
  uint8_t native;         // both operands CSC: add sums A's and B's entries in one running sum; a dense outcome has +0.0 for -0.0
  uint8_t pad;
  int32_t* colcnt;        // count pass: [cols] kept entries of each column
  unsigned long long* total;  // count pass: kept entries of the pair (pre-zeroed)
  const int32_t* optr;    // fill pass, sparse outcome: column pointers (scanned from colcnt), row indices, values
  int32_t* oidx;
  double* oval;
  double* dense;          // fill pass, dense outcome: column-major rows x cols, every element written (nullptr: sparse outcome)
};
struct SpEwLaunchShape {
  bool acc_in_smem;       // per-warp column accumulators in shared memory, else in the caller's scratch (scratch_bytes)
  size_t smem_bytes;
  int max_ctas;           // persistent grid
  size_t scratch_bytes;
};
constexpr int kSpEwMaxSmem = 200 * 1024;
SpEwLaunchShape sparse_ew_shape(int max_rows);
// op: EW_ADD / EW_MUL / EW_DIV.  fill = false: the count pass (colcnt, total); fill = true: the entries.  Every pair's rows <= max_rows.
cudaError_t launch_sparse_ew(int op, bool fill, const SpEwPair* d_pairs, int npairs, int max_rows, int max_cols, void* d_scratch,
                             const SpEwLaunchShape& s, cudaStream_t stream);
// dense (+) sparse: C = op(D, S) (op(S, D) when sparse_left) at the stored positions of S, the last stored value of a position;
// the rest of C (op with an absent operand) is written before by launch_ew_batched
struct DsEwDesc {
  const int32_t* ptr;     // S: CSC, or CSR when sT
  const int32_t* idx;
  const double* val;
  const double* D;        // rows x cols, row-major when dT
  double* C;              // rows x cols, column-major
  int32_t rows, cols;
  uint8_t sT, dT, sparse_left;
  uint8_t pad[5];
};
cudaError_t launch_sparse_ew_scatter(int op, const DsEwDesc* d_descs, int ndescs, int max_lines, cudaStream_t stream);

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
// ---- dense x low-density sparse partials C (+)= A S on the same kernels, as C^T = S^T A^T (spmm.cu, DESIGN section 4.5.2).  The
// prepared block is S^T: its CSC arrays (ptrs = column pointers, n + 1; idx = row indices), m = n columns of S, kdim = rows of S.
struct DspmmPrep {        // Spmm2Prep's fields, then:
  const int32_t* ptrs;
  const int32_t* idx;
  const double* vals;
  int32_t m, kdim;
  unsigned char* ent;
  int32_t* rp;
  int32_t* segoff;
  uint8_t* kref;          // out: [strips * chunks][KC] the distinct indices of each segment, by slot (unused slots zero)
  int32_t repeats_reversed;  // repeated indices of a row are in reverse storage order (a CSR block after launch_sptrans), so the
                             // first of them is the stored one that counts
  int32_t pad;
};
struct DspmmPair {        // A(i,k) (column-major, lda even, 16-byte aligned) x S(k,j) (prepared)
  const unsigned char* ent;
  const int32_t* rp;      // rp[segment][TM + 1]: distinct indices of the segment
  const int32_t* segoff;
  const uint8_t* kref;
  const double* A;
  int32_t kdim, lda;      // lda = rows of A = Spmm2Out::n
};
size_t dspmm_aux_bytes(int n, int kdim, int64_t nnz, size_t* ent_off, size_t* rp_off, size_t* seg_off, size_t* kref_off);
cudaError_t launch_dspmm_prep(const DspmmPrep* d_preps, int nblocks, int max_n, int max_kdim, cudaStream_t stream);
// Spmm2Out of an output block C (m x n, column-major): {C, n, m, ...}; items: (out, strip of 256 columns of C, tile of 64 rows)
cudaError_t launch_dspmm(const Spmm2Item* d_items, int nitems, const Spmm2Out* d_outs, const DspmmPair* d_pairs, cudaStream_t stream);
constexpr int DS_KW = kSpmmMaxDim / 32;  // words of a row's non-finite set / a column's stored set
struct DsFlagDesc {       // one left block (column-major image, lda = m)
  const double* A;
  int32_t m, kdim;
  uint32_t* bits;         // out: [m][DS_KW]
  uint32_t* rowflags;     // out: [(m + 31) / 32]
  int32_t* any;           // out: 1 when a bit is set (pre-zeroed)
};
struct DsFixPair {        // one routed pair, after every partial of its output block
  const uint32_t* bits;
  const uint32_t* rowflags;
  const int32_t* any;
  const int32_t* ptr;     // CSC of S
  const int32_t* idx;
  double* C;              // m x n, column-major
  int32_t m, n;
};
cudaError_t launch_ds_flags(const DsFlagDesc* d_descs, int ndescs, int max_m, cudaStream_t stream);
cudaError_t launch_ds_fixup(const DsFixPair* d_pairs, int npairs, cudaStream_t stream);
bool spmm2_encode_b_tmap(void* out128, const double* base, int64_t kdim, int64_t n, int64_t ld);
cudaError_t launch_spmm2_prep(const Spmm2Prep* d_preps, int nblocks, int max_m, int max_kdim, cudaStream_t stream);
cudaError_t launch_spmm2(const Spmm2Item* d_items, int nitems, const Spmm2Out* d_outs, const Spmm2Pair* d_pairs, const void* d_tmaps,
                         cudaStream_t stream);

// Aggregates (RowSum / ColumnSum / Sum / TraceDirectExecution, MatfastExecution.scala:239-463), batched over blocks;
// the cross-block reduceByKey(LocalMatrix.add) is fused in: every block adds straight into its output vector / scalar
// (fp64 atomics; the reference's reduce order is arbitrary as well).  Outputs must be zeroed before the launch.
struct AggDesc {
  const double* v;        // dense values (sparse blocks go to launch_sparse_agg)
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

// ---- aggregates and slicing of sparse blocks on their stored entries (sparse_agg.cu, DESIGN section 4.5.4) -----------------------
// A block's lines are the columns of a CSC block and the rows of a CSR one (colPtrs, rowIndices, values as stored).
enum SpAggMode {
  SPAGG_ALONG = 0,   // the output index is the line (colSum of CSC, rowSum of CSR): one lane per line
  SPAGG_ACROSS = 1,  // the output index is the stored index (rowSum of CSC, colSum of CSR): one warp per block
  SPAGG_DIAG = 2,    // trace: the entries whose index equals their line's, one scalar per block
};
struct SpAggDesc {
  const int32_t* ptr;     // nlines + 1
  const int32_t* idx;
  const double* val;
  double* part;           // out: the block's partial, len doubles, every element written
  int32_t nlines, len;    // len: output length (rows for rowSum, columns for colSum, 1 for trace)
  int32_t mode;           // SpAggMode
  int32_t pad;
};
// One output vector and the partials of its sparse blocks, in ascending block index
struct SpAggOut {
  double* out;
  const double* part;     // nparts x len, consecutive
  int32_t len, nparts;
  int32_t accumulate;     // 1: the line also has dense blocks, the total is added with an atomic; 0: stored
  int32_t pad;
};
constexpr int kSpAggSmemLen = 2048;  // longest SPAGG_ACROSS output a warp accumulates in shared memory; longer ones in `part`
// max_nlines: the most lines of any block; max_across_len: the longest SPAGG_ACROSS output (0: none)
cudaError_t launch_sparse_agg(const SpAggDesc* d_descs, int ndescs, int max_nlines, int max_across_len, cudaStream_t stream);
cudaError_t launch_sparse_agg_combine(const SpAggOut* d_outs, int nouts, int max_len, cudaStream_t stream);
// project / selection: out[0, len) of one sparse block, the last stored entry of a position or 0.0 (every element written)
struct SpSliceDesc {
  const int32_t* ptr;
  const int32_t* idx;
  const double* val;
  double* out;
  int32_t len;
  int32_t line;           // target < 0: the line copied into out; else the first of the len lines searched (out[l - line])
  int32_t target;         // the index searched in each line, -1 = along one line
  int32_t pad;
};
cudaError_t launch_sparse_slice(const SpSliceDesc* d_descs, int ndescs, int max_len, cudaStream_t stream);

// ---- matrix x thin-matrix products C = M X over dense, CSC and CSR blocks (matvec.cu, DESIGN section 4.5.5) -----------------------
// M = A for C = A X, M = A^T for C = X A.  X has cols <= kMvMaxCols columns (rows for X A), the kernels run a width W in {1, 2, 4, 8}
// >= cols, and column j of C is computed exactly as the width-1 product M X(:, j).  Each output block has its pairs (k-blocks) in
// ascending k; x is a pair's X block: kdim contiguous doubles at width 1, x(c, j) at x[c xl.c + j xl.j] (MvXLayout) above.
constexpr int kMvMaxCols = 8;
enum MvKind {
  MV_DENSE_ICONT = 0,  // dense, M(i, c) at A[i + c sc]
  MV_DENSE_KCONT = 1,  // dense, M(i, c) at A[i si + c]
  MV_CSR = 2,          // the CSR arrays of M (A X with a CSR block)
  MV_PART = 3,         // the partial launch_matvec_parts wrote
};
struct MvPair {
  const double* A;
  const int32_t* ptr;     // MV_CSR: row pointers, column indices, values
  const int32_t* idx;
  const double* val;
  const double* x;
  const double* part;     // MV_PART: column j of the partial at part[j len], len doubles each
  int64_t si, sc;
  int32_t kdim, kind;
};
// The strides of an X block, one per MvPair / MvPartDesc in an array of their own: the width-1 kernels read neither it nor `cols`,
// so their code and the descriptors' sizes are those of the single-vector route.
struct MvXLayout {
  int32_t c, j;
};
struct MvOut {
  double* C;              // len x cols column-major (A X: (i, j) at i + j len) or cols x len (X A: (j, i) at j + i cols), every
                          // element written
  int32_t len, pair_begin, pair_count, cols;
};
constexpr int kMvTile = 32;  // outputs per CTA
struct MvItem {           // one CTA: outputs [tile * kMvTile, +kMvTile) of one output block
  int32_t out, tile;
};
// max_cols: the widest output block (picks W); d_xls: one MvXLayout per pair, unread (may be null) when max_cols == 1; xa: C = X A
cudaError_t launch_matvec(const MvOut* d_outs, const MvPair* d_pairs, const MvItem* d_items, int nitems, int max_cols,
                          const MvXLayout* d_xls, int xa, cudaStream_t stream);
enum MvPartMode {
  MV_ALONG = 0,   // the output index is the line (X S with a CSC block): one lane per line, x indexed by the stored index
  MV_ACROSS = 1,  // the output index is the stored index (A X with a CSC block, X S with a CSR block): one warp, x indexed by the line
};
struct MvPartDesc {
  const int32_t* ptr;     // nlines + 1, as stored
  const int32_t* idx;
  const double* val;
  const double* x;        // X block: xlen rows (c) x cols
  double* part;           // out: column j at part[j len], len doubles each, every element written
  int32_t nlines, len, xlen;
  int32_t mode;           // MvPartMode
  int32_t image;          // 1 (X S): the dense image's terms (the last stored entry of a position; NaN in column j where a non-finite
                          // x(r, j) meets an unstored position)
  int32_t cols;
};
cudaError_t launch_matvec_parts(const MvPartDesc* d_descs, int ndescs, int max_nlines, int max_across_len, int max_cols,
                                const MvXLayout* d_xls, cudaStream_t stream);

// Small table upload that does NOT go through the copy engines: an SM-driven copy from mapped pinned host memory.  The
// descriptor tables of an operator must not queue behind gigabytes of block ingest on the H2D engine.
cudaError_t launch_copy_words(void* dst, const void* src_mapped, size_t bytes, cudaStream_t stream);

// Cross-GPU sum of the K-split multiply's partial products (abi_grid.cpp, mr_dmatrix_multiply_ksplit):
//   out[e] = parts[0][offset + e] + parts[1][offset + e] + ... + parts[nparts - 1][offset + e],  e < count,
// added left to right in part order (deterministic, independent of timing).  Part pointers may be peer-device pointers: the
// reads go over NVLink, so the roof is NVLink read bandwidth, not HBM.  `parts` is a device array of nparts (<= kKsplitMaxParts)
// base pointers; descriptors are device memory.
struct KsplitDesc {
  double* out;
  int64_t offset;  // elements, the same for every part
  int64_t count;
};
constexpr int kKsplitMaxParts = 64;
cudaError_t launch_ksplit_reduce(const KsplitDesc* d_descs, int ndescs, const double* const* d_parts, int nparts, int64_t max_count,
                                 cudaStream_t stream);

// Whole dense matrices <-> blocks (dense_io.cu, abi_dense.cpp).  A window: rows x cols logical elements; a row-major side (rm = 1)
// holds element (r, c) at p[r * ld + c], a column-major one at p[r + c * ld].
struct DenseIoDesc {
  const double* src;      // nullptr (assemble only): the window is zero-filled
  double* dst;
  int64_t lds, ldd;       // leading dimensions, elements
  int32_t rows, cols;
  uint8_t src_rm, dst_rm;
  uint8_t pad[6];
};
// gather: src and dst share one layout (src_rm == dst_rm); assemble: any pair of layouts (any_transposed: some src_rm != dst_rm)
cudaError_t launch_dense_gather(const DenseIoDesc* d_descs, int ndescs, int max_rows, int max_cols, cudaStream_t stream);
cudaError_t launch_dense_assemble(const DenseIoDesc* d_descs, int ndescs, int max_rows, int max_cols, bool any_transposed,
                                  cudaStream_t stream);
// The entries of a CSC (csr = 0) or CSR (csr = 1) block into its window of dst, after that window was zero-filled.
struct DenseScatterDesc {
  const int32_t* ptrs;    // nlines + 1
  const int32_t* idx;
  const double* vals;
  double* dst;            // the window's element (0, 0)
  int64_t ldd;
  int32_t nlines;         // columns (CSC) or rows (CSR)
  uint8_t csr, dst_rm;
  uint8_t pad[2];
};
cudaError_t launch_dense_scatter(const DenseScatterDesc* d_descs, int ndescs, int max_lines, cudaStream_t stream);

// ---- sparse x sparse block products and their partial sums (spgemm.cu) ---------------------------------------------------------
// A chain: one output block whose partials are all low-density sparse x sparse, computed in a CSC frame (the CSR arrays of a block
// are the CSC arrays of its transpose, so an all-CSR chain runs as C^T = B^T A^T).  Level l: P_l = L_l * R_l (L: m x kdim,
// R: kdim x n, both CSC), S <- S + P_l.  Products and sums rounded one by one, zeros dropped after each (see DESIGN section 4.5.1).
struct SpgemmPair {
  const int32_t* lp;      // L column pointers (kdim + 1), row indices, values
  const int32_t* li;
  const double* lv;
  const int32_t* rp;      // R column pointers (n + 1), row indices, values
  const int32_t* ri;
  const double* rv;
};
struct SpgemmChain {
  int32_t m, n;           // frame dims of the output
  int32_t pair_begin, levels;
  int32_t count_off;      // counters of level l: counts[count_off + l] = nnz(P_l), counts[count_off + levels + l] = nnz(S_l) - nnz(S_l-1);
                          // tri: then the same two counts over the diagonal at count_off + 2 levels and count_off + 3 levels
  int32_t tri;            // a diagonal block of a Gram product: rows r <= c of column c only (its P_l are symmetric)
  int32_t* colcnt;        // count pass: [n] entries of each column of the final S
  const int32_t* optr;    // fill pass, sparse output: column pointers [n + 1] ...
  int32_t* oidx;          // ... row indices (nullptr: dense output) ...
  double* oval;           // ... values
  double* dense;          // fill pass, dense output: frame element (r, c) at dense[r * drs + c * dcs], every element written
  int64_t drs, dcs;
};
struct SpgemmItem {       // one CTA's work: columns col0 .. col0 + spgemm_columns_per_item() - 1 of a chain
  int32_t chain, col0;
};
struct SpgemmLaunchShape {
  int smem_counters;      // per-level counters in shared memory (levels <= this), else global atomics
  int cnt_lines;          // counters per level: 2, or 4 when a chain is triangular
  bool acc_in_smem;       // per-warp column accumulators in shared memory, else in the caller's scratch (scratch_bytes)
  int max_ctas;           // persistent grid
  size_t scratch_bytes;
};
constexpr int kSpgemmMaxSmem = 200 * 1024;
int spgemm_columns_per_item();
SpgemmLaunchShape spgemm_shape(int max_m, int max_levels, bool tri);
// fill = false: the count pass (colcnt, counts, *d_products += scalar products; counts and products pre-zeroed; *d_unsorted = 1
// when d_unsorted is given and a walked R column's row indices do not ascend); fill = true: writes the entries.  Every chain's
// m <= max_m.
cudaError_t launch_spgemm(bool fill, const SpgemmItem* d_items, int nitems, const SpgemmChain* d_chains, const SpgemmPair* d_pairs,
                          int* d_counts, unsigned long long* d_products, void* d_scratch, int max_m, const SpgemmLaunchShape& s,
                          int* d_unsorted, cudaStream_t stream);
// out[0] = 0, out[t + 1] = in[0] + ... + in[t], t < n; one CTA per descriptor
struct ScanDesc {
  const int32_t* in;
  int32_t* out;
  int32_t n;
  int32_t pad;
};
cudaError_t launch_exclusive_scan(const ScanDesc* d_descs, int ndescs, cudaStream_t stream);
// Stable CSR <-> CSC conversion: the nl input lines (ptr, idx, val; indices < no) become the no lines of the transpose (optr, oidx,
// oval), indices ascending in every line.  cur: [no] zeroed ints; scans[t] = {cur, optr, no} of descriptor t.
struct SpTransDesc {
  const int32_t* ptr;
  const int32_t* idx;
  const double* val;
  int32_t nl, no, nnz;
  int32_t pad;
  int32_t* optr;
  int32_t* oidx;
  double* oval;
  int32_t* cur;
};
cudaError_t launch_sptrans(const SpTransDesc* d_descs, const ScanDesc* d_scans, int ndescs, int max_nnz, int max_nl, int max_no,
                           cudaStream_t stream);

// java.util.Random-compatible U(0,1) fill: out[i] = i-th nextDouble() of new Random(seed), batched over blocks
struct RandDesc {
  double* out;
  int64_t n;
  int64_t seed;
};
cudaError_t launch_java_rand_batched(const RandDesc* d_descs, int nblocks, int64_t max_n, cudaStream_t stream);

}  // namespace matrel
