// matrel.hpp -- header-only C++17 mirror of the reference's Dataset operator API over the C ABI
// (include/matrel.h).  Method names and argument order follow
// <reference>/src/main/scala/org/apache/spark/sql/matfast/Dataset.scala:57-152; `require`
// failures surface as matfast::IllegalArgumentException carrying the reference's message text.
#pragma once
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <tuple>
#include <vector>

#include "matrel.h"

namespace matfast {

struct IllegalArgumentException : std::invalid_argument {
  using std::invalid_argument::invalid_argument;
};
struct MatrelError : std::runtime_error {
  int code;
  MatrelError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

inline void check(mr_status st) {
  if (st == MR_OK) return;
  const std::string msg = mr_last_error();
  if (st == MR_EINVAL || st == MR_EDIM) throw IllegalArgumentException(msg);
  throw MatrelError(st, msg);
}

// MLMatrix.scala:234-241 / :525-543 -- host containers for block ingest/egress
struct DenseMatrix {
  int32_t numRows = 0, numCols = 0;
  std::vector<double> values;  // column-major; row-major when isTransposed
  bool isTransposed = false;
};
struct SparseMatrix {
  int32_t numRows = 0, numCols = 0;
  std::vector<int32_t> colPtrs, rowIndices;
  std::vector<double> values;
  bool isTransposed = false;
};

class MatfastSession {
 public:
  explicit MatfastSession(int device = -1, bool compat_bugs = true, void* stream = nullptr) {
    mr_options o{};
    o.device = device;
    o.compat_bugs = compat_bugs ? 1 : 0;
    o.stream = stream;
    check(mr_init(&o, &ctx_));
  }
  ~MatfastSession() {
    if (ctx_) mr_shutdown(ctx_);
  }
  MatfastSession(const MatfastSession&) = delete;
  MatfastSession& operator=(const MatfastSession&) = delete;
  void sync() { check(mr_sync(ctx_)); }
  mr_context* raw() const { return ctx_; }

 private:
  mr_context* ctx_ = nullptr;
};

class Dataset {
 public:
  explicit Dataset(MatfastSession& s) : session_(&s) {
    mr_matrix* h = nullptr;
    check(mr_matrix_create(s.raw(), &h));
    h_.reset(h, [](mr_matrix* m) { mr_matrix_free(m); });
  }
  // Seq(MatrixBlock(rid, cid, matrix)).toDS()
  void putBlock(int32_t rid, int32_t cid, const DenseMatrix& m) {
    mr_block_desc d{};
    d.type = 1;
    d.numRows = m.numRows;
    d.numCols = m.numCols;
    d.values = const_cast<double*>(m.values.data());
    d.valuesLen = static_cast<int64_t>(m.values.size());
    d.isTransposed = m.isTransposed;
    check(mr_matrix_put_block(h_.get(), rid, cid, &d));
  }
  void putBlock(int32_t rid, int32_t cid, const SparseMatrix& m) {
    mr_block_desc d{};
    d.type = 0;
    d.numRows = m.numRows;
    d.numCols = m.numCols;
    d.colPtrs = const_cast<int32_t*>(m.colPtrs.data());
    d.colPtrsLen = static_cast<int64_t>(m.colPtrs.size());
    d.rowIndices = const_cast<int32_t*>(m.rowIndices.data());
    d.rowIndicesLen = static_cast<int64_t>(m.rowIndices.size());
    d.values = const_cast<double*>(m.values.data());
    d.valuesLen = static_cast<int64_t>(m.values.size());
    d.isTransposed = m.isTransposed;
    check(mr_matrix_put_block(h_.get(), rid, cid, &d));
  }
  bool hasBlock(int32_t rid, int32_t cid) const {
    int32_t present = 0;
    check(mr_matrix_has_block(h_.get(), rid, cid, &present));
    return present != 0;
  }
  std::vector<std::pair<int32_t, int32_t>> blockIds() const {
    int64_t n = 0;
    check(mr_matrix_num_blocks(h_.get(), &n));
    std::vector<int32_t> r(n), c(n);
    if (n) check(mr_matrix_block_ids(h_.get(), r.data(), c.data(), n));
    std::vector<std::pair<int32_t, int32_t>> out(n);
    for (int64_t i = 0; i < n; ++i) out[i] = {r[i], c[i]};
    return out;
  }
  // dense blocks only; sparse results are fetched with the two-call mr_matrix_get_block protocol
  DenseMatrix getDenseBlock(int32_t rid, int32_t cid) const {
    mr_block_desc d{};
    check(mr_matrix_get_block(h_.get(), rid, cid, &d));
    if (d.type != 1) throw MatrelError(MR_ENOTSUP, "block is sparse");
    DenseMatrix m;
    m.numRows = d.numRows;
    m.numCols = d.numCols;
    m.isTransposed = d.isTransposed != 0;
    m.values.resize(static_cast<size_t>(d.valuesLen));
    d.values = m.values.data();
    check(mr_matrix_get_block(h_.get(), rid, cid, &d));
    return m;
  }

  // ---- operators (Dataset.scala:57-152) -----------------------------------------------------
  Dataset matrixMultiply(int64_t leftRowNum, int64_t leftColNum, const Dataset& right, int64_t rightRowNum,
                         int64_t rightColNum, int32_t blkSize) const {
    return binary(mr_matrix_multiply, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize);
  }
  Dataset addElement(int64_t lr, int64_t lc, const Dataset& right, int64_t rr, int64_t rc, int32_t blkSize) const {
    return binary(mr_add_element, lr, lc, right, rr, rc, blkSize);
  }
  Dataset multiplyElement(int64_t lr, int64_t lc, const Dataset& right, int64_t rr, int64_t rc, int32_t blkSize) const {
    return binary(mr_multiply_element, lr, lc, right, rr, rc, blkSize);
  }
  Dataset divideElement(int64_t lr, int64_t lc, const Dataset& right, int64_t rr, int64_t rc, int32_t blkSize) const {
    return binary(mr_divide_element, lr, lc, right, rr, rc, blkSize);
  }
  Dataset matrixRankOneUpdate(int64_t lr, int64_t lc, const Dataset& right, int64_t rr, int64_t rc, int32_t blkSize) const {
    return binary(mr_rank_one_update, lr, lc, right, rr, rc, blkSize);
  }
  Dataset transpose() const {
    mr_matrix* o = nullptr;
    check(mr_transpose(h_.get(), &o));
    return Dataset(*session_, o);
  }
  Dataset t() const { return transpose(); }
  Dataset addScalar(double alpha) const { return unary(mr_add_scalar, alpha); }
  Dataset multiplyScalar(double alpha) const { return unary(mr_multiply_scalar, alpha); }
  Dataset power(double alpha) const { return unary(mr_power, alpha); }
  // aggregates and slicing (Dataset.scala:38-87)
  Dataset rowSum(int64_t nrows, int64_t ncols) const { return shaped(mr_row_sum, nrows, ncols); }
  Dataset colSum(int64_t nrows, int64_t ncols) const { return shaped(mr_col_sum, nrows, ncols); }
  Dataset sum(int64_t nrows, int64_t ncols) const { return shaped(mr_sum, nrows, ncols); }
  Dataset trace(int64_t nrows, int64_t ncols) const { return shaped(mr_trace, nrows, ncols); }
  Dataset project(int64_t nrows, int64_t ncols, int32_t blkSize, bool rowOrCol, int64_t index) const {
    mr_matrix* o = nullptr;
    check(mr_project(h_.get(), nrows, ncols, blkSize, rowOrCol ? 1 : 0, index, &o));
    return Dataset(*session_, o);
  }
  Dataset selection(int64_t nrows, int64_t ncols, int32_t blkSize, int64_t rowIdx, int64_t colIdx) const {
    mr_matrix* o = nullptr;
    check(mr_selection(h_.get(), nrows, ncols, blkSize, rowIdx, colIdx, &o));
    return Dataset(*session_, o);
  }
  Dataset vec(int64_t nrows, int64_t ncols, int32_t blkSize) const {
    mr_matrix* o = nullptr;
    check(mr_vec(h_.get(), nrows, ncols, blkSize, &o));
    return Dataset(*session_, o);
  }
  // Dataset.collect(): every dense block as (rid, cid, matrix); sparse results go through the two-call mr_matrix_get_block protocol
  std::vector<std::tuple<int32_t, int32_t, DenseMatrix>> collect() const {
    std::vector<std::tuple<int32_t, int32_t, DenseMatrix>> out;
    for (const auto& id : blockIds()) out.emplace_back(id.first, id.second, getDenseBlock(id.first, id.second));
    return out;
  }
  mr_matrix* raw() const { return h_.get(); }

 private:
  Dataset(MatfastSession& s, mr_matrix* h) : session_(&s), h_(h, [](mr_matrix* m) { mr_matrix_free(m); }) {}
  using BinFn = mr_status (*)(mr_matrix*, int64_t, int64_t, mr_matrix*, int64_t, int64_t, int32_t, mr_matrix**);
  using UnFn = mr_status (*)(mr_matrix*, double, mr_matrix**);
  using ShapedFn = mr_status (*)(mr_matrix*, int64_t, int64_t, mr_matrix**);
  Dataset shaped(ShapedFn f, int64_t nrows, int64_t ncols) const {
    mr_matrix* o = nullptr;
    check(f(h_.get(), nrows, ncols, &o));
    return Dataset(*session_, o);
  }
  Dataset binary(BinFn f, int64_t lr, int64_t lc, const Dataset& right, int64_t rr, int64_t rc, int32_t blk) const {
    mr_matrix* o = nullptr;
    check(f(h_.get(), lr, lc, right.h_.get(), rr, rc, blk, &o));
    return Dataset(*session_, o);
  }
  Dataset unary(UnFn f, double alpha) const {
    mr_matrix* o = nullptr;
    check(f(h_.get(), alpha, &o));
    return Dataset(*session_, o);
  }
  MatfastSession* session_;
  std::shared_ptr<mr_matrix> h_;
};

// ---- one process, all GPUs of the box (mr_init_grid): the placement grid replaces the Spark cluster --------------------------
class GridSession {
 public:
  explicit GridSession(int32_t ngpus, bool compat_bugs = true) {
    mr_options o{};
    o.device = -1;
    o.compat_bugs = compat_bugs ? 1 : 0;
    check(mr_init_grid(&o, ngpus, &g_));
  }
  ~GridSession() {
    if (g_) mr_grid_shutdown(g_);
  }
  GridSession(const GridSession&) = delete;
  GridSession& operator=(const GridSession&) = delete;
  void sync() { check(mr_grid_sync(g_)); }
  int32_t gpus() const {
    int32_t n = 0, pr = 0, pc = 0, nccl = 0;
    check(mr_grid_info(g_, &n, &pr, &pc, &nccl));
    return n;
  }
  mr_grid* raw() const { return g_; }

 private:
  mr_grid* g_ = nullptr;
};

// A Dataset whose blocks live on the GPUs of a GridSession (rank (rid % pr, cid % pc) owns block (rid, cid)).
class DistributedDataset {
 public:
  DistributedDataset(GridSession& g, int64_t nrows, int64_t ncols, int32_t blkSize) : grid_(&g) {
    mr_dmatrix* h = nullptr;
    check(mr_dmatrix_create(g.raw(), nrows, ncols, blkSize, &h));
    h_.reset(h, [](mr_dmatrix* m) { mr_dmatrix_free(m); });
  }
  // per-block java.util.Random(seed0 + rid * nbc + cid) streams, generated where the blocks live
  static DistributedDataset rand(GridSession& g, int64_t nrows, int64_t ncols, int32_t blkSize, int64_t seed0) {
    mr_dmatrix* h = nullptr;
    check(mr_dmatrix_rand(g.raw(), nrows, ncols, blkSize, seed0, &h));
    return DistributedDataset(g, h);
  }
  void putBlock(int32_t rid, int32_t cid, const DenseMatrix& m) {  // routed to the owner
    mr_block_desc d{};
    d.type = 1;
    d.numRows = m.numRows;
    d.numCols = m.numCols;
    d.values = const_cast<double*>(m.values.data());
    d.valuesLen = static_cast<int64_t>(m.values.size());
    d.isTransposed = m.isTransposed;
    check(mr_dmatrix_put_block(h_.get(), rid, cid, &d));
  }
  bool hasBlock(int32_t rid, int32_t cid) const {
    int32_t present = 0;
    check(mr_dmatrix_has_block(h_.get(), rid, cid, &present));
    return present != 0;
  }
  DenseMatrix getDenseBlock(int32_t rid, int32_t cid) const {
    mr_block_desc d{};
    check(mr_dmatrix_get_block(h_.get(), rid, cid, &d));
    DenseMatrix m;
    m.numRows = d.numRows;
    m.numCols = d.numCols;
    m.isTransposed = d.isTransposed != 0;
    m.values.resize(static_cast<size_t>(d.valuesLen));
    d.values = m.values.data();
    check(mr_dmatrix_get_block(h_.get(), rid, cid, &d));
    return m;
  }
  int32_t owner(int32_t rid, int32_t cid) const {
    int32_t rank = 0;
    check(mr_dmatrix_owner(h_.get(), rid, cid, &rank));
    return rank;
  }
  // Dataset.matrixMultiply :134-142 on the grid: peers' blocks are pulled over NVLink, no reduction
  DistributedDataset matrixMultiply(const DistributedDataset& right) const {
    mr_dmatrix* o = nullptr;
    check(mr_dmatrix_multiply(h_.get(), right.h_.get(), &o));
    return DistributedDataset(*grid_, o);
  }
  DistributedDataset addElement(const DistributedDataset& right) const { return elementwise(0, right); }
  DistributedDataset multiplyElement(const DistributedDataset& right) const { return elementwise(1, right); }
  DistributedDataset divideElement(const DistributedDataset& right) const { return elementwise(2, right); }
  double sum() const { return reduce(0); }
  double trace() const { return reduce(1); }
  // repartitionWithTargetPartitioner: (P, 1) = RowPartitioner, (1, P) = ColumnPartitioner
  DistributedDataset repartition(int32_t new_pr, int32_t new_pc) const {
    mr_dmatrix* o = nullptr;
    check(mr_dmatrix_repartition(h_.get(), new_pr, new_pc, &o));
    return DistributedDataset(*grid_, o);
  }
  // Dataset.t / transpose :57-61: blocks swap ids and move to their new owners; payloads untouched, isTransposed flipped
  DistributedDataset t() const { return transpose(); }
  DistributedDataset transpose() const {
    mr_dmatrix* o = nullptr;
    check(mr_dmatrix_transpose(h_.get(), &o));
    return DistributedDataset(*grid_, o);
  }
  // Dataset.addScalar / multiplyScalar / power :89-103: a map over the blocks each GPU owns
  DistributedDataset addScalar(double alpha) const { return scalar(0, alpha); }
  DistributedDataset multiplyScalar(double alpha) const { return scalar(1, alpha); }
  DistributedDataset power(double alpha) const { return scalar(2, alpha); }
  // Dataset.rowSum / colSum :63-72: local line sums + one ncclAllReduce; the result is nrows x 1 / 1 x ncols on the same grid
  DistributedDataset rowSum() const { return axisSum(0); }
  DistributedDataset colSum() const { return axisSum(1); }
  // Dataset.project :38-47 / selection :49-55; dimensions and block size travel with the handle
  DistributedDataset project(bool rowOrCol, int64_t index) const {
    mr_dmatrix* o = nullptr;
    check(mr_dmatrix_project(h_.get(), rowOrCol ? 1 : 0, index, &o));
    return DistributedDataset(*grid_, o);
  }
  DistributedDataset selection(int64_t rowIdx, int64_t colIdx) const {
    mr_dmatrix* o = nullptr;
    check(mr_dmatrix_selection(h_.get(), rowIdx, colIdx, &o));
    return DistributedDataset(*grid_, o);
  }
  mr_dmatrix* raw() const { return h_.get(); }

 private:
  DistributedDataset axisSum(int32_t axis) const {
    mr_dmatrix* o = nullptr;
    check(mr_dmatrix_axis_sum(h_.get(), axis, &o));
    return DistributedDataset(*grid_, o);
  }
  DistributedDataset scalar(int32_t op, double alpha) const {
    mr_dmatrix* o = nullptr;
    check(mr_dmatrix_scalar(op, h_.get(), alpha, &o));
    return DistributedDataset(*grid_, o);
  }
  DistributedDataset(GridSession& g, mr_dmatrix* h) : grid_(&g), h_(h, [](mr_dmatrix* m) { mr_dmatrix_free(m); }) {}
  DistributedDataset elementwise(int32_t op, const DistributedDataset& right) const {
    mr_dmatrix* o = nullptr;
    check(mr_dmatrix_elementwise(op, h_.get(), right.h_.get(), &o));
    return DistributedDataset(*grid_, o);
  }
  double reduce(int32_t what) const {
    double v = 0.0;
    check(mr_dmatrix_reduce_scalar(h_.get(), what, &v));
    return v;
  }
  GridSession* grid_;
  std::shared_ptr<mr_dmatrix> h_;
};

}  // namespace matfast
