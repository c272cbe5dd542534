// Element-wise operators (add / multiply / divide joins, scalar maps, rank-one update), transpose and materialisation.
#include "host.h"

using namespace matrel;
using namespace mrhost;

namespace mrhost {
void check_same_dims(int64_t lr, int64_t lc, int64_t rr, int64_t rc) {
  // MatfastExecution.scala:584-587 (and :621-624, :658-661)
  MR_REQUIRE(lr == rr, MR_EDIM, "Row number not match, leftRowNum = %lld, rightRowNum = %lld", (long long)lr,
             (long long)rr);
  MR_REQUIRE(lc == rc, MR_EDIM, "Col number not match, leftColNum = %lld, rightColNum = %lld", (long long)lc,
             (long long)rc);
}

}  // namespace mrhost

namespace {

// ------------------------------------------------------------------------------------------------
// element-wise operator plumbing
// ------------------------------------------------------------------------------------------------
struct EwBatch {
  mr_context* ctx;
  int op;
  std::vector<EwDesc> descs;
  std::vector<Block> keep;  // densified temporaries
  std::vector<std::pair<std::pair<int32_t, int32_t>, std::pair<int32_t, int32_t>>> shapes;  // key -> (rows, cols)
  int max_rows = 0, max_cols = 0;
  bool any_T = false;
  size_t total = 0;
  std::vector<size_t> sparse_rule;  // indices of results that follow the sparse (op) sparse output-format rule

  void add(std::pair<int32_t, int32_t> key, const Block* a, const Block* b, const double* y, int rows, int cols) {
    EwDesc d{};
    d.A = a ? a->values.ptr<double>() : nullptr;
    d.B = b ? b->values.ptr<double>() : nullptr;
    d.Y = y;
    d.rows = rows;
    d.cols = cols;
    d.aT = a ? a->isT : 0;
    d.bT = (b && op != EW_RANK1 && op != EW_RANK1_COMPAT) ? b->isT : 0;
    any_T = any_T || d.aT || d.bT;
    max_rows = std::max(max_rows, rows);
    max_cols = std::max(max_cols, cols);
    total += align_up(static_cast<size_t>(rows) * cols * sizeof(double));
    descs.push_back(d);
    shapes.push_back({key, {rows, cols}});
  }

  void run(mr_matrix* result) {
    if (descs.empty()) return;
    Slab slab(ctx, total);
    for (size_t i = 0; i < descs.size(); ++i) {
      const int rows = shapes[i].second.first, cols = shapes[i].second.second;
      Span s = slab.take(static_cast<size_t>(rows) * cols * sizeof(double));
      descs[i].C = s.ptr<double>();
      result->blocks[shapes[i].first] = dense_block(rows, cols, s, false);  // always column-major (LocalMatrix.scala:62)
    }
    Buf d = upload(ctx, descs);
    CUDA_CHECK(launch_ew_batched(op, static_cast<const EwDesc*>(d->p), static_cast<int>(descs.size()), max_rows,
                                 max_cols, any_T, ctx->stream));
    note_launch(ctx);
    if (!sparse_rule.empty()) apply_sparse_rule(result);
  }

  // LocalMatrix.addSparseSparse / elementWiseOpSparseSparse output format (LocalMatrix.scala:74-139, 521-602): the
  // dense result is converted with toSparse (CSC, isTransposed = false) iff rows*cols > 2*nnz + cols + 1, where nnz
  // counts entries != 0.0 (NaN included).  Both the transposed and the native branch reduce to this rule.
  void apply_sparse_rule(mr_matrix* result) {
    std::vector<DenseWin> wins;
    for (size_t bi : sparse_rule) wins.push_back(DenseWin{descs[bi].C, shapes[bi].second.first, shapes[bi].second.second});
    const auto counts = column_counts(ctx, wins);
    std::vector<DenseWin> chosen;
    std::vector<std::vector<int32_t>> chosen_counts;
    std::vector<std::pair<int32_t, int32_t>> keys;
    for (size_t i = 0; i < wins.size(); ++i) {
      if (static_cast<int64_t>(wins[i].rows) * wins[i].cols > 2 * total_count(counts[i]) + wins[i].cols + 1) {
        chosen.push_back(wins[i]);
        chosen_counts.push_back(counts[i]);
        keys.push_back(shapes[sparse_rule[i]].first);
      }
    }
    std::vector<Block> fresh = compact_csc(ctx, chosen, chosen_counts);
    for (size_t i = 0; i < fresh.size(); ++i) result->blocks[keys[i]] = std::move(fresh[i]);  // replaces the dense window
  }
};

void check_block_dims_add(const Block& a, const Block& b) {
  // LocalMatrix.add (LocalMatrix.scala:36-41)
  MR_REQUIRE(a.numRows == b.numRows, MR_EDIM,
             "Matrix A and B must have the same number of rows. But found A.numRows = %d, B.numRows = %d", a.numRows,
             b.numRows);
  MR_REQUIRE(a.numCols == b.numCols, MR_EDIM,
             "Matrix A and B must have the same number of cols. But found A.numCols = %d, B.numCols = %d", a.numCols,
             b.numCols);
}

void check_block_dims_ew(const Block& a, const Block& b) {
  // LocalMatrix.elementWiseMultiply / Divide (LocalMatrix.scala:467-470, 480-483)
  MR_REQUIRE(a.numRows == b.numRows, MR_EDIM, "mat1.numRows = %d, mat2.numRows = %d", a.numRows, b.numRows);
  MR_REQUIRE(a.numCols == b.numCols, MR_EDIM, "mat1.numCols = %d, mat2.numCols = %d", a.numCols, b.numCols);
}

void elementwise_join(int op, mr_matrix* left, mr_matrix* right, mr_matrix* result) {
  mr_context* ctx = left->ctx;
  EwBatch batch{ctx, op};
  batch.keep.reserve(2 * (left->blocks.size() + right->blocks.size()) + 2);
  auto dense_view = [&](const Block& b) -> const Block* {
    if (b.dense()) return &b;
    batch.keep.push_back(densify(ctx, b));
    return &batch.keep.back();
  };
  for (auto& kv : left->blocks) {
    auto it = right->blocks.find(kv.first);
    if (it == right->blocks.end()) {
      if (op == EW_ADD) result->blocks[kv.first] = kv.second;  // outer join: one-sided blocks pass through
      continue;
    }
    const Block& a = kv.second;
    const Block& b = it->second;
    if (op == EW_ADD) check_block_dims_add(a, b);
    else check_block_dims_ew(a, b);
    const bool both_sparse = !a.dense() && !b.dense();
    const Block* x = dense_view(a);
    const Block* y = dense_view(b);
    // defect B4 (LocalMatrix.scala:474,487): (Sparse, Dense) swaps the operands; visible for divide only
    if (op == EW_DIV && !a.dense() && b.dense() && ctx->compat_bugs) std::swap(x, y);
    batch.add(kv.first, x, y, nullptr, a.numRows, a.numCols);
    if (both_sparse) batch.sparse_rule.push_back(batch.descs.size() - 1);
  }
  if (op == EW_ADD)
    for (auto& kv : right->blocks)
      if (!left->blocks.count(kv.first)) result->blocks[kv.first] = kv.second;
  batch.run(result);
}

void map_values(int op, mr_matrix* a, double alpha, mr_matrix* result) {
  mr_context* ctx = a->ctx;
  std::vector<MapDesc> descs;
  size_t total = 0;
  int64_t max_n = 0;
  for (auto& kv : a->blocks) total += align_up(static_cast<size_t>(kv.second.valuesLen) * sizeof(double));
  Slab slab(ctx, total);
  for (auto& kv : a->blocks) {
    const Block& b = kv.second;
    Block o = b;  // same type, dims, flag and (shared) index arrays: the map touches stored values only
    o.values = slab.take(static_cast<size_t>(b.valuesLen) * sizeof(double));
    if (b.valuesLen > 0) {
      descs.push_back(MapDesc{b.values.ptr<double>(), o.values.ptr<double>(), b.valuesLen});
      max_n = std::max(max_n, b.valuesLen);
    }
    result->blocks[kv.first] = std::move(o);
  }
  if (descs.empty()) return;
  Buf d = upload(ctx, descs);
  CUDA_CHECK(launch_map_batched(op, static_cast<const MapDesc*>(d->p), static_cast<int>(descs.size()), max_n, alpha,
                                ctx->stream));
  note_launch(ctx);
}

}  // namespace

extern "C" {

mr_status mr_transpose(mr_matrix* a, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(a && out, MR_EINVAL, "null argument");
    require_device(a, "mr_transpose");
    std::unique_ptr<mr_matrix> r(new_matrix(a->ctx));
    for (auto& kv : a->blocks) {
      Block b = kv.second;  // shares the device arrays (DenseMatrix.transpose, MLMatrix.scala:312; Sparse :634-635)
      std::swap(b.numRows, b.numCols);
      b.isT = !b.isT;
      r->blocks[{kv.first.second, kv.first.first}] = std::move(b);  // (rid, cid) -> (cid, rid), MatfastExecution.scala:230-231
    }
    *out = r.release();
  });
}

static mr_status ew_operator(int op, mr_matrix* left, int64_t lr, int64_t lc, mr_matrix* right, int64_t rr, int64_t rc,
                             mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(left && right && out, MR_EINVAL, "null argument");
    const char* name = op == EW_ADD ? "mr_add_element" : op == EW_MUL ? "mr_multiply_element" : "mr_divide_element";
    require_device(left, name);
    require_device(right, name);
    MR_REQUIRE(left->ctx == right->ctx, MR_EINVAL, "operands belong to different contexts");
    check_same_dims(lr, lc, rr, rc);
    std::lock_guard<std::mutex> lock(left->ctx->mu);
    wait_ready_all(left->ctx, left);
    wait_ready_all(left->ctx, right);
    std::unique_ptr<mr_matrix> r(new_matrix(left->ctx));
    elementwise_join(op, left, right, r.get());
    *out = r.release();
  });
}

mr_status mr_add_element(mr_matrix* left, int64_t lr, int64_t lc, mr_matrix* right, int64_t rr, int64_t rc,
                         int32_t blkSize, mr_matrix** out) {
  (void)blkSize;
  return ew_operator(EW_ADD, left, lr, lc, right, rr, rc, out);
}
mr_status mr_multiply_element(mr_matrix* left, int64_t lr, int64_t lc, mr_matrix* right, int64_t rr, int64_t rc,
                              int32_t blkSize, mr_matrix** out) {
  (void)blkSize;
  return ew_operator(EW_MUL, left, lr, lc, right, rr, rc, out);
}
mr_status mr_divide_element(mr_matrix* left, int64_t lr, int64_t lc, mr_matrix* right, int64_t rr, int64_t rc,
                            int32_t blkSize, mr_matrix** out) {
  (void)blkSize;
  return ew_operator(EW_DIV, left, lr, lc, right, rr, rc, out);
}

static mr_status map_operator(int op, mr_matrix* a, double alpha, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(a && out, MR_EINVAL, "null argument");
    require_device(a, op == MAP_ADD_SCALAR ? "mr_add_scalar" : op == MAP_MUL_SCALAR ? "mr_multiply_scalar" : "mr_power");
    std::lock_guard<std::mutex> lock(a->ctx->mu);
    wait_ready_all(a->ctx, a);
    std::unique_ptr<mr_matrix> r(new_matrix(a->ctx));
    map_values(op, a, alpha, r.get());
    *out = r.release();
  });
}
mr_status mr_add_scalar(mr_matrix* a, double alpha, mr_matrix** out) { return map_operator(MAP_ADD_SCALAR, a, alpha, out); }
mr_status mr_multiply_scalar(mr_matrix* a, double alpha, mr_matrix** out) { return map_operator(MAP_MUL_SCALAR, a, alpha, out); }
mr_status mr_power(mr_matrix* a, double alpha, mr_matrix** out) { return map_operator(MAP_POW, a, alpha, out); }

mr_status mr_rank_one_update(mr_matrix* left, int64_t lr, int64_t lc, mr_matrix* right, int64_t rr, int64_t rc,
                             int32_t blkSize, mr_matrix** out) {
  (void)blkSize;
  return guarded([&] {
    MR_REQUIRE(left && right && out, MR_EINVAL, "null argument");
    require_device(left, "mr_rank_one_update");
    require_device(right, "mr_rank_one_update");
    MR_REQUIRE(left->ctx == right->ctx, MR_EINVAL, "operands belong to different contexts");
    mr_context* ctx = left->ctx;
    if (ctx->compat_bugs) {
      // the reference's own `require`s (MatfastExecution.scala:741-744), which only admit 1-row matrices
      MR_REQUIRE(rr == 1, MR_EDIM, "Vector column size is not 1, but #cols = %lld", (long long)rr);
      MR_REQUIRE(lr == rr, MR_EDIM,
                 "Dimension not match for matrix addition, A.nrows = %lld, A.ncols = %lld, B.nrows = %lld, B.ncols = %lld",
                 (long long)lr, (long long)lc, (long long)rr, (long long)rc);
    } else {
      // intended semantics: A (n x n) + v v^T with v an n x 1 block column (MatrixOperator.scala:151-152)
      MR_REQUIRE(rc == 1, MR_EDIM, "Vector column size is not 1, but #cols = %lld", (long long)rc);
      MR_REQUIRE(lr == rr && lc == rr, MR_EDIM,
                 "Dimension not match for matrix addition, A.nrows = %lld, A.ncols = %lld, B.nrows = %lld, B.ncols = %lld",
                 (long long)lr, (long long)lc, (long long)rr, (long long)rc);
    }
    std::lock_guard<std::mutex> lock(ctx->mu);
    wait_ready_all(ctx, left);
    wait_ready_all(ctx, right);
    std::unique_ptr<mr_matrix> r(new_matrix(ctx));
    EwBatch batch{ctx, ctx->compat_bugs ? EW_RANK1_COMPAT : EW_RANK1};
    batch.keep.reserve(left->blocks.size() + 2 * right->blocks.size() + 2);
    std::map<const Block*, const Block*> dense_cache;
    auto dense_view = [&](const Block& b) -> const Block* {
      if (b.dense()) return &b;
      auto it = dense_cache.find(&b);
      if (it != dense_cache.end()) return it->second;
      batch.keep.push_back(densify(ctx, b));
      return dense_cache[&b] = &batch.keep.back();
    };
    for (auto& kv : left->blocks) {
      const int32_t i = kv.first.first, j = kv.first.second;
      const Block& a = kv.second;
      // helper :271-275: x2.rid == i, x3.rid == j (vector blocks are looked up by their row-block id)
      const Block *x = nullptr, *y = nullptr;
      for (auto& vb : right->blocks) {
        if (vb.first.first == i) x = &vb.second;
        if (vb.first.first == j) y = &vb.second;
      }
      if (!x || !y) continue;
      MR_REQUIRE(static_cast<int64_t>(x->numRows) * x->numCols >= a.numRows &&
                     static_cast<int64_t>(y->numRows) * y->numCols >= a.numCols,
                 MR_EDIM, "vector block shorter than matrix block (%d x %d)", a.numRows, a.numCols);
      if (ctx->compat_bugs && !a.dense())
        fail(MR_ENOTSUP, "rankOneAdd on a sparse block in compat mode (LocalMatrix.scala:1079-1081 indexes the "
                         "dense result with the sparse value index) is not reproduced");
      const Block* xd = dense_view(*x);
      const Block* yd = dense_view(*y);
      const Block* ad = ctx->compat_bugs ? &a : dense_view(a);
      // mat2(i, 0) of an n x 1 (or, transposed, 1 x n flagged) dense block is values[i] either way
      batch.add(kv.first, ad, xd, yd->values.ptr<double>(), a.numRows, a.numCols);
    }
    batch.run(r.get());
    *out = r.release();
  });
}


mr_status mr_materialize(mr_matrix* a, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(a && out, MR_EINVAL, "null argument");
    require_device(a, "mr_materialize");
    mr_context* ctx = a->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    wait_ready_all(ctx, a);
    std::unique_ptr<mr_matrix> r(new_matrix(ctx));
    EwBatch batch{ctx, EW_COPY};
    for (auto& kv : a->blocks) {
      const Block& b = kv.second;
      if (!b.dense()) {
        r->blocks[kv.first] = densify(ctx, b);
      } else if (!b.isT) {
        r->blocks[kv.first] = b;  // already canonical: share
      } else {
        batch.add(kv.first, &b, nullptr, nullptr, b.numRows, b.numCols);
      }
    }
    batch.run(r.get());
    *out = r.release();
  });
}


}  // extern "C"
