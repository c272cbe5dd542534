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
  std::vector<Block> keep;  // densified temporaries (rank-one update)
  std::vector<std::pair<std::pair<int32_t, int32_t>, std::pair<int32_t, int32_t>>> shapes;  // key -> (rows, cols)
  int max_rows = 0, max_cols = 0;
  bool any_T = false;
  size_t total = 0;

  // a or b may be null: an absent operand (0.0 everywhere) of EW_ADD / EW_MUL / EW_DIV
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
  }
};

// ------------------------------------------------------------------------------------------------
// sparse (+) sparse on the stored entries (sparse_ew.cu, DESIGN section 4.5.3): a count pass over every pair of the call, one
// host synchronisation for the per-pair totals, the reference's output rule, exactly sized results from one slab, a fill pass.
// ------------------------------------------------------------------------------------------------
struct SparsePair {
  std::pair<int32_t, int32_t> key;
  const Block* a;
  const Block* b;
};

void sparse_sparse_join(mr_context* ctx, int op, const std::vector<SparsePair>& jobs, mr_matrix* result) {
  if (jobs.empty()) return;
  const size_t np = jobs.size();
  // ---- CSR operands through sptrans, once per block
  std::map<const Block*, size_t> conv;  // block -> offset of its CSC copy in the scratch
  size_t conv_bytes = 0;
  for (auto& j : jobs)
    for (const Block* b : {j.a, j.b})
      if (b->isT && !conv.count(b)) {
        conv.emplace(b, conv_bytes);
        conv_bytes += CscLayout(b->numCols, b->valuesLen).bytes;
      }
  Buf cbuf;
  if (!conv.empty()) {
    cbuf = std::make_shared<DevBuf>(ctx, conv_bytes);
    std::vector<CsrToCsc> cv;
    for (auto& kv : conv) {
      const Block* b = kv.first;
      cv.push_back(CsrToCsc{b->colPtrs.ptr<int32_t>(), b->rowIndices.ptr<int32_t>(), b->values.ptr<double>(), b->numRows, b->numCols,
                            b->valuesLen, static_cast<char*>(cbuf->p) + kv.second});
    }
    csr_to_csc(ctx, cv);
  }
  // ---- the pairs in the CSC frame
  size_t col_total = 0;
  for (auto& j : jobs) col_total += static_cast<size_t>(j.a->numCols);
  const size_t tot_off = 0, cnt_off = align_up(np * sizeof(unsigned long long));
  Buf meta = std::make_shared<DevBuf>(ctx, cnt_off + std::max<size_t>(col_total, 1) * sizeof(int32_t));
  CUDA_CHECK(cudaMemsetAsync(meta->p, 0, cnt_off, ctx->stream));
  auto* d_total = reinterpret_cast<unsigned long long*>(static_cast<char*>(meta->p) + tot_off);
  int32_t* d_colcnt = reinterpret_cast<int32_t*>(static_cast<char*>(meta->p) + cnt_off);
  std::vector<SpEwPair> pairs(np);
  int max_rows = 0, max_cols = 0;
  size_t coff = 0;
  for (size_t i = 0; i < np; ++i) {
    const Block* a = jobs[i].a;
    const Block* b = jobs[i].b;
    const bool native = !a->isT && !b->isT;
    SpEwPair& q = pairs[i];
    auto csc_of = [&](const Block* x, const int32_t*& p, const int32_t*& ix, const double*& v, uint8_t& mode) {
      if (x->isT) {
        const char* w = static_cast<const char*>(cbuf->p) + conv.at(x);
        const CscLayout L(x->numCols, x->valuesLen);
        p = reinterpret_cast<const int32_t*>(w + L.ptr);
        ix = reinterpret_cast<const int32_t*>(w + L.idx);
        v = reinterpret_cast<const double*>(w + L.val);
        mode = SPEW_FIRST;
      } else {
        p = x->colPtrs.ptr<int32_t>();
        ix = x->rowIndices.ptr<int32_t>();
        v = x->values.ptr<double>();
        mode = native ? SPEW_SUM : SPEW_LAST;
      }
    };
    csc_of(a, q.ap, q.ai, q.av, q.amode);
    csc_of(b, q.bp, q.bi, q.bv, q.bmode);
    q.rows = a->numRows;
    q.cols = a->numCols;
    q.native = native ? 1 : 0;
    q.colcnt = d_colcnt + coff;
    q.total = d_total + i;
    coff += static_cast<size_t>(q.cols);
    max_rows = std::max(max_rows, q.rows);
    max_cols = std::max(max_cols, q.cols);
    ctx->stats.ew_sparse_pairs += 1;
    ctx->stats.ew_sparse_entries += a->valuesLen + b->valuesLen;
  }
  // ---- count pass, the per-pair totals
  const SpEwLaunchShape shape = sparse_ew_shape(max_rows);
  Buf scratch = shape.scratch_bytes ? std::make_shared<DevBuf>(ctx, shape.scratch_bytes) : nullptr;
  Buf d_pairs = upload(ctx, pairs);
  CUDA_CHECK(launch_sparse_ew(op, false, static_cast<const SpEwPair*>(d_pairs->p), static_cast<int>(np), max_rows, max_cols,
                              scratch ? scratch->p : nullptr, shape, ctx->stream));
  note_launch(ctx);
  std::vector<unsigned long long> nnz(np);
  CUDA_CHECK(cudaMemcpyAsync(nnz.data(), d_total, np * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  ctx->stats.d2h_bytes += static_cast<int64_t>(np * sizeof(unsigned long long));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  // ---- the reference's output rule (LocalMatrix.scala:82-88, :131-138): CSC (isTransposed = false) iff rows * cols > 2 nnz + cols + 1
  std::vector<bool> sparse_out(np);
  size_t bytes = 0;
  for (size_t i = 0; i < np; ++i) {
    const SpEwPair& q = pairs[i];
    sparse_out[i] = static_cast<int64_t>(q.rows) * q.cols > 2 * static_cast<int64_t>(nnz[i]) + q.cols + 1;
    if (sparse_out[i])
      bytes += align_up((static_cast<size_t>(q.cols) + 1) * sizeof(int32_t)) + align_up(nnz[i] * sizeof(int32_t)) +
               align_up(nnz[i] * sizeof(double));
    else
      bytes += align_up(static_cast<size_t>(q.rows) * q.cols * sizeof(double));
  }
  Slab slab(ctx, bytes);
  std::vector<ScanDesc> scans;
  for (size_t i = 0; i < np; ++i) {
    SpEwPair& q = pairs[i];
    Block& out = result->blocks[jobs[i].key];
    if (!sparse_out[i]) {
      Span s = slab.take(static_cast<size_t>(q.rows) * q.cols * sizeof(double));
      q.dense = s.ptr<double>();
      out = dense_block(q.rows, q.cols, s, false);
      continue;
    }
    Span ptr = slab.take((static_cast<size_t>(q.cols) + 1) * sizeof(int32_t)), idx = slab.take(nnz[i] * sizeof(int32_t)),
         val = slab.take(nnz[i] * sizeof(double));
    q.optr = ptr.ptr<int32_t>();
    q.oidx = idx.ptr<int32_t>();
    q.oval = val.ptr<double>();
    scans.push_back(ScanDesc{q.colcnt, ptr.ptr<int32_t>(), q.cols, 0});
    Block b;
    b.type = 0;
    b.numRows = q.rows;
    b.numCols = q.cols;
    b.isT = false;
    b.valuesLen = static_cast<int64_t>(nnz[i]);
    b.colPtrsLen = q.cols + 1;
    b.colPtrs = ptr;
    b.rowIndices = idx;
    b.values = val;
    out = std::move(b);
  }
  // ---- fill pass
  if (!scans.empty()) {
    Buf d_scans = upload(ctx, scans);
    CUDA_CHECK(launch_exclusive_scan(static_cast<const ScanDesc*>(d_scans->p), static_cast<int>(scans.size()), ctx->stream));
    note_launch(ctx);
  }
  Buf d_pairs2 = upload(ctx, pairs);
  CUDA_CHECK(launch_sparse_ew(op, true, static_cast<const SpEwPair*>(d_pairs2->p), static_cast<int>(np), max_rows, max_cols,
                              scratch ? scratch->p : nullptr, shape, ctx->stream));
  note_launch(ctx);
}

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
  ctx->stats.ew_sparse_pairs = 0;
  ctx->stats.ew_sparse_entries = 0;
  EwBatch batch{ctx, op};           // dense (+) dense, and the unstored positions of dense (+) sparse
  std::vector<DsEwDesc> scatter;    // dense (+) sparse: the stored positions, after the batch (its index in batch.descs in .C)
  std::vector<size_t> scatter_at;
  std::vector<SparsePair> spsp;     // sparse (+) sparse
  int max_lines = 0;
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
    if (!a.dense() && !b.dense()) {
      spsp.push_back(SparsePair{kv.first, &a, &b});
      continue;
    }
    if (a.dense() && b.dense()) {
      batch.add(kv.first, &a, &b, nullptr, a.numRows, a.numCols);
      continue;
    }
    // dense (+) sparse: op(x, y) with the sparse operand absent from the batch; defect B4 (LocalMatrix.scala:474,487): (Sparse,
    // Dense) swaps the operands, visible for divide only
    const Block& s = a.dense() ? b : a;
    const Block& d = a.dense() ? a : b;
    const bool sparse_left = !a.dense() && !(op == EW_DIV && ctx->compat_bugs);
    if (sparse_left) batch.add(kv.first, nullptr, &d, nullptr, a.numRows, a.numCols);
    else batch.add(kv.first, &d, nullptr, nullptr, a.numRows, a.numCols);
    ctx->stats.ew_sparse_pairs += 1;
    ctx->stats.ew_sparse_entries += s.valuesLen;
    if (s.valuesLen == 0) continue;
    DsEwDesc e{};
    e.ptr = s.colPtrs.ptr<int32_t>();
    e.idx = s.rowIndices.ptr<int32_t>();
    e.val = s.values.ptr<double>();
    e.D = d.values.ptr<double>();
    e.rows = a.numRows;
    e.cols = a.numCols;
    e.sT = s.isT ? 1 : 0;
    e.dT = d.isT ? 1 : 0;
    e.sparse_left = sparse_left ? 1 : 0;
    scatter.push_back(e);
    scatter_at.push_back(batch.descs.size() - 1);
    max_lines = std::max(max_lines, s.isT ? s.numRows : s.numCols);
  }
  if (op == EW_ADD)
    for (auto& kv : right->blocks)
      if (!left->blocks.count(kv.first)) result->blocks[kv.first] = kv.second;
  batch.run(result);
  if (!scatter.empty()) {
    for (size_t i = 0; i < scatter.size(); ++i) scatter[i].C = batch.descs[scatter_at[i]].C;
    Buf d = upload(ctx, scatter);
    CUDA_CHECK(launch_sparse_ew_scatter(op, static_cast<const DsEwDesc*>(d->p), static_cast<int>(scatter.size()), max_lines, ctx->stream));
    note_launch(ctx);
  }
  sparse_sparse_join(ctx, op, spsp, result);
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
