// Aggregates (rowSum / colSum / sum / trace), slicing (project / selection) and vec.
#include "host.h"

using namespace matrel;
using namespace mrhost;

extern "C" {

static mr_status aggregate_operator(int op, mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(a && out, MR_EINVAL, "null argument");
    require_device(a, op == AGG_ROW_SUM ? "mr_row_sum" : op == AGG_COL_SUM ? "mr_col_sum" : op == AGG_SUM ? "mr_sum" : "mr_trace");
    if (op == AGG_TRACE)  // Dataset.scala:80
      MR_REQUIRE(nrows == ncols, MR_EDIM, "Cannot perform trace() on a rectangle matrix");
    mr_context* ctx = a->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    wait_ready_all(ctx, a);
    std::unique_ptr<mr_matrix> r(new_matrix(ctx));
    // output blocks: one per block-row (rowSum), block-column (colSum), or a single scalar
    std::map<std::pair<int32_t, int32_t>, int32_t> out_len;
    for (auto& kv : a->blocks) {
      const Block& b = kv.second;
      if (op == AGG_TRACE && kv.first.first != kv.first.second) continue;
      if (op == AGG_TRACE && b.dense())  // MatfastExecution.scala:428
        MR_REQUIRE(b.numRows == b.numCols, MR_EDIM, "block is not square, row_num=%d, col_num=%d", b.numRows, b.numCols);
      std::pair<int32_t, int32_t> key = op == AGG_ROW_SUM ? std::make_pair(kv.first.first, 0)
                                        : op == AGG_COL_SUM ? std::make_pair(0, kv.first.second)
                                                            : std::make_pair(0, 0);
      const int32_t len = op == AGG_ROW_SUM ? b.numRows : op == AGG_COL_SUM ? b.numCols : 1;
      auto it = out_len.find(key);
      if (it == out_len.end()) out_len[key] = len;
      else if (op == AGG_ROW_SUM)  // LocalMatrix.add requires of the reduceByKey (LocalMatrix.scala:36-41)
        MR_REQUIRE(it->second == len, MR_EDIM,
                   "Matrix A and B must have the same number of rows. But found A.numRows = %d, B.numRows = %d", it->second, len);
      else if (op == AGG_COL_SUM)
        MR_REQUIRE(it->second == len, MR_EDIM,
                   "Matrix A and B must have the same number of cols. But found A.numCols = %d, B.numCols = %d", it->second, len);
    }
    if (out_len.empty()) {
      *out = r.release();
      return;
    }
    size_t total = 0;
    for (auto& kv : out_len) total += align_up(static_cast<size_t>(kv.second) * sizeof(double));
    Slab slab(ctx, total);
    CUDA_CHECK(cudaMemsetAsync(slab.buf->p, 0, std::max<size_t>(total, kAlign), ctx->stream));
    std::map<std::pair<int32_t, int32_t>, double*> out_ptr;
    for (auto& kv : out_len) {
      Span s = slab.take(static_cast<size_t>(kv.second) * sizeof(double));
      out_ptr[kv.first] = s.ptr<double>();
      r->blocks[kv.first] = op == AGG_ROW_SUM ? dense_block(kv.second, 1, s) : op == AGG_COL_SUM ? dense_block(1, kv.second, s)
                                                                                                  : dense_block(1, 1, s);
    }
    // dense blocks: one batched launch that adds into the zeroed outputs; sparse blocks (not for sum, which adds the stored
    // values of both kinds): per-block partials on their stored entries, combined per output in ascending block index
    std::vector<AggDesc> descs;
    std::set<std::pair<int32_t, int32_t>> has_dense;
    std::map<std::pair<int32_t, int32_t>, std::vector<const Block*>> sparse_of;
    if (op != AGG_SUM) {
      ctx->stats.agg_sparse_blocks = 0;
      ctx->stats.agg_sparse_entries = 0;
    }
    int max_r = 1, max_c = 1;
    for (auto& kv : a->blocks) {
      const Block& b = kv.second;
      if (op == AGG_TRACE && kv.first.first != kv.first.second) continue;
      const std::pair<int32_t, int32_t> key = op == AGG_ROW_SUM ? std::make_pair(kv.first.first, 0)
                                              : op == AGG_COL_SUM ? std::make_pair(0, kv.first.second)
                                                                  : std::make_pair(0, 0);
      AggDesc d{};
      if (op == AGG_SUM) {  // values.sum over the STORED values, dense or sparse (:381-384)
        // a dense block may hold 2^31 values or more, so it is described by its shape; a sparse block's int32 colPtrs bound its
        // valuesLen by INT32_MAX
        d.v = b.values.ptr<double>();
        d.rows = b.dense() ? b.numRows : static_cast<int32_t>(b.valuesLen);
        d.cols = b.dense() ? b.numCols : 1;
        d.isT = 0;
        if (b.valuesLen == 0) continue;
      } else if (!b.dense()) {
        ctx->stats.agg_sparse_blocks += 1;
        ctx->stats.agg_sparse_entries += b.valuesLen;
        if (b.valuesLen > 0) sparse_of[key].push_back(&b);  // an empty block adds nothing to its zeroed output
        continue;
      } else {
        d.v = b.values.ptr<double>();
        d.rows = b.numRows;
        d.cols = b.numCols;
        d.isT = b.isT;
      }
      d.out = out_ptr[key];
      has_dense.insert(key);
      max_r = std::max(max_r, d.rows);
      max_c = std::max(max_c, d.cols);
      descs.push_back(d);
    }
    if (!descs.empty()) {
      Buf dd = upload(ctx, descs);
      CUDA_CHECK(launch_aggregate(op, static_cast<const AggDesc*>(dd->p), static_cast<int>(descs.size()), max_r, max_c, ctx->stream));
      note_launch(ctx);
    }
    if (!sparse_of.empty()) {
      size_t bytes = 0;
      for (auto& kv : sparse_of) bytes += align_up(kv.second.size() * static_cast<size_t>(out_len[kv.first]) * sizeof(double));
      Slab scratch(ctx, bytes);  // the partials, nparts x len per output
      std::vector<SpAggDesc> sd;
      std::vector<SpAggOut> so;
      int max_lines = 1, max_across = 0, max_len = 1;
      for (auto& kv : sparse_of) {
        const int32_t len = out_len[kv.first];
        const std::vector<const Block*>& parts = kv.second;
        Span sp = scratch.take(parts.size() * static_cast<size_t>(len) * sizeof(double));
        so.push_back(SpAggOut{out_ptr[kv.first], sp.ptr<double>(), len, static_cast<int32_t>(parts.size()),
                              has_dense.count(kv.first) ? 1 : 0, 0});
        max_len = std::max(max_len, len);
        for (size_t i = 0; i < parts.size(); ++i) {
          const Block& b = *parts[i];
          SpAggDesc d{};
          d.ptr = b.colPtrs.ptr<int32_t>();
          d.idx = b.rowIndices.ptr<int32_t>();
          d.val = b.values.ptr<double>();
          d.part = sp.ptr<double>() + i * static_cast<size_t>(len);
          d.nlines = b.isT ? b.numRows : b.numCols;
          d.len = len;
          d.mode = op == AGG_TRACE ? SPAGG_DIAG : (op == AGG_ROW_SUM) == b.isT ? SPAGG_ALONG : SPAGG_ACROSS;
          if (d.mode == SPAGG_ACROSS) max_across = std::max(max_across, len);
          max_lines = std::max(max_lines, d.nlines);
          sd.push_back(d);
        }
      }
      Buf d_sd = upload(ctx, sd), d_so = upload(ctx, so);
      CUDA_CHECK(launch_sparse_agg(static_cast<const SpAggDesc*>(d_sd->p), static_cast<int>(sd.size()), max_lines, max_across,
                                   ctx->stream));
      note_launch(ctx);
      CUDA_CHECK(launch_sparse_agg_combine(static_cast<const SpAggOut*>(d_so->p), static_cast<int>(so.size()), max_len, ctx->stream));
      note_launch(ctx);
    }
    *out = r.release();
  });
}
mr_status mr_row_sum(mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out) { return aggregate_operator(AGG_ROW_SUM, a, nrows, ncols, out); }
mr_status mr_col_sum(mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out) { return aggregate_operator(AGG_COL_SUM, a, nrows, ncols, out); }
mr_status mr_sum(mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out) { return aggregate_operator(AGG_SUM, a, nrows, ncols, out); }
mr_status mr_trace(mr_matrix* a, int64_t nrows, int64_t ncols, mr_matrix** out) { return aggregate_operator(AGG_TRACE, a, nrows, ncols, out); }

static mr_status slice_operator(mr_matrix* a, int32_t blkSize, bool take_row, int64_t index, int64_t index2, mr_matrix** out) {
  return guarded([&] {
    require_device(a, index2 >= 0 ? "mr_selection" : "mr_project");
    MR_REQUIRE(blkSize > 0, MR_EINVAL, "blkSize must be positive, got %d", blkSize);
    mr_context* ctx = a->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    wait_ready_all(ctx, a);
    std::unique_ptr<mr_matrix> r(new_matrix(ctx));
    const int32_t blkid = static_cast<int32_t>(index / blkSize), offset = static_cast<int32_t>(index % blkSize);  // :40-41
    const int32_t blkid2 = index2 >= 0 ? static_cast<int32_t>(index2 / blkSize) : -1;
    const int32_t offset2 = index2 >= 0 ? static_cast<int32_t>(index2 % blkSize) : -1;
    ctx->stats.agg_sparse_blocks = 0;
    ctx->stats.agg_sparse_entries = 0;
    std::vector<LineDesc> descs;      // dense blocks
    std::vector<SpSliceDesc> sdescs;  // sparse blocks, on their stored entries
    struct Out {
      std::pair<int32_t, int32_t> key;
      int32_t rows, cols;
      bool sparse;
      size_t at;  // index into descs / sdescs
    };
    std::vector<Out> outs;
    size_t total = 0;
    int max_len = 1, max_slen = 1;
    for (auto& kv : a->blocks) {
      const int32_t rid = kv.first.first, cid = kv.first.second;
      if ((take_row ? rid : cid) != blkid) continue;                       // filter(tuple => tuple._1 == rowblkID), :48
      if (index2 >= 0 && (take_row ? cid : rid) != blkid2) continue;
      const Block& b = kv.second;
      if (offset >= (take_row ? b.numRows : b.numCols)) continue;
      if (index2 >= 0 && offset2 >= (take_row ? b.numCols : b.numRows)) continue;
      const int32_t len = index2 >= 0 ? 1 : (take_row ? b.numCols : b.numRows);
      Out o{index2 >= 0 ? std::make_pair(0, 0) : take_row ? std::make_pair(0, cid) : std::make_pair(rid, 0),
            index2 >= 0 ? 1 : take_row ? 1 : len, index2 >= 0 ? 1 : take_row ? len : 1, !b.dense(), 0};
      if (b.dense()) {
        LineDesc d{};
        d.v = b.values.ptr<double>();
        d.rows = b.numRows;
        d.cols = b.numCols;
        d.offset = offset;
        d.offset2 = offset2;
        d.len = len;
        d.isT = b.isT;
        d.take_row = take_row;
        o.at = descs.size();
        descs.push_back(d);
        max_len = std::max(max_len, len);
      } else {
        // the block's lines are its columns (CSC) or rows (CSR): a row of a CSR block or a column of a CSC one is one line; the
        // other way, and an entry, are one index searched in each of the lines
        SpSliceDesc d{};
        d.ptr = b.colPtrs.ptr<int32_t>();
        d.idx = b.rowIndices.ptr<int32_t>();
        d.val = b.values.ptr<double>();
        d.len = len;
        if (index2 >= 0) {
          d.line = b.isT ? offset : offset2;
          d.target = b.isT ? offset2 : offset;
        } else if (take_row == b.isT) {
          d.line = offset;
          d.target = -1;
        } else {
          d.line = 0;
          d.target = offset;
        }
        o.at = sdescs.size();
        sdescs.push_back(d);
        max_slen = std::max(max_slen, len);
        ctx->stats.agg_sparse_blocks += 1;
        ctx->stats.agg_sparse_entries += b.valuesLen;
      }
      outs.push_back(o);
      total += align_up(static_cast<size_t>(len) * sizeof(double));
    }
    if (!outs.empty()) {
      Slab slab(ctx, total);
      for (const Out& o : outs) {
        Span sp = slab.take(static_cast<size_t>(o.rows) * o.cols * sizeof(double));
        if (o.sparse) sdescs[o.at].out = sp.ptr<double>();
        else descs[o.at].out = sp.ptr<double>();
        r->blocks[o.key] = dense_block(o.rows, o.cols, sp);
      }
    }
    if (!descs.empty()) {
      Buf dd = upload(ctx, descs);
      CUDA_CHECK(launch_extract_lines(static_cast<const LineDesc*>(dd->p), static_cast<int>(descs.size()), max_len, ctx->stream));
      note_launch(ctx);
    }
    if (!sdescs.empty()) {
      Buf dd = upload(ctx, sdescs);
      CUDA_CHECK(launch_sparse_slice(static_cast<const SpSliceDesc*>(dd->p), static_cast<int>(sdescs.size()), max_slen, ctx->stream));
      note_launch(ctx);
    }
    *out = r.release();
  });
}

mr_status mr_project(mr_matrix* a, int64_t nrows, int64_t ncols, int32_t blkSize, int32_t rowOrCol, int64_t index, mr_matrix** out) {
  mr_status st = guarded([&] {
    MR_REQUIRE(a && out, MR_EINVAL, "null argument");
    if (rowOrCol)  // Dataset.scala:42,44
      MR_REQUIRE(index >= 0 && index < nrows, MR_EINVAL, "row index should be smaller than #rows, index=%lld, #rows=%lld",
                 (long long)index, (long long)nrows);
    else
      MR_REQUIRE(index >= 0 && index < ncols, MR_EINVAL, "col index should be smaller than #cols, index=%lld, #cols=%lld",
                 (long long)index, (long long)ncols);
  });
  if (st != MR_OK) return st;
  return slice_operator(a, blkSize, rowOrCol != 0, index, -1, out);
}

mr_status mr_selection(mr_matrix* a, int64_t nrows, int64_t ncols, int32_t blkSize, int64_t rowIdx, int64_t colIdx, mr_matrix** out) {
  mr_status st = guarded([&] {
    MR_REQUIRE(a && out, MR_EINVAL, "null argument");
    // Dataset.scala:52-53
    MR_REQUIRE(rowIdx >= 0 && rowIdx < nrows, MR_EINVAL, "row index should be smaller than #rows, rid=%lld, #rows=%lld",
               (long long)rowIdx, (long long)nrows);
    MR_REQUIRE(colIdx >= 0 && colIdx < ncols, MR_EINVAL, "col index should be smaller than #cols, cid=%lld, #cols=%lld",
               (long long)colIdx, (long long)ncols);
  });
  if (st != MR_OK) return st;
  return slice_operator(a, blkSize, true, rowIdx, colIdx, out);
}

mr_status mr_vec(mr_matrix* a, int64_t nrows, int64_t ncols, int32_t blkSize, mr_matrix** out) {
  (void)ncols;
  mr_matrix* canon = nullptr;
  mr_status st = guarded([&] {
    MR_REQUIRE(a && out, MR_EINVAL, "null argument");
    MR_REQUIRE(blkSize > 0 && nrows > 0, MR_EINVAL, "nrows and blkSize must be positive");
    require_device(a, "mr_vec");
  });
  if (st != MR_OK) return st;
  st = mr_materialize(a, &canon);  // column-major, non-transposed dense blocks (shares already canonical ones)
  if (st != MR_OK) return st;
  st = guarded([&] {
    mr_context* ctx = a->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    std::unique_ptr<mr_matrix> r(new_matrix(ctx));
    const int64_t ROW_BLK_NUM = ceil_div(nrows, blkSize);  // MatfastExecution.scala:543
    for (auto& kv : canon->blocks) {
      const Block& b = kv.second;
      const int64_t i = kv.first.first, j = kv.first.second;
      for (int32_t t = 0; t < b.numCols; ++t) {
        const int64_t key = (j * blkSize + t) * ROW_BLK_NUM + i;  // :552 with the block-column offset in elements
        MR_REQUIRE(key <= INT32_MAX, MR_EINVAL, "vec(): block id %lld does not fit an Int", (long long)key);
        Span col{b.values.buf, b.values.off + static_cast<size_t>(t) * b.numRows * sizeof(double)};
        Block v = dense_block(b.numRows, 1, col, false);
        v.ready = b.ready;
        r->blocks[{static_cast<int32_t>(key), 0}] = std::move(v);
      }
    }
    *out = r.release();
  });
  mr_matrix_free(canon);
  return st;
}


}  // extern "C"
