// The streamed multiply: C = A B when A, B or both are host-resident (mr_matrix_create_host / mr_matrix_to_host), for products
// whose operands and result do not fit on the device together.  C is cut into tiles (a run of block rows x a run of block
// columns); every tile is one multiply_impl call over device copies of the panels it reads, with the output written into one of
// two device C-tile buffers and copied back into the host-resident result while the next tile computes.
//
//   outer loop: panels of the outer operand (B(:, J) or A(I, :), whichever makes fewer host -> device bytes), uploaded once;
//   inner loop: panels of the other operand, uploaded into one of two buffers so that the next is on the wire while a tile
//               computes.  Every uploaded block has its own event and ingest number: the chunked launch of multiply_impl starts
//               on the first pieces of a panel.
// A buffer is only rewritten after an event recorded behind everything that reads it; there is no host synchronisation in the
// loop.  The whole product's engine and kernel-variant choices are taken once (multiply_decisions) and handed to every tile, so
// a streamed C is bit-identical to the resident one (DESIGN.md section 4.6).
#include "host.h"

using namespace matrel;
using namespace mrhost;

namespace mrhost {

size_t stream_budget(mr_context* ctx, size_t enough) {
  if (ctx->stream_budget_mb > 0) return static_cast<size_t>(ctx->stream_budget_mb) << 20;
  size_t free_b = 0, total_b = 0;
  if (enough != SIZE_MAX) {  // the pool's cache stays when the memory free without it is enough
    CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    if (free_b > (1ull << 30) && free_b - (1ull << 30) >= enough) return free_b - (1ull << 30);
  }
  // free memory at the call, with what this device's pool caches handed back first, minus 1 GiB of headroom
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
  (void)cudaGetLastError();
  CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
  return free_b > (1ull << 30) ? free_b - (1ull << 30) : 0;
}

// The tiling rule.  Inputs: nr block rows of A and nc block columns of B take part; a_row / b_col = device bytes of the largest
// block row of A / block column of B when that operand is host-resident (0 when it is used in place); a_bytes / b_bytes = its
// host -> device payload (0 in place); c_block = device bytes of the largest output block; scratch(tr, tc) = what a tr x tc tile
// call allocates besides: the Ozaki-II residue scratch, and with sparse operands the dense images of sparse blocks, the row-major
// copies of dense right blocks and the re-packed CSR segments of the sparse x dense kernels.  A tile of tr x tc blocks with B
// outer needs
//     2 tr a_row + tc b_col + 2 tr tc c_block + scratch(tr, tc)
// (A outer: tr a_row + 2 tc b_col + ...) and moves |B| + ceil(nc / tc) |A| (A outer: |A| + ceil(nr / tr) |B|) to the device.
// Among the tiles that fit the budget the rule takes the fewest host -> device bytes, then the fewest tiles.
struct StreamTiling {
  bool ok = false;
  int64_t tr = 0, tc = 0;
  bool outer_b = true;       // B(:, J) is the outer panel
  int64_t h2d_bytes = 0;
  int64_t tiles = 0;
  size_t device_bytes = 0;   // of the chosen tile; when !ok, of the smallest one
};

StreamTiling choose_tiling(int64_t nr, int64_t nc, size_t a_row, size_t b_col, int64_t a_bytes, int64_t b_bytes, size_t c_block,
                           size_t budget, const std::function<size_t(int64_t, int64_t)>& scratch) {
  StreamTiling best;
  best.device_bytes = SIZE_MAX;
  auto sizes = [](int64_t n) {  // one tile extent per distinct panel count
    std::vector<int64_t> v;
    for (int64_t p = 1; p <= n; ++p) {
      const int64_t t = ceil_div(n, p);
      if (v.empty() || v.back() != t) v.push_back(t);
    }
    return v;
  };
  for (int64_t tr : sizes(nr))
    for (int64_t tc : sizes(nc)) {
      const size_t common = 2 * static_cast<size_t>(tr) * tc * c_block + scratch(tr, tc);
      for (bool outer_b : {true, false}) {
        const size_t dev = common + (outer_b ? 2 * tr * a_row + tc * b_col : tr * a_row + 2 * tc * b_col);
        const int64_t bytes = outer_b ? b_bytes + ceil_div(nc, tc) * a_bytes : a_bytes + ceil_div(nr, tr) * b_bytes;
        const int64_t tiles = ceil_div(nr, tr) * ceil_div(nc, tc);
        if (dev > budget) {
          if (!best.ok && dev < best.device_bytes) best.device_bytes = dev;
          continue;
        }
        if (!best.ok || bytes < best.h2d_bytes || (bytes == best.h2d_bytes && tiles < best.tiles)) {
          best.ok = true;
          best.tr = tr;
          best.tc = tc;
          best.outer_b = outer_b;
          best.h2d_bytes = bytes;
          best.tiles = tiles;
          best.device_bytes = dev;
        }
      }
    }
  return best;
}

namespace {

size_t footprint(const Block& b) {  // device bytes of a block staged into a panel buffer
  size_t n = align_up(static_cast<size_t>(b.valuesLen) * sizeof(double));
  if (!b.dense()) n += align_up(static_cast<size_t>(b.colPtrsLen) * 4) + align_up(static_cast<size_t>(b.valuesLen) * 4);
  return n;
}
int64_t payload(const Block& b) {  // bytes of a block's arrays
  int64_t n = b.valuesLen * 8;
  if (!b.dense()) n += b.colPtrsLen * 4 + b.valuesLen * 4;
  return n;
}

}  // namespace

mr_matrix* multiply_streamed(mr_context* ctx, mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right,
                             int64_t rightRowNum, int64_t rightColNum, int32_t blkSize) {
  const MultiplyDecisions dec = multiply_decisions(ctx, left, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize);
  // ---- the block rows of A and block columns of B (ascending ids): a panel is a run of consecutive entries
  std::map<int32_t, size_t> row_dev, col_dev;  // device bytes per block row of A / block column of B
  std::map<int32_t, size_t> row_fp, row_dense, col_dense;  // stored and dense-image bytes of a block row of A / column of B
  std::map<int32_t, int32_t> row_m, col_n;     // largest block height / width
  int64_t a_bytes = 0, b_bytes = 0;
  bool a_sparse = false, b_sparse = false;
  auto dense_bytes = [](const Block& b) { return align_up(static_cast<size_t>(b.numRows) * b.numCols * sizeof(double)); };
  for (auto& kv : left->blocks) {
    row_dev[kv.first.first] += left->host ? footprint(kv.second) : 0;
    row_fp[kv.first.first] += footprint(kv.second);
    row_dense[kv.first.first] += dense_bytes(kv.second);
    row_m[kv.first.first] = std::max(row_m[kv.first.first], kv.second.numRows);
    if (left->host) a_bytes += payload(kv.second);
    a_sparse = a_sparse || !kv.second.dense();
  }
  for (auto& kv : right->blocks) {
    col_dev[kv.first.second] += right->host ? footprint(kv.second) : 0;
    col_dense[kv.first.second] += dense_bytes(kv.second);
    col_n[kv.first.second] = std::max(col_n[kv.first.second], kv.second.numCols);
    if (right->host) b_bytes += payload(kv.second);
    b_sparse = b_sparse || !kv.second.dense();
  }
  std::unique_ptr<mr_matrix> C(new_matrix(ctx));
  C->host = std::make_shared<HostStore>(ctx);
  ctx->stats.stream_tiles = 0;
  ctx->stats.stream_h2d_bytes = 0;
  ctx->stats.stream_d2h_bytes = 0;
  if (row_m.empty() || col_n.empty()) return C.release();
  std::vector<int32_t> rows, cols;
  size_t a_row = 0, b_col = 0, a_row_fp = 0, a_row_dense = 0, b_col_dense = 0;
  int32_t max_m = 0, max_n = 0;
  for (auto& kv : row_m) {
    rows.push_back(kv.first);
    max_m = std::max(max_m, kv.second);
    a_row = std::max(a_row, row_dev[kv.first]);
    a_row_fp = std::max(a_row_fp, row_fp[kv.first]);
    a_row_dense = std::max(a_row_dense, row_dense[kv.first]);
  }
  for (auto& kv : col_n) {
    cols.push_back(kv.first);
    max_n = std::max(max_n, kv.second);
    b_col = std::max(b_col, col_dev[kv.first]);
    b_col_dense = std::max(b_col_dense, col_dense[kv.first]);
  }
  // per block row of A / column of B, what the dense x sparse route allocates for its blocks (b_col_ds: the B blocks' dense images
  // where they are densified, as before)
  std::map<int32_t, size_t> a_ds, b_col_ds;
  for (auto& kv : left->blocks)
    if (dec.ds_left.count(kv.first)) a_ds[kv.first.first] += dspmm_left_scratch(kv.second);
  for (auto& kv : right->blocks) {
    const bool routed = dec.ds_right.count(kv.first) != 0;
    size_t& n = b_col_ds[kv.first.second];
    if (!routed || dec.ds_dense_right.count(kv.first)) n += dense_bytes(kv.second);
    if (routed) n += dspmm_right_scratch(kv.second);
  }
  size_t a_ds_max = 0, b_col_ds_max = 0;
  for (auto& kv : a_ds) a_ds_max = std::max(a_ds_max, kv.second);
  for (auto& kv : b_col_ds) b_col_ds_max = std::max(b_col_ds_max, kv.second);
  // per block row of A / column of B, the sparse paths of a tile call allocate at most: dense images of sparse A blocks (pairs the
  // reference multiplies densely) and the re-packed CSR segments (bounded by the stored row); dense images of sparse B blocks, and
  // row-major copies of the column-major dense B blocks a sparse x dense kernel reads
  // Right blocks of dense x sparse pairs that take the stored-entry route get no dense image: their prepared segments (and CSC
  // copy) instead, and their left blocks a column-major copy and non-finite sets (DESIGN section 4.5.2).
  // The matrix x vector route (DESIGN section 4.5.5) makes no images: its scratch is at most one output block per pair.
  const bool mv = dec.mv != MV_NONE;
  const size_t a_scratch = mv ? 0 : (a_sparse ? a_row_dense + a_row_fp : 0) + a_ds_max;
  const size_t b_scratch = mv ? 0 : (a_sparse ? 1 : 0) * b_col_dense + (b_sparse ? b_col_ds_max : 0);
  const int64_t kblocks = ceil_div(leftColNum, blkSize);
  // ---- device budget and the tile
  const size_t budget = stream_budget(ctx);
  const size_t c_block = align_up(static_cast<size_t>(max_m) * max_n * sizeof(double));
  const StreamTiling T = choose_tiling(
      static_cast<int64_t>(rows.size()), static_cast<int64_t>(cols.size()), a_row, b_col, a_bytes, b_bytes, c_block, budget,
      [&](int64_t tr, int64_t tc) {
        const size_t oz2 = dec.oz2 ? oz2_scratch_for(ctx, blkSize, leftColNum, static_cast<int>(tr), static_cast<int>(tc)) : 0;
        const size_t mv_parts = mv ? static_cast<size_t>(tr) * tc * kblocks * c_block : 0;
        return oz2 + mv_parts + static_cast<size_t>(tr) * a_scratch + static_cast<size_t>(tc) * b_scratch;
      });
  if (!T.ok)
    fail(MR_ENOMEM,
         "streamed multiply: one block row x one block column with full K needs %zu bytes of device memory, the budget is %zu bytes "
         "(option stream_budget_mb, 0 = free device memory minus 1 GiB)",
         T.device_bytes, budget);

  // ---- panels and buffers
  auto runs = [](const std::vector<int32_t>& ids, int64_t t) {
    std::vector<std::pair<int32_t, int32_t>> out;  // [first id, last id] of each run
    for (size_t p = 0; p < ids.size(); p += static_cast<size_t>(t))
      out.emplace_back(ids[p], ids[std::min(ids.size(), p + static_cast<size_t>(t)) - 1]);
    return out;
  };
  const auto rpanels = runs(rows, T.tr), cpanels = runs(cols, T.tc);
  auto panel_dev = [](const std::map<int32_t, size_t>& per, const std::pair<int32_t, int32_t>& run) {
    size_t n = 0;
    for (auto it = per.lower_bound(run.first); it != per.end() && it->first <= run.second; ++it) n += it->second;
    return n;
  };
  auto window = [&](int32_t i, int32_t j) { return align_up(static_cast<size_t>(row_m[i]) * col_n[j] * sizeof(double)); };
  size_t a_cap = 0, b_cap = 0, c_cap = 0;
  for (auto& r : rpanels) a_cap = std::max(a_cap, panel_dev(row_dev, r));
  for (auto& c : cpanels) b_cap = std::max(b_cap, panel_dev(col_dev, c));
  for (auto& r : rpanels)
    for (auto& c : cpanels) {
      size_t n = 0;
      for (auto i = row_m.lower_bound(r.first); i != row_m.end() && i->first <= r.second; ++i)
        for (auto j = col_n.lower_bound(c.first); j != col_n.end() && j->first <= c.second; ++j) n += window(i->first, j->first);
      c_cap = std::max(c_cap, n);
    }
  const bool outer_b = T.outer_b;
  mr_matrix* outer_op = outer_b ? right : left;
  mr_matrix* inner_op = outer_b ? left : right;
  const auto& outer_panels = outer_b ? cpanels : rpanels;
  const auto& inner_panels = outer_b ? rpanels : cpanels;
  const size_t outer_cap = outer_b ? b_cap : a_cap, inner_cap = outer_b ? a_cap : b_cap;
  Buf outer_buf = std::make_shared<DevBuf>(ctx, outer_cap);
  Buf inner_buf[2] = {std::make_shared<DevBuf>(ctx, inner_cap), std::make_shared<DevBuf>(ctx, inner_cap)};
  Buf c_buf[2] = {std::make_shared<DevBuf>(ctx, c_cap), std::make_shared<DevBuf>(ctx, c_cap)};
  cudaStream_t cs = ctx->pipeline ? ctx->h2d_stream : ctx->stream;
  if (cs != ctx->stream) {  // the buffers are allocated on the context stream: the ingest stream must see them
    CUDA_CHECK(cudaEventRecord(ctx->ev_alloc, ctx->stream));
    CUDA_CHECK(cudaStreamWaitEvent(cs, ctx->ev_alloc, 0));
  }
  cudaStream_t rs = ctx->pipeline ? ctx->d2h_stream : ctx->stream;

  // The blocks of `src` whose row (by_row) or column id lies in `run`: host blocks are copied into `buf` on the ingest stream,
  // each with its own event and ingest number; device blocks are used in place.
  auto stage = [&](const mr_matrix* src, bool by_row, const std::pair<int32_t, int32_t>& run, const Buf& buf, mr_matrix* dst) {
    size_t off = 0;
    for (auto& kv : src->blocks) {
      const int32_t id = by_row ? kv.first.first : kv.first.second;
      if (id < run.first || id > run.second) continue;
      if (!src->host) {
        dst->blocks[kv.first] = kv.second;
        continue;
      }
      const Block& b = kv.second;
      if (b.ready) CUDA_CHECK(cudaStreamWaitEvent(cs, b.ready->ev, 0));  // the host block is still being written back
      Block d = b;
      d.settled = false;
      auto copy_in = [&](const Span& from, size_t bytes) {
        Span s{buf, off};
        off += align_up(bytes);
        if (bytes) {
          CUDA_CHECK(cudaMemcpyAsync(s.ptr<char>(), from.buf->p, bytes, cudaMemcpyHostToDevice, cs));
          ctx->stats.h2d_bytes += static_cast<int64_t>(bytes);
          ctx->stats.stream_h2d_bytes += static_cast<int64_t>(bytes);
        }
        return s;
      };
      d.values = copy_in(b.values, static_cast<size_t>(b.valuesLen) * sizeof(double));
      if (!b.dense()) {
        d.colPtrs = copy_in(b.colPtrs, static_cast<size_t>(b.colPtrsLen) * sizeof(int32_t));
        d.rowIndices = copy_in(b.rowIndices, static_cast<size_t>(b.valuesLen) * sizeof(int32_t));
      }
      d.ready = std::make_shared<Ready>();
      CUDA_CHECK(cudaEventRecord(d.ready->ev, cs));
      d.seq = ++ctx->ingest_seq;
      buf->ready = d.ready;  // the copies into a buffer are in order: its last one covers them all
      dst->blocks[kv.first] = std::move(d);
    }
  };

  ReadyPtr outer_free, inner_free[2], c_free[2];  // behind the last reader of each buffer (null: never read yet)
  int64_t t = 0;
  for (const auto& op : outer_panels) {
    std::unique_ptr<mr_matrix> outer_tile(new_matrix(ctx));
    if (outer_op->host && outer_free) CUDA_CHECK(cudaStreamWaitEvent(cs, outer_free->ev, 0));
    stage(outer_op, !outer_b, op, outer_buf, outer_tile.get());
    for (const auto& ip : inner_panels) {
      const int s = static_cast<int>(t & 1);
      std::unique_ptr<mr_matrix> inner_tile(new_matrix(ctx));
      if (inner_op->host && inner_free[s]) CUDA_CHECK(cudaStreamWaitEvent(cs, inner_free[s]->ev, 0));
      stage(inner_op, outer_b, ip, inner_buf[s], inner_tile.get());
      // C windows of this tile in c_buf[s], once the copies out of it two tiles ago are done
      if (c_free[s]) CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, c_free[s]->ev, 0));
      const auto& rp = outer_b ? ip : op;
      const auto& cp = outer_b ? op : ip;
      std::map<std::pair<int32_t, int32_t>, size_t> woff;
      size_t off = 0;
      for (auto i = row_m.lower_bound(rp.first); i != row_m.end() && i->first <= rp.second; ++i)
        for (auto j = col_n.lower_bound(cp.first); j != col_n.end() && j->first <= cp.second; ++j) {
          woff[{i->first, j->first}] = off;
          off += window(i->first, j->first);
        }
      const Buf cb = c_buf[s];
      const OutWindowFn win = [&](int32_t rid, int32_t cid) { return Span{cb, woff.at({rid, cid})}; };
      mr_matrix* A_tile = outer_b ? inner_tile.get() : outer_tile.get();
      mr_matrix* B_tile = outer_b ? outer_tile.get() : inner_tile.get();
      std::unique_ptr<mr_matrix> part(
          multiply_impl(ctx, A_tile, leftRowNum, leftColNum, B_tile, rightRowNum, rightColNum, blkSize, nullptr, &win, &dec));
      ReadyPtr done = std::make_shared<Ready>();  // behind the whole tile: every chunk joins the context stream
      CUDA_CHECK(cudaEventRecord(done->ev, ctx->stream));
      inner_free[s] = done;
      outer_free = done;
      // egress: the tile's blocks into the host-resident result
      if (rs != ctx->stream) CUDA_CHECK(cudaStreamWaitEvent(rs, done->ev, 0));
      std::vector<Block*> landed;
      auto copy_out = [&](const Span& from, size_t bytes) {
        Span h = C->host->take(bytes);
        if (bytes) {
          CUDA_CHECK(cudaMemcpyAsync(h.buf->p, from.ptr<char>(), bytes, cudaMemcpyDeviceToHost, rs));
          ctx->stats.d2h_bytes += static_cast<int64_t>(bytes);
          ctx->stats.stream_d2h_bytes += static_cast<int64_t>(bytes);
        }
        return h;
      };
      for (auto& kv : part->blocks) {
        const Block& b = kv.second;
        Block h = b;
        h.ready.reset();
        h.seq = 0;
        h.settled = false;
        h.values = copy_out(b.values, static_cast<size_t>(b.valuesLen) * sizeof(double));
        if (!b.dense()) {
          h.colPtrs = copy_out(b.colPtrs, static_cast<size_t>(b.colPtrsLen) * sizeof(int32_t));
          h.rowIndices = copy_out(b.rowIndices, static_cast<size_t>(b.valuesLen) * sizeof(int32_t));
        }
        Block& slot = C->blocks[kv.first];
        slot = std::move(h);
        landed.push_back(&slot);
      }
      ReadyPtr copied = std::make_shared<Ready>();
      CUDA_CHECK(cudaEventRecord(copied->ev, rs));
      for (Block* b : landed) b->ready = copied;
      c_free[s] = copied;
      // device arrays of the tile's result (sparse blocks have their own) are released after the copies out of them
      for (auto& kv : part->blocks)
        for (const Span* sp : {&kv.second.values, &kv.second.colPtrs, &kv.second.rowIndices})
          if (sp->buf) sp->buf->ready = copied;
      ++t;
    }
  }
  ctx->stats.stream_tiles = t;
  return C.release();
}

}  // namespace mrhost
