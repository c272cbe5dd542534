// Whole dense matrices in and out of datasets (include/matrel.h: mr_matrix_from_dense, mr_matrix_to_dense): Seq(MatrixBlock) of
// DenseMatrix blocks cut from one array, and DenseMatrix.toArray (MLMatrix.scala:55-61) for a whole dataset.
//   from_dense, host src    one 2D copy per block on the ingest stream, each block with its own event and ingest number (as
//                           mr_matrix_put_block), so a multiply issued next pipelines behind the ingest (DESIGN.md section 4.4)
//   from_dense, device src  the ingest stream waits for the caller's stream, then one dense_gather_kernel launch (dense_io.cu)
//   from_dense, host target plain copies into the dataset's page-locked store (2D copies on the egress stream for a device src)
//   to_dense                dense_assemble_kernel (+ dense_scatter_kernel for sparse blocks) over block-row or block-column panels:
//                           straight into a device dst, or into two device panel buffers in turn, each copied out by one 2D copy on
//                           the egress stream while the next panel is assembled; host-resident blocks are staged to the device first
// The host only copies; every layout change runs on the GPU.
#include <climits>

#include "host.h"

using namespace matrel;
using namespace mrhost;

namespace {

// true for memory of a device (then *dev is its ordinal); host memory, page-locked or not, and managed memory go the host path
bool device_memory(const void* p, int* dev) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  *dev = a.device;
  return a.type == cudaMemoryTypeDevice;
}

void check_dense_shape(int64_t nrows, int64_t ncols, int64_t ld, int32_t rowMajor, int32_t blkSize) {
  MR_REQUIRE(nrows > 0 && ncols > 0 && blkSize > 0, MR_EINVAL, "nrows, ncols, blkSize must be positive, got %lld, %lld, %d",
             (long long)nrows, (long long)ncols, blkSize);
  MR_REQUIRE(rowMajor == 0 || rowMajor == 1, MR_EINVAL, "rowMajor must be 0 or 1, got %d", rowMajor);
  const int64_t contiguous = rowMajor ? ncols : nrows;
  MR_REQUIRE(ld >= contiguous, MR_EINVAL, "ld = %lld is smaller than the contiguous dimension %lld (%s)", (long long)ld,
             (long long)contiguous, rowMajor ? "ncols of a row-major matrix" : "nrows of a column-major matrix");
  MR_REQUIRE(ceil_div(nrows, blkSize) <= INT_MAX && ceil_div(ncols, blkSize) <= INT_MAX, MR_EINVAL,
             "a %lld x %lld matrix in blocks of %d has block ids beyond Int", (long long)nrows, (long long)ncols, blkSize);
}

void check_device(const mr_context* ctx, bool on_device, int dev, const char* what) {
  MR_REQUIRE(!on_device || dev == ctx->device, MR_EINVAL, "%s is memory of device %d; this context runs on device %d", what, dev,
             ctx->device);
}

// offset of element (r, c) in a matrix of leading dimension ld
int64_t at(bool rm, int64_t ld, int64_t r, int64_t c) { return rm ? r * ld + c : r + c * ld; }

size_t payload_bytes(const Block& b) {
  size_t n = align_up(static_cast<size_t>(b.valuesLen) * sizeof(double));
  if (!b.dense()) n += align_up(static_cast<size_t>(b.colPtrsLen) * 4) + align_up(static_cast<size_t>(b.valuesLen) * 4);
  return n;
}

}  // namespace

extern "C" {

mr_status mr_matrix_from_dense(mr_context* ctx, const double* src, int64_t nrows, int64_t ncols, int64_t ld, int32_t rowMajor,
                               int32_t blkSize, int32_t host_resident, void* stream, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && src != nullptr && out != nullptr, MR_EINVAL, "ctx/src/out is null");
    check_dense_shape(nrows, ncols, ld, rowMajor, blkSize);
    // DenseMatrix.rand `require` (MLMatrix.scala:454-455): a block's values must be one JVM array
    const int64_t br = std::min<int64_t>(blkSize, nrows), bc = std::min<int64_t>(blkSize, ncols);
    MR_REQUIRE(br * bc <= INT32_MAX, MR_EINVAL, "%lld x %lld dense matrix is too large to allocate", (long long)br, (long long)bc);
    DeviceScope dev(ctx);
    int sdev = -1;
    const bool dsrc = device_memory(src, &sdev);
    check_device(ctx, dsrc, sdev, "src");
    std::lock_guard<std::mutex> lock(ctx->mu);
    const bool rm = rowMajor != 0;
    const int64_t nbr = ceil_div(nrows, blkSize), nbc = ceil_div(ncols, blkSize);
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    struct Piece {
      int32_t rid, cid, rows, cols;
      const double* from;  // the block's window of src
    };
    std::vector<Piece> pieces;
    pieces.reserve(static_cast<size_t>(nbr * nbc));
    for (int64_t i = 0; i < nbr; ++i)
      for (int64_t j = 0; j < nbc; ++j) {
        const int32_t r = static_cast<int32_t>(std::min<int64_t>(blkSize, nrows - i * blkSize));
        const int32_t c = static_cast<int32_t>(std::min<int64_t>(blkSize, ncols - j * blkSize));
        pieces.push_back(Piece{static_cast<int32_t>(i), static_cast<int32_t>(j), r, c, src + at(rm, ld, i * blkSize, j * blkSize)});
      }
    // a block keeps src's layout: `fast` contiguous elements per line, `slow` lines
    auto fast = [&](const Piece& p) { return static_cast<size_t>(rm ? p.cols : p.rows); };
    auto slow = [&](const Piece& p) { return static_cast<size_t>(rm ? p.rows : p.cols); };
    auto wait_user = [&](cudaStream_t s) {  // `s` after the producer of a device src
      if (user && user != s) {
        CUDA_CHECK(cudaEventRecord(ctx->ev_order, user));
        CUDA_CHECK(cudaStreamWaitEvent(s, ctx->ev_order, 0));
      }
    };
    std::unique_ptr<mr_matrix> m(new_matrix(ctx));

    if (host_resident) {
      m->host = std::make_shared<HostStore>(ctx);
      cudaStream_t rs = ctx->pipeline ? ctx->d2h_stream : ctx->stream;
      if (dsrc) wait_user(rs);
      for (const Piece& p : pieces) {
        const size_t bytes = static_cast<size_t>(p.rows) * p.cols * sizeof(double);
        Span h = m->host->take(bytes);
        double* d = h.ptr<double>();
        if (dsrc) {
          CUDA_CHECK(cudaMemcpy2DAsync(d, fast(p) * 8, p.from, static_cast<size_t>(ld) * 8, fast(p) * 8, slow(p), cudaMemcpyDeviceToHost, rs));
          ctx->stats.d2h_bytes += static_cast<int64_t>(bytes);
        } else {
          for (size_t l = 0; l < slow(p); ++l) std::memcpy(d + l * fast(p), p.from + static_cast<int64_t>(l) * ld, fast(p) * 8);
        }
        m->blocks[{p.rid, p.cid}] = dense_block(p.rows, p.cols, h, rm);
      }
      if (dsrc) {  // readers of the host blocks wait for exactly these copies (as after mr_matrix_to_host)
        ReadyPtr done = std::make_shared<Ready>();
        CUDA_CHECK(cudaEventRecord(done->ev, rs));
        for (auto& kv : m->blocks) kv.second.ready = done;
      }
      *out = m.release();
      return;
    }

    size_t total = 0;
    for (const Piece& p : pieces) total += align_up(static_cast<size_t>(p.rows) * p.cols * sizeof(double));
    Slab slab(ctx, total);
    std::vector<Span> spans;
    spans.reserve(pieces.size());
    for (const Piece& p : pieces) spans.push_back(slab.take(static_cast<size_t>(p.rows) * p.cols * sizeof(double)));
    cudaStream_t cs = ctx->pipeline ? ctx->h2d_stream : ctx->stream;
    Buf table;
    if (dsrc) {
      std::vector<DenseIoDesc> descs;
      int max_r = 0, max_c = 0;
      for (size_t k = 0; k < pieces.size(); ++k) {
        const Piece& p = pieces[k];
        descs.push_back(DenseIoDesc{p.from, spans[k].ptr<double>(), ld, static_cast<int64_t>(fast(p)), p.rows, p.cols,
                                    static_cast<uint8_t>(rm), static_cast<uint8_t>(rm), {}});
        max_r = std::max(max_r, p.rows);
        max_c = std::max(max_c, p.cols);
      }
      table = upload(ctx, descs);
      if (cs != ctx->stream) {  // the slab and the table are ordered on the context stream: the ingest stream must see them
        CUDA_CHECK(cudaEventRecord(ctx->ev_alloc, ctx->stream));
        CUDA_CHECK(cudaStreamWaitEvent(cs, ctx->ev_alloc, 0));
      }
      wait_user(cs);
      CUDA_CHECK(launch_dense_gather(static_cast<const DenseIoDesc*>(table->p), static_cast<int>(descs.size()), max_r, max_c, cs));
      note_launch(ctx);
    } else if (cs != ctx->stream) {
      CUDA_CHECK(cudaEventRecord(ctx->ev_alloc, ctx->stream));
      CUDA_CHECK(cudaStreamWaitEvent(cs, ctx->ev_alloc, 0));
    }
    ReadyPtr last;
    for (size_t k = 0; k < pieces.size(); ++k) {
      const Piece& p = pieces[k];
      if (!dsrc) {
        CUDA_CHECK(cudaMemcpy2DAsync(spans[k].ptr<double>(), fast(p) * 8, p.from, static_cast<size_t>(ld) * 8, fast(p) * 8, slow(p),
                                     cudaMemcpyDefault, cs));
        ctx->stats.h2d_bytes += static_cast<int64_t>(static_cast<size_t>(p.rows) * p.cols * sizeof(double));
      }
      Block b = dense_block(p.rows, p.cols, spans[k], rm);
      if (ctx->pipeline) {
        if (!dsrc || !last) {  // a device src lands in one launch: one event covers every block
          last = std::make_shared<Ready>();
          CUDA_CHECK(cudaEventRecord(last->ev, cs));
        }
        b.ready = last;
        b.seq = ++ctx->ingest_seq;
      }
      m->blocks[{p.rid, p.cid}] = std::move(b);
    }
    slab.buf->ready = last;  // the ingest stream is in order: the last event covers every write into the slab
    if (table) table->ready = last;
    *out = m.release();
  });
}

mr_status mr_matrix_to_dense(mr_matrix* m, int64_t nrows, int64_t ncols, int32_t blkSize, double* dst, int64_t ld, int32_t rowMajor,
                             void* stream) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && dst != nullptr, MR_EINVAL, "matrix/dst is null");
    check_dense_shape(nrows, ncols, ld, rowMajor, blkSize);
    for (auto& kv : m->blocks) {
      const int64_t rid = kv.first.first, cid = kv.first.second;
      const Block& b = kv.second;
      MR_REQUIRE(rid >= 0 && cid >= 0 && b.numRows <= blkSize && b.numCols <= blkSize && rid * blkSize + b.numRows <= nrows &&
                     cid * blkSize + b.numCols <= ncols,
                 MR_EDIM, "block (%lld, %lld) of %d x %d does not lie inside the %lld x %lld matrix in blocks of %d", (long long)rid,
                 (long long)cid, b.numRows, b.numCols, (long long)nrows, (long long)ncols, blkSize);
    }
    mr_context* ctx = m->ctx;
    DeviceScope dev(ctx);
    int ddev = -1;
    const bool ddst = device_memory(dst, &ddev);
    check_device(ctx, ddst, ddev, "dst");
    std::lock_guard<std::mutex> lock(ctx->mu);
    const bool rm = rowMajor != 0, hostb = m->host != nullptr;
    const int64_t nbr = ceil_div(nrows, blkSize), nbc = ceil_div(ncols, blkSize);
    // Panels are runs of block rows (row-major dst) or block columns (column-major dst): each is one contiguous range of dst's lines.
    const int64_t nlines = rm ? nbr : nbc, n_slow = rm ? nrows : ncols, n_fast = rm ? ncols : nrows;
    std::vector<size_t> line_stage(static_cast<size_t>(nlines), 0);  // host-resident payload per block line
    if (hostb)
      for (auto& kv : m->blocks) line_stage[static_cast<size_t>(rm ? kv.first.first : kv.first.second)] += payload_bytes(kv.second);
    const size_t out_line = ddst ? 0 : static_cast<size_t>(blkSize) * n_fast * sizeof(double);
    auto stage_max = [&](int64_t p) {  // the largest payload of p consecutive block lines
      size_t run = 0, best = 0;
      for (int64_t l = 0; l < nlines; ++l) {
        run += line_stage[l];
        if (l >= p) run -= line_stage[l - p];
        best = std::max(best, run);
      }
      return best;
    };
    auto need = [&](int64_t p) { return 2 * (static_cast<size_t>(p) * out_line + stage_max(p)); };  // two buffers of each kind
    // a host dst goes through several panels, so that copies overlap assembly; a device dst takes as few panels as fit
    const int64_t p_want = ddst ? nlines : std::max<int64_t>(1, ceil_div(nlines, 8));
    int64_t p = nlines;
    if (!ddst || hostb) {
      const size_t budget = stream_budget(ctx, need(p_want));
      if (need(1) > budget)
        fail(MR_ENOMEM,
             "to_dense: one block-%s panel needs %zu bytes of device memory (two buffers), the budget is %zu bytes (option "
             "stream_budget_mb, 0 = free device memory minus 1 GiB)",
             rm ? "row" : "column", need(1), budget);
      int64_t lo = 1, hi = nlines;  // need() grows with p: the largest p that fits
      while (lo < hi) {
        const int64_t mid = lo + (hi - lo + 1) / 2;
        if (need(mid) <= budget) lo = mid;
        else hi = mid - 1;
      }
      p = std::min(lo, p_want);
    }
    const int64_t npanels = ceil_div(nlines, p);
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    if (user && user != ctx->stream) {  // dst's previous users (a freshly allocated torch tensor's stream) come first
      CUDA_CHECK(cudaEventRecord(ctx->ev_order, user));
      CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_order, 0));
    }
    if (!hostb)
      for (auto& kv : m->blocks) wait_ready(ctx, kv.second);
    cudaStream_t cs = ctx->pipeline ? ctx->h2d_stream : ctx->stream;  // staging of host-resident blocks
    cudaStream_t rs = ctx->pipeline ? ctx->d2h_stream : ctx->stream;  // panel copies into a host dst
    const int nbuf = static_cast<int>(std::min<int64_t>(2, npanels));
    Buf outbuf[2], stage[2];
    ReadyPtr out_free[2], stage_free[2];  // buffer k may be rewritten once its event has completed
    for (int k = 0; k < nbuf; ++k) {
      if (!ddst) outbuf[k] = std::make_shared<DevBuf>(ctx, static_cast<size_t>(p) * out_line);
      if (hostb) stage[k] = std::make_shared<DevBuf>(ctx, std::max<size_t>(stage_max(p), 16));
    }
    if (cs != ctx->stream || rs != ctx->stream) {  // the buffers are allocated on the context stream
      CUDA_CHECK(cudaEventRecord(ctx->ev_alloc, ctx->stream));
      if (hostb) CUDA_CHECK(cudaStreamWaitEvent(cs, ctx->ev_alloc, 0));
      if (!ddst) CUDA_CHECK(cudaStreamWaitEvent(rs, ctx->ev_alloc, 0));
    }
    for (int64_t k = 0; k < npanels; ++k) {
      const int q = static_cast<int>(k % 2);
      const int64_t l0 = k * p, l1 = std::min(nlines, l0 + p);
      const int64_t s0 = l0 * blkSize, s1 = std::min(n_slow, l1 * blkSize);  // dst lines of the panel
      // where each block's arrays are read from: in place, or the panel's staging buffer
      std::map<std::pair<int32_t, int32_t>, Block> staged;
      auto in_panel = [&](int32_t rid, int32_t cid) {
        const int64_t l = rm ? rid : cid;
        return l >= l0 && l < l1;
      };
      if (hostb) {
        if (stage_free[q]) CUDA_CHECK(cudaStreamWaitEvent(cs, stage_free[q]->ev, 0));
        size_t off = 0;
        auto copy_in = [&](const Span& from, size_t bytes) {
          Span d{stage[q], off};
          off += align_up(bytes);
          if (bytes) {
            CUDA_CHECK(cudaMemcpyAsync(d.ptr<char>(), from.buf->p, bytes, cudaMemcpyHostToDevice, cs));
            ctx->stats.h2d_bytes += static_cast<int64_t>(bytes);
          }
          return d;
        };
        for (auto& kv : m->blocks) {
          if (!in_panel(kv.first.first, kv.first.second)) continue;
          const Block& b = kv.second;
          if (b.ready) CUDA_CHECK(cudaStreamWaitEvent(cs, b.ready->ev, 0));  // a write-back still in flight
          Block d = b;
          d.values = copy_in(b.values, static_cast<size_t>(b.valuesLen) * sizeof(double));
          if (!b.dense()) {
            d.colPtrs = copy_in(b.colPtrs, static_cast<size_t>(b.colPtrsLen) * 4);
            d.rowIndices = copy_in(b.rowIndices, static_cast<size_t>(b.valuesLen) * 4);
          }
          staged[kv.first] = std::move(d);
        }
        if (cs != ctx->stream) {
          CUDA_CHECK(cudaEventRecord(ctx->ev_order, cs));
          CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_order, 0));
        }
      }
      // the panel's windows: dst itself, or the panel buffer (its own lines s0 .. s1, leading dimension n_fast)
      double* base = ddst ? dst : static_cast<double*>(outbuf[q]->p);
      const int64_t wld = ddst ? ld : n_fast, shift = ddst ? 0 : s0;
      auto window = [&](int64_t r0, int64_t c0) { return base + at(rm, wld, r0 - (rm ? shift : 0), c0 - (rm ? 0 : shift)); };
      if (!ddst && out_free[q]) CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, out_free[q]->ev, 0));
      std::vector<DenseIoDesc> descs;
      std::vector<DenseScatterDesc> scat;
      int max_r = 0, max_c = 0, max_lines = 0;
      bool any_t = false;
      auto zero = [&](int64_t r0, int64_t c0, int64_t rows, int64_t cols) {
        if (rows <= 0 || cols <= 0) return;
        descs.push_back(DenseIoDesc{nullptr, window(r0, c0), 0, wld, static_cast<int32_t>(rows), static_cast<int32_t>(cols), 0,
                                    static_cast<uint8_t>(rm), {}});
        max_r = std::max<int>(max_r, static_cast<int>(rows));
        max_c = std::max<int>(max_c, static_cast<int>(cols));
      };
      for (int64_t l = l0; l < l1; ++l)
        for (int64_t o = 0; o < (rm ? nbc : nbr); ++o) {
          const int32_t rid = static_cast<int32_t>(rm ? l : o), cid = static_cast<int32_t>(rm ? o : l);
          const int64_t r0 = static_cast<int64_t>(rid) * blkSize, c0 = static_cast<int64_t>(cid) * blkSize;
          const int64_t cr = std::min<int64_t>(blkSize, nrows - r0), cc = std::min<int64_t>(blkSize, ncols - c0);  // the cell
          auto it = m->blocks.find({rid, cid});
          if (it == m->blocks.end()) {
            zero(r0, c0, cr, cc);
            continue;
          }
          const Block& b = hostb ? staged.at({rid, cid}) : it->second;
          if (b.dense()) {
            if (b.numRows > 0 && b.numCols > 0) {
              const int64_t lds = b.isT ? b.numCols : b.numRows;
              descs.push_back(DenseIoDesc{b.values.ptr<double>(), window(r0, c0), lds, wld, b.numRows, b.numCols,
                                          static_cast<uint8_t>(b.isT), static_cast<uint8_t>(rm), {}});
              max_r = std::max(max_r, b.numRows);
              max_c = std::max(max_c, b.numCols);
              any_t = any_t || b.isT != rm;
            }
            // the rest of the cell a smaller block leaves uncovered
            zero(r0 + b.numRows, c0, cr - b.numRows, cc);
            zero(r0, c0 + b.numCols, b.numRows, cc - b.numCols);
          } else {
            zero(r0, c0, cr, cc);
            if (b.valuesLen > 0) {
              scat.push_back(DenseScatterDesc{b.colPtrs.ptr<int32_t>(), b.rowIndices.ptr<int32_t>(), b.values.ptr<double>(),
                                              window(r0, c0), wld, static_cast<int32_t>(b.colPtrsLen - 1), static_cast<uint8_t>(b.isT),
                                              static_cast<uint8_t>(rm), {}});
              max_lines = std::max(max_lines, static_cast<int>(b.colPtrsLen - 1));
            }
          }
        }
      if (!descs.empty()) {
        Buf t = upload(ctx, descs);
        CUDA_CHECK(launch_dense_assemble(static_cast<const DenseIoDesc*>(t->p), static_cast<int>(descs.size()), max_r, max_c, any_t,
                                         ctx->stream));
        note_launch(ctx);
      }
      if (!scat.empty()) {  // after the zero fill of the same windows (same stream)
        Buf t = upload(ctx, scat);
        CUDA_CHECK(launch_dense_scatter(static_cast<const DenseScatterDesc*>(t->p), static_cast<int>(scat.size()), max_lines, ctx->stream));
        note_launch(ctx);
      }
      if (hostb && cs != ctx->stream) {
        stage_free[q] = std::make_shared<Ready>();
        CUDA_CHECK(cudaEventRecord(stage_free[q]->ev, ctx->stream));
      }
      if (!ddst) {
        if (rs != ctx->stream) {
          CUDA_CHECK(cudaEventRecord(ctx->ev_order, ctx->stream));
          CUDA_CHECK(cudaStreamWaitEvent(rs, ctx->ev_order, 0));
        }
        const size_t lines = static_cast<size_t>(s1 - s0);
        CUDA_CHECK(cudaMemcpy2DAsync(dst + s0 * ld, static_cast<size_t>(ld) * 8, outbuf[q]->p, static_cast<size_t>(n_fast) * 8,
                                     static_cast<size_t>(n_fast) * 8, lines, cudaMemcpyDeviceToHost, rs));
        ctx->stats.d2h_bytes += static_cast<int64_t>(lines * n_fast * sizeof(double));
        out_free[q] = std::make_shared<Ready>();
        CUDA_CHECK(cudaEventRecord(out_free[q]->ev, rs));
      }
    }
    // the panel buffers are released on the context stream, after the copies that read them
    for (int k = 0; k < nbuf; ++k)
      if (outbuf[k]) outbuf[k]->ready = out_free[k];
    Ready done;
    CUDA_CHECK(cudaEventRecord(done.ev, ddst ? ctx->stream : rs));
    if (user) CUDA_CHECK(cudaStreamWaitEvent(user, done.ev, 0));
    else CUDA_CHECK(cudaEventSynchronize(done.ev));
  });
}

}  // extern "C"
