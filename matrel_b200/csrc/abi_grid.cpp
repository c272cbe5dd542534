// Multi-GPU layer of the C ABI: datasets sharded over a pr x pc process grid, the grid multiply, and the single-process grid
// (one process drives all GPUs of the box).
//
// What it replaces in the reference (M/ = <reference>/src/main/scala/org/apache/spark/sql/matfast/):
//   * RowPartitioner / ColumnPartitioner placement (M/partitioner/RowPartitioner.scala:34, ColumnPartitioner.scala:34): rank (r, c)
//     owns the blocks with rid % pr == r and cid % pc == c -- of A, B and C alike (C-stationary);
//   * the two groupByKey + join of matrixMultiplyGeneral (M/execution/MatfastExecutionHelper.scala:236-249) that co-locate A(:, k)
//     with B(k, :): every rank PULLS the A blocks of its block rows from the ranks of its grid row and the B blocks of its block
//     columns from the ranks of its grid column, straight out of their device slabs over NVLink with the copy engines
//     (cudaMemcpyAsync on peer-mapped / IPC-opened pointers -- no SM is taken from the GEMM), block row by block row, each
//     chunk tagged with an event; the multiply (abi_multiply.cpp) starts on the first chunk while the rest is on the wire;
//   * reduceByKey(LocalMatrix.add) (:255): nothing -- every rank owns whole output blocks and keeps the K reduction in the kernel.
//   * duplicateCrossPartitions (:224-233): the same pull with a single k-block.
// One process per GPU (torch.distributed launches, matrel_b200/distributed.py): peers' slabs are opened through CUDA IPC
// (mr_ipc_export / mr_ipc_open).  One process for all GPUs (mr_init_grid): peers' slabs are plain peer-accessible pointers and
// the cross-device ordering is done with events; NCCL (ncclCommInitAll, loaded at run time) carries the collectives that are
// reductions (aggregates).
#include "host.h"

#include <dlfcn.h>

using namespace matrel;
using namespace mrhost;

namespace mrhost {

ShardLayout make_layout(int64_t nrows, int64_t ncols, int32_t blk, int32_t pr, int32_t pc, int32_t r, int32_t c) {
  ShardLayout L{};
  L.nrows = nrows;
  L.ncols = ncols;
  L.blk = blk;
  L.pr = pr;
  L.pc = pc;
  L.r = r;
  L.c = c;
  L.nbr = ceil_div(nrows, blk);
  L.nbc = ceil_div(ncols, blk);
  L.slots_r = ceil_div(L.nbr, pr);
  L.slots_c = ceil_div(L.nbc, pc);
  L.slot_elems = static_cast<int64_t>(blk) * blk;
  return L;
}

void validate_layout(const mr_grid_layout* g) {
  MR_REQUIRE(g != nullptr, MR_EINVAL, "layout is null");
  MR_REQUIRE(g->nrows > 0 && g->ncols > 0 && g->blkSize > 0, MR_EINVAL, "nrows, ncols, blkSize must be positive");
  MR_REQUIRE(g->pr > 0 && g->pc > 0 && g->r >= 0 && g->r < g->pr && g->c >= 0 && g->c < g->pc, MR_EINVAL,
             "bad process grid %d x %d / (%d, %d)", g->pr, g->pc, g->r, g->c);
  MR_REQUIRE(static_cast<int64_t>(g->blkSize) * g->blkSize <= INT32_MAX, MR_EINVAL, "%d x %d dense matrix is too large to allocate",
             g->blkSize, g->blkSize);
}

// Registers every block this rank owns as a window of the slab (a sharded dataset is dense over its block grid).
void register_owned_blocks(mr_matrix* m) {
  const ShardLayout& L = m->shard->L;
  for (int64_t i = L.r; i < L.nbr; i += L.pr)
    for (int64_t j = L.c; j < L.nbc; j += L.pc) {
      const int32_t br = static_cast<int32_t>(std::min<int64_t>(L.blk, L.nrows - i * L.blk));
      const int32_t bc = static_cast<int32_t>(std::min<int64_t>(L.blk, L.ncols - j * L.blk));
      Span s{m->shard->slab, static_cast<size_t>(L.slot(i, j)) * L.slot_elems * sizeof(double)};
      m->blocks[{static_cast<int32_t>(i), static_cast<int32_t>(j)}] = dense_block(br, bc, s, m->shard->isT);
    }
}

mr_matrix* new_sharded(mr_context* ctx, const ShardLayout& L, bool ipc_capable, bool zero, bool isT) {
  std::unique_ptr<mr_matrix> m(new_matrix(ctx));
  auto sh = std::make_shared<ShardInfo>();
  sh->L = L;
  sh->isT = isT;
  const size_t bytes = std::max<size_t>(static_cast<size_t>(L.local_slots()) * L.slot_elems * sizeof(double), 16);
  sh->slab = ipc_capable ? std::make_shared<DevBuf>(ctx, bytes, DevBuf::SyncAlloc{}) : std::make_shared<DevBuf>(ctx, bytes);
  sh->ipc_capable = ipc_capable;
  if (zero) CUDA_CHECK(cudaMemsetAsync(sh->slab->p, 0, bytes, ctx->stream));
  m->shard = sh;
  register_owned_blocks(m.get());
  return m.release();
}

// ---- driver entry point needed for IPC of interior pointers
using AddrRangeFn = int (*)(unsigned long long*, size_t*, unsigned long long);
AddrRangeFn addr_range_fn() {
  static AddrRangeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<AddrRangeFn>(p);
  }();
  return fn;
}

}  // namespace mrhost

namespace {

// The A blocks of my block rows / the B blocks of my block columns, pulled from the grid row / grid column.
struct PanelPull {
  Buf buf;                 // [nsrc][peer local slots][slot_elems] for the peers (own slab is used in place)
  std::vector<ReadyPtr> chunk_ready;
};

}  // namespace

extern "C" {

mr_status mr_matrix_create_sharded(mr_context* ctx, const mr_grid_layout* g, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && out != nullptr, MR_EINVAL, "ctx/out is null");
    validate_layout(g);
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    *out = new_sharded(ctx, make_layout(g->nrows, g->ncols, g->blkSize, g->pr, g->pc, g->r, g->c), true, true);
  });
}

mr_status mr_matrix_layout(const mr_matrix* m, mr_grid_layout* out) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && out != nullptr, MR_EINVAL, "null argument");
    MR_REQUIRE(m->shard != nullptr, MR_EINVAL, "not a sharded dataset");
    const ShardLayout& L = m->shard->L;
    *out = mr_grid_layout{L.nrows, L.ncols, L.blk, L.pr, L.pc, L.r, L.c};
  });
}

mr_status mr_matrix_slab(mr_matrix* m, double** dslab, int64_t* bytes) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && dslab != nullptr, MR_EINVAL, "null argument");
    MR_REQUIRE(m->shard != nullptr, MR_EINVAL, "not a sharded dataset");
    *dslab = static_cast<double*>(m->shard->slab->p);
    if (bytes) *bytes = static_cast<int64_t>(m->shard->slab->bytes);
  });
}

// Adopts a caller-owned device slab (e.g. a torch tensor) as a sharded dataset: the blocks this rank owns are windows of it.
mr_status mr_matrix_adopt_sharded(mr_context* ctx, const mr_grid_layout* g, double* dslab, uint8_t isTransposed, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && out != nullptr && dslab != nullptr, MR_EINVAL, "null argument");
    validate_layout(g);
    std::unique_ptr<mr_matrix> m(new_matrix(ctx));
    auto sh = std::make_shared<ShardInfo>();
    sh->L = make_layout(g->nrows, g->ncols, g->blkSize, g->pr, g->pc, g->r, g->c);
    sh->slab = std::make_shared<DevBuf>(ctx, dslab, static_cast<size_t>(sh->L.local_slots()) * sh->L.slot_elems * sizeof(double));
    sh->ipc_capable = true;  // up to the caller's allocator (cudaMalloc-backed memory is)
    sh->isT = isTransposed != 0;
    m->shard = sh;
    register_owned_blocks(m.get());
    *out = m.release();
  });
}

mr_status mr_ipc_export(const void* dptr, void* handle64, int64_t* offset) {
  return guarded([&] {
    MR_REQUIRE(dptr != nullptr && handle64 != nullptr && offset != nullptr, MR_EINVAL, "null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    AddrRangeFn fn = addr_range_fn();
    if (!fn) fail(MR_ECUDA, "cuMemGetAddressRange is unavailable");
    unsigned long long base = 0;
    size_t size = 0;
    if (fn(&base, &size, reinterpret_cast<unsigned long long>(dptr)) != 0) fail(MR_ECUDA, "cuMemGetAddressRange failed for %p", dptr);
    cudaIpcMemHandle_t h;
    CUDA_CHECK(cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(base)));
    std::memcpy(handle64, &h, 64);
    *offset = static_cast<int64_t>(reinterpret_cast<unsigned long long>(dptr) - base);
  });
}

mr_status mr_ipc_open(mr_context* ctx, const void* handle64, int64_t offset, void** dptr) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && handle64 != nullptr && dptr != nullptr && offset >= 0, MR_EINVAL, "bad argument");
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    std::string key(static_cast<const char*>(handle64), 64);
    auto it = ctx->ipc_open.find(key);
    if (it == ctx->ipc_open.end()) {
      cudaIpcMemHandle_t h;
      std::memcpy(&h, handle64, 64);
      void* base = nullptr;
      CUDA_CHECK(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
      it = ctx->ipc_open.emplace(key, base).first;
    }
    *dptr = static_cast<char*>(it->second) + offset;
  });
}

// Reads `bytes` at a device pointer valid in this process (own, peer-mapped or IPC-opened memory) into host memory, ordered after
// everything enqueued on the context so far.  Used by checks that need a peer's operand blocks on the host.
mr_status mr_memcpy_d2h(mr_context* ctx, const void* dptr, void* host, int64_t bytes) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && dptr != nullptr && host != nullptr && bytes >= 0, MR_EINVAL, "bad argument");
    DeviceScope dev(ctx);
    CUDA_CHECK(cudaStreamSynchronize(ctx->p2p_stream));
    CUDA_CHECK(cudaMemcpyAsync(host, dptr, static_cast<size_t>(bytes), cudaMemcpyDefault, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->stats.d2h_bytes += bytes;
  });
}

mr_status mr_ipc_close_all(mr_context* ctx) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr, MR_EINVAL, "ctx is null");
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    CUDA_CHECK(cudaStreamSynchronize(ctx->p2p_stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    for (auto& kv : ctx->ipc_open) cudaIpcCloseMemHandle(kv.second);
    ctx->ipc_open.clear();
  });
}

// C(local) = A B on the process grid, C-stationary.  slabsA_row[c'] (c' = 0 .. pc-1) = base of the slab of rank (r, c') of A;
// slabsB_col[r'] (r' = 0 .. pr-1) = base of the slab of rank (r', c) of B; both valid in THIS process (own slab, peer-mapped or
// IPC-opened).  The caller guarantees that the peers' slabs are complete and stay untouched until this rank's pulls have run
// (one process per GPU: a barrier on the stream before, one after; mr_init_grid does it with events).  nchunks = number of pieces
// the A pull is cut into along this rank's block rows (>= 1): the multiply starts on piece 0 while the others are on the wire.
static mr_status grid_multiply_impl(mr_matrix* A, mr_matrix* B, const double* const* slabsA_row, const double* const* slabsB_col,
                                    int32_t nchunks, const void* const* gates, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(A && B && out && slabsA_row && slabsB_col, MR_EINVAL, "null argument");
    MR_REQUIRE(A->shard && B->shard, MR_EINVAL, "operands must be sharded datasets (mr_matrix_create_sharded)");
    MR_REQUIRE(A->ctx == B->ctx, MR_EINVAL, "operands belong to different contexts");
    const ShardLayout LA = A->shard->L, LB = B->shard->L;
    MR_REQUIRE(LA.pr == LB.pr && LA.pc == LB.pc && LA.r == LB.r && LA.c == LB.c && LA.blk == LB.blk, MR_EINVAL,
               "operands are laid out on different grids");
    // MatfastExecution.scala:702-703
    MR_REQUIRE(LA.ncols == LB.nrows, MR_EDIM, "Matrix dimension not match, leftColNum = %lld, rightRowNum = %lld",
               (long long)LA.ncols, (long long)LB.nrows);
    MR_REQUIRE(!A->shard->isT && !B->shard->isT, MR_ENOTSUP, "grid multiply of a flag-transposed sharded dataset: materialise it first");
    mr_context* ctx = A->ctx;
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    const int pr = LA.pr, pc = LA.pc, r = LA.r, c = LA.c;
    const size_t slot_bytes = static_cast<size_t>(LA.slot_elems) * sizeof(double);
    const size_t a_local = static_cast<size_t>(LA.local_slots()) * slot_bytes, b_local = static_cast<size_t>(LB.local_slots()) * slot_bytes;
    cudaStream_t ps = ctx->p2p_stream;
    // the pull stream starts after everything enqueued so far on the context stream (operand producers, the panel allocations)
    Buf panelA = pc > 1 ? std::make_shared<DevBuf>(ctx, a_local * (pc - 1)) : nullptr;
    Buf panelB = pr > 1 ? std::make_shared<DevBuf>(ctx, b_local * (pr - 1)) : nullptr;
    CUDA_CHECK(cudaEventRecord(ctx->ev_order, ctx->stream));
    CUDA_CHECK(cudaStreamWaitEvent(ps, ctx->ev_order, 0));
    auto peer_index = [](int p, int self) { return p < self ? p : p - 1; };  // position of peer p in the panel buffer
    auto gate = [&](int idx) {  // caller-provided "the peers' data for this piece is in place" event
      if (gates != nullptr && gates[idx] != nullptr) CUDA_CHECK(cudaStreamWaitEvent(ps, static_cast<cudaEvent_t>(const_cast<void*>(gates[idx])), 0));
    };
    // ---- pulls, piece by piece: block rows [rows * ch / n, rows * (ch + 1) / n) of A from the grid row, then block columns
    //      [cols * ch / n, cols * (ch + 1) / n) of B from the grid column, ch = 0 .. n - 1.  Alternating the two operands lets the
    //      multiply start on the leading (1 / n) x (1 / n) corner of C and grow it piece by piece, instead of waiting for all of B.
    //      The k-blocks a peer owns of one block row are contiguous in its slab (one copy per peer and piece of A); a piece of B is
    //      one run per local k-row.  Pulled blocks carry the event of their piece and an ingest sequence number in pull order,
    //      which is what the multiply groups its launches by; own blocks keep whatever event / number their host ingest gave them.
    const int64_t my_rows = LA.slots_r_of(r);
    const int64_t my_cols = LB.nbc > c ? (LB.nbc - c + pc - 1) / pc : 0;
    nchunks = static_cast<int32_t>(std::max<int32_t>(1, std::min<int32_t>(nchunks, 64)));
    std::vector<ReadyPtr> readyA(nchunks), readyB(nchunks);
    std::vector<uint64_t> seqA(nchunks), seqB(nchunks);
    std::vector<int> chunk_of_row(static_cast<size_t>(std::max<int64_t>(my_rows, 1)), 0), chunk_of_col(static_cast<size_t>(std::max<int64_t>(my_cols, 1)), 0);
    for (int ch = 0; ch < nchunks; ++ch) {
      {
        const int64_t lo = my_rows * ch / nchunks, hi = my_rows * (ch + 1) / nchunks;
        for (int64_t li = lo; li < hi; ++li) chunk_of_row[li] = ch;
        gate(2 * ch);
        if (pc > 1 && hi > lo) {
          const size_t off = static_cast<size_t>(lo) * LA.slots_c * slot_bytes, len = static_cast<size_t>(hi - lo) * LA.slots_c * slot_bytes;
          for (int cc = 0; cc < pc; ++cc) {
            if (cc == c) continue;
            MR_REQUIRE(slabsA_row[cc] != nullptr, MR_EINVAL, "slabsA_row[%d] is null", cc);
            CUDA_CHECK(cudaMemcpyAsync(static_cast<char*>(panelA->p) + a_local * peer_index(cc, c) + off,
                                       reinterpret_cast<const char*>(slabsA_row[cc]) + off, len, cudaMemcpyDefault, ps));
          }
        }
        readyA[ch] = std::make_shared<Ready>();
        CUDA_CHECK(cudaEventRecord(readyA[ch]->ev, ps));
        seqA[ch] = ++ctx->ingest_seq;
      }
      {
        const int64_t lo = my_cols * ch / nchunks, hi = my_cols * (ch + 1) / nchunks;
        for (int64_t lj = lo; lj < hi; ++lj) chunk_of_col[lj] = ch;
        gate(2 * ch + 1);
        if (pr > 1 && hi > lo) {
          const size_t len = static_cast<size_t>(hi - lo) * slot_bytes;
          for (int rr = 0; rr < pr; ++rr) {
            if (rr == r) continue;
            MR_REQUIRE(slabsB_col[rr] != nullptr, MR_EINVAL, "slabsB_col[%d] is null", rr);
            for (int64_t lk = 0; lk < LB.slots_r_of(rr); ++lk) {
              const size_t off = static_cast<size_t>(lk * LB.slots_c + lo) * slot_bytes;
              CUDA_CHECK(cudaMemcpyAsync(static_cast<char*>(panelB->p) + b_local * peer_index(rr, r) + off,
                                         reinterpret_cast<const char*>(slabsB_col[rr]) + off, len, cudaMemcpyDefault, ps));
            }
          }
        }
        readyB[ch] = std::make_shared<Ready>();
        CUDA_CHECK(cudaEventRecord(readyB[ch]->ev, ps));
        seqB[ch] = ++ctx->ingest_seq;
      }
    }
    if (panelA) panelA->ready = readyA[nchunks - 1];
    if (panelB) panelB->ready = readyB[nchunks - 1];
    ctx->stats.p2p_bytes += static_cast<int64_t>((pc > 1 ? a_local * (pc - 1) : 0) + (pr > 1 ? b_local * (pr - 1) : 0));
    std::unique_ptr<mr_matrix> tA(new_matrix(ctx)), tB(new_matrix(ctx));
    for (int64_t i = r; i < LA.nbr; i += pr) {
      const int64_t li = i / pr;
      for (int64_t k = 0; k < LA.nbc; ++k) {
        const int src = static_cast<int>(k % pc);
        const int32_t br = static_cast<int32_t>(std::min<int64_t>(LA.blk, LA.nrows - i * LA.blk));
        const int32_t bc = static_cast<int32_t>(std::min<int64_t>(LA.blk, LA.ncols - k * LA.blk));
        const size_t slot_off = static_cast<size_t>(li * LA.slots_c + k / pc) * slot_bytes;
        const std::pair<int32_t, int32_t> key{static_cast<int32_t>(i), static_cast<int32_t>(k)};
        if (src == c) {
          Block b = dense_block(br, bc, Span{A->shard->slab, slot_off}, false);
          auto it = A->blocks.find(key);
          if (it != A->blocks.end()) {  // own block possibly still being ingested from the host: it keeps its own event, and
            b.ready = it->second.ready;  // counts as part of its piece for the order the multiply works in (a gated caller
            b.seq = seqA[chunk_of_row[li]];  // uploads piece by piece in pull order, so the piece number is its arrival order)
            b.settled = it->second.settled;
          }
          tA->blocks[key] = std::move(b);
        } else {
          Block b = dense_block(br, bc, Span{panelA, a_local * peer_index(src, c) + slot_off}, false);
          b.ready = readyA[chunk_of_row[li]];
          b.seq = seqA[chunk_of_row[li]];
          tA->blocks[key] = std::move(b);
        }
      }
    }
    for (int64_t k = 0; k < LB.nbr; ++k) {
      const int src = static_cast<int>(k % pr);
      for (int64_t j = c; j < LB.nbc; j += pc) {
        const int32_t br = static_cast<int32_t>(std::min<int64_t>(LB.blk, LB.nrows - k * LB.blk));
        const int32_t bc = static_cast<int32_t>(std::min<int64_t>(LB.blk, LB.ncols - j * LB.blk));
        const size_t slot_off = static_cast<size_t>((k / pr) * LB.slots_c + j / pc) * slot_bytes;
        const std::pair<int32_t, int32_t> key{static_cast<int32_t>(k), static_cast<int32_t>(j)};
        if (src == r) {
          Block b = dense_block(br, bc, Span{B->shard->slab, slot_off}, false);
          auto it = B->blocks.find(key);
          if (it != B->blocks.end()) {
            b.ready = it->second.ready;
            b.seq = seqB[chunk_of_col[j / pc]];
            b.settled = it->second.settled;
          }
          tB->blocks[key] = std::move(b);
        } else {
          Block b = dense_block(br, bc, Span{panelB, b_local * peer_index(src, r) + slot_off}, false);
          b.ready = readyB[chunk_of_col[j / pc]];
          b.seq = seqB[chunk_of_col[j / pc]];
          tB->blocks[key] = std::move(b);
        }
      }
    }
    const ShardLayout LC = make_layout(LA.nrows, LB.ncols, LA.blk, pr, pc, r, c);
    std::unique_ptr<mr_matrix> result(multiply_impl(ctx, tA.get(), LA.nrows, LA.ncols, tB.get(), LB.nrows, LB.ncols, LA.blk, &LC));
    *out = result.release();
  });
}

mr_status mr_grid_multiply(mr_matrix* A, mr_matrix* B, const double* const* slabsA_row, const double* const* slabsB_col,
                           int32_t nchunks, mr_matrix** out) {
  return grid_multiply_impl(A, B, slabsA_row, slabsB_col, nchunks, nullptr, out);
}

// The same with one caller-provided CUDA event per piece of the pull, 2 * nchunks of them: gates[2 ch] guards the pull of piece
// ch of A (this rank's block rows [rows * ch / nchunks, rows * (ch + 1) / nchunks)), gates[2 ch + 1] the pull of piece ch of B (its
// block columns [cols * ch / nchunks, cols * (ch + 1) / nchunks)); pieces may be empty.  A null entry means "already in place".  This is how a multi-process caller overlaps its peers' host->device ingest with the multiply:
// every rank uploads piece after piece, puts a stream barrier behind each, records an event, and hands the events in here.
mr_status mr_grid_multiply_gated(mr_matrix* A, mr_matrix* B, const double* const* slabsA_row, const double* const* slabsB_col,
                                 int32_t nchunks, const void* const* gates, mr_matrix** out) {
  return grid_multiply_impl(A, B, slabsA_row, slabsB_col, nchunks, gates, out);
}

// The blocks of a dataset that a partition owns: rid % row_mod == row_rem and cid % col_mod == col_rem (RowPartitioner /
// ColumnPartitioner arithmetic); the result shares the device arrays with the source (no copy).
mr_status mr_matrix_filter_blocks(mr_matrix* a, int32_t row_mod, int32_t row_rem, int32_t col_mod, int32_t col_rem, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(a && out, MR_EINVAL, "null argument");
    MR_REQUIRE(row_mod >= 1 && col_mod >= 1 && row_rem >= 0 && row_rem < row_mod && col_rem >= 0 && col_rem < col_mod, MR_EINVAL,
               "bad partition (%d mod %d, %d mod %d)", row_rem, row_mod, col_rem, col_mod);
    std::lock_guard<std::mutex> lock(a->ctx->mu);
    std::unique_ptr<mr_matrix> m(new_matrix(a->ctx));
    for (auto& kv : a->blocks)
      if (kv.first.first % row_mod == row_rem && kv.first.second % col_mod == col_rem) m->blocks[kv.first] = kv.second;
    *out = m.release();
  });
}

// The same with a LEFT operand that is not sharded: `A_rows` holds every block A(i, k) -- sparse or dense, any k -- of the block
// rows i this rank owns (rid % pr == r).  This is how a thin / sparse operand travels: the reference replicates it with
// duplicateCrossPartitions (MatfastExecutionHelper.scala:224-233); here the caller generates or ingests the block rows where they
// are needed, and only the dense B is pulled from the grid column (BASELINE configs[4]: CSR blocks x dense on 4 GPUs).
mr_status mr_grid_multiply_rows(mr_matrix* A_rows, int64_t leftRowNum, int64_t leftColNum, mr_matrix* B, const double* const* slabsB_col,
                                mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(A_rows && B && out && slabsB_col, MR_EINVAL, "null argument");
    MR_REQUIRE(B->shard, MR_EINVAL, "the right operand must be a sharded dataset (mr_matrix_create_sharded)");
    MR_REQUIRE(A_rows->ctx == B->ctx, MR_EINVAL, "operands belong to different contexts");
    const ShardLayout LB = B->shard->L;
    MR_REQUIRE(leftColNum == LB.nrows, MR_EDIM, "Matrix dimension not match, leftColNum = %lld, rightRowNum = %lld",
               (long long)leftColNum, (long long)LB.nrows);
    MR_REQUIRE(!B->shard->isT, MR_ENOTSUP, "grid multiply of a flag-transposed sharded dataset: materialise it first");
    mr_context* ctx = B->ctx;
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    const int pr = LB.pr, pc = LB.pc, r = LB.r, c = LB.c;
    for (auto& kv : A_rows->blocks)
      MR_REQUIRE(kv.first.first % pr == r, MR_EINVAL, "left block (%d, %d) is not in a block row of rank (%d, %d)", kv.first.first,
                 kv.first.second, r, c);
    const size_t slot_bytes = static_cast<size_t>(LB.slot_elems) * sizeof(double);
    const size_t b_local = static_cast<size_t>(LB.local_slots()) * slot_bytes;
    cudaStream_t ps = ctx->p2p_stream;
    Buf panelB = pr > 1 ? std::make_shared<DevBuf>(ctx, b_local * (pr - 1)) : nullptr;
    CUDA_CHECK(cudaEventRecord(ctx->ev_order, ctx->stream));
    CUDA_CHECK(cudaStreamWaitEvent(ps, ctx->ev_order, 0));
    auto peer_index = [](int p, int self) { return p < self ? p : p - 1; };
    ReadyPtr readyB;
    if (pr > 1) {
      for (int rr = 0; rr < pr; ++rr) {
        if (rr == r) continue;
        MR_REQUIRE(slabsB_col[rr] != nullptr, MR_EINVAL, "slabsB_col[%d] is null", rr);
        CUDA_CHECK(cudaMemcpyAsync(static_cast<char*>(panelB->p) + b_local * peer_index(rr, r), slabsB_col[rr], b_local, cudaMemcpyDefault, ps));
      }
      readyB = std::make_shared<Ready>();
      CUDA_CHECK(cudaEventRecord(readyB->ev, ps));
      panelB->ready = readyB;
      ctx->stats.p2p_bytes += static_cast<int64_t>(b_local * (pr - 1));
    }
    const uint64_t seqB = ++ctx->ingest_seq;
    std::unique_ptr<mr_matrix> tB(new_matrix(ctx));
    for (int64_t k = 0; k < LB.nbr; ++k) {
      const int src = static_cast<int>(k % pr);
      for (int64_t j = c; j < LB.nbc; j += pc) {
        const int32_t br = static_cast<int32_t>(std::min<int64_t>(LB.blk, LB.nrows - k * LB.blk));
        const int32_t bc = static_cast<int32_t>(std::min<int64_t>(LB.blk, LB.ncols - j * LB.blk));
        const size_t slot_off = static_cast<size_t>((k / pr) * LB.slots_c + j / pc) * slot_bytes;
        const std::pair<int32_t, int32_t> key{static_cast<int32_t>(k), static_cast<int32_t>(j)};
        if (src == r) {
          Block b = dense_block(br, bc, Span{B->shard->slab, slot_off}, false);
          auto it = B->blocks.find(key);
          if (it != B->blocks.end()) {
            b.ready = it->second.ready;
            b.seq = it->second.seq;
            b.settled = it->second.settled;
          }
          tB->blocks[key] = std::move(b);
        } else {
          Block b = dense_block(br, bc, Span{panelB, b_local * peer_index(src, r) + slot_off}, false);
          b.ready = readyB;
          b.seq = seqB;
          tB->blocks[key] = std::move(b);
        }
      }
    }
    const ShardLayout LC = make_layout(leftRowNum, LB.ncols, LB.blk, pr, pc, r, c);
    *out = multiply_impl(ctx, A_rows, leftRowNum, leftColNum, tB.get(), LB.nrows, LB.ncols, LB.blk, &LC);
  });
}

}  // extern "C"

// =================================================================================================
// Single-process grid: one host process drives every GPU of the box (SURVEY.md 8b "one process drives all 8 GPUs").
// =================================================================================================
#include <nccl.h>

namespace {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok() const { return lib != nullptr; }
};

NcclApi& nccl_api() {
  static NcclApi api = [] {
    NcclApi a;
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      a.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (a.lib) break;
    }
    if (!a.lib) return a;
    auto sym = [&](const char* n) { return dlsym(a.lib, n); };
    a.CommInitAll = reinterpret_cast<decltype(a.CommInitAll)>(sym("ncclCommInitAll"));
    a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(sym("ncclCommDestroy"));
    a.AllReduce = reinterpret_cast<decltype(a.AllReduce)>(sym("ncclAllReduce"));
    a.Send = reinterpret_cast<decltype(a.Send)>(sym("ncclSend"));
    a.Recv = reinterpret_cast<decltype(a.Recv)>(sym("ncclRecv"));
    a.GroupStart = reinterpret_cast<decltype(a.GroupStart)>(sym("ncclGroupStart"));
    a.GroupEnd = reinterpret_cast<decltype(a.GroupEnd)>(sym("ncclGroupEnd"));
    a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(sym("ncclGetErrorString"));
    if (!a.CommInitAll || !a.CommDestroy || !a.AllReduce || !a.Send || !a.Recv || !a.GroupStart || !a.GroupEnd) a.lib = nullptr;
    return a;
  }();
  return api;
}

#define NCCL_CHECK(expr)                                                                                       \
  do {                                                                                                         \
    ncclResult_t _r = (expr);                                                                                  \
    if (_r != ncclSuccess)                                                                                     \
      fail(MR_ENCCL, "NCCL error %d at %s:%d (%s)", static_cast<int>(_r), __FILE__, __LINE__,                  \
           nccl_api().GetErrorString ? nccl_api().GetErrorString(_r) : "?");                                  \
  } while (0)

void grid_shape_of(int n, int* pr, int* pc) {
  switch (n) {
    case 1: *pr = 1; *pc = 1; return;
    case 2: *pr = 1; *pc = 2; return;
    case 4: *pr = 2; *pc = 2; return;
    case 8: *pr = 2; *pc = 4; return;
    default: break;
  }
  int r = 1;
  for (int d = 1; d * d <= n; ++d)
    if (n % d == 0) r = d;
  *pr = r;
  *pc = n / r;
}

}  // namespace

struct mr_grid {
  int n = 0, pr = 1, pc = 1;
  std::vector<mr_context*> ctx;       // rank -> context; rank = r * pc + c runs on device `rank`
  std::vector<ncclComm_t> comms;      // empty when NCCL could not be loaded
  std::vector<cudaEvent_t> ev_ready;  // rank -> "my slabs are complete" / "my pulls are done"
  std::vector<cudaEvent_t> ev_done;
};

struct mr_dmatrix {
  mr_grid* g = nullptr;
  int64_t nrows = 0, ncols = 0;
  int32_t blk = 0;
  int32_t pr = 1, pc = 1;             // the placement grid of THIS dataset (the grid's own shape unless re-partitioned)
  int owner(int32_t rid, int32_t cid) const { return (rid % pr) * pc + (cid % pc); }
  std::vector<mr_matrix*> part;       // rank -> the blocks that rank owns (sharded dataset)
  ~mr_dmatrix() {
    for (size_t i = 0; i < part.size(); ++i)
      if (part[i]) {
        DeviceScope dev(part[i]->ctx);
        delete part[i];
      }
  }
};

namespace {

ShardLayout layout_of(const mr_dmatrix* m, int rank) { return make_layout(m->nrows, m->ncols, m->blk, m->pr, m->pc, rank / m->pc, rank % m->pc); }

std::unique_ptr<mr_dmatrix> new_dmatrix(mr_grid* g, int64_t nrows, int64_t ncols, int32_t blk, int pr = 0, int pc = 0) {
  std::unique_ptr<mr_dmatrix> m(new mr_dmatrix);
  m->g = g;
  m->nrows = nrows;
  m->ncols = ncols;
  m->blk = blk;
  m->pr = pr > 0 ? pr : g->pr;
  m->pc = pc > 0 ? pc : g->pc;
  m->part.assign(g->n, nullptr);
  return m;
}

// An operand that lives on another placement grid is first moved to (pr, pc): repartitionWithTargetPartitioner
// (MatfastExecutionHelper.scala:34-44) -- what the reference does before every co-partitioned operator.
struct OnGrid {
  mr_dmatrix* m;
  mr_dmatrix* owned = nullptr;
  OnGrid(mr_dmatrix* a, int pr, int pc) : m(a) {
    if (a->pr != pr || a->pc != pc) {
      const mr_status st = mr_dmatrix_repartition(a, pr, pc, &owned);
      if (st != MR_OK) throw MrError{st, g_last_error};
      m = owned;
    }
  }
  ~OnGrid() {
    if (owned) mr_dmatrix_free(owned);
  }
  OnGrid(const OnGrid&) = delete;
  OnGrid& operator=(const OnGrid&) = delete;
};

// A part that is not backed by a slab in this layout (e.g. the result of an element-wise operator) is copied into one.
mr_matrix* ensure_sharded(mr_matrix* part, const ShardLayout& L, std::unique_ptr<mr_matrix>& keep) {
  if (part->shard && !part->shard->isT && part->shard->L.same_as(L)) return part;
  mr_context* ctx = part->ctx;
  keep.reset(new_sharded(ctx, L, false, true));
  std::vector<EwDesc> descs;
  int max_r = 0, max_c = 0;
  bool any_t = false;
  for (auto& kv : keep->blocks) {
    auto it = part->blocks.find(kv.first);
    if (it == part->blocks.end()) continue;  // absent block = zeros (already cleared)
    const Block& src = it->second.dense() ? it->second : it->second;  // sparse parts are densified below
    Block dense_src = src.dense() ? src : densify(ctx, src);
    wait_ready(ctx, dense_src);
    MR_REQUIRE(dense_src.numRows == kv.second.numRows && dense_src.numCols == kv.second.numCols, MR_EDIM,
               "block (%d, %d) is %d x %d, the layout expects %d x %d", kv.first.first, kv.first.second, dense_src.numRows,
               dense_src.numCols, kv.second.numRows, kv.second.numCols);
    EwDesc d{};
    d.A = dense_src.values.ptr<double>();
    d.C = kv.second.values.ptr<double>();
    d.rows = dense_src.numRows;
    d.cols = dense_src.numCols;
    d.aT = dense_src.isT;
    any_t = any_t || dense_src.isT;
    max_r = std::max(max_r, d.rows);
    max_c = std::max(max_c, d.cols);
    descs.push_back(d);
    keep->temps.push_back(dense_src.values.buf);  // densified temporaries live until the copy has run
  }
  if (!descs.empty()) {
    Buf dd = upload(ctx, descs);
    CUDA_CHECK(launch_ew_batched(EW_COPY, static_cast<const EwDesc*>(dd->p), static_cast<int>(descs.size()), max_r, max_c, any_t, ctx->stream));
    note_launch(ctx);
  }
  return keep.get();
}


// Moves every block of `A` into the slab of its owner in `res` (same GPUs, `res` carries its own dims and placement): block
// (i, j) keeps its id (re-partitioning) or becomes block (j, i) (transpose; the payload is reinterpreted, not rewritten, and the
// result's shared layout flag is set).  Blocks that stay on their GPU are copied on its stream; the others travel as one
// ncclSend / ncclRecv pair per block inside ONE group, each on its endpoint's context stream.
void move_blocks(mr_dmatrix* A, mr_dmatrix* res, bool swap_ids) {
  mr_grid* g = A->g;
  const int n = g->n;
  if (n > 1 && g->comms.empty()) fail(MR_ENCCL, "NCCL is not available (libnccl.so.2 could not be loaded or ncclCommInitAll failed)");
  std::vector<std::unique_ptr<mr_matrix>> keep(n);
  std::vector<mr_matrix*> src(n);
  for (int i = 0; i < n; ++i) {   // sources as column-major slabs
    DeviceScope dev(g->ctx[i]);
    std::lock_guard<std::mutex> lock(g->ctx[i]->mu);
    src[i] = ensure_sharded(A->part[i], A->part[i]->shard ? A->part[i]->shard->L : layout_of(A, i), keep[i]);
    wait_ready_all(g->ctx[i], src[i]);
  }
  for (int i = 0; i < n; ++i) {
    DeviceScope dev(g->ctx[i]);
    res->part[i] = new_sharded(g->ctx[i], layout_of(res, i), false, true, /*isT=*/swap_ids);
  }
  const int64_t nbr = ceil_div(A->nrows, A->blk), nbc = ceil_div(A->ncols, A->blk);
  if (n > 1) NCCL_CHECK(nccl_api().GroupStart());
  for (int64_t i = 0; i < nbr; ++i)
    for (int64_t j = 0; j < nbc; ++j) {
      const std::pair<int32_t, int32_t> sid{static_cast<int32_t>(i), static_cast<int32_t>(j)};
      const std::pair<int32_t, int32_t> did = swap_ids ? std::make_pair(sid.second, sid.first) : sid;
      const int from = A->owner(sid.first, sid.second);
      if (!src[from]->blocks.count(sid)) continue;
      const int to = res->owner(did.first, did.second);
      const Block& sb = src[from]->blocks.at(sid);
      const Block& db = res->part[to]->blocks.at(did);
      const size_t cnt = static_cast<size_t>(sb.numRows) * sb.numCols;
      if (from == to) {
        DeviceScope dev(g->ctx[to]);
        CUDA_CHECK(cudaMemcpyAsync(db.values.ptr<double>(), sb.values.ptr<double>(), cnt * sizeof(double), cudaMemcpyDeviceToDevice, g->ctx[to]->stream));
      } else {
        NCCL_CHECK(nccl_api().Send(sb.values.ptr<double>(), cnt, ncclDouble, to, g->comms[from], g->ctx[from]->stream));
        NCCL_CHECK(nccl_api().Recv(db.values.ptr<double>(), cnt, ncclDouble, from, g->comms[to], g->ctx[to]->stream));
      }
    }
  if (n > 1) NCCL_CHECK(nccl_api().GroupEnd());
  // the sources' temporaries (keep) are released stream-ordered behind the copies / sends enqueued above
}

// The common shape of rowSum / colSum / project / selection on the grid: a per-GPU operator yields pieces keyed (line, 0) (axis 0:
// the result is len x 1) or (0, line) (axis 1: 1 x len); pieces with the same key are ADDED across the GPUs and the sum becomes
// result block (line, 0) / (0, line) at its owner under A's placement.  Every GPU writes its pieces into a zeroed vector covering
// the axis (one 256-byte aligned segment per block line), ONE ncclAllReduce adds the vectors, and each owner registers its
// segments as blocks (zero-copy windows of the vector).  A line without a piece on any GPU produces no block, as in the reference.
template <typename LocalOp>
std::unique_ptr<mr_dmatrix> collect_lines(mr_dmatrix* A, int axis, int64_t len, LocalOp&& local) {
  mr_grid* g = A->g;
  const int n = g->n;
  if (n > 1 && g->comms.empty()) fail(MR_ENCCL, "NCCL is not available (libnccl.so.2 could not be loaded or ncclCommInitAll failed)");
  const int64_t nlines = ceil_div(len, A->blk);
  const int64_t seg = static_cast<int64_t>(align_up(static_cast<size_t>(A->blk) * sizeof(double)) / sizeof(double));  // doubles per segment
  const size_t bytes = static_cast<size_t>(nlines) * seg * sizeof(double);
  std::vector<Buf> vec(n);
  std::vector<char> present(static_cast<size_t>(nlines), 0);
  for (int i = 0; i < n; ++i) {
    mr_context* ctx = g->ctx[i];
    DeviceScope dev(ctx);
    mr_matrix* s = nullptr;
    const mr_status st = local(A->part[i], &s);
    if (st != MR_OK) throw MrError{st, g_last_error};
    std::unique_ptr<mr_matrix> hold(s);
    vec[i] = std::make_shared<DevBuf>(ctx, std::max<size_t>(bytes, 16));
    CUDA_CHECK(cudaMemsetAsync(vec[i]->p, 0, bytes, ctx->stream));
    for (auto& kv : s->blocks) {
      const int64_t line = axis == 0 ? kv.first.first : kv.first.second;
      const int64_t cnt = static_cast<int64_t>(kv.second.numRows) * kv.second.numCols;
      MR_REQUIRE(line >= 0 && line < nlines && cnt == std::min<int64_t>(A->blk, len - line * A->blk), MR_EDIM,
                 "piece (%d, %d) holds %lld elements, the %lld x %lld matrix in %d-blocks expects %lld", kv.first.first, kv.first.second,
                 (long long)cnt, (long long)A->nrows, (long long)A->ncols, A->blk, (long long)std::min<int64_t>(A->blk, len - line * A->blk));
      present[static_cast<size_t>(line)] = 1;
      wait_ready(ctx, kv.second);
      CUDA_CHECK(cudaMemcpyAsync(static_cast<double*>(vec[i]->p) + line * seg, kv.second.values.ptr<double>(),
                                 static_cast<size_t>(cnt) * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    }
  }
  if (n > 1) {
    NCCL_CHECK(nccl_api().GroupStart());
    for (int i = 0; i < n; ++i)
      NCCL_CHECK(nccl_api().AllReduce(vec[i]->p, vec[i]->p, static_cast<size_t>(nlines * seg), ncclDouble, ncclSum, g->comms[i], g->ctx[i]->stream));
    NCCL_CHECK(nccl_api().GroupEnd());
  }
  auto res = new_dmatrix(g, axis == 0 ? len : 1, axis == 0 ? 1 : len, A->blk, A->pr, A->pc);
  for (int i = 0; i < n; ++i) {
    DeviceScope dev(g->ctx[i]);
    std::unique_ptr<mr_matrix> p(new_matrix(g->ctx[i]));
    for (int64_t line = 0; line < nlines; ++line) {
      if (!present[static_cast<size_t>(line)]) continue;
      const int32_t rid = axis == 0 ? static_cast<int32_t>(line) : 0, cid = axis == 0 ? 0 : static_cast<int32_t>(line);
      if (res->owner(rid, cid) != i) continue;
      const int32_t cnt = static_cast<int32_t>(std::min<int64_t>(A->blk, len - line * A->blk));
      Span sp{vec[i], static_cast<size_t>(line * seg) * sizeof(double)};
      p->blocks[{rid, cid}] = axis == 0 ? dense_block(cnt, 1, sp) : dense_block(1, cnt, sp);
    }
    res->part[i] = p.release();
  }
  return res;
}

}  // namespace

extern "C" {

mr_status mr_init_grid(const mr_options* opts, int32_t ngpus, mr_grid** out) {
  return guarded([&] {
    MR_REQUIRE(out != nullptr && ngpus >= 1, MR_EINVAL, "bad argument");
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
      (void)cudaGetLastError();
      fail(MR_ECUDA, "no usable CUDA device: the engine has no CPU fallback");
    }
    MR_REQUIRE(ngpus <= count, MR_EINVAL, "grid of %d GPUs requested, %d visible", ngpus, count);
    std::unique_ptr<mr_grid> g(new mr_grid);
    g->n = ngpus;
    grid_shape_of(ngpus, &g->pr, &g->pc);
    for (int i = 0; i < ngpus; ++i) {
      mr_options o{};
      if (opts) o = *opts;
      o.device = i;
      o.stream = nullptr;
      mr_context* c = nullptr;
      const mr_status st = mr_init(&o, &c);
      if (st != MR_OK) {
        for (mr_context* x : g->ctx) mr_shutdown(x);
        throw MrError{st, g_last_error};
      }
      g->ctx.push_back(c);
    }
    // peer access in both directions, for plain allocations and for the stream-ordered pools the operator results come from
    for (int i = 0; i < ngpus; ++i) {
      CUDA_CHECK(cudaSetDevice(i));
      cudaMemPool_t pool;
      CUDA_CHECK(cudaDeviceGetDefaultMemPool(&pool, i));
      for (int j = 0; j < ngpus; ++j) {
        if (i == j) continue;
        int can = 0;
        CUDA_CHECK(cudaDeviceCanAccessPeer(&can, j, i));
        if (!can) fail(MR_ECUDA, "device %d cannot access device %d: the grid needs NVLink / PCIe peer access", j, i);
        cudaError_t e = cudaDeviceEnablePeerAccess(j, 0);  // i may read j
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CUDA_CHECK(e);
        (void)cudaGetLastError();
        cudaMemAccessDesc d{};
        d.location.type = cudaMemLocationTypeDevice;
        d.location.id = j;
        d.flags = cudaMemAccessFlagsProtReadWrite;
        CUDA_CHECK(cudaMemPoolSetAccess(pool, &d, 1));  // j may access i's pool
      }
      cudaEvent_t e1, e2;
      CUDA_CHECK(cudaEventCreateWithFlags(&e1, cudaEventDisableTiming));
      CUDA_CHECK(cudaEventCreateWithFlags(&e2, cudaEventDisableTiming));
      g->ev_ready.push_back(e1);
      g->ev_done.push_back(e2);
    }
    if (ngpus > 1 && nccl_api().ok()) {
      std::vector<int> devs(ngpus);
      for (int i = 0; i < ngpus; ++i) devs[i] = i;
      g->comms.assign(ngpus, nullptr);
      ncclResult_t r = nccl_api().CommInitAll(g->comms.data(), ngpus, devs.data());
      if (r != ncclSuccess) g->comms.clear();  // the pulls do not need it; the reductions report MR_ENCCL
    }
    CUDA_CHECK(cudaSetDevice(0));
    *out = g.release();
  });
}

mr_status mr_grid_shutdown(mr_grid* g) {
  return guarded([&] {
    if (!g) return;
    for (int i = 0; i < g->n; ++i) {
      cudaSetDevice(i);
      if (i < static_cast<int>(g->comms.size()) && g->comms[i]) nccl_api().CommDestroy(g->comms[i]);
      cudaEventDestroy(g->ev_ready[i]);
      cudaEventDestroy(g->ev_done[i]);
    }
    for (mr_context* c : g->ctx) mr_shutdown(c);
    cudaSetDevice(0);
    delete g;
  });
}

mr_status mr_grid_info(const mr_grid* g, int32_t* ngpus, int32_t* pr, int32_t* pc, int32_t* has_nccl) {
  return guarded([&] {
    MR_REQUIRE(g != nullptr, MR_EINVAL, "grid is null");
    if (ngpus) *ngpus = g->n;
    if (pr) *pr = g->pr;
    if (pc) *pc = g->pc;
    if (has_nccl) *has_nccl = g->comms.empty() ? 0 : 1;
  });
}

mr_status mr_grid_context(mr_grid* g, int32_t rank, mr_context** ctx) {
  return guarded([&] {
    MR_REQUIRE(g != nullptr && ctx != nullptr && rank >= 0 && rank < g->n, MR_EINVAL, "bad argument");
    *ctx = g->ctx[rank];
  });
}

mr_status mr_grid_sync(mr_grid* g) {
  return guarded([&] {
    MR_REQUIRE(g != nullptr, MR_EINVAL, "grid is null");
    for (mr_context* c : g->ctx) {
      DeviceScope dev(c);
      CUDA_CHECK(cudaStreamSynchronize(c->p2p_stream));
      const mr_status st = mr_sync(c);
      if (st != MR_OK) throw MrError{st, g_last_error};
    }
  });
}

mr_status mr_dmatrix_create(mr_grid* g, int64_t nrows, int64_t ncols, int32_t blkSize, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(g != nullptr && out != nullptr, MR_EINVAL, "null argument");
    mr_grid_layout chk{nrows, ncols, blkSize, g->pr, g->pc, 0, 0};
    validate_layout(&chk);
    auto m = new_dmatrix(g, nrows, ncols, blkSize);
    for (int i = 0; i < g->n; ++i) {
      DeviceScope dev(g->ctx[i]);
      m->part[i] = new_sharded(g->ctx[i], layout_of(m.get(), i), false, true);
    }
    *out = m.release();
  });
}

mr_status mr_dmatrix_free(mr_dmatrix* m) {
  return guarded([&] { delete m; });
}

mr_status mr_dmatrix_part(mr_dmatrix* m, int32_t rank, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && out != nullptr && rank >= 0 && rank < m->g->n, MR_EINVAL, "bad argument");
    *out = m->part[rank];
  });
}

mr_status mr_dmatrix_dims(const mr_dmatrix* m, int64_t* nrows, int64_t* ncols, int32_t* blkSize) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr, MR_EINVAL, "null argument");
    if (nrows) *nrows = m->nrows;
    if (ncols) *ncols = m->ncols;
    if (blkSize) *blkSize = m->blk;
  });
}

// The rank that owns block (rid, cid): RowPartitioner x ColumnPartitioner arithmetic on the grid.
mr_status mr_dmatrix_owner(const mr_dmatrix* m, int32_t rid, int32_t cid, int32_t* rank) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && rank != nullptr && rid >= 0 && cid >= 0, MR_EINVAL, "bad argument");
    *rank = m->owner(rid, cid);
  });
}

mr_status mr_dmatrix_put_block(mr_dmatrix* m, int32_t rid, int32_t cid, const mr_block_desc* blk) {
  if (!m || rid < 0 || cid < 0) {
    g_last_error = "requirement failed: bad argument";
    return MR_EINVAL;
  }
  return mr_matrix_put_block(m->part[m->owner(rid, cid)], rid, cid, blk);
}

mr_status mr_dmatrix_has_block(const mr_dmatrix* m, int32_t rid, int32_t cid, int32_t* out) {
  if (!m || rid < 0 || cid < 0) {
    g_last_error = "requirement failed: bad argument";
    return MR_EINVAL;
  }
  return mr_matrix_has_block(m->part[m->owner(rid, cid)], rid, cid, out);
}

mr_status mr_dmatrix_get_block(mr_dmatrix* m, int32_t rid, int32_t cid, mr_block_desc* inout) {
  if (!m || rid < 0 || cid < 0) {
    g_last_error = "requirement failed: bad argument";
    return MR_EINVAL;
  }
  return mr_matrix_get_block(m->part[m->owner(rid, cid)], rid, cid, inout);
}

mr_status mr_dmatrix_num_blocks(const mr_dmatrix* m, int64_t* out) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && out != nullptr, MR_EINVAL, "null argument");
    int64_t n = 0;
    for (mr_matrix* p : m->part) n += static_cast<int64_t>(p->blocks.size());
    *out = n;
  });
}

mr_status mr_dmatrix_rand(mr_grid* g, int64_t nrows, int64_t ncols, int32_t blkSize, int64_t seed0, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(g != nullptr && out != nullptr, MR_EINVAL, "null argument");
    mr_grid_layout chk{nrows, ncols, blkSize, g->pr, g->pc, 0, 0};
    validate_layout(&chk);
    auto m = new_dmatrix(g, nrows, ncols, blkSize);
    for (int i = 0; i < g->n; ++i) {
      mr_context* ctx = g->ctx[i];
      DeviceScope dev(ctx);
      const ShardLayout L = layout_of(m.get(), i);
      m->part[i] = new_sharded(ctx, L, false, true);
      std::vector<RandDesc> descs;
      int64_t max_n = 0;
      for (auto& kv : m->part[i]->blocks) {
        const int64_t cnt = static_cast<int64_t>(kv.second.numRows) * kv.second.numCols;
        descs.push_back(RandDesc{kv.second.values.ptr<double>(), cnt, seed0 + static_cast<int64_t>(kv.first.first) * L.nbc + kv.first.second});
        max_n = std::max(max_n, cnt);
      }
      for (size_t off = 0; off < descs.size(); off += 65535) {
        std::vector<RandDesc> chunk(descs.begin() + off, descs.begin() + std::min(descs.size(), off + 65535));
        Buf d = upload(ctx, chunk);
        CUDA_CHECK(launch_java_rand_batched(static_cast<const RandDesc*>(d->p), static_cast<int>(chunk.size()), max_n, ctx->stream));
        note_launch(ctx);
      }
    }
    *out = m.release();
  });
}

// Dataset.matrixMultiply (M/Dataset.scala:134-142) on the grid: dimensions and block size come from the handles.
mr_status mr_dmatrix_multiply(mr_dmatrix* A_in, mr_dmatrix* B_in, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(A_in && B_in && out, MR_EINVAL, "null argument");
    MR_REQUIRE(A_in->g == B_in->g, MR_EINVAL, "operands live on different grids");
    MR_REQUIRE(A_in->blk == B_in->blk, MR_EINVAL, "operands have different block sizes (%d, %d)", A_in->blk, B_in->blk);
    MR_REQUIRE(A_in->ncols == B_in->nrows, MR_EDIM, "Matrix dimension not match, leftColNum = %lld, rightRowNum = %lld",
               (long long)A_in->ncols, (long long)B_in->nrows);
    mr_grid* g = A_in->g;
    OnGrid ga(A_in, g->pr, g->pc), gb(B_in, g->pr, g->pc);   // the multiply runs on the grid's own (C-stationary) placement
    mr_dmatrix *A = ga.m, *B = gb.m;
    const int n = g->n, pr = g->pr, pc = g->pc;
    // operands in slab form on every rank
    std::vector<std::unique_ptr<mr_matrix>> keepA(n), keepB(n);
    std::vector<mr_matrix*> pa(n), pb(n);
    for (int i = 0; i < n; ++i) {
      DeviceScope dev(g->ctx[i]);
      std::lock_guard<std::mutex> lock(g->ctx[i]->mu);
      pa[i] = ensure_sharded(A->part[i], layout_of(A, i), keepA[i]);
      pb[i] = ensure_sharded(B->part[i], layout_of(B, i), keepB[i]);
      // "my slabs are complete once everything enqueued so far on my streams has run"
      CUDA_CHECK(cudaStreamWaitEvent(g->ctx[i]->stream, [&] {
        CUDA_CHECK(cudaEventRecord(g->ctx[i]->ev_alloc, g->ctx[i]->h2d_stream));
        return g->ctx[i]->ev_alloc;
      }(), 0));
      CUDA_CHECK(cudaEventRecord(g->ev_ready[i], g->ctx[i]->stream));
    }
    auto res = new_dmatrix(g, A->nrows, B->ncols, A->blk);
    for (int i = 0; i < n; ++i) {
      mr_context* ctx = g->ctx[i];
      DeviceScope dev(ctx);
      const int r = i / pc, c = i % pc;
      std::vector<const double*> rowA(pc), colB(pr);
      for (int cc = 0; cc < pc; ++cc) {
        const int peer = r * pc + cc;
        rowA[cc] = static_cast<const double*>(pa[peer]->shard->slab->p);
        if (peer != i) CUDA_CHECK(cudaStreamWaitEvent(ctx->p2p_stream, g->ev_ready[peer], 0));
      }
      for (int rr = 0; rr < pr; ++rr) {
        const int peer = rr * pc + c;
        colB[rr] = static_cast<const double*>(pb[peer]->shard->slab->p);
        if (peer != i) CUDA_CHECK(cudaStreamWaitEvent(ctx->p2p_stream, g->ev_ready[peer], 0));
      }
      mr_matrix* cpart = nullptr;
      const mr_status st = mr_grid_multiply(pa[i], pb[i], rowA.data(), colB.data(), 4, &cpart);
      if (st != MR_OK) throw MrError{st, g_last_error};
      res->part[i] = cpart;
      CUDA_CHECK(cudaEventRecord(g->ev_done[i], ctx->p2p_stream));
    }
    // nobody may release / overwrite an operand slab before every peer's pulls from it have run
    for (int i = 0; i < n; ++i) {
      DeviceScope dev(g->ctx[i]);
      const int r = i / pc, c = i % pc;
      for (int cc = 0; cc < pc; ++cc)
        if (cc != c) CUDA_CHECK(cudaStreamWaitEvent(g->ctx[i]->stream, g->ev_done[r * pc + cc], 0));
      for (int rr = 0; rr < pr; ++rr)
        if (rr != r) CUDA_CHECK(cudaStreamWaitEvent(g->ctx[i]->stream, g->ev_done[rr * pc + c], 0));
    }
    *out = res.release();
  });
}

// Co-partitioned element-wise operators (MatrixElement{Add,Multiply,Divide}Execution, the zipPartitions fast path of
// MatfastExecutionHelper.scala:64-173): op 0 = add, 1 = multiply, 2 = divide.  Both operands live on the same grid with the same
// placement function, so no block moves.
mr_status mr_dmatrix_elementwise(int32_t op, mr_dmatrix* A, mr_dmatrix* B_in, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(A && B_in && out, MR_EINVAL, "null argument");
    MR_REQUIRE(A->g == B_in->g, MR_EINVAL, "operands live on different grids");
    MR_REQUIRE(op >= 0 && op <= 2, MR_EINVAL, "unknown element-wise op %d", op);
    // MatrixElementAddExecution picks the left operand's partitioner (MatfastExecution.scala:590-606) and re-partitions the right
    OnGrid gb(B_in, A->pr, A->pc);
    mr_dmatrix* B = gb.m;
    auto res = new_dmatrix(A->g, A->nrows, A->ncols, A->blk, A->pr, A->pc);
    for (int i = 0; i < A->g->n; ++i) {
      DeviceScope dev(A->g->ctx[i]);
      mr_matrix* o = nullptr;
      auto fn = op == 0 ? mr_add_element : (op == 1 ? mr_multiply_element : mr_divide_element);
      const mr_status st = fn(A->part[i], A->nrows, A->ncols, B->part[i], B->nrows, B->ncols, A->blk, &o);
      if (st != MR_OK) throw MrError{st, g_last_error};
      res->part[i] = o;
    }
    *out = res.release();
  });
}

// Dataset.sum / trace (M/Dataset.scala:73-82; SumDirectExecution / TraceDirectExecution + reduceByKey(add)): the local reduction
// kernel on every GPU, then ONE ncclAllReduce of a scalar over the grid (the reference reduces through a shuffle).
mr_status mr_dmatrix_reduce_scalar(mr_dmatrix* A, int32_t what /* 0 = sum, 1 = trace */, double* value) {
  return guarded([&] {
    MR_REQUIRE(A && value, MR_EINVAL, "null argument");
    mr_grid* g = A->g;
    const int n = g->n;
    std::vector<Buf> acc(n);
    for (int i = 0; i < n; ++i) {
      mr_context* ctx = g->ctx[i];
      DeviceScope dev(ctx);
      mr_matrix* s = nullptr;
      const mr_status st = what == 0 ? mr_sum(A->part[i], A->nrows, A->ncols, &s) : mr_trace(A->part[i], A->nrows, A->ncols, &s);
      if (st != MR_OK) throw MrError{st, g_last_error};
      std::unique_ptr<mr_matrix> hold(s);
      acc[i] = std::make_shared<DevBuf>(ctx, sizeof(double));
      CUDA_CHECK(cudaMemsetAsync(acc[i]->p, 0, sizeof(double), ctx->stream));
      auto it = s->blocks.find({0, 0});
      if (it != s->blocks.end())
        CUDA_CHECK(cudaMemcpyAsync(acc[i]->p, it->second.values.ptr<double>(), sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    }
    if (n > 1) {
      if (g->comms.empty()) fail(MR_ENCCL, "NCCL is not available (libnccl.so.2 could not be loaded or ncclCommInitAll failed)");
      NCCL_CHECK(nccl_api().GroupStart());
      for (int i = 0; i < n; ++i) NCCL_CHECK(nccl_api().AllReduce(acc[i]->p, acc[i]->p, 1, ncclDouble, ncclSum, g->comms[i], g->ctx[i]->stream));
      NCCL_CHECK(nccl_api().GroupEnd());
    }
    DeviceScope dev(g->ctx[0]);
    CUDA_CHECK(cudaMemcpyAsync(value, acc[0]->p, sizeof(double), cudaMemcpyDeviceToHost, g->ctx[0]->stream));
    CUDA_CHECK(cudaStreamSynchronize(g->ctx[0]->stream));
  });
}

// Dataset.rowSum / colSum (M/Dataset.scala:63-72; RowSumDirectExecution / ColumnSumDirectExecution, M/execution/MatfastExecution.scala
// :239-370: per-block line sums, then reduceByKey(add) over the block row / block column): axis 0 = rowSum (nrows x 1), 1 = colSum
// (1 x ncols).  collect_lines() does the work: local kernels, ONE ncclAllReduce of a vector -- the shuffle of the reference.
mr_status mr_dmatrix_axis_sum(mr_dmatrix* A, int32_t axis, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(A && out, MR_EINVAL, "null argument");
    MR_REQUIRE(axis == 0 || axis == 1, MR_EINVAL, "axis must be 0 (rowSum) or 1 (colSum), got %d", axis);
    *out = collect_lines(A, axis, axis == 0 ? A->nrows : A->ncols, [&](mr_matrix* part, mr_matrix** o) {
             return axis == 0 ? mr_row_sum(part, A->nrows, A->ncols, o) : mr_col_sum(part, A->nrows, A->ncols, o);
           }).release();
  });
}

// Dataset.project (M/Dataset.scala:38-47; ProjectRow / ProjectColumnDirectExecution, M/execution/MatfastExecution.scala:31-169): row
// `index` as a 1 x ncols dataset (rowOrCol != 0) or column `index` as nrows x 1.  The GPUs that own blocks of the block row /
// block column extract their pieces; the same vector all-reduce brings every piece to the owner of its result block (the other
// GPUs contribute zeros), which is the re-keying to (0, cid) / (rid, 0) plus the shuffle the reference's next operator would do.
mr_status mr_dmatrix_project(mr_dmatrix* A, int32_t rowOrCol, int64_t index, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(A && out, MR_EINVAL, "null argument");
    *out = collect_lines(A, rowOrCol ? 1 : 0, rowOrCol ? A->ncols : A->nrows, [&](mr_matrix* part, mr_matrix** o) {
             return mr_project(part, A->nrows, A->ncols, A->blk, rowOrCol, index, o);
           }).release();
  });
}

// Dataset.selection (M/Dataset.scala:49-55; SelectDirectExecution, M/execution/MatfastExecution.scala:171-213): entry (rowIdx, colIdx)
// as a 1 x 1 dataset whose block (0, 0) lives on rank 0.
mr_status mr_dmatrix_selection(mr_dmatrix* A, int64_t rowIdx, int64_t colIdx, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(A && out, MR_EINVAL, "null argument");
    *out = collect_lines(A, 0, 1, [&](mr_matrix* part, mr_matrix** o) {
             return mr_selection(part, A->nrows, A->ncols, A->blk, rowIdx, colIdx, o);
           }).release();
  });
}

// repartitionWithTargetPartitioner (M/execution/MatfastExecutionHelper.scala:34-44) between two grids of the same GPUs: every
// block moves from its owner under (pr, pc) to its owner under (new_pr, new_pc) -- the all-to-all permutation that replaces the
// reference's ShuffledRDD, as grouped ncclSend / ncclRecv straight between the slabs (one message per block).  new_pr x new_pc
// must cover the same GPUs: (P, 1) = RowPartitioner, (1, P) = ColumnPartitioner, (pr, pc) = the multiply's grid.
mr_status mr_dmatrix_repartition(mr_dmatrix* A, int32_t new_pr, int32_t new_pc, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(A && out, MR_EINVAL, "null argument");
    mr_grid* g = A->g;
    MR_REQUIRE(new_pr > 0 && new_pc > 0 && new_pr * new_pc == g->n, MR_EINVAL, "%d x %d does not cover the %d GPUs of the grid", new_pr,
               new_pc, g->n);
    auto res = new_dmatrix(g, A->nrows, A->ncols, A->blk, new_pr, new_pc);
    move_blocks(A, res.get(), /*swap_ids=*/false);
    *out = res.release();
  });
}

// Dataset.t / transpose (M/Dataset.scala:57-61; MatrixTransposeExecution, M/execution/MatfastExecution.scala:215-236: a key swap
// (rid, cid) -> (cid, rid) plus the isTransposed flag flip of MLMatrix.scala:312) on the grid: block (i, j) of A becomes block
// (j, i) of the result on the SAME placement function, i.e. it moves from rank (i % pr, j % pc) to rank (j % pr, i % pc) -- the
// re-placement the reference's next shuffle would do -- as grouped ncclSend / ncclRecv between the slabs.  Payloads are not
// touched: a column-major block IS the row-major block of the transpose, so the result is a sharded dataset whose shared
// isTransposed flag is set (operators that need column-major slabs normalise it on the device, ensure_sharded).
mr_status mr_dmatrix_transpose(mr_dmatrix* A, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(A && out, MR_EINVAL, "null argument");
    auto res = new_dmatrix(A->g, A->ncols, A->nrows, A->blk, A->pr, A->pc);
    move_blocks(A, res.get(), /*swap_ids=*/true);
    *out = res.release();
  });
}

// Dataset.addScalar / multiplyScalar / power (M/Dataset.scala:89-103; MatrixScalar{Add,Multiply}Execution, MatrixPowerExecution,
// M/execution/MatfastExecution.scala:465-532: a map over the blocks, no shuffle): op 0 = add, 1 = multiply, 2 = power.  Every
// GPU maps the blocks it owns; placement, layout flags and sparsity structure are preserved (LocalMatrix.scala:411-426,931-980).
mr_status mr_dmatrix_scalar(int32_t op, mr_dmatrix* A, double alpha, mr_dmatrix** out) {
  return guarded([&] {
    MR_REQUIRE(A && out, MR_EINVAL, "null argument");
    MR_REQUIRE(op >= 0 && op <= 2, MR_EINVAL, "unknown scalar op %d", op);
    auto res = new_dmatrix(A->g, A->nrows, A->ncols, A->blk, A->pr, A->pc);
    for (int i = 0; i < A->g->n; ++i) {
      DeviceScope dev(A->g->ctx[i]);
      mr_matrix* o = nullptr;
      auto fn = op == 0 ? mr_add_scalar : (op == 1 ? mr_multiply_scalar : mr_power);
      const mr_status st = fn(A->part[i], alpha, &o);
      if (st != MR_OK) throw MrError{st, g_last_error};
      res->part[i] = o;
    }
    *out = res.release();
  });
}

}  // extern "C"
