// C-ABI host layer of the H100 block-matrix engine (see include/matrel.h): context lifetime, device memory, block ingest /
// egress and the helpers shared by the operator files (abi_multiply.cpp, abi_elementwise.cpp, abi_aggregate.cpp,
// abi_partition.cpp).
//
// This file is the replacement for the reference's L2 physical operators and their helpers:
//   MatfastExecution.scala   (MatrixMatrixMultiplicationExecution :688-726, MatrixTransposeExecution
//                             :215-236, MatrixElement*Execution :571-686, MatrixScalar*/Power :465-532,
//                             RankOneUpdateExecution :728-747)
//   MatfastExecutionHelper.scala (matrixMultiplyGeneral :235-263, multiplyOuterProductDuplicate* :175-221,
//                             add/multiply/divideWithPartitioner :64-173, matrixRankOneUpdate :265-285,
//                             genBlockCyclicPartitioner :46-62)
//   LocalMatrix.scala        (matrixMultiplication dispatch :889-914 and the per-block kernels)
//   MLMatrixSerializer.scala (block <-> 7-field struct, :26-69)
// The Spark shuffles (groupByKey / join / reduceByKey / zipPartitions) become index arithmetic over a
// device-resident block table; every arithmetic step is a CUDA kernel (gemm_f64.cu, ew.cu).
// There is no CPU compute path in this file: host code only validates, builds descriptor tables
// and launches.
#include <cstdlib>

#include "host.h"

using namespace matrel;
using namespace mrhost;

namespace mrhost {

thread_local std::string g_last_error;

// release threshold of each device's default memory pool before the first context on it raised it (restored by the last one)
constexpr int kMaxPoolDevices = 64;
std::mutex g_pool_mu;
int g_pool_users[kMaxPoolDevices] = {};
uint64_t g_pool_threshold_before[kMaxPoolDevices] = {};

[[noreturn]] void fail(mr_status code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  throw MrError{code, buf};
}

void note_launch(mr_context* ctx, int n) { ctx->stats.kernel_launches += n; }

// Order the context stream after the producer of a block.  Returns true when the producer was still running.
bool wait_ready(mr_context* ctx, const Block& b) {
  if (!b.ready) return false;
  const cudaError_t q = cudaEventQuery(b.ready->ev);
  if (q == cudaSuccess) {
    b.ready.reset();  // never query this block again
    b.settled = true;
    return false;
  }
  (void)cudaGetLastError();
  cudaStreamWaitEvent(ctx->stream, b.ready->ev, 0);
  return true;
}
bool wait_ready_on(cudaStream_t stream, const Block& b) {  // same, ordering `stream` instead of the context stream
  if (!b.ready) return false;
  const cudaError_t q = cudaEventQuery(b.ready->ev);
  if (q == cudaSuccess) {
    b.ready.reset();
    b.settled = true;
    return false;
  }
  (void)cudaGetLastError();
  cudaStreamWaitEvent(stream, b.ready->ev, 0);
  return true;
}
// true when the block's producer has finished (and forgets the event so it is not queried again)
bool block_done(const Block& b) {
  if (!b.ready) return true;
  if (cudaEventQuery(b.ready->ev) == cudaSuccess) {
    b.ready.reset();
    b.settled = true;
    return true;
  }
  (void)cudaGetLastError();
  return false;
}
bool wait_ready_all(mr_context* ctx, const mr_matrix* m) {
  bool any = false;
  for (auto& kv : m->blocks) any = wait_ready(ctx, kv.second) || any;
  return any;
}

// Descriptor tables (a few hundred KB per operator) travel through a mapped pinned staging ring and an SM-driven copy
// kernel instead of cudaMemcpyAsync: on the H2D copy engine they would queue behind every block upload already
// submitted on the ingest stream, and the first chunk of a pipelined multiply could not start until ALL operands had
// landed.  Ring regions are only reused after a stream synchronisation (on wrap-around).
Buf upload_bytes(mr_context* ctx, const void* data, size_t bytes) {
  Buf b = std::make_shared<DevBuf>(ctx, std::max<size_t>((bytes + 3) / 4 * 4, 16));
  if (bytes == 0) return b;
  const size_t need = align_up(bytes);
  if (ctx->stage_host != nullptr && need <= ctx->stage_cap / 2) {
    if (ctx->stage_off + need > ctx->stage_cap) {
      CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
      ctx->stage_off = 0;
    }
    std::memcpy(ctx->stage_host + ctx->stage_off, data, bytes);
    CUDA_CHECK(launch_copy_words(b->p, ctx->stage_dev + ctx->stage_off, bytes, ctx->stream));
    ctx->stage_off += need;
  } else {
    CUDA_CHECK(cudaMemcpyAsync(b->p, data, bytes, cudaMemcpyHostToDevice, ctx->stream));
  }
  ctx->stats.h2d_bytes += static_cast<int64_t>(bytes);
  return b;
}

Block dense_block(int32_t rows, int32_t cols, Span values, bool isT) {
  Block b;
  b.type = 1;
  b.numRows = rows;
  b.numCols = cols;
  b.isT = isT;
  b.values = std::move(values);
  b.valuesLen = static_cast<int64_t>(rows) * cols;
  return b;
}

// SparseMatrix.toDense (MLMatrix.scala:669-671) on the device: zero fill + scatter.
Block densify(mr_context* ctx, const Block& s) {
  const size_t bytes = static_cast<size_t>(s.numRows) * s.numCols * sizeof(double);
  Span v{std::make_shared<DevBuf>(ctx, std::max<size_t>(bytes, 16)), 0};
  if (bytes) CUDA_CHECK(cudaMemsetAsync(v.ptr<double>(), 0, bytes, ctx->stream));
  if (s.valuesLen > 0) {
    CUDA_CHECK(launch_sparse_to_dense(s.colPtrs.ptr<int32_t>(), s.rowIndices.ptr<int32_t>(), s.values.ptr<double>(),
                                      s.isT, v.ptr<double>(), s.numRows, s.numCols, ctx->stream));
    note_launch(ctx);
  }
  return dense_block(s.numRows, s.numCols, v, false);
}

const char* type_name(const Block& b) { return b.dense() ? "DenseMatrix" : "SparseMatrix"; }

int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
// ------------------------------------------------------------------------------------------------
// dense window -> CSC compaction (DenseMatrix.toSparse, MLMatrix.scala:392-420), batched
// ------------------------------------------------------------------------------------------------
// Per-column counts of entries != 0.0 (NaN counts, as in the reference's `arr(i) != 0`): one launch + one sync.
std::vector<std::vector<int32_t>> column_counts(mr_context* ctx, const std::vector<DenseWin>& wins) {
  std::vector<std::vector<int32_t>> out(wins.size());
  if (wins.empty()) return out;
  size_t ncols_total = 0;
  int maxc = 0;
  for (auto& w : wins) {
    ncols_total += static_cast<size_t>(w.cols);
    maxc = std::max(maxc, w.cols);
  }
  Buf counts = std::make_shared<DevBuf>(ctx, std::max<size_t>(ncols_total * sizeof(int32_t), 16));
  std::vector<CscDesc> cd(wins.size());
  size_t off = 0;
  for (size_t i = 0; i < wins.size(); ++i) {
    cd[i] = CscDesc{wins[i].p, wins[i].rows, wins[i].cols, static_cast<int32_t*>(counts->p) + off, nullptr, nullptr, nullptr};
    off += static_cast<size_t>(wins[i].cols);
  }
  Buf dcd = upload(ctx, cd);
  CUDA_CHECK(launch_csc_count(static_cast<const CscDesc*>(dcd->p), static_cast<int>(cd.size()), maxc, ctx->stream));
  note_launch(ctx);
  std::vector<int32_t> h(ncols_total);
  if (ncols_total) {
    CUDA_CHECK(cudaMemcpyAsync(h.data(), counts->p, ncols_total * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    ctx->stats.d2h_bytes += static_cast<int64_t>(ncols_total * sizeof(int32_t));
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  off = 0;
  for (size_t i = 0; i < wins.size(); ++i) {
    out[i].assign(h.begin() + static_cast<std::ptrdiff_t>(off), h.begin() + static_cast<std::ptrdiff_t>(off + wins[i].cols));
    off += static_cast<size_t>(wins[i].cols);
  }
  return out;
}

int64_t total_count(const std::vector<int32_t>& counts) {
  int64_t n = 0;
  for (int32_t c : counts) n += c;
  return n;
}

// CSC blocks (isTransposed = false) of the windows, given their column counts: one launch.
std::vector<Block> compact_csc(mr_context* ctx, const std::vector<DenseWin>& wins, const std::vector<std::vector<int32_t>>& counts) {
  std::vector<Block> out;
  std::vector<CscDesc> fill;
  int maxc = 0;
  for (size_t i = 0; i < wins.size(); ++i) {
    const int rows = wins[i].rows, cols = wins[i].cols;
    std::vector<int32_t> ptrs(static_cast<size_t>(cols) + 1, 0);
    for (int c = 0; c < cols; ++c) ptrs[c + 1] = ptrs[c] + counts[i][c];
    const int64_t nnz = ptrs[cols];
    Block sb;
    sb.type = 0;
    sb.numRows = rows;
    sb.numCols = cols;
    sb.isT = false;
    sb.valuesLen = nnz;
    sb.colPtrsLen = cols + 1;
    sb.colPtrs = upload_raw(ctx, ptrs.data(), ptrs.size() * sizeof(int32_t));
    sb.rowIndices = Span{std::make_shared<DevBuf>(ctx, std::max<size_t>(nnz * sizeof(int32_t), 16)), 0};
    sb.values = Span{std::make_shared<DevBuf>(ctx, std::max<size_t>(nnz * sizeof(double), 16)), 0};
    fill.push_back(CscDesc{wins[i].p, rows, cols, nullptr, sb.colPtrs.ptr<int32_t>(), sb.rowIndices.ptr<int32_t>(),
                           sb.values.ptr<double>()});
    maxc = std::max(maxc, cols);
    out.push_back(std::move(sb));
  }
  if (!fill.empty()) {
    Buf dfill = upload(ctx, fill);
    CUDA_CHECK(launch_csc_fill(static_cast<const CscDesc*>(dfill->p), static_cast<int>(fill.size()), maxc, ctx->stream));
    note_launch(ctx);
  }
  return out;
}
mr_matrix* new_matrix(mr_context* ctx) {
  auto* m = new mr_matrix;
  m->ctx = ctx;
  return m;
}

void validate_desc(const mr_block_desc* d) {
  MR_REQUIRE(d != nullptr, MR_EINVAL, "block descriptor is null");
  MR_REQUIRE(d->numRows >= 0 && d->numCols >= 0, MR_EINVAL, "negative block dimensions %d x %d", d->numRows, d->numCols);
  if (d->type == 1) {
    // DenseMatrix ctor (MLMatrix.scala:240)
    MR_REQUIRE(d->valuesLen == static_cast<int64_t>(d->numRows) * d->numCols, MR_EINVAL,
               "The number of values supplied doesn't match the size of the matrix! values.length: %lld, "
               "numRows * numCols: %lld",
               (long long)d->valuesLen, (long long)(static_cast<int64_t>(d->numRows) * d->numCols));
    MR_REQUIRE(d->valuesLen == 0 || d->values != nullptr, MR_EINVAL, "values is null");
  } else if (d->type == 0) {
    // SparseMatrix ctor (MLMatrix.scala:533-542)
    MR_REQUIRE(d->valuesLen == d->rowIndicesLen, MR_EINVAL,
               "The number of row indices and values don't match! values.length: %lld, rowIndices.length: %lld",
               (long long)d->valuesLen, (long long)d->rowIndicesLen);
    if (d->isTransposed)
      MR_REQUIRE(d->colPtrsLen == d->numRows + 1, MR_EINVAL, "Expecting %d colPtrs when numRows = %d but got %lld",
                 d->numRows + 1, d->numRows, (long long)d->colPtrsLen);
    else
      MR_REQUIRE(d->colPtrsLen == d->numCols + 1, MR_EINVAL, "Expecting %d colPtrs when numCols = %d but got %lld",
                 d->numCols + 1, d->numCols, (long long)d->colPtrsLen);
    MR_REQUIRE(d->colPtrs != nullptr, MR_EINVAL, "colPtrs is null");
    MR_REQUIRE(d->valuesLen == d->colPtrs[d->colPtrsLen - 1], MR_EINVAL,
               "The last value of colPtrs must equal the number of elements. values.length: %lld, colPtrs.last: %d",
               (long long)d->valuesLen, d->colPtrs[d->colPtrsLen - 1]);
    MR_REQUIRE(d->valuesLen == 0 || (d->values != nullptr && d->rowIndices != nullptr), MR_EINVAL,
               "values / rowIndices is null");
  } else {
    fail(MR_ENOTSUP, "Unsupported matrix type %d", static_cast<int>(d->type));
  }
}

Span upload_raw(mr_context* ctx, const void* host, size_t bytes) {
  Span s{std::make_shared<DevBuf>(ctx, std::max<size_t>(bytes, 16)), 0};
  if (bytes) {
    CUDA_CHECK(cudaMemcpyAsync(s.buf->p, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    ctx->stats.h2d_bytes += static_cast<int64_t>(bytes);
  }
  return s;
}

}  // namespace mrhost

// ------------------------------------------------------------------------------------------------
// ABI: lifetime
// ------------------------------------------------------------------------------------------------
extern "C" {

const char* mr_last_error(void) { return g_last_error.c_str(); }
const char* mr_version(void) { return "matrel-b200 0.1 (sm_90a)"; }

mr_status mr_init(const mr_options* opts, mr_context** out) {
  return guarded([&] {
    MR_REQUIRE(out != nullptr, MR_EINVAL, "out is null");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
      (void)cudaGetLastError();
      fail(MR_ECUDA, "no usable CUDA device (%s): the engine has no CPU fallback",
           e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    auto ctx = std::unique_ptr<mr_context>(new mr_context);
    int dev = opts ? opts->device : -1;
    if (dev < 0) CUDA_CHECK(cudaGetDevice(&dev));
    MR_REQUIRE(dev < count, MR_EINVAL, "device ordinal %d out of range (have %d)", dev, count);
    CUDA_CHECK(cudaSetDevice(dev));
    ctx->device = dev;
    cudaDeviceProp prop{};
    CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0)
      fail(MR_ECUDA, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", dev, prop.major, prop.minor);
    if (opts) {
      ctx->compat_bugs = opts->compat_bugs;
      ctx->gemm_algo = opts->gemm_algo;
      ctx->ozaki_slices = opts->ozaki_slices;
    }
    if (const char* ks = std::getenv("MATREL_OZ2_KSPLIT")) ctx->oz2_ksplit = std::atoi(ks);  // A/B switch for measurements; option "oz2_ksplit"
    if (opts && opts->stream) {
      ctx->stream = static_cast<cudaStream_t>(opts->stream);
    } else {
      CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
      ctx->own_stream = true;
    }
    CUDA_CHECK(cudaEventCreate(&ctx->ev0));
    CUDA_CHECK(cudaEventCreate(&ctx->ev1));
    CUDA_CHECK(cudaEventCreate(&ctx->ev2));
    CUDA_CHECK(cudaEventCreate(&ctx->ev3));
    CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_alloc, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_order, cudaEventDisableTiming));
    CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->h2d_stream, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->p2p_stream, cudaStreamNonBlocking));
    for (int i = 0; i < mr_context::kChunkStreams; ++i) {
      CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->chunk_stream[i], cudaStreamNonBlocking));
      CUDA_CHECK(cudaEventCreateWithFlags(&ctx->chunk_join[i], cudaEventDisableTiming));
    }
    {
      void* hp = nullptr;
      const size_t cap = 16u << 20;
      if (cudaHostAlloc(&hp, cap, cudaHostAllocMapped) == cudaSuccess) {
        void* dp = nullptr;
        if (cudaHostGetDevicePointer(&dp, hp, 0) == cudaSuccess) {
          ctx->stage_host = static_cast<char*>(hp);
          ctx->stage_dev = static_cast<char*>(dp);
          ctx->stage_cap = cap;
        } else {
          cudaFreeHost(hp);
        }
      }
      (void)cudaGetLastError();
    }
    // keep freed blocks in the pool: operators allocate result slabs on every call
    cudaMemPool_t pool;
    CUDA_CHECK(cudaDeviceGetDefaultMemPool(&pool, dev));
    {  // the pool setting is per device, shared by every context on it: the first context saves it, the last one restores it
      std::lock_guard<std::mutex> g(g_pool_mu);
      if (dev < kMaxPoolDevices && g_pool_users[dev]++ == 0)
        CUDA_CHECK(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &g_pool_threshold_before[dev]));
    }
    uint64_t thr = UINT64_MAX;
    CUDA_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    *out = ctx.release();
  });
}

mr_status mr_shutdown(mr_context* ctx) {
  return guarded([&] {
    if (!ctx) return;
    DeviceScope dev(ctx);
    cudaStreamSynchronize(ctx->h2d_stream);
    cudaStreamSynchronize(ctx->p2p_stream);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->d2h_stream);
    for (auto& kv : ctx->ipc_open) cudaIpcCloseMemHandle(kv.second);
    cudaStreamDestroy(ctx->h2d_stream);
    cudaStreamDestroy(ctx->d2h_stream);
    cudaStreamDestroy(ctx->p2p_stream);
    for (int i = 0; i < mr_context::kChunkStreams; ++i) {
      if (ctx->chunk_stream[i]) cudaStreamDestroy(ctx->chunk_stream[i]);
      if (ctx->chunk_join[i]) cudaEventDestroy(ctx->chunk_join[i]);
    }
    if (ctx->stage_host) cudaFreeHost(ctx->stage_host);
    if (ctx->ev_alloc) cudaEventDestroy(ctx->ev_alloc);
    if (ctx->ev_order) cudaEventDestroy(ctx->ev_order);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->ev2) cudaEventDestroy(ctx->ev2);
    if (ctx->ev3) cudaEventDestroy(ctx->ev3);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    {  // the last context on the device hands the cached operator memory back and undoes the pool setting of mr_init
      std::lock_guard<std::mutex> g(g_pool_mu);
      cudaMemPool_t pool;
      if (ctx->device < kMaxPoolDevices && --g_pool_users[ctx->device] == 0 && cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) {
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &g_pool_threshold_before[ctx->device]);
        cudaMemPoolTrimTo(pool, 0);
      }
      (void)cudaGetLastError();
    }
    delete ctx;
  });
}

mr_status mr_set_stream(mr_context* ctx, void* cuda_stream) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr, MR_EINVAL, "ctx is null");
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (ctx->own_stream) {
      cudaStreamDestroy(ctx->stream);
      ctx->own_stream = false;
    }
    if (cuda_stream) {
      ctx->stream = static_cast<cudaStream_t>(cuda_stream);
    } else {
      CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
      ctx->own_stream = true;
    }
  });
}

mr_status mr_set_option(mr_context* ctx, const char* key, int64_t value) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && key != nullptr, MR_EINVAL, "ctx/key is null");
    std::string k(key);
    if (k == "compat_bugs") ctx->compat_bugs = static_cast<int>(value);
    else if (k == "gemm_algo") ctx->gemm_algo = static_cast<int>(value);
    else if (k == "ozaki_slices") ctx->ozaki_slices = static_cast<int>(value);
    else if (k == "crt_moduli") ctx->crt_moduli = static_cast<int>(value);
    else if (k == "ozaki_scratch_mb") ctx->ozaki_scratch_mb = static_cast<int>(value);
    else if (k == "spmm_algo") ctx->spmm_algo = static_cast<int>(value);
    else if (k == "time_kernels") ctx->time_kernels = static_cast<int>(value);
    else if (k == "gemm_variant") ctx->force_variant = static_cast<int>(value);
    else if (k == "oz2_ksplit") ctx->oz2_ksplit = static_cast<int>(value);
    else if (k == "pipeline") ctx->pipeline = static_cast<int>(value);
    else fail(MR_EINVAL, "unknown option '%s'", key);
  });
}

mr_status mr_sync(mr_context* ctx) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr, MR_EINVAL, "ctx is null");
    DeviceScope dev(ctx);
    CUDA_CHECK(cudaStreamSynchronize(ctx->h2d_stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->p2p_stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->d2h_stream));
  });
}

// Orders the context stream after every host->device block copy submitted so far (they run on a private ingest stream):
// what a caller needs before a cross-process barrier that tells peers "my blocks are in place".
mr_status mr_wait_ingest(mr_context* ctx) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr, MR_EINVAL, "ctx is null");
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    CUDA_CHECK(cudaEventRecord(ctx->ev_alloc, ctx->h2d_stream));
    CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_alloc, 0));
  });
}

// The same for a caller-owned stream (e.g. the side stream a cross-process barrier runs on).
mr_status mr_wait_ingest_on(mr_context* ctx, void* cuda_stream) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr, MR_EINVAL, "ctx is null");
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    CUDA_CHECK(cudaEventRecord(ctx->ev_alloc, ctx->h2d_stream));
    CUDA_CHECK(cudaStreamWaitEvent(static_cast<cudaStream_t>(cuda_stream), ctx->ev_alloc, 0));
  });
}

mr_status mr_get_stats(mr_context* ctx, mr_stats* out) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && out != nullptr, MR_EINVAL, "ctx/out is null");
    *out = ctx->stats;
  });
}

mr_status mr_reset_stats(mr_context* ctx) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr, MR_EINVAL, "ctx is null");
    ctx->stats = mr_stats{};
  });
}

// ------------------------------------------------------------------------------------------------
// ABI: datasets
// ------------------------------------------------------------------------------------------------
mr_status mr_matrix_create(mr_context* ctx, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && out != nullptr, MR_EINVAL, "ctx/out is null");
    *out = new_matrix(ctx);
  });
}

mr_status mr_matrix_free(mr_matrix* m) {
  return guarded([&] {
    if (!m) return;
    DeviceScope dev(m->ctx);
    delete m;
  });
}

mr_status mr_matrix_put_block(mr_matrix* m, int32_t rid, int32_t cid, const mr_block_desc* d) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr, MR_EINVAL, "matrix is null");
    validate_desc(d);
    mr_context* ctx = m->ctx;
    DeviceScope dev(ctx);
    if (m->shard) {
      // a sharded dataset is dense over its block grid: the block is copied into its slot of the slab
      const ShardLayout& L = m->shard->L;
      MR_REQUIRE(d->type == 1, MR_ENOTSUP, "sharded datasets hold dense blocks; got a SparseMatrix for block (%d, %d)", rid, cid);
      MR_REQUIRE(rid >= 0 && cid >= 0 && rid < L.nbr && cid < L.nbc, MR_EINVAL, "block (%d, %d) outside the %lld x %lld block grid", rid,
                 cid, (long long)L.nbr, (long long)L.nbc);
      MR_REQUIRE(rid % L.pr == L.r && cid % L.pc == L.c, MR_EINVAL, "block (%d, %d) belongs to rank (%d, %d) of the %d x %d grid, not (%d, %d)",
                 rid, cid, rid % L.pr, cid % L.pc, L.pr, L.pc, L.r, L.c);
      auto it = m->blocks.find({rid, cid});
      MR_REQUIRE(it != m->blocks.end(), MR_EINVAL, "block (%d, %d) is not registered", rid, cid);
      Block& tgt = it->second;
      MR_REQUIRE(d->numRows == tgt.numRows && d->numCols == tgt.numCols, MR_EDIM, "block (%d, %d) is %d x %d, the layout expects %d x %d",
                 rid, cid, d->numRows, d->numCols, tgt.numRows, tgt.numCols);
      MR_REQUIRE((d->isTransposed != 0) == m->shard->isT, MR_ENOTSUP,
                 "block (%d, %d): isTransposed differs from the dataset's (all blocks of a sharded dataset share one layout flag)", rid, cid);
      cudaStream_t cs = ctx->pipeline ? ctx->h2d_stream : ctx->stream;
      if (ctx->pipeline) {  // the slab (and whatever produced its previous content) is ordered on the context stream
        CUDA_CHECK(cudaEventRecord(ctx->ev_alloc, ctx->stream));
        CUDA_CHECK(cudaStreamWaitEvent(cs, ctx->ev_alloc, 0));
      }
      const size_t bytes = static_cast<size_t>(d->valuesLen) * sizeof(double);
      if (bytes) {
        CUDA_CHECK(cudaMemcpyAsync(tgt.values.ptr<double>(), d->values, bytes, cudaMemcpyHostToDevice, cs));
        ctx->stats.h2d_bytes += static_cast<int64_t>(bytes);
      }
      if (ctx->pipeline) {
        ReadyPtr r = std::make_shared<Ready>();
        CUDA_CHECK(cudaEventRecord(r->ev, cs));
        tgt.ready = r;
        tgt.settled = false;
        tgt.seq = ++ctx->ingest_seq;
        m->shard->slab->ready = r;
      }
      return;
    }
    Block b;
    b.type = d->type;
    b.numRows = d->numRows;
    b.numCols = d->numCols;
    b.isT = d->isTransposed != 0;
    b.valuesLen = d->valuesLen;
    // Ingest on its own stream: the copy of block k+1 overlaps whatever the context stream is computing, and
    // operators wait per block (Block::ready), so a multiply can start on the row panels that have landed.
    cudaStream_t cs = ctx->pipeline ? ctx->h2d_stream : ctx->stream;
    auto put = [&](const void* host, size_t bytes) {
      Span sp{std::make_shared<DevBuf>(ctx, std::max<size_t>(bytes, 16)), 0};
      return std::make_pair(sp, bytes ? host : nullptr);
    };
    auto vals = put(d->values, static_cast<size_t>(d->valuesLen) * sizeof(double));
    std::pair<Span, const void*> cp{}, ri{};
    if (d->type == 0) {
      b.colPtrsLen = d->colPtrsLen;
      cp = put(d->colPtrs, static_cast<size_t>(d->colPtrsLen) * sizeof(int32_t));
      ri = put(d->rowIndices, static_cast<size_t>(d->rowIndicesLen) * sizeof(int32_t));
    }
    if (ctx->pipeline) {  // allocations are ordered on the context stream: the ingest stream must see them
      CUDA_CHECK(cudaEventRecord(ctx->ev_alloc, ctx->stream));
      CUDA_CHECK(cudaStreamWaitEvent(cs, ctx->ev_alloc, 0));
    }
    auto copy = [&](std::pair<Span, const void*>& x, size_t bytes) {
      if (x.second && bytes) {
        CUDA_CHECK(cudaMemcpyAsync(x.first.buf->p, x.second, bytes, cudaMemcpyHostToDevice, cs));
        ctx->stats.h2d_bytes += static_cast<int64_t>(bytes);
      }
    };
    copy(vals, static_cast<size_t>(d->valuesLen) * sizeof(double));
    b.values = vals.first;
    if (d->type == 0) {
      copy(cp, static_cast<size_t>(d->colPtrsLen) * sizeof(int32_t));
      copy(ri, static_cast<size_t>(d->rowIndicesLen) * sizeof(int32_t));
      b.colPtrs = cp.first;
      b.rowIndices = ri.first;
    }
    if (ctx->pipeline) {
      ReadyPtr r = std::make_shared<Ready>();
      CUDA_CHECK(cudaEventRecord(r->ev, cs));
      b.ready = r;
      b.seq = ++ctx->ingest_seq;
      b.values.buf->ready = r;
      if (d->type == 0) {
        b.colPtrs.buf->ready = r;
        b.rowIndices.buf->ready = r;
      }
    }
    m->blocks[{rid, cid}] = std::move(b);
  });
}

mr_status mr_matrix_put_blocks(mr_matrix* m, int64_t count, const int32_t* rids, const int32_t* cids, const mr_block_desc* blks) {
  if (count < 0 || (count > 0 && (!rids || !cids || !blks))) {
    g_last_error = "requirement failed: null argument";
    return MR_EINVAL;
  }
  for (int64_t i = 0; i < count; ++i) {
    const mr_status st = mr_matrix_put_block(m, rids[i], cids[i], &blks[i]);
    if (st != MR_OK) return st;
  }
  return MR_OK;
}

mr_status mr_matrix_wait_ingest(mr_matrix* m) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr, MR_EINVAL, "matrix is null");
    DeviceScope dev(m->ctx);
    std::vector<ReadyPtr> pending;
    {
      std::lock_guard<std::mutex> lock(m->ctx->mu);
      for (auto& kv : m->blocks)
        if (kv.second.ready) pending.push_back(kv.second.ready);
    }
    for (auto& r : pending) CUDA_CHECK(cudaEventSynchronize(r->ev));
  });
}

mr_status mr_matrix_put_block_device(mr_matrix* m, int32_t rid, int32_t cid, int32_t numRows, int32_t numCols,
                                     const double* dvalues, uint8_t isTransposed) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr, MR_EINVAL, "matrix is null");
    MR_REQUIRE(numRows >= 0 && numCols >= 0, MR_EINVAL, "negative block dimensions %d x %d", numRows, numCols);
    MR_REQUIRE(dvalues != nullptr || static_cast<int64_t>(numRows) * numCols == 0, MR_EINVAL, "device pointer is null");
    Span s{std::make_shared<DevBuf>(m->ctx, const_cast<double*>(dvalues),
                                    static_cast<size_t>(numRows) * numCols * sizeof(double)),
           0};
    m->blocks[{rid, cid}] = dense_block(numRows, numCols, s, isTransposed != 0);
  });
}

mr_status mr_matrix_put_blocks_device(mr_matrix* m, int64_t count, const int32_t* rids, const int32_t* cids,
                                      const int32_t* numRows, const int32_t* numCols, const double* const* dvalues,
                                      const uint8_t* isTransposed) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr, MR_EINVAL, "matrix is null");
    MR_REQUIRE(count == 0 || (rids && cids && numRows && numCols && dvalues), MR_EINVAL, "null argument");
    for (int64_t i = 0; i < count; ++i) {
      MR_REQUIRE(numRows[i] >= 0 && numCols[i] >= 0, MR_EINVAL, "negative block dimensions %d x %d", numRows[i], numCols[i]);
      Span s{std::make_shared<DevBuf>(m->ctx, const_cast<double*>(dvalues[i]),
                                      static_cast<size_t>(numRows[i]) * numCols[i] * sizeof(double)),
             0};
      m->blocks[{rids[i], cids[i]}] = dense_block(numRows[i], numCols[i], s, isTransposed ? isTransposed[i] != 0 : false);
    }
  });
}

mr_status mr_matrix_num_blocks(const mr_matrix* m, int64_t* out) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && out != nullptr, MR_EINVAL, "matrix/out is null");
    *out = static_cast<int64_t>(m->blocks.size());
  });
}

mr_status mr_matrix_has_block(const mr_matrix* m, int32_t rid, int32_t cid, int32_t* out) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && out != nullptr, MR_EINVAL, "matrix/out is null");
    *out = m->blocks.count({rid, cid}) ? 1 : 0;
  });
}

mr_status mr_matrix_block_ids(const mr_matrix* m, int32_t* rids, int32_t* cids, int64_t cap) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && rids != nullptr && cids != nullptr, MR_EINVAL, "null argument");
    MR_REQUIRE(cap >= static_cast<int64_t>(m->blocks.size()), MR_EINVAL, "capacity %lld < number of blocks %zu",
               (long long)cap, m->blocks.size());
    int64_t i = 0;
    for (auto& kv : m->blocks) {
      rids[i] = kv.first.first;
      cids[i] = kv.first.second;
      ++i;
    }
  });
}

mr_status mr_matrix_get_block(mr_matrix* m, int32_t rid, int32_t cid, mr_block_desc* io) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && io != nullptr, MR_EINVAL, "null argument");
    auto it = m->blocks.find({rid, cid});
    if (it == m->blocks.end()) fail(MR_ENOTFOUND, "no block (%d, %d) in this dataset", rid, cid);
    const Block& b = it->second;
    mr_context* ctx = m->ctx;
    DeviceScope dev(ctx);
    ReadyPtr ready;
    bool settled;
    {
      std::lock_guard<std::mutex> lock(ctx->mu);
      ready = b.ready;  // snapshot: operators on other threads may drop completed events
      settled = b.settled;
    }
    const int64_t rowIndicesLen = b.dense() ? 0 : b.valuesLen;
    // Egress on its own stream, ordered after this block's producer only (one chunk of a chunked multiply, or
    // everything enqueued on the context stream so far when the block has no event of its own).
    cudaStream_t rs = ctx->pipeline ? ctx->d2h_stream : ctx->stream;
    if (ctx->pipeline && (io->values || io->colPtrs || io->rowIndices)) {
      if (ready) {
        CUDA_CHECK(cudaStreamWaitEvent(rs, ready->ev, 0));
      } else if (!settled) {
        CUDA_CHECK(cudaEventRecord(ctx->ev_order, ctx->stream));
        CUDA_CHECK(cudaStreamWaitEvent(rs, ctx->ev_order, 0));
      }
    }
    if (io->values != nullptr) {
      MR_REQUIRE(io->valuesLen >= b.valuesLen, MR_EINVAL, "values capacity %lld < %lld", (long long)io->valuesLen,
                 (long long)b.valuesLen);
      if (b.valuesLen)
        CUDA_CHECK(cudaMemcpyAsync(io->values, b.values.ptr<double>(), static_cast<size_t>(b.valuesLen) * sizeof(double),
                                   cudaMemcpyDeviceToHost, rs));
      ctx->stats.d2h_bytes += b.valuesLen * 8;
    }
    if (!b.dense() && io->colPtrs != nullptr) {
      MR_REQUIRE(io->colPtrsLen >= b.colPtrsLen, MR_EINVAL, "colPtrs capacity too small");
      CUDA_CHECK(cudaMemcpyAsync(io->colPtrs, b.colPtrs.ptr<int32_t>(), static_cast<size_t>(b.colPtrsLen) * 4,
                                 cudaMemcpyDeviceToHost, rs));
      ctx->stats.d2h_bytes += b.colPtrsLen * 4;
    }
    if (!b.dense() && io->rowIndices != nullptr) {
      MR_REQUIRE(io->rowIndicesLen >= rowIndicesLen, MR_EINVAL, "rowIndices capacity too small");
      if (rowIndicesLen)
        CUDA_CHECK(cudaMemcpyAsync(io->rowIndices, b.rowIndices.ptr<int32_t>(), static_cast<size_t>(rowIndicesLen) * 4,
                                   cudaMemcpyDeviceToHost, rs));
      ctx->stats.d2h_bytes += rowIndicesLen * 4;
    }
    if (io->values || io->colPtrs || io->rowIndices) CUDA_CHECK(cudaStreamSynchronize(rs));
    io->type = b.type;
    io->numRows = b.numRows;
    io->numCols = b.numCols;
    io->isTransposed = b.isT ? 1 : 0;
    io->valuesLen = b.valuesLen;
    io->colPtrsLen = b.dense() ? 0 : b.colPtrsLen;
    io->rowIndicesLen = rowIndicesLen;
  });
}

mr_status mr_matrix_block_device_ptr(mr_matrix* m, int32_t rid, int32_t cid, double** dptr) {
  return guarded([&] {
    MR_REQUIRE(m != nullptr && dptr != nullptr, MR_EINVAL, "null argument");
    auto it = m->blocks.find({rid, cid});
    if (it == m->blocks.end()) fail(MR_ENOTFOUND, "no block (%d, %d) in this dataset", rid, cid);
    *dptr = it->second.values.ptr<double>();
  });
}

mr_status mr_matrix_rand(mr_context* ctx, int64_t nrows, int64_t ncols, int32_t blkSize, int64_t seed0,
                         mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && out != nullptr, MR_EINVAL, "ctx/out is null");
    MR_REQUIRE(nrows > 0 && ncols > 0 && blkSize > 0, MR_EINVAL, "nrows, ncols, blkSize must be positive");
    // DenseMatrix.rand `require` (MLMatrix.scala:454-455)
    MR_REQUIRE(static_cast<int64_t>(blkSize) * blkSize <= INT32_MAX, MR_EINVAL,
               "%d x %d dense matrix is too large to allocate", blkSize, blkSize);
    const int64_t nbr = ceil_div(nrows, blkSize), nbc = ceil_div(ncols, blkSize);
    std::unique_ptr<mr_matrix> m(new_matrix(ctx));
    size_t total = 0;
    for (int64_t i = 0; i < nbr; ++i)
      for (int64_t j = 0; j < nbc; ++j) {
        const int64_t r = std::min<int64_t>(blkSize, nrows - i * blkSize), c = std::min<int64_t>(blkSize, ncols - j * blkSize);
        total += align_up(static_cast<size_t>(r * c) * sizeof(double));
      }
    Slab slab(ctx, total);
    std::vector<RandDesc> descs;
    int64_t max_n = 0;
    for (int64_t i = 0; i < nbr; ++i)
      for (int64_t j = 0; j < nbc; ++j) {
        const int32_t r = static_cast<int32_t>(std::min<int64_t>(blkSize, nrows - i * blkSize));
        const int32_t c = static_cast<int32_t>(std::min<int64_t>(blkSize, ncols - j * blkSize));
        Span s = slab.take(static_cast<size_t>(r) * c * sizeof(double));
        descs.push_back(RandDesc{s.ptr<double>(), static_cast<int64_t>(r) * c, seed0 + i * nbc + j});
        max_n = std::max<int64_t>(max_n, static_cast<int64_t>(r) * c);
        m->blocks[{static_cast<int32_t>(i), static_cast<int32_t>(j)}] = dense_block(r, c, s, false);
      }
    // gridDim.y limit: launch in chunks of 65535 blocks
    for (size_t off = 0; off < descs.size(); off += 65535) {
      std::vector<RandDesc> chunk(descs.begin() + off, descs.begin() + std::min(descs.size(), off + 65535));
      Buf d = upload(ctx, chunk);
      CUDA_CHECK(launch_java_rand_batched(static_cast<const RandDesc*>(d->p), static_cast<int>(chunk.size()), max_n, ctx->stream));
      note_launch(ctx);
    }
    *out = m.release();
  });
}

mr_status mr_matrix_rand_partition(mr_context* ctx, int64_t nrows, int64_t ncols, int32_t blkSize, int64_t seed0,
                                   int32_t pr, int32_t pc, int32_t r, int32_t c, double* dslab, int64_t slotElems,
                                   mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && out != nullptr && dslab != nullptr, MR_EINVAL, "null argument");
    MR_REQUIRE(nrows > 0 && ncols > 0 && blkSize > 0, MR_EINVAL, "nrows, ncols, blkSize must be positive");
    MR_REQUIRE(pr > 0 && pc > 0 && r >= 0 && r < pr && c >= 0 && c < pc, MR_EINVAL, "bad process grid %d x %d / (%d, %d)",
               pr, pc, r, c);
    MR_REQUIRE(slotElems >= static_cast<int64_t>(blkSize) * blkSize, MR_EINVAL, "slotElems %lld < blkSize^2",
               (long long)slotElems);
    const int64_t nbr = ceil_div(nrows, blkSize), nbc = ceil_div(ncols, blkSize);
    const int64_t slots_c = ceil_div(nbc, pc);
    std::unique_ptr<mr_matrix> m(new_matrix(ctx));
    std::vector<RandDesc> descs;
    int64_t max_n = 0;
    for (int64_t i = r; i < nbr; i += pr)
      for (int64_t j = c; j < nbc; j += pc) {
        const int32_t br = static_cast<int32_t>(std::min<int64_t>(blkSize, nrows - i * blkSize));
        const int32_t bc = static_cast<int32_t>(std::min<int64_t>(blkSize, ncols - j * blkSize));
        double* p = dslab + ((i / pr) * slots_c + (j / pc)) * slotElems;
        descs.push_back(RandDesc{p, static_cast<int64_t>(br) * bc, seed0 + i * nbc + j});
        max_n = std::max<int64_t>(max_n, static_cast<int64_t>(br) * bc);
        Span s{std::make_shared<DevBuf>(ctx, p, static_cast<size_t>(br) * bc * sizeof(double)), 0};
        m->blocks[{static_cast<int32_t>(i), static_cast<int32_t>(j)}] = dense_block(br, bc, s, false);
      }
    for (size_t off = 0; off < descs.size(); off += 65535) {
      std::vector<RandDesc> chunk(descs.begin() + off, descs.begin() + std::min(descs.size(), off + 65535));
      Buf d = upload(ctx, chunk);
      CUDA_CHECK(launch_java_rand_batched(static_cast<const RandDesc*>(d->p), static_cast<int>(chunk.size()), max_n, ctx->stream));
      note_launch(ctx);
    }
    *out = m.release();
  });
}

// SparseMatrix.sprand(r, c, density, new java.util.Random(seed0 + rid * nbc + cid)) for every block of an nrows x ncols matrix
// (M/matrix/MLMatrix.scala:791-856), generated on the device bit-identically to the JVM.  csr != 0: block (rid, cid) is
// sprand(c, r, ...).transpose, i.e. the r x c block in CSR form (isTransposed = true) -- the BASELINE configs[4] operand.
mr_status mr_matrix_sprand(mr_context* ctx, int64_t nrows, int64_t ncols, int32_t blkSize, double density, int64_t seed0, uint8_t csr,
                           mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(ctx != nullptr && out != nullptr, MR_EINVAL, "ctx/out is null");
    MR_REQUIRE(nrows > 0 && ncols > 0 && blkSize > 0, MR_EINVAL, "nrows, ncols, blkSize must be positive");
    // genRandMatrix `require` (MLMatrix.scala:798-799)
    MR_REQUIRE(density >= 0.0 && density <= 1.0, MR_EINVAL,
               "density must be a double in the range 0.0 <= d <= 1.0. Currently, density: %g", density);
    MR_REQUIRE(density > 0.0 && density < 0.34, MR_ENOTSUP, "device sprand restates the draw-by-draw branch (0 < density < 0.34), got %g", density);
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    const int64_t nbr = ceil_div(nrows, blkSize), nbc = ceil_div(ncols, blkSize);
    struct Plan {
      int32_t rid, cid, r, c, gr, gc;  // logical dims (r, c); generator dims (gr, gc)
      int64_t nnz;
      size_t off_ptr, off_idx, off_val;
    };
    std::vector<Plan> plans;
    size_t total = 0;
    int max_cols = 1;
    for (int64_t i = 0; i < nbr; ++i)
      for (int64_t j = 0; j < nbc; ++j) {
        Plan p{};
        p.rid = static_cast<int32_t>(i);
        p.cid = static_cast<int32_t>(j);
        p.r = static_cast<int32_t>(std::min<int64_t>(blkSize, nrows - i * blkSize));
        p.c = static_cast<int32_t>(std::min<int64_t>(blkSize, ncols - j * blkSize));
        p.gr = csr ? p.c : p.r;
        p.gc = csr ? p.r : p.c;
        MR_REQUIRE((p.gr & (p.gr - 1)) == 0 && (p.gc & (p.gc - 1)) == 0, MR_ENOTSUP,
                   "device sprand needs power-of-two block dimensions (java.util.Random.nextInt consumes one draw per call only then); "
                   "block (%d, %d) is %d x %d", p.rid, p.cid, p.r, p.c);
        p.nnz = static_cast<int64_t>(std::ceil(static_cast<double>(p.gr) * p.gc * density));
        MR_REQUIRE(sprand_draws(p.nnz) > 0, MR_ENOTSUP, "device sprand handles up to ~14000 non-zeros per block, block (%d, %d) needs %lld",
                   p.rid, p.cid, (long long)p.nnz);
        p.off_ptr = total;
        total += align_up(static_cast<size_t>(p.gc + 1) * 4);
        p.off_idx = total;
        total += align_up(static_cast<size_t>(p.nnz) * 4);
        p.off_val = total;
        total += align_up(static_cast<size_t>(p.nnz) * 8);
        max_cols = std::max(max_cols, p.gc);
        plans.push_back(p);
      }
    Slab slab(ctx, total);
    Buf status = std::make_shared<DevBuf>(ctx, sizeof(int));
    CUDA_CHECK(cudaMemsetAsync(status->p, 0, sizeof(int), ctx->stream));
    std::unique_ptr<mr_matrix> m(new_matrix(ctx));
    std::vector<SprandDesc> descs;
    for (const Plan& p : plans) {
      Block b;
      b.type = 0;
      b.numRows = p.r;
      b.numCols = p.c;
      b.isT = csr != 0;
      b.valuesLen = p.nnz;
      b.colPtrsLen = p.gc + 1;
      b.colPtrs = Span{slab.buf, p.off_ptr};
      b.rowIndices = Span{slab.buf, p.off_idx};
      b.values = Span{slab.buf, p.off_val};
      SprandDesc d{};
      d.rows = p.gr;
      d.cols = p.gc;
      d.nnz = static_cast<int32_t>(p.nnz);
      d.draws = sprand_draws(p.nnz);
      d.seed = seed0 + static_cast<int64_t>(p.rid) * nbc + p.cid;
      d.colPtrs = b.colPtrs.ptr<int32_t>();
      d.rowIndices = b.rowIndices.ptr<int32_t>();
      d.values = b.values.ptr<double>();
      d.status = static_cast<int*>(status->p);
      descs.push_back(d);
      m->blocks[{p.rid, p.cid}] = std::move(b);
    }
    for (size_t off = 0; off < descs.size(); off += 65535) {
      std::vector<SprandDesc> chunk(descs.begin() + off, descs.begin() + std::min(descs.size(), off + 65535));
      Buf d = upload(ctx, chunk);
      CUDA_CHECK(launch_sprand(static_cast<const SprandDesc*>(d->p), static_cast<int>(chunk.size()), max_cols, ctx->stream));
      note_launch(ctx);
    }
    int h_status = 0;
    CUDA_CHECK(cudaMemcpyAsync(&h_status, status->p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (h_status) fail(MR_ECUDA, "device sprand ran out of draws before reaching the requested number of distinct coordinates");
    *out = m.release();
  });
}

}  // extern "C"
