// Internal header of the C-ABI host layer (abi_*.cpp): error plumbing, the context, device buffers, blocks and the
// helpers the operator files share.  Nothing here is exported (the library is built with -fvisibility=hidden; only the
// MR_API entry points of include/matrel.h are visible).
#pragma once
#include "../../include/matrel.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <set>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "kernels.h"

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
namespace mrhost {

extern thread_local std::string g_last_error;   // what mr_last_error() returns (abi_core.cpp)

struct MrError {
  mr_status code;
  std::string msg;
};

[[noreturn]] void fail(mr_status code, const char* fmt, ...);

// Scala `require(cond, msg)` -> IllegalArgumentException("requirement failed: " + msg)
#define MR_REQUIRE(cond, code, ...)                                           \
  do {                                                                        \
    if (!(cond)) {                                                            \
      char _b[900];                                                           \
      snprintf(_b, sizeof(_b), __VA_ARGS__);                                  \
      fail((code), "requirement failed: %s", _b);                             \
    }                                                                         \
  } while (0)

#define CUDA_CHECK(expr)                                                                         \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) fail(MR_ECUDA, "CUDA error %s at %s:%d (%s)", cudaGetErrorName(_e), __FILE__, __LINE__, \
                                cudaGetErrorString(_e));                                         \
  } while (0)

template <typename F>
mr_status guarded(F&& f) {
  try {
    f();
    return MR_OK;
  } catch (const MrError& e) {
    g_last_error = e.msg;
    return e.code;
  } catch (const std::bad_alloc&) {
    g_last_error = "out of host memory";
    return MR_ENOMEM;
  } catch (const std::exception& e) {
    g_last_error = std::string("internal error: ") + e.what();
    return MR_EINVAL;
  } catch (...) {
    g_last_error = "unknown internal error";
    return MR_EINVAL;
  }
}

}  // namespace mrhost

// ------------------------------------------------------------------------------------------------
// context, device buffers, blocks
// ------------------------------------------------------------------------------------------------
struct mr_context {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int compat_bugs = 1;
  int gemm_algo = 0;
  int ozaki_slices = 0;
  int crt_moduli = 0;
  int ozaki_scratch_mb = 0;  // budget of the Ozaki-II residue scratch (0 = 16 GiB)
  int spmm_algo = 0;         // 0 = auto (pipelined TMA kernel when the blocks are large enough), 1 = the simple shared-memory kernel
  int time_kernels = 0;
  int force_variant = -1;
  int oz2_strassen = 1;   // option "oz2_strassen": one Strassen level for eligible resident Ozaki-II multiplies (DESIGN section 4.1.3):
                          // 1 = from M, N, K >= 16384 on, 2 = at every eligible size, 0 = off
  int oz2_ksplit = 0;     // option "oz2_ksplit" (default: environment MATREL_OZ2_KSPLIT, else 0): K-split item order of the CTA-pair GEMM
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr, ev_alloc = nullptr, ev_order = nullptr;
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;  // ingest / egress overlap with compute on `stream`
  // The chunks of a pipelined multiply are independent launches: issued round-robin on these side streams, the last
  // (partial) wave of one chunk overlaps the first waves of the next instead of leaving SMs idle between launches.
  static constexpr int kChunkStreams = 3;
  cudaStream_t chunk_stream[kChunkStreams] = {nullptr, nullptr, nullptr};
  cudaEvent_t chunk_join[kChunkStreams] = {nullptr, nullptr, nullptr};
  uint64_t ingest_seq = 0;
  // mapped pinned staging ring for descriptor tables (see upload())
  char* stage_host = nullptr;
  char* stage_dev = nullptr;
  size_t stage_cap = 0, stage_off = 0;
  int pipeline = 1;
  cudaStream_t p2p_stream = nullptr;             // pulls of peers' blocks over NVLink (copy engines), see abi_grid.cpp
  std::map<std::string, void*> ipc_open;         // CUDA IPC handles opened by this context (handle bytes -> mapped base)
  int64_t stream_budget_mb = 0;  // device budget of a streamed multiply (0 = free device memory at the call minus 1 GiB)
  // page-locked chunks of freed host-resident datasets, kept for the next one (pinning is slow); released by mr_shutdown
  std::multimap<size_t, void*> pinned_free;
  std::mutex pinned_mu;
  mr_stats stats{};
  std::mutex mu;
};

namespace mrhost {

// Completion event of an asynchronous producer of a block (an H2D copy on the ingest stream, or one chunk of a
// chunked multiply); consumers on other streams wait on it instead of on whole streams.
struct Ready {
  cudaEvent_t ev = nullptr;
  Ready() { cudaEventCreateWithFlags(&ev, cudaEventDisableTiming); }
  ~Ready() {
    if (ev) cudaEventDestroy(ev);
  }
  Ready(const Ready&) = delete;
  Ready& operator=(const Ready&) = delete;
};
using ReadyPtr = std::shared_ptr<Ready>;

struct DevBuf {
  mr_context* ctx;
  ReadyPtr ready;  // set when another stream writes or reads this buffer: the free must be ordered after it
  void* p = nullptr;
  size_t bytes = 0;
  bool owned = true;
  bool sync_alloc = false;  // cudaMalloc / cudaFree (exportable through CUDA IPC) instead of the stream-ordered pool
  struct SyncAlloc {};
  DevBuf(mr_context* c, size_t n, SyncAlloc) : ctx(c), bytes(n), sync_alloc(true) {
    cudaError_t e = cudaMalloc(&p, n ? n : 16);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      fail(e == cudaErrorMemoryAllocation ? MR_ENOMEM : MR_ECUDA, "cudaMalloc(%zu bytes) failed: %s", n, cudaGetErrorString(e));
    }
  }
  DevBuf(mr_context* c, size_t n) : ctx(c), bytes(n) {
    if (n == 0) return;
    cudaError_t e = cudaMallocAsync(&p, n, ctx->stream);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      fail(e == cudaErrorMemoryAllocation ? MR_ENOMEM : MR_ECUDA, "cudaMallocAsync(%zu bytes) failed: %s", n,
           cudaGetErrorString(e));
    }
  }
  DevBuf(mr_context* c, void* borrowed, size_t n) : ctx(c), p(borrowed), bytes(n), owned(false) {}
  ~DevBuf() {
    if (owned && p) {
      if (sync_alloc) {
        cudaFree(p);  // synchronises the device: nothing can still be using it
      } else {
        if (ready) cudaStreamWaitEvent(ctx->stream, ready->ev, 0);
        cudaFreeAsync(p, ctx->stream);
      }
    }
  }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
};
using Buf = std::shared_ptr<DevBuf>;

struct Span {  // a typed window into a (possibly shared) device buffer
  Buf buf;
  size_t off = 0;  // bytes
  template <typename T>
  T* ptr() const {
    return buf ? reinterpret_cast<T*>(static_cast<char*>(buf->p) + off) : nullptr;
  }
};

struct Block {
  uint8_t type = 1;  // 0 sparse, 1 dense (MLMatrixSerializer.scala:31,40)
  int32_t numRows = 0, numCols = 0;
  bool isT = false;
  Span values;
  int64_t valuesLen = 0;
  Span colPtrs, rowIndices;  // sparse only
  int64_t colPtrsLen = 0;
  mutable ReadyPtr ready;    // producer still in flight on another stream (nullptr = ordered on the context stream);
                             // dropped (under the context mutex) once the event is seen complete
  uint64_t seq = 0;              // ingest order of the block's H2D copy (0 = not produced by the ingest stream)
  mutable bool settled = false;  // the dropped event had completed: the block's data needs no further ordering
  bool dense() const { return type == 1; }
};

constexpr size_t kAlign = 256;
inline size_t align_up(size_t x) { return (x + kAlign - 1) / kAlign * kAlign; }

// Page-locked host memory of a host-resident dataset (abi_core.cpp): chunks of up to 1 GiB carved into 256-byte aligned
// windows.  Blocks of such a dataset are ordinary Blocks whose Spans borrow windows of these chunks.  The chunks go back to
// the context's cache when the last dataset sharing the store is freed (after every copy that may still touch them).
struct HostStore {
  mr_context* ctx;
  std::vector<std::pair<void*, size_t>> chunks;
  size_t used = 0, total = 0;  // bytes taken from the last chunk, bytes of all chunks
  explicit HostStore(mr_context* c) : ctx(c) {}
  ~HostStore();
  Span take(size_t bytes);
  HostStore(const HostStore&) = delete;
  HostStore& operator=(const HostStore&) = delete;
};

}  // namespace mrhost

namespace mrhost {
// Placement of a dataset sharded over a pr x pc process grid: rank (r, c) owns the blocks with rid % pr == r (RowPartitioner.scala:34)
// and cid % pc == c (ColumnPartitioner.scala:34); block (rid, cid) is slot (rid / pr) * slots_c + cid / pc of its owner's slab.
struct ShardLayout {
  int64_t nrows = 0, ncols = 0;
  int32_t blk = 0, pr = 1, pc = 1, r = 0, c = 0;
  int64_t nbr = 0, nbc = 0, slots_r = 0, slots_c = 0, slot_elems = 0;
  int64_t slot(int64_t rid, int64_t cid) const { return (rid / pr) * slots_c + cid / pc; }
  int64_t local_slots() const { return slots_r * slots_c; }
  int64_t slots_r_of(int rr) const { return nbr > rr ? (nbr - rr + pr - 1) / pr : 0; }  // block rows owned by grid row rr
  bool same_as(const ShardLayout& o) const {
    return nrows == o.nrows && ncols == o.ncols && blk == o.blk && pr == o.pr && pc == o.pc && r == o.r && c == o.c;
  }
};
struct ShardInfo {
  ShardLayout L;
  Buf slab;             // local_slots x blk^2 doubles; every owned block is a window of it
  bool ipc_capable = false;
  bool isT = false;     // the isTransposed flag shared by all blocks of the dataset
};
}  // namespace mrhost

struct mr_matrix {
  mr_context* ctx;
  std::map<std::pair<int32_t, int32_t>, mrhost::Block> blocks;
  std::shared_ptr<mrhost::ShardInfo> shard;   // set for datasets laid out on a process grid (abi_grid.cpp)
  std::vector<mrhost::Buf> temps;             // scratch that must outlive work enqueued on behalf of this dataset
  std::shared_ptr<mrhost::HostStore> host;    // set for host-resident datasets: every block lives in this page-locked store
};

namespace mrhost {
// One process may drive several GPUs (mr_init_grid): every entry point that launches or allocates runs on its context's device.
struct DeviceScope {
  int prev = -1;
  explicit DeviceScope(const mr_context* ctx) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != ctx->device) cudaSetDevice(ctx->device);
    else prev = -1;
  }
  ~DeviceScope() {
    if (prev >= 0) cudaSetDevice(prev);
  }
  DeviceScope(const DeviceScope&) = delete;
  DeviceScope& operator=(const DeviceScope&) = delete;
};
ShardLayout make_layout(int64_t nrows, int64_t ncols, int32_t blk, int32_t pr, int32_t pc, int32_t r, int32_t c);
mr_matrix* new_sharded(mr_context* ctx, const ShardLayout& L, bool ipc_capable, bool zero, bool isT = false);
// Where a multiply writes output block (rid, cid): a dense column-major window the caller has allocated (at least m x n doubles).
using OutWindowFn = std::function<Span(int32_t rid, int32_t cid)>;
// The body of mr_matrix_multiply (abi_multiply.cpp).  out_layout != nullptr: the result is a sharded dataset in that layout
// (its blocks are windows of one slab at their slots) instead of a packed one.  out_windows != nullptr (with out_layout ==
// nullptr): every output block is written into the caller's window and the result's blocks are those windows.  The caller
// holds ctx->mu.
// The choices multiply_impl otherwise derives from the shape it is given.  A streamed multiply computes them once for the whole
// product and hands them to every tile, so that each output element takes the same engine and kernel variant as in the resident
// call: oz2 = try the Ozaki-II engine, variant = DMMA tile variant (gemm_variant still overrides it).
enum MvSide { MV_NONE = 0, MV_AX = 1, MV_XA = 2 };  // no matrix x vector route, C = A x, C = x A (abi_multiply.cpp, run_matvec)
struct MultiplyDecisions {
  int mv = MV_NONE;  // the matrix x vector route (then nothing else below applies)
  bool oz2 = false;
  int variant = 0;
  // dense x sparse pairs (ids of their blocks): left and right blocks of the pairs that take the stored-entry route, and right
  // blocks of the pairs densified next to GEMM pairs (the streamed multiply's scratch bound)
  std::set<std::pair<int32_t, int32_t>> ds_left, ds_right, ds_dense_right;
};
// gram: left x right is a Gram product (gram_route in abi_multiply.cpp, DESIGN section 4.1.2), decided by mr_matrix_multiply only:
// every block dense (the dense engines), or every block sparse (the sparse x sparse chains, when every output block is one).
enum GramKind { GRAM_NONE = 0, GRAM_DENSE = 1, GRAM_SPARSE = 2 };
mr_matrix* multiply_impl(mr_context* ctx, mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right, int64_t rightRowNum,
                         int64_t rightColNum, int32_t blkSize, const ShardLayout* out_layout, const OutWindowFn* out_windows = nullptr,
                         const MultiplyDecisions* decisions = nullptr, GramKind gram = GRAM_NONE);
// The decisions multiply_impl would take for left x right, from block metadata only (the blocks may be host-resident).
MultiplyDecisions multiply_decisions(const mr_context* ctx, const mr_matrix* left, int64_t leftRowNum, int64_t leftColNum,
                                     const mr_matrix* right, int64_t rightRowNum, int64_t rightColNum, int32_t blkSize);
// Scratch the dense x low-density sparse route allocates for one left / right block of its pairs (upper bounds).
size_t dspmm_left_scratch(const Block& a);
size_t dspmm_right_scratch(const Block& b);
// Bytes of Ozaki-II residue scratch multiply_impl allocates for an nr x nc grid of output blocks (the ozaki_scratch_mb rule).
size_t oz2_scratch_for(const mr_context* ctx, int32_t blk, int64_t K, int nr, int nc);
// The streamed multiply (abi_stream.cpp): at least one operand is host-resident; the result is host-resident.
mr_matrix* multiply_streamed(mr_context* ctx, mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right,
                             int64_t rightRowNum, int64_t rightColNum, int32_t blkSize);
// Device memory a streamed multiply or a panelled mr_matrix_to_dense may use (abi_stream.cpp): the option stream_budget_mb, or
// when it is 0 the free device memory at the call minus 1 GiB, counted after the device's memory pool has handed its cache back
// (a synchronisation of the context stream) unless the memory free without that is already `enough`.
size_t stream_budget(mr_context* ctx, size_t enough = SIZE_MAX);
// MR_ENOTSUP for a host-resident operand of an operator that only runs on device datasets.
void require_device(const mr_matrix* m, const char* op);
}  // namespace mrhost

namespace mrhost {

// ---- shared host helpers (abi_core.cpp)
void note_launch(mr_context* ctx, int n = 1);
// Order the context stream (or `stream`) after the producer of a block.  Returns true when the producer was still running.
bool wait_ready(mr_context* ctx, const Block& b);
bool wait_ready_on(cudaStream_t stream, const Block& b);
bool block_done(const Block& b);
bool wait_ready_all(mr_context* ctx, const mr_matrix* m);
Buf upload_bytes(mr_context* ctx, const void* data, size_t bytes);
template <typename T>
Buf upload(mr_context* ctx, const std::vector<T>& v) {
  return upload_bytes(ctx, v.data(), v.size() * sizeof(T));
}
Span upload_raw(mr_context* ctx, const void* host, size_t bytes);
Block dense_block(int32_t rows, int32_t cols, Span values, bool isT = false);
Block densify(mr_context* ctx, const Block& s);
const char* type_name(const Block& b);
int64_t ceil_div(int64_t a, int64_t b);
mr_matrix* new_matrix(mr_context* ctx);
void validate_desc(const mr_block_desc* d);
void check_same_dims(int64_t lr, int64_t lc, int64_t rr, int64_t rc);

// The CSC copy of a CSR block (csr_to_csc): byte offsets of its arrays in a window of `bytes` bytes.
struct CscLayout {
  size_t ptr, idx, val, bytes;
  CscLayout(int32_t cols, int64_t nnz);
};
// One CSR -> CSC conversion: the CSR arrays of a rows x cols block with nnz entries, and the window its CSC copy goes to.
struct CsrToCsc {
  const int32_t* ptr;
  const int32_t* idx;
  const double* val;
  int32_t rows, cols;
  int64_t nnz;
  char* out;  // CscLayout(cols, nnz).bytes
};
// Runs the conversions in one launch_sptrans (indices ascending in every column; a repeated coordinate's entries end up next to
// each other, the last stored first).  Nothing when `convs` is empty.
void csr_to_csc(mr_context* ctx, const std::vector<CsrToCsc>& convs);

// A slab allocator for operator results: one device allocation, blocks are windows into it.
struct Slab {
  Buf buf;
  size_t used = 0;
  Slab(mr_context* ctx, size_t total) : buf(std::make_shared<DevBuf>(ctx, std::max<size_t>(total, kAlign))) {}
  Span take(size_t bytes) {
    Span s{buf, used};
    used += align_up(bytes);
    return s;
  }
};

}  // namespace mrhost
