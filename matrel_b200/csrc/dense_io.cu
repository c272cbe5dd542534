// Whole dense matrices in and out of datasets (mr_matrix_from_dense / mr_matrix_to_dense, abi_dense.cpp), batched over the blocks
// of a matrix or of one panel of it (one launch, a descriptor per window):
//   dense_gather_kernel    a device matrix -> its blocks, each in the matrix's own layout (a row-major sub-block is the reference's
//                          transposed dense block, MLMatrix.scala:285-289), so both sides are read and written along lines
//   dense_assemble_kernel  blocks -> windows of a matrix (DenseMatrix.toArray, MLMatrix.scala:55-61, for a whole dataset): line
//                          copies when the layouts agree, a 32x32 tile through padded shared memory when they differ, zero fill for
//                          windows with no dense data
//   dense_scatter_kernel   the entries of sparse blocks into their zero-filled windows (SparseMatrix.toArray, MLMatrix.scala:637-663)
// Line copies use 128-bit loads and stores whenever a line's source and destination share their 16-byte phase (an 8-byte aligned
// torch slice, an odd leading dimension: one scalar element first), 64-bit ones otherwise; both stay coalesced.
#include "kernels.h"

namespace matrel {
namespace {

constexpr int IO_THREADS = 256;
constexpr int IO_WARPS = IO_THREADS / 32;
constexpr int IO_CHUNK = 512;  // elements of one line a warp copies per work unit

// One warp copies n elements s[0..n) -> d[0..n) (s == nullptr: writes zeros).
__device__ __forceinline__ void copy_line(const double* __restrict__ s, double* __restrict__ d, int n, int lane) {
  const bool zero = (s == nullptr);
  const uintptr_t pd = reinterpret_cast<uintptr_t>(d);
  if (!zero && ((reinterpret_cast<uintptr_t>(s) ^ pd) & 15) != 0) {
    for (int i = lane; i < n; i += 32) d[i] = __ldcs(s + i);
    return;
  }
  const int head = (pd & 15) != 0 ? 1 : 0;
  if (lane == 0 && head && n > 0) d[0] = zero ? 0.0 : __ldcs(s);
  const int nvec = n > head ? (n - head) >> 1 : 0;
  double2* d2 = reinterpret_cast<double2*>(d + head);
  if (zero) {
    for (int i = lane; i < nvec; i += 32) __stcs(d2 + i, make_double2(0.0, 0.0));
  } else {
    const double2* s2 = reinterpret_cast<const double2*>(s + head);
    int i = lane;
    for (; i + 96 < nvec; i += 128) {  // four independent 128-bit loads in flight per lane
      const double2 a = __ldcs(s2 + i), b = __ldcs(s2 + i + 32), c = __ldcs(s2 + i + 64), e = __ldcs(s2 + i + 96);
      __stcs(d2 + i, a);
      __stcs(d2 + i + 32, b);
      __stcs(d2 + i + 64, c);
      __stcs(d2 + i + 96, e);
    }
    for (; i < nvec; i += 32) __stcs(d2 + i, __ldcs(s2 + i));
  }
  const int t = head + 2 * nvec;  // at most one element left
  if (lane == 0 && t < n) d[t] = zero ? 0.0 : __ldcs(s + t);
}

// Same layout on both sides: the window is `slow` lines of `fast` elements; a work unit is up to IO_CHUNK elements of one line,
// one warp per unit, grid-stride over the units of the descriptor.
__device__ __forceinline__ void copy_window(const DenseIoDesc& d) {
  const bool rm = d.dst_rm != 0;
  const int fast = rm ? d.cols : d.rows, slow = rm ? d.rows : d.cols;
  if (fast <= 0 || slow <= 0) return;
  const int chunks = (fast + IO_CHUNK - 1) / IO_CHUNK;
  const int64_t units = static_cast<int64_t>(slow) * chunks;
  const int lane = threadIdx.x & 31;
  for (int64_t u = static_cast<int64_t>(blockIdx.x) * IO_WARPS + (threadIdx.x >> 5); u < units;
       u += static_cast<int64_t>(gridDim.x) * IO_WARPS) {
    const int64_t line = u / chunks;
    const int f0 = static_cast<int>(u % chunks) * IO_CHUNK;
    copy_line(d.src ? d.src + line * d.lds + f0 : nullptr, d.dst + line * d.ldd + f0, min(IO_CHUNK, fast - f0), lane);
  }
}

// Layouts differ: src element (a, b) at src[a + b * lds] (a along src's contiguous dimension) goes to dst[b + a * ldd].  32x32 tiles,
// read along a and written along b, both coalesced; the 33-double row pitch spreads the column reads over the banks.
__device__ __forceinline__ void transpose_window(const DenseIoDesc& d, double (&sm)[32][33]) {
  const int fa = d.src_rm ? d.cols : d.rows, fb = d.src_rm ? d.rows : d.cols;
  const int ta = (fa + 31) / 32, tb = (fb + 31) / 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int t = blockIdx.x; t < ta * tb; t += gridDim.x) {  // uniform across the CTA: the __syncthreads below are safe
    const int a0 = (t % ta) * 32, b0 = (t / ta) * 32;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int a = a0 + tx, b = b0 + ty + 8 * j;
      if (a < fa && b < fb) sm[ty + 8 * j][tx] = __ldcs(d.src + a + static_cast<int64_t>(b) * d.lds);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int a = a0 + ty + 8 * j, b = b0 + tx;
      if (a < fa && b < fb) __stcs(d.dst + b + static_cast<int64_t>(a) * d.ldd, sm[tx][ty + 8 * j]);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(IO_THREADS) dense_gather_kernel(const DenseIoDesc* __restrict__ descs) {
  copy_window(descs[blockIdx.y]);
}

__global__ void __launch_bounds__(IO_THREADS) dense_assemble_kernel(const DenseIoDesc* __restrict__ descs) {
  __shared__ double sm[32][33];
  const DenseIoDesc& d = descs[blockIdx.y];
  if (d.src != nullptr && d.src_rm != d.dst_rm) transpose_window(d, sm);
  else copy_window(d);
}

// One warp per compressed line (a column of a CSC block, a row of a CSR one), grid-stride over the lines.
__global__ void __launch_bounds__(IO_THREADS) dense_scatter_kernel(const DenseScatterDesc* __restrict__ descs) {
  const DenseScatterDesc d = descs[blockIdx.y];
  const int lane = threadIdx.x & 31;
  for (int line = blockIdx.x * IO_WARPS + (threadIdx.x >> 5); line < d.nlines; line += gridDim.x * IO_WARPS) {
    const int beg = d.ptrs[line], end = d.ptrs[line + 1];
    for (int e = beg + lane; e < end; e += 32) {
      const int64_t r = d.csr ? line : d.idx[e], c = d.csr ? d.idx[e] : line;
      d.dst[d.dst_rm ? r * d.ldd + c : r + c * d.ldd] = d.vals[e];
    }
  }
}

unsigned io_grid_x(int64_t ctas) { return static_cast<unsigned>(ctas < 1 ? 1 : (ctas > 65535 ? 65535 : ctas)); }

// CTAs that cover the largest window of a launch under either path (the rest of a grid-stride loop picks up what a cap leaves)
int64_t io_ctas(int max_rows, int max_cols, bool transposes) {
  const int64_t by_rows = static_cast<int64_t>(max_rows) * ((max_cols + IO_CHUNK - 1) / IO_CHUNK);  // row-major windows
  const int64_t by_cols = static_cast<int64_t>(max_cols) * ((max_rows + IO_CHUNK - 1) / IO_CHUNK);  // column-major windows
  const int64_t copy = ((by_rows > by_cols ? by_rows : by_cols) + IO_WARPS - 1) / IO_WARPS;
  const int64_t tiles = transposes ? ((max_rows + 31) / 32) * static_cast<int64_t>((max_cols + 31) / 32) : 0;
  return copy > tiles ? copy : tiles;
}

}  // namespace

cudaError_t launch_dense_gather(const DenseIoDesc* d_descs, int ndescs, int max_rows, int max_cols, cudaStream_t stream) {
  if (ndescs <= 0 || max_rows <= 0 || max_cols <= 0) return cudaSuccess;
  const unsigned gx = io_grid_x(io_ctas(max_rows, max_cols, false));
  for (int off = 0; off < ndescs; off += 65535)  // gridDim.y limit
    dense_gather_kernel<<<dim3(gx, ndescs - off < 65535 ? ndescs - off : 65535), IO_THREADS, 0, stream>>>(d_descs + off);
  return cudaGetLastError();
}

cudaError_t launch_dense_assemble(const DenseIoDesc* d_descs, int ndescs, int max_rows, int max_cols, bool any_transposed,
                                  cudaStream_t stream) {
  if (ndescs <= 0 || max_rows <= 0 || max_cols <= 0) return cudaSuccess;
  const unsigned gx = io_grid_x(io_ctas(max_rows, max_cols, any_transposed));
  for (int off = 0; off < ndescs; off += 65535)
    dense_assemble_kernel<<<dim3(gx, ndescs - off < 65535 ? ndescs - off : 65535), IO_THREADS, 0, stream>>>(d_descs + off);
  return cudaGetLastError();
}

cudaError_t launch_dense_scatter(const DenseScatterDesc* d_descs, int ndescs, int max_lines, cudaStream_t stream) {
  if (ndescs <= 0 || max_lines <= 0) return cudaSuccess;
  const unsigned gx = io_grid_x((max_lines + IO_WARPS - 1) / IO_WARPS);
  for (int off = 0; off < ndescs; off += 65535)
    dense_scatter_kernel<<<dim3(gx, ndescs - off < 65535 ? ndescs - off : 65535), IO_THREADS, 0, stream>>>(d_descs + off);
  return cudaGetLastError();
}

}  // namespace matrel
