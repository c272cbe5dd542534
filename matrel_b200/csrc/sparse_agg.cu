// Aggregates (rowSum / colSum / trace) and slicing (project / selection) of sparse blocks on their stored entries, without dense
// images of them (DESIGN section 4.5.4).
//
// The arithmetic, which these kernels reproduce bit for bit (NaN payloads aside).  Every add is one __dadd_rn.
//   1. rowSum / colSum: a block's partial at output index t is p[t] = ((0.0 + v1) + v2) + ... over its stored entries at index t,
//      in storage order (repeats each count; explicit zeros, -0.0 and non-finite values take part).  The partials of one output
//      line are combined in ascending block index, S[t] = ((0.0 + p_b0[t]) + p_b1[t]) + ..., and S is stored into the output, or
//      added with an fp64 atomic when the line also has dense blocks.
//   2. trace: t_b = ((0.0 + v1) + v2) + ... over the stored entries whose index equals their line's, in storage order; the
//      diagonal blocks are combined as in 1.
//   3. project / selection: the value at a position is its LAST stored entry in storage order, 0.0 where nothing is stored.
//
// sparse_agg_kernel: a persistent grid over (32-line group, block) work items, so any number of blocks is one launch.  The items
//   are group-major: the first item of every block comes first, so the one-warp-per-block items spread over all warps of the grid.
//   SPAGG_ALONG  (colSum of CSC, rowSum of CSR): one lane per line sums the line in storage order and writes p[line].
//   SPAGG_ACROSS (rowSum of CSC, colSum of CSR): one warp walks the block's entries in storage order, 32 at a time, into an
//     accumulator of the output length (shared memory, or the block's partial slot in global memory above kSpAggSmemLen).  Lanes
//     whose indices are distinct in a step update at once; lanes sharing an index are applied by the lowest of them in lane
//     (= storage) order.  Steps are separated by __syncwarp, so every index sees its entries in storage order.  The loads of
//     kSpAggUnroll steps are issued before their updates.
//   SPAGG_DIAG   (trace): lanes find the diagonal entries of 32 lines at once; the warp adds them line after line.
// sparse_agg_combine_kernel: one thread per output element walks that line's partials in ascending block index.
// sparse_slice_kernel: along a line, the warp zero-fills the output and scatters the line (spread over the lanes when its
//   indices strictly ascend, else one lane in storage order so that the last entry wins); across lines, one lane per line scans
//   it for the index, keeps the last match and writes its output element once.
#include "kernels.h"

namespace matrel {

namespace {

constexpr int kSpAggWarps = 4;   // warps per CTA
constexpr int kSpAggUnroll = 4;  // steps of 32 entries whose loads are in flight together
constexpr unsigned kFull = 0xffffffffu;

// p[t] = 0.0 + v1 + ... over the entries of line t (one lane per line)
__device__ __forceinline__ void along_sum(const SpAggDesc& d, int line) {
  if (line >= d.nlines) return;
  const int s0 = d.ptr[line], s1 = d.ptr[line + 1];
  double s = 0.0;
  for (int e = s0; e < s1; ++e) s = __dadd_rn(s, d.val[e]);
  d.part[line] = s;
}

// acc[t] = 0.0 + v1 + ... over the entries at index t, in storage order (one warp per block)
__device__ __forceinline__ void across_sum(const SpAggDesc& d, double* acc, int lane) {
  for (int t = lane; t < d.len; t += 32) acc[t] = 0.0;
  __syncwarp();
  const int e0 = d.ptr[0], e1 = d.ptr[d.nlines];
  for (int base = e0; base < e1; base += 32 * kSpAggUnroll) {
    int ti[kSpAggUnroll];
    double tv[kSpAggUnroll];
#pragma unroll
    for (int u = 0; u < kSpAggUnroll; ++u) {
      const int e = base + u * 32 + lane;
      ti[u] = e < e1 ? d.idx[e] : -1;
      tv[u] = e < e1 ? d.val[e] : 0.0;
    }
#pragma unroll
    for (int u = 0; u < kSpAggUnroll; ++u) {
      const unsigned grp = __match_any_sync(kFull, ti[u]);
      if (ti[u] >= 0 && lane == __ffs(grp) - 1) {  // the lowest lane of its index: its own entry, then its peers' in lane order
        double a = __dadd_rn(acc[ti[u]], tv[u]);
        for (unsigned m = grp & (grp - 1); m; m &= m - 1) a = __dadd_rn(a, d.val[base + u * 32 + __ffs(m) - 1]);
        acc[ti[u]] = a;
      }
      __syncwarp();
    }
  }
}

// t_b = 0.0 + v1 + ... over the entries with index == line, in storage order (one warp per block; the sum is warp-uniform)
__device__ __forceinline__ void diag_sum(const SpAggDesc& d, int lane) {
  double s = 0.0;
  for (int l0 = 0; l0 < d.nlines; l0 += 32) {
    const int l = l0 + lane;
    int s0 = 0, s1 = 0, cnt = 0;
    double v = 0.0;
    if (l < d.nlines) {
      s0 = d.ptr[l];
      s1 = d.ptr[l + 1];
      for (int e = s0; e < s1; ++e)
        if (d.idx[e] == l) {
          if (cnt == 0) v = d.val[e];
          ++cnt;
        }
    }
    for (unsigned has = __ballot_sync(kFull, cnt > 0); has; has &= has - 1) {
      const int k = __ffs(has) - 1;
      const int ck = __shfl_sync(kFull, cnt, k);
      const double vk = __shfl_sync(kFull, v, k);
      if (ck == 1) {
        s = __dadd_rn(s, vk);
      } else {  // a repeated diagonal position: walk the line in storage order
        const int a = __shfl_sync(kFull, s0, k), b = __shfl_sync(kFull, s1, k);
        for (int e = a; e < b; ++e)
          if (d.idx[e] == l0 + k) s = __dadd_rn(s, d.val[e]);
      }
    }
  }
  if (lane == 0) d.part[0] = s;
}

__global__ void __launch_bounds__(kSpAggWarps * 32) sparse_agg_kernel(const SpAggDesc* __restrict__ descs, int ndescs,
                                                                      int64_t nitems, int smem_len) {
  extern __shared__ __align__(16) double spagg_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* wacc = spagg_smem + static_cast<size_t>(warp) * smem_len;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kSpAggWarps;
  for (int64_t it = static_cast<int64_t>(blockIdx.x) * kSpAggWarps + warp; it < nitems; it += stride) {
    const SpAggDesc d = descs[it % ndescs];
    const int g = static_cast<int>(it / ndescs);
    if (d.mode == SPAGG_ALONG) {
      along_sum(d, g * 32 + lane);
    } else if (g == 0 && d.mode == SPAGG_ACROSS) {
      const bool in_smem = d.len <= smem_len;
      across_sum(d, in_smem ? wacc : d.part, lane);
      if (in_smem) {
        __syncwarp();
        for (int t = lane; t < d.len; t += 32) d.part[t] = wacc[t];
        __syncwarp();
      }
    } else if (g == 0) {
      diag_sum(d, lane);
    }
  }
}

constexpr int kCombineThreads = 256;

__global__ void __launch_bounds__(kCombineThreads) sparse_agg_combine_kernel(const SpAggOut* __restrict__ outs, int64_t nitems,
                                                                             int chunks) {
  for (int64_t it = blockIdx.x; it < nitems; it += gridDim.x) {
    const SpAggOut o = outs[it / chunks];
    const int t = static_cast<int>(it % chunks) * kCombineThreads + threadIdx.x;
    if (t >= o.len) continue;
    double s = 0.0;
#pragma unroll 4
    for (int p = 0; p < o.nparts; ++p) s = __dadd_rn(s, o.part[static_cast<size_t>(p) * o.len + t]);
    if (o.accumulate) atomicAdd(o.out + t, s);
    else o.out[t] = s;
  }
}

__global__ void __launch_bounds__(kSpAggWarps * 32) sparse_slice_kernel(const SpSliceDesc* __restrict__ descs, int ndescs,
                                                                        int64_t nitems) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kSpAggWarps;
  for (int64_t it = static_cast<int64_t>(blockIdx.x) * kSpAggWarps + warp; it < nitems; it += stride) {
    const SpSliceDesc d = descs[it % ndescs];
    const int g = static_cast<int>(it / ndescs);
    if (d.target < 0) {  // along the line: zero-fill, then the entries
      if (g != 0) continue;
      for (int t = lane; t < d.len; t += 32) d.out[t] = 0.0;
      __syncwarp();
      const int s0 = d.ptr[d.line], s1 = d.ptr[d.line + 1];
      bool asc = true;
      for (int e = s0 + lane; e + 1 < s1; e += 32) asc = asc && d.idx[e] < d.idx[e + 1];
      if (__all_sync(kFull, asc)) {
        for (int e = s0 + lane; e < s1; e += 32) d.out[d.idx[e]] = d.val[e];
      } else if (lane == 0) {
        for (int e = s0; e < s1; ++e) d.out[d.idx[e]] = d.val[e];
      }
      __syncwarp();
    } else {  // across lines: one lane per line, the last match
      const int t = g * 32 + lane;
      if (t >= d.len) continue;
      const int l = d.line + t;
      const int s0 = d.ptr[l], s1 = d.ptr[l + 1];
      double v = 0.0;
      for (int e = s0; e < s1; ++e)
        if (d.idx[e] == d.target) v = d.val[e];
      d.out[t] = v;
    }
  }
}

PerDeviceOnce g_spagg_attr;

int persistent_ctas(const void* kernel, int threads, size_t smem) {
  int dev = 0, sms = 132, per_sm = 1;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) {
    (void)cudaGetLastError();
    per_sm = 1;
  }
  return sms * per_sm;
}

int capped(int64_t need, int max_ctas) { return static_cast<int>(need < max_ctas ? (need > 0 ? need : 1) : max_ctas); }

}  // namespace

cudaError_t launch_sparse_agg(const SpAggDesc* d_descs, int ndescs, int max_nlines, int max_across_len, cudaStream_t stream) {
  if (ndescs <= 0) return cudaSuccess;
  const int smem_len = max_across_len < kSpAggSmemLen ? max_across_len : kSpAggSmemLen;
  const size_t smem = static_cast<size_t>(kSpAggWarps) * smem_len * sizeof(double);
  cudaError_t e = g_spagg_attr.run([] {
    return cudaFuncSetAttribute(sparse_agg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(kSpAggWarps * kSpAggSmemLen * sizeof(double)));
  });
  if (e != cudaSuccess) return e;
  const int groups = max_nlines > 32 ? (max_nlines + 31) / 32 : 1;
  const int64_t nitems = static_cast<int64_t>(ndescs) * groups;
  const int ctas = capped((nitems + kSpAggWarps - 1) / kSpAggWarps,
                          persistent_ctas(reinterpret_cast<const void*>(sparse_agg_kernel), kSpAggWarps * 32, smem));
  sparse_agg_kernel<<<ctas, kSpAggWarps * 32, smem, stream>>>(d_descs, ndescs, nitems, smem_len);
  return cudaGetLastError();
}

cudaError_t launch_sparse_agg_combine(const SpAggOut* d_outs, int nouts, int max_len, cudaStream_t stream) {
  if (nouts <= 0 || max_len <= 0) return cudaSuccess;
  const int chunks = (max_len + kCombineThreads - 1) / kCombineThreads;
  const int64_t nitems = static_cast<int64_t>(nouts) * chunks;
  const int ctas = capped(nitems, persistent_ctas(reinterpret_cast<const void*>(sparse_agg_combine_kernel), kCombineThreads, 0));
  sparse_agg_combine_kernel<<<ctas, kCombineThreads, 0, stream>>>(d_outs, nitems, chunks);
  return cudaGetLastError();
}

cudaError_t launch_sparse_slice(const SpSliceDesc* d_descs, int ndescs, int max_len, cudaStream_t stream) {
  if (ndescs <= 0) return cudaSuccess;
  const int groups = max_len > 32 ? (max_len + 31) / 32 : 1;
  const int64_t nitems = static_cast<int64_t>(ndescs) * groups;
  const int ctas = capped((nitems + kSpAggWarps - 1) / kSpAggWarps,
                          persistent_ctas(reinterpret_cast<const void*>(sparse_slice_kernel), kSpAggWarps * 32, 0));
  sparse_slice_kernel<<<ctas, kSpAggWarps * 32, 0, stream>>>(d_descs, ndescs, nitems);
  return cudaGetLastError();
}

}  // namespace matrel
