// Matrix x vector products C = A x and C = x A over dense, CSC and CSR blocks, without dense images (DESIGN section 4.5.5).
//
// Both forms run as C = M x: for A x, M = A; for x A, M = A^T (so a CSC block of A is a CSR block of M and the other way round,
// and a column-major dense block of A is a row-major one of M).  An output block's pairs are its k-blocks in ascending k.
//
// The arithmetic, which these kernels reproduce bit for bit (NaN payloads aside).  Every product is one __dmul_rn, every add one
// __dadd_rn.
//   1. A pair's partial p_k[i] starts at +0.0 and adds its terms M(i, c) x[c] one by one:
//      - dense M and CSR M (A x): c ascending, in storage order (repeats each count);
//      - CSC A (A x): the columns in ascending order, within a column in storage order (LocalMatrix.multiplySparseMatDenseVec);
//      - x S (sparse S): the terms of the dense image S.toDense: the last stored entry of a position counts, and p_k[j] is NaN
//        where a non-finite x[r] meets a position (r, j) that is not stored.
//   2. The partials are combined in ascending k: S = p_k0, then S + p_k1, and so on.
//
// matvec_kernel: one CTA of 8 warps per (output block, tile of 32 outputs).  Warp w computes the partial of pair g + w for the tile,
//   one lane per output; warp 0 then folds the 8 partials into S in pair order.  Dense pairs stream M with 32 loads in flight per
//   lane: a column-major tile (outputs contiguous) column by column, a row-major one (k contiguous) through a 32 x 33 shared tile.
//   CSR pairs walk their row.  Precomputed pairs read the partial matvec_part_kernel wrote.
// matvec_part_kernel: the pairs whose terms of one output are scattered across the stored lines (CSC A x, CSR x S) and the x S
//   pairs of CSC blocks, into a partial per pair.  MV_ALONG: one lane per output line.  MV_ACROSS: one warp per pair walks the
//   entries in storage order into an accumulator (shared memory up to kMvPartSmemLen outputs, else the partial itself); lanes sharing
//   an output index in a step are applied by the lowest of them in lane (= storage) order, as sparse_agg_kernel does.
#include <cuda_pipeline.h>

#include "kernels.h"

namespace matrel {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kMvWarps = 8;
constexpr int kMvTileLd = kMvTile + 1;   // row stride of the shared tile of a row-major pair (no bank conflicts)
constexpr int kMvHalf = 16;              // loads in flight per lane and step of a column-major pair
constexpr int kMvPartWarps = 4;
constexpr int kMvPartUnroll = 4;

__device__ __forceinline__ double pair_partial(const MvPair& p, int i0, int len, int lane, double* tile) {
  const int i = i0 + lane;
  const bool live = i < len;
  double s = 0.0;
  if (p.kind == MV_PART) return live ? p.part[i] : 0.0;
  if (p.kind == MV_CSR) {
    if (live)
      for (int e = p.ptr[i], e1 = p.ptr[i + 1]; e < e1; ++e) s = __dadd_rn(s, __dmul_rn(p.val[e], __ldg(p.x + p.idx[e])));
    return s;
  }
  for (int c0 = 0; c0 < p.kdim; c0 += kMvTile) {
    const int nc = min(kMvTile, p.kdim - c0);
    const double xv = lane < nc ? __ldg(p.x + c0 + lane) : 0.0;
    if (p.kind == MV_DENSE_ICONT) {  // M(i, c) at A[i + c sc]
      const double* a = p.A + i + static_cast<int64_t>(c0) * p.sc;
#pragma unroll
      for (int h = 0; h < kMvTile; h += kMvHalf) {
        double v[kMvHalf];
#pragma unroll
        for (int u = 0; u < kMvHalf; ++u) v[u] = (live && h + u < nc) ? a[static_cast<int64_t>(h + u) * p.sc] : 0.0;
#pragma unroll
        for (int u = 0; u < kMvHalf; ++u) {
          const double w = __shfl_sync(kFull, xv, h + u);
          if (h + u < nc) s = __dadd_rn(s, __dmul_rn(v[u], w));
        }
      }
    } else {  // MV_DENSE_KCONT: M(i, c) at A[i si + c]; the warp copies 32 rows x 32 columns coalesced (cp.async: all 32 copies of a
              // lane in flight), lane r sums row r.  Elements outside the block are not copied: no live lane reads them.
      const int rows = lane < nc ? min(kMvTile, len - i0) : 0;
      const double* src = p.A + static_cast<int64_t>(i0) * p.si + c0 + lane;
      for (int r = 0; r < rows; ++r, src += p.si) __pipeline_memcpy_async(tile + r * kMvTileLd + lane, src, sizeof(double));
      __pipeline_commit();
      __pipeline_wait_prior(0);
      __syncwarp();
      for (int j = 0; j < kMvTile; ++j) {
        const double w = __shfl_sync(kFull, xv, j);
        if (j < nc) s = __dadd_rn(s, __dmul_rn(tile[lane * kMvTileLd + j], w));
      }
      __syncwarp();
    }
  }
  return s;
}

__global__ void __launch_bounds__(kMvWarps * 32) matvec_kernel(const MvOut* __restrict__ outs, const MvPair* __restrict__ pairs,
                                                               const MvItem* __restrict__ items) {
  extern __shared__ __align__(16) double mv_smem[];
  __shared__ double part[kMvWarps][kMvTile];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* tile = mv_smem + warp * kMvTile * kMvTileLd;
  const MvItem it = items[blockIdx.x];
  const MvOut o = outs[it.out];
  const int i0 = it.tile * kMvTile;
  double S = 0.0;
  for (int g = 0; g < o.pair_count; g += kMvWarps) {
    if (g + warp < o.pair_count) {
      const MvPair p = pairs[o.pair_begin + g + warp];
      part[warp][lane] = pair_partial(p, i0, o.len, lane, tile);
    }
    __syncthreads();
    if (warp == 0) {
      const int n = min(kMvWarps, o.pair_count - g);
      for (int w = 0; w < n; ++w) S = (g + w == 0) ? part[w][lane] : __dadd_rn(S, part[w][lane]);
    }
    __syncthreads();
  }
  if (warp == 0 && i0 + lane < o.len) o.C[i0 + lane] = S;
}

// The line of stored entry e: the last c with ptr[c] <= e
__device__ __forceinline__ int line_of(const int32_t* ptr, int nlines, int e) {
  int lo = 0, hi = nlines;  // ptr[lo] <= e < ptr[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(ptr + mid) <= e) lo = mid;
    else hi = mid;
  }
  return lo;
}

// A later entry of the same line stores the same position (the dense image keeps the last one)
__device__ __forceinline__ bool overwritten(const MvPartDesc& d, int e, int line) {
  const int t = d.idx[e];
  for (int f = e + 1, f1 = d.ptr[line + 1]; f < f1; ++f)
    if (d.idx[f] == t) return true;
  return false;
}

__device__ __forceinline__ bool stores(const MvPartDesc& d, int line, int t) {
  for (int f = d.ptr[line], f1 = d.ptr[line + 1]; f < f1; ++f)
    if (d.idx[f] == t) return true;
  return false;
}

// MV_ALONG: p[line] over the entries of one line (one lane per line); x is indexed by the stored index
__device__ __forceinline__ void along(const MvPartDesc& d, int line, int lane) {
  const bool live = line < d.nlines;
  double s = 0.0;
  if (live)
    for (int e = d.ptr[line], e1 = d.ptr[line + 1]; e < e1; ++e)
      if (!d.image || !overwritten(d, e, line)) s = __dadd_rn(s, __dmul_rn(d.val[e], __ldg(d.x + d.idx[e])));
  if (d.image)  // non-finite x[r] facing an unstored (r, line)
    for (int r0 = 0; r0 < d.xlen; r0 += 32) {
      const int r = r0 + lane;
      for (unsigned nf = __ballot_sync(kFull, r < d.xlen && !isfinite(__ldg(d.x + r))); nf; nf &= nf - 1) {
        const int rr = r0 + __ffs(nf) - 1;
        if (live && !stores(d, line, rr)) s = __longlong_as_double(0x7ff8000000000000ll);
      }
    }
  if (live) d.part[line] = s;
}

// MV_ACROSS: acc[t] over the entries with index t, in storage order (one warp per pair); x is indexed by the line
__device__ __forceinline__ void across(const MvPartDesc& d, double* acc, double* stage, int lane) {
  for (int t = lane; t < d.len; t += 32) acc[t] = 0.0;
  __syncwarp();
  const int e0 = d.ptr[0], e1 = d.ptr[d.nlines];
  for (int base = e0; base < e1; base += 32 * kMvPartUnroll) {
    int ti[kMvPartUnroll];
#pragma unroll
    for (int u = 0; u < kMvPartUnroll; ++u) {
      const int e = base + u * 32 + lane;
      ti[u] = -1;
      double tv = 0.0;
      if (e < e1) {
        const int line = line_of(d.ptr, d.nlines, e);
        if (!d.image || !overwritten(d, e, line)) {
          ti[u] = d.idx[e];
          tv = __dmul_rn(d.val[e], __ldg(d.x + line));
        }
      }
      stage[u * 32 + lane] = tv;
    }
    __syncwarp();
#pragma unroll
    for (int u = 0; u < kMvPartUnroll; ++u) {
      const unsigned grp = __match_any_sync(kFull, ti[u]);
      if (ti[u] >= 0 && lane == __ffs(grp) - 1) {  // the lowest lane of its index: its own term, then its peers' in lane order
        double a = __dadd_rn(acc[ti[u]], stage[u * 32 + lane]);
        for (unsigned m = grp & (grp - 1); m; m &= m - 1) a = __dadd_rn(a, stage[u * 32 + __ffs(m) - 1]);
        acc[ti[u]] = a;
      }
      __syncwarp();
    }
  }
  if (d.image)  // non-finite x[line] facing an unstored (line, t)
    for (int r0 = 0; r0 < d.nlines; r0 += 32) {
      const int r = r0 + lane;
      for (unsigned nf = __ballot_sync(kFull, r < d.nlines && !isfinite(__ldg(d.x + r))); nf; nf &= nf - 1) {
        const int rr = r0 + __ffs(nf) - 1;
        for (int t = lane; t < d.len; t += 32)
          if (!stores(d, rr, t)) acc[t] = __longlong_as_double(0x7ff8000000000000ll);
        __syncwarp();
      }
    }
  __syncwarp();
}

__global__ void __launch_bounds__(kMvPartWarps * 32) matvec_part_kernel(const MvPartDesc* __restrict__ descs, int ndescs,
                                                                        int nitems, int smem_len) {
  extern __shared__ __align__(16) double mvp_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* wacc = mvp_smem + static_cast<size_t>(warp) * (smem_len + 32 * kMvPartUnroll);
  double* stage = wacc + smem_len;
  const int stride = gridDim.x * kMvPartWarps;
  for (int it = blockIdx.x * kMvPartWarps + warp; it < nitems; it += stride) {
    const MvPartDesc d = descs[it % ndescs];
    const int g = it / ndescs;
    if (d.mode == MV_ALONG) {
      if (g * 32 < d.nlines) along(d, g * 32 + lane, lane);
    } else if (g == 0) {
      const bool in_smem = d.len <= smem_len;
      across(d, in_smem ? wacc : d.part, stage, lane);
      if (in_smem) {
        for (int t = lane; t < d.len; t += 32) d.part[t] = wacc[t];
        __syncwarp();
      }
    }
  }
}

PerDeviceOnce g_mv_attr, g_mvp_attr;

int resident_ctas(const void* kernel, int threads, size_t smem) {
  int dev = 0, sms = 132, per_sm = 1;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) {
    (void)cudaGetLastError();
    per_sm = 1;
  }
  return sms * per_sm;
}

}  // namespace

cudaError_t launch_matvec(const MvOut* d_outs, const MvPair* d_pairs, const MvItem* d_items, int nitems, cudaStream_t stream) {
  if (nitems <= 0) return cudaSuccess;
  const size_t smem = static_cast<size_t>(kMvWarps) * kMvTile * kMvTileLd * sizeof(double);
  cudaError_t e = g_mv_attr.run([smem] {
    return cudaFuncSetAttribute(matvec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  });
  if (e != cudaSuccess) return e;
  matvec_kernel<<<nitems, kMvWarps * 32, smem, stream>>>(d_outs, d_pairs, d_items);
  return cudaGetLastError();
}

cudaError_t launch_matvec_parts(const MvPartDesc* d_descs, int ndescs, int max_nlines, int max_across_len, cudaStream_t stream) {
  if (ndescs <= 0) return cudaSuccess;
  const int smem_len = max_across_len < kMvPartSmemLen ? max_across_len : kMvPartSmemLen;
  const size_t smem = static_cast<size_t>(kMvPartWarps) * (smem_len + 32 * kMvPartUnroll) * sizeof(double);
  cudaError_t e = g_mvp_attr.run([] {
    return cudaFuncSetAttribute(matvec_part_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(kMvPartWarps * (kMvPartSmemLen + 32 * kMvPartUnroll) * sizeof(double)));
  });
  if (e != cudaSuccess) return e;
  const int groups = max_nlines > 32 ? (max_nlines + 31) / 32 : 1;
  if (static_cast<int64_t>(ndescs) * groups > INT32_MAX) return cudaErrorInvalidValue;
  const int nitems = ndescs * groups;
  const int need = (nitems + kMvPartWarps - 1) / kMvPartWarps;
  const int cap = resident_ctas(reinterpret_cast<const void*>(matvec_part_kernel), kMvPartWarps * 32, smem);
  const int ctas = need < cap ? (need > 0 ? need : 1) : cap;
  matvec_part_kernel<<<ctas, kMvPartWarps * 32, smem, stream>>>(d_descs, ndescs, nitems, smem_len);
  return cudaGetLastError();
}

}  // namespace matrel
