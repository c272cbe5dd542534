// Matrix x thin-matrix products C = A X and C = X A over dense, CSC and CSR blocks, without dense images (DESIGN section 4.5.5).
// X has 1 to kMvMaxCols columns (A X) or rows (X A); 1 is the matrix x vector product.
//
// Both forms run as C = M X: for A X, M = A; for X A, M = A^T (so a CSC block of A is a CSR block of M and the other way round,
// and a column-major dense block of A is a row-major one of M).  An output block's pairs are its k-blocks in ascending k.
//
// The arithmetic, which these kernels reproduce bit for bit (NaN payloads aside), column by column: column j of C is the width-1
// product M X(:, j).  Every product is one __dmul_rn, every add one __dadd_rn.
//   1. A pair's partial p_k[i] starts at +0.0 and adds its terms M(i, c) x[c] one by one:
//      - dense M and CSR M (A x): c ascending, in storage order (repeats each count);
//      - CSC A (A x): the columns in ascending order, within a column in storage order (LocalMatrix.multiplySparseMatDenseVec);
//      - x S (sparse S): the terms of the dense image S.toDense: the last stored entry of a position counts, and p_k[j] is NaN
//        where a non-finite x[r] meets a position (r, j) that is not stored.
//   2. The partials are combined in ascending k: S = p_k0, then S + p_k1, and so on.
//
// Both kernels are templates on the width W in {1, 2, 4, 8}; a call with cols < W runs W with the columns >= cols reading column
// cols - 1 and never stored.  A lane keeps W accumulators, so every matrix element, stored entry and index is read once for all
// columns.
// matvec_kernel: one CTA of 8 warps per (output block, tile of 32 outputs).  Warp w computes the partial of pair g + w for the tile,
//   one lane per output; warp 0 then folds the 8 partials into S in pair order.  Dense pairs stream M with 32 loads in flight per
//   lane: a column-major tile (outputs contiguous) column by column, a row-major one (k contiguous) through a 32 x 33 shared tile.
//   CSR pairs walk their row.  Precomputed pairs read the partial matvec_part_kernel wrote.  X A tiles of C (j fastest) are staged
//   in shared memory so that the stores are contiguous.
// matvec_part_kernel: the pairs whose terms of one output are scattered across the stored lines (CSC A x, CSR x S) and the x S
//   pairs of CSC blocks, into a partial per pair.  MV_ALONG: one lane per output line.  MV_ACROSS: one warp per pair walks the
//   entries in storage order into an accumulator (shared memory up to kMvPartSmemLen<W> outputs, else the partial itself); lanes
//   sharing an output index in a step are applied by the lowest of them in lane (= storage) order, as sparse_agg_kernel does.
#include <cuda_pipeline.h>

#include "kernels.h"

namespace matrel {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kMvWarps = 8;
constexpr int kMvTileLd = kMvTile + 1;   // row stride of the shared tile of a row-major pair (no bank conflicts)
constexpr int kMvHalf = 16;              // loads in flight per lane and step of a column-major pair
constexpr int kMvPartUnroll = 4;
// Longest MV_ACROSS output a warp accumulates in shared memory at width W (W doubles per output; longer ones in the partial), and
// the warps per CTA that keep a pre-pass CTA near 72 KiB of shared memory: 2048 outputs x 4 warps at W = 1, 1024 outputs x 4, 2 and
// 1 warps at W = 2, 4 and 8 (so blocks of 1024 stay in shared memory at every width).
template <int W>
constexpr int kMvPartSmemLen = W == 1 ? 2048 : 1024;
template <int W>
constexpr int kMvPartWarps = W <= 2 ? 4 : 8 / W;

// The column offsets of an X block: x(c, j) at x[c xl.c + xo[j]]; columns >= cols read column cols - 1 (never stored)
template <int W>
__device__ __forceinline__ void column_offsets(const MvXLayout& xl, int cols, int (&xo)[W]) {
#pragma unroll
  for (int j = 0; j < W; ++j) xo[j] = W == 1 ? 0 : min(j, cols - 1) * xl.j;
}

template <int W>
__device__ __forceinline__ double xat(const double* x, const MvXLayout& xl, const int (&xo)[W], int c, int j) {
  return W == 1 ? __ldg(x + c) : __ldg(x + c * xl.c + xo[j]);
}

template <int W>
__device__ __forceinline__ void pair_partial(const MvPair& p, const MvXLayout& xl, int cols, int i0, int len, int lane, double* tile,
                                             double (&s)[W]) {
  const int i = i0 + lane;
  const bool live = i < len;
  int xo[W];
  column_offsets<W>(xl, cols, xo);
#pragma unroll
  for (int j = 0; j < W; ++j) s[j] = 0.0;
  if (p.kind == MV_PART) {
#pragma unroll
    for (int j = 0; j < W; ++j) s[j] = live && (W == 1 || j < cols) ? p.part[i + j * len] : 0.0;
    return;
  }
  if (p.kind == MV_CSR) {
    if (live)
      for (int e = p.ptr[i], e1 = p.ptr[i + 1]; e < e1; ++e)
#pragma unroll
        for (int j = 0; j < W; ++j) s[j] = __dadd_rn(s[j], __dmul_rn(p.val[e], xat<W>(p.x, xl, xo, p.idx[e], j)));
    return;
  }
  for (int c0 = 0; c0 < p.kdim; c0 += kMvTile) {
    const int nc = min(kMvTile, p.kdim - c0);
    double xv[W];
#pragma unroll
    for (int j = 0; j < W; ++j) xv[j] = lane < nc ? xat<W>(p.x, xl, xo, c0 + lane, j) : 0.0;
    if (p.kind == MV_DENSE_ICONT) {  // M(i, c) at A[i + c sc]
      const double* a = p.A + i + static_cast<int64_t>(c0) * p.sc;
#pragma unroll
      for (int h = 0; h < kMvTile; h += kMvHalf) {
        double v[kMvHalf];
#pragma unroll
        for (int u = 0; u < kMvHalf; ++u) v[u] = (live && h + u < nc) ? a[static_cast<int64_t>(h + u) * p.sc] : 0.0;
#pragma unroll
        for (int u = 0; u < kMvHalf; ++u)
#pragma unroll
          for (int j = 0; j < W; ++j) {
            const double w = __shfl_sync(kFull, xv[j], h + u);
            if (h + u < nc) s[j] = __dadd_rn(s[j], __dmul_rn(v[u], w));
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
      for (int c = 0; c < kMvTile; ++c)
#pragma unroll
        for (int j = 0; j < W; ++j) {
          const double w = __shfl_sync(kFull, xv[j], c);
          if (c < nc) s[j] = __dadd_rn(s[j], __dmul_rn(tile[lane * kMvTileLd + c], w));
        }
      __syncwarp();
    }
  }
}

template <int W>
__global__ void __launch_bounds__(kMvWarps * 32, W == 1 ? 0 : 1) matvec_kernel(const MvOut* __restrict__ outs, const MvPair* __restrict__ pairs,
                                                               const MvItem* __restrict__ items, const MvXLayout* __restrict__ xls,
                                                               int xa) {
  extern __shared__ __align__(16) double mv_smem[];
  __shared__ double part[kMvWarps][W][kMvTile];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* tile = mv_smem + warp * kMvTile * kMvTileLd;
  const MvItem it = items[blockIdx.x];
  const MvOut o = outs[it.out];
  const int i0 = it.tile * kMvTile;
  double S[W];
#pragma unroll
  for (int j = 0; j < W; ++j) S[j] = 0.0;
  for (int g = 0; g < o.pair_count; g += kMvWarps) {
    if (g + warp < o.pair_count) {
      const int pi = o.pair_begin + g + warp;
      const MvPair p = pairs[pi];
      double s[W];
      pair_partial<W>(p, W == 1 ? MvXLayout{} : xls[pi], o.cols, i0, o.len, lane, tile, s);
#pragma unroll
      for (int j = 0; j < W; ++j) part[warp][j][lane] = s[j];
    }
    __syncthreads();
    if (warp == 0) {
      const int n = min(kMvWarps, o.pair_count - g);
      for (int w = 0; w < n; ++w)
#pragma unroll
        for (int j = 0; j < W; ++j) S[j] = (g + w == 0) ? part[w][j][lane] : __dadd_rn(S[j], part[w][j][lane]);
    }
    __syncthreads();
  }
  if (W == 1 || !xa) {  // (i, j) at i + j len
#pragma unroll
    for (int j = 0; j < W; ++j)
      if (warp == 0 && (W == 1 || j < o.cols) && i0 + lane < o.len) o.C[i0 + lane + j * o.len] = S[j];
  } else if (warp == 0) {  // (j, i) at j + i cols: the tile's outputs are one contiguous run, written through part[0] (free after the last fold)
    double* st = &part[0][0][0];
#pragma unroll
    for (int j = 0; j < W; ++j) st[lane * W + j] = S[j];
    __syncwarp();
    const int n = min(kMvTile, o.len - i0) * o.cols;
    for (int e = lane; e < n; e += 32) o.C[i0 * o.cols + e] = st[e / o.cols * W + e % o.cols];
  }
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
template <int W>
__device__ __forceinline__ void along(const MvPartDesc& d, const MvXLayout& xl, int line, int lane) {
  const bool live = line < d.nlines;
  int xo[W];
  column_offsets<W>(xl, d.cols, xo);
  double s[W];
#pragma unroll
  for (int j = 0; j < W; ++j) s[j] = 0.0;
  if (live)
    for (int e = d.ptr[line], e1 = d.ptr[line + 1]; e < e1; ++e)
      if (!d.image || !overwritten(d, e, line))
#pragma unroll
        for (int j = 0; j < W; ++j) s[j] = __dadd_rn(s[j], __dmul_rn(d.val[e], xat<W>(d.x, xl, xo, d.idx[e], j)));
  if (d.image)  // non-finite x(r, j) facing an unstored (r, line)
#pragma unroll
    for (int j = 0; j < W; ++j)
      if (W == 1 || j < d.cols)
      for (int r0 = 0; r0 < d.xlen; r0 += 32) {
        const int r = r0 + lane;
        for (unsigned nf = __ballot_sync(kFull, r < d.xlen && !isfinite(xat<W>(d.x, xl, xo, r, j))); nf; nf &= nf - 1) {
          const int rr = r0 + __ffs(nf) - 1;
          if (live && !stores(d, line, rr)) s[j] = __longlong_as_double(0x7ff8000000000000ll);
        }
      }
  if (live)
#pragma unroll
    for (int j = 0; j < W; ++j)
      if (W == 1 || j < d.cols) d.part[line + j * d.len] = s[j];
}

// MV_ACROSS: acc[t + j ld] over the entries with index t, in storage order (one warp per pair); x is indexed by the line
template <int W>
__device__ __forceinline__ void across(const MvPartDesc& d, const MvXLayout& xl, double* acc, int ld, double* stage, int lane) {
  int xo[W];
  column_offsets<W>(xl, d.cols, xo);
  const int cols = W == 1 ? 1 : d.cols;
#pragma unroll
  for (int j = 0; j < W; ++j)
    if (j < cols)
      for (int t = lane; t < d.len; t += 32) acc[t + j * ld] = 0.0;
  __syncwarp();
  const int e0 = d.ptr[0], e1 = d.ptr[d.nlines];
  for (int base = e0; base < e1; base += 32 * kMvPartUnroll) {
    int ti[kMvPartUnroll];
#pragma unroll
    for (int u = 0; u < kMvPartUnroll; ++u) {
      const int e = base + u * 32 + lane;
      ti[u] = -1;
      double tv[W];
#pragma unroll
      for (int j = 0; j < W; ++j) tv[j] = 0.0;
      if (e < e1) {
        const int line = line_of(d.ptr, d.nlines, e);
        if (!d.image || !overwritten(d, e, line)) {
          ti[u] = d.idx[e];
#pragma unroll
          for (int j = 0; j < W; ++j) tv[j] = __dmul_rn(d.val[e], xat<W>(d.x, xl, xo, line, j));
        }
      }
#pragma unroll
      for (int j = 0; j < W; ++j) stage[(u * W + j) * 32 + lane] = tv[j];
    }
    __syncwarp();
#pragma unroll
    for (int u = 0; u < kMvPartUnroll; ++u) {
      const unsigned grp = __match_any_sync(kFull, ti[u]);
      if (ti[u] >= 0 && lane == __ffs(grp) - 1)  // the lowest lane of its index: its own term, then its peers' in lane order
#pragma unroll
        for (int j = 0; j < W; ++j) {
          if (j >= cols) break;
          double a = __dadd_rn(acc[ti[u] + j * ld], stage[(u * W + j) * 32 + lane]);
          for (unsigned m = grp & (grp - 1); m; m &= m - 1) a = __dadd_rn(a, stage[(u * W + j) * 32 + __ffs(m) - 1]);
          acc[ti[u] + j * ld] = a;
        }
      __syncwarp();
    }
  }
  if (d.image)  // non-finite x(line, j) facing an unstored (line, t)
#pragma unroll
    for (int j = 0; j < W; ++j)
      if (j < cols)
      for (int r0 = 0; r0 < d.nlines; r0 += 32) {
        const int r = r0 + lane;
        for (unsigned nf = __ballot_sync(kFull, r < d.nlines && !isfinite(xat<W>(d.x, xl, xo, r, j))); nf; nf &= nf - 1) {
          const int rr = r0 + __ffs(nf) - 1;
          for (int t = lane; t < d.len; t += 32)
            if (!stores(d, rr, t)) acc[t + j * ld] = __longlong_as_double(0x7ff8000000000000ll);
          __syncwarp();
        }
      }
  __syncwarp();
}

template <int W>
__global__ void __launch_bounds__(kMvPartWarps<W> * 32, W == 1 ? 0 : 1) matvec_part_kernel(const MvPartDesc* __restrict__ descs, int ndescs,
                                                                            int nitems, int smem_len,
                                                                            const MvXLayout* __restrict__ xls) {
  constexpr int kWarps = kMvPartWarps<W>;
  extern __shared__ __align__(16) double mvp_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* wacc = mvp_smem + static_cast<size_t>(warp) * (smem_len + 32 * kMvPartUnroll) * W;
  double* stage = wacc + smem_len * W;
  const int stride = gridDim.x * kWarps;
  for (int it = blockIdx.x * kWarps + warp; it < nitems; it += stride) {
    const MvPartDesc d = descs[it % ndescs];
    const MvXLayout xl = W == 1 ? MvXLayout{} : xls[it % ndescs];
    const int g = it / ndescs;
    if (d.mode == MV_ALONG) {
      if (g * 32 < d.nlines) along<W>(d, xl, g * 32 + lane, lane);
    } else if (g == 0) {
      const bool in_smem = d.len <= smem_len;
      across<W>(d, xl, in_smem ? wacc : d.part, in_smem ? smem_len : d.len, stage, lane);
      if (in_smem) {
#pragma unroll
        for (int j = 0; j < W; ++j)
          if (W == 1 || j < d.cols)
            for (int t = lane; t < d.len; t += 32) d.part[t + j * d.len] = wacc[t + j * smem_len];
        __syncwarp();
      }
    }
  }
}

PerDeviceOnce g_mv_attr[4], g_mvp_attr[4];  // per width 1, 2, 4, 8

int resident_ctas(const void* kernel, int threads, size_t smem) {
  int dev = 0, sms = 132, per_sm = 1;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) {
    (void)cudaGetLastError();
    per_sm = 1;
  }
  return sms * per_sm;
}

template <int W, int L>
cudaError_t matvec_w(const MvOut* d_outs, const MvPair* d_pairs, const MvItem* d_items, int nitems, const MvXLayout* d_xls, int xa,
                     cudaStream_t stream) {
  const size_t smem = static_cast<size_t>(kMvWarps) * kMvTile * kMvTileLd * sizeof(double);
  cudaError_t e = g_mv_attr[L].run([smem] {
    return cudaFuncSetAttribute(matvec_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  });
  if (e != cudaSuccess) return e;
  matvec_kernel<W><<<nitems, kMvWarps * 32, smem, stream>>>(d_outs, d_pairs, d_items, d_xls, xa);
  return cudaGetLastError();
}

template <int W, int L>
cudaError_t matvec_parts_w(const MvPartDesc* d_descs, int ndescs, int max_nlines, int max_across_len, const MvXLayout* d_xls,
                           cudaStream_t stream) {
  constexpr int kWarps = kMvPartWarps<W>, kLen = kMvPartSmemLen<W>;
  const int smem_len = max_across_len < kLen ? max_across_len : kLen;
  const size_t smem = static_cast<size_t>(kWarps) * (smem_len + 32 * kMvPartUnroll) * W * sizeof(double);
  cudaError_t e = g_mvp_attr[L].run([] {
    return cudaFuncSetAttribute(matvec_part_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(kWarps * (kLen + 32 * kMvPartUnroll) * W * sizeof(double)));
  });
  if (e != cudaSuccess) return e;
  const int groups = max_nlines > 32 ? (max_nlines + 31) / 32 : 1;
  if (static_cast<int64_t>(ndescs) * groups > INT32_MAX) return cudaErrorInvalidValue;
  const int nitems = ndescs * groups;
  const int need = (nitems + kWarps - 1) / kWarps;
  const int cap = resident_ctas(reinterpret_cast<const void*>(matvec_part_kernel<W>), kWarps * 32, smem);
  const int ctas = need < cap ? (need > 0 ? need : 1) : cap;
  matvec_part_kernel<W><<<ctas, kWarps * 32, smem, stream>>>(d_descs, ndescs, nitems, smem_len, d_xls);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_matvec(const MvOut* d_outs, const MvPair* d_pairs, const MvItem* d_items, int nitems, int max_cols,
                          const MvXLayout* d_xls, int xa, cudaStream_t stream) {
  if (nitems <= 0) return cudaSuccess;
  if (max_cols <= 1) return matvec_w<1, 0>(d_outs, d_pairs, d_items, nitems, d_xls, xa, stream);
  if (max_cols <= 2) return matvec_w<2, 1>(d_outs, d_pairs, d_items, nitems, d_xls, xa, stream);
  if (max_cols <= 4) return matvec_w<4, 2>(d_outs, d_pairs, d_items, nitems, d_xls, xa, stream);
  if (max_cols <= kMvMaxCols) return matvec_w<8, 3>(d_outs, d_pairs, d_items, nitems, d_xls, xa, stream);
  return cudaErrorInvalidValue;
}

cudaError_t launch_matvec_parts(const MvPartDesc* d_descs, int ndescs, int max_nlines, int max_across_len, int max_cols,
                                const MvXLayout* d_xls, cudaStream_t stream) {
  if (ndescs <= 0) return cudaSuccess;
  if (max_cols <= 1) return matvec_parts_w<1, 0>(d_descs, ndescs, max_nlines, max_across_len, d_xls, stream);
  if (max_cols <= 2) return matvec_parts_w<2, 1>(d_descs, ndescs, max_nlines, max_across_len, d_xls, stream);
  if (max_cols <= 4) return matvec_parts_w<4, 2>(d_descs, ndescs, max_nlines, max_across_len, d_xls, stream);
  if (max_cols <= kMvMaxCols) return matvec_parts_w<8, 3>(d_descs, ndescs, max_nlines, max_across_len, d_xls, stream);
  return cudaErrorInvalidValue;
}

}  // namespace matrel
