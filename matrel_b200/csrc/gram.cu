// The mirror pass of Gram products C = A^T A and C = A A^T (DESIGN section 4.1.2).  The dense engines compute the output blocks on
// and above the block diagonal; this kernel writes every strictly-lower element from its transpose, for all blocks in ONE launch.
//
// One CTA of 32 x 8 threads moves 32 x 32 tiles of dst: it reads the matching tile of src with the lanes along src's columns (its
// contiguous dimension), transposes it through a padded shared tile, and writes dst with the lanes along dst's columns, so both
// sides are coalesced.  Tiles are addressed within an item as (tile row, tile column), grid-strided by blockIdx.x; items by
// blockIdx.y.  A diagonal item skips the tiles wholly above its diagonal and, in the tiles it crosses, reads only the elements
// strictly above it and writes only those strictly below it: the engines may not have stored anything below.
//
// gram_sym_kernel: the sparse counterpart for a diagonal block of a sparse Gram product, whose chain produced its upper triangle U
// only (spgemm.cu, triangular chains).  One warp per column c of the full block: U(:, c) (rows <= c), then U^T(:, c) past its
// diagonal entry (rows > c).  Both segments ascend, so the column does too.
#include "kernels.h"

namespace matrel {

namespace {

constexpr int kMirTile = 32, kMirRows = 8;

__global__ void __launch_bounds__(kMirTile * kMirRows) gram_mirror_kernel(const GramMirror* __restrict__ items, int nitems) {
  __shared__ double sh[kMirTile][kMirTile + 1];
  const int x = threadIdx.x, y0 = threadIdx.y;
  for (int d = blockIdx.y; d < nitems; d += gridDim.y) {
    const GramMirror g = items[d];
    const int tiles_r = (g.m + kMirTile - 1) / kMirTile, tiles_c = (g.n + kMirTile - 1) / kMirTile;
    const int64_t ntiles = static_cast<int64_t>(tiles_r) * tiles_c;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const int tr = static_cast<int>(t % tiles_r), tc = static_cast<int>(t / tiles_r);
      if (g.diag && tr < tc) continue;  // uniform over the CTA
      const int r0 = tr * kMirTile, c0 = tc * kMirTile;
      // sh[y][x] = src(c0 + x, r0 + y) = dst(r0 + y, c0 + x)
      for (int y = y0; y < kMirTile; y += kMirRows) {
        const int p = r0 + y, q = c0 + x;
        if (p < g.m && q < g.n && (!g.diag || q < p)) sh[y][x] = g.src[q + static_cast<size_t>(g.n) * p];
      }
      __syncthreads();
      for (int y = y0; y < kMirTile; y += kMirRows) {
        const int p = r0 + x, q = c0 + y;
        if (p < g.m && q < g.n && (!g.diag || q < p)) g.dst[p + static_cast<size_t>(g.m) * q] = sh[x][y];
      }
      __syncthreads();
    }
  }
}

// diagonal entry of column c present in U (its last entry, rows ascending)
__device__ __forceinline__ int gram_sym_diag(const GramSym& g, int c) {
  const int e = g.up[c + 1];
  return e > g.up[c] && g.ui[e - 1] == c ? 1 : 0;
}

constexpr int kSymWarps = 8;

template <bool FILL>
__global__ void __launch_bounds__(kSymWarps * 32) gram_sym_kernel(const GramSym* __restrict__ items) {
  const GramSym g = items[blockIdx.y];
  const int lane = threadIdx.x & 31;
  for (int c = blockIdx.x * kSymWarps + (threadIdx.x >> 5); c < g.n; c += gridDim.x * kSymWarps) {
    const int u0 = g.up[c], u1 = g.up[c + 1];
    const int t0 = g.tp[c] + gram_sym_diag(g, c), t1 = g.tp[c + 1];
    if (!FILL) {
      if (lane == 0) g.cnt[c] = (u1 - u0) + (t1 - t0);
      continue;
    }
    const int o = g.optr[c];
    for (int e = u0 + lane; e < u1; e += 32) {
      g.oidx[o + e - u0] = g.ui[e];
      g.oval[o + e - u0] = g.uv[e];
    }
    const int o2 = o + (u1 - u0);
    for (int e = t0 + lane; e < t1; e += 32) {
      g.oidx[o2 + e - t0] = g.ti[e];
      g.oval[o2 + e - t0] = g.tv[e];
    }
  }
}

}  // namespace

cudaError_t launch_gram_sym(bool fill, const GramSym* d_items, int nitems, int max_n, cudaStream_t stream) {
  if (nitems <= 0 || max_n <= 0) return cudaSuccess;
  const int bx = std::min((max_n + kSymWarps - 1) / kSymWarps, 1024);
  for (int off = 0; off < nitems; off += 65535) {
    const dim3 grid(bx, std::min(nitems - off, 65535));
    if (fill) gram_sym_kernel<true><<<grid, kSymWarps * 32, 0, stream>>>(d_items + off);
    else gram_sym_kernel<false><<<grid, kSymWarps * 32, 0, stream>>>(d_items + off);
  }
  return cudaGetLastError();
}

cudaError_t launch_gram_mirror(const GramMirror* d_items, int nitems, int max_m, int max_n, cudaStream_t stream) {
  if (nitems <= 0 || max_m <= 0 || max_n <= 0) return cudaSuccess;
  const int64_t tiles = static_cast<int64_t>((max_m + kMirTile - 1) / kMirTile) * ((max_n + kMirTile - 1) / kMirTile);
  const dim3 grid(static_cast<unsigned>(std::min<int64_t>(tiles, 4096)), static_cast<unsigned>(std::min(nitems, 65535)));
  gram_mirror_kernel<<<grid, dim3(kMirTile, kMirRows), 0, stream>>>(d_items, nitems);
  return cudaGetLastError();
}

}  // namespace matrel
