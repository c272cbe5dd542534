// Element-wise joins with a sparse side (LocalMatrix.add / elementWiseMultiply / elementWiseDivide, LocalMatrix.scala:34-139,
// 464-602) on the stored entries of the sparse blocks, without dense images of them (DESIGN section 4.5.3).
//
// The reference's loops, which these kernels reproduce bit for bit (NaN payloads aside).  op is one IEEE operation rounded to
// nearest (__dadd_rn / __dmul_rn / __ddiv_rn, so that nothing is contracted):
//   1. sparse (+) sparse, both CSC (addSparseSparseNative :98-139, elementWiseOpSparseSparseNative :548-602).  An operand's value at
//      (r, j) is 0.0 + v1 + v2 + ... over its stored entries at (r, j) in storage order: repeats are summed and a stored -0.0 becomes
//      +0.0.  add keeps ONE running sum per row, A's entries then B's (coltmp(r) += ...); multiply / divide take op(a, b).  The
//      result is op over the union of stored positions, op(0, 0) elsewhere (0 for add and multiply, NaN for divide).
//   2. sparse (+) sparse, either CSR (the toArray branch, :74-91, :521-541).  An operand's value is its LAST stored entry at the
//      position (foreachActive overwrites, MLMatrix.scala:637-663), sign kept.  A CSR operand arrives here through launch_sptrans,
//      which puts repeated entries of a position in reverse storage order, so there the FIRST of them counts.
//   In both cases an entry is kept iff it is != 0.0 (NaN kept, -0.0 dropped), rows ascending.  The host applies the output rule
//   (CSC iff rows * cols > 2 nnz + cols + 1, else dense) from the per-pair totals of the count pass.  A dense outcome of case 1 is
//   the toDense of that CSC (a -0.0 result is +0.0); of case 2 it is the array itself (-0.0 kept).
//   3. dense (+) sparse, either order (addDenseSparse, elementWiseOpDenseSparse, :65-72, :507-519): always dense, column-major.
//      op(d, 0) at unstored positions is written by the batched ew kernels with an absent operand; sparse_ew_scatter_kernel then
//      writes op(d, s) (or op(s, d)) at the stored positions, s the last stored value.
//
// sparse_ew_kernel: one warp per 32 consecutive output columns of a pair, the columns one after another, in a CSC frame, on a
// persistent grid over (pair, 32-column group) work items, so any number of pairs is one launch.  Each warp owns a column
// accumulator (as spgemm_chain_kernel's): the two operand values sa[M], sb[M] and a bitmap of the rows the column's union touched,
// in shared memory, or in global scratch for tall blocks.  A line whose indices strictly ascend is spread over the lanes; any other
// line (unsorted, or with repeats) is walked in storage order by one lane, so the result never depends on scheduling.  The kept
// entries come out of the bitmap in ascending row order.  COUNT writes per-column counts and adds each pair's total; FILL writes
// the CSC entries at the scanned column pointers, or every element of a dense window.
#include "kernels.h"

namespace matrel {

namespace {

constexpr int kSpEwWarps = 4;  // warps per CTA

template <int OP>
__device__ __forceinline__ double spew_op(double a, double b) {
  if (OP == EW_ADD) return __dadd_rn(a, b);
  if (OP == EW_MUL) return __dmul_rn(a, b);
  return __ddiv_rn(a, b);
}

__device__ __forceinline__ size_t spew_words(int M) { return static_cast<size_t>((M + 31) / 32); }
__host__ __device__ __forceinline__ size_t spew_acc_bytes(int M) {
  return (static_cast<size_t>(M) * 2 * sizeof(double) + static_cast<size_t>((M + 31) / 32) * sizeof(uint32_t) + 15) / 16 * 16;
}

// true when idx[s0 .. s1) strictly ascends (warp-uniform)
__device__ __forceinline__ bool strictly_ascending(const int32_t* __restrict__ idx, int s0, int s1, int lane) {
  bool ok = true;
  for (int e = s0 + lane; e + 1 < s1; e += 32) ok = ok && idx[e] < idx[e + 1];
  return __all_sync(0xffffffffu, ok);
}

// One operand's entries of a column into the accumulator: tgt[r] = 0.0 + v1 + ... (SPEW_SUM), the last stored v (SPEW_LAST) or
// the first stored v of an ascending line whose repeats are adjacent (SPEW_FIRST).  A row the column's union had not touched yet
// starts with sa = sb = 0.0.
__device__ __forceinline__ void spew_scatter(const int32_t* __restrict__ idx, const double* __restrict__ val, int s0, int s1, int mode,
                                             double* sa, double* sb, double* tgt, uint32_t* bits, int lane) {
  if (s0 == s1) return;
  auto put = [&](int r, double x) {
    const uint32_t bit = 1u << (r & 31);
    const uint32_t old = atomicOr(bits + (r >> 5), bit);
    if (!(old & bit)) {
      sa[r] = 0.0;
      sb[r] = 0.0;
    }
    tgt[r] = mode == SPEW_SUM ? __dadd_rn(tgt[r], x) : x;
  };
  if (mode == SPEW_FIRST || strictly_ascending(idx, s0, s1, lane)) {
    for (int e = s0 + lane; e < s1; e += 32) {
      const int r = idx[e];
      if (mode == SPEW_FIRST && e > s0 && idx[e - 1] == r) continue;
      put(r, val[e]);
    }
  } else if (lane == 0) {
    for (int e = s0; e < s1; ++e) put(idx[e], val[e]);
  }
  __syncwarp();
}

template <int OP, bool FILL>
__global__ void __launch_bounds__(kSpEwWarps * 32, 1) sparse_ew_kernel(const SpEwPair* __restrict__ pairs, int64_t nitems, int groups_per_pair,
                                                                   char* scratch, int M) {
  extern __shared__ __align__(16) char spew_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t acc_bytes = spew_acc_bytes(M);
  char* base = scratch ? scratch + (static_cast<size_t>(blockIdx.x) * kSpEwWarps + warp) * acc_bytes : spew_smem + warp * acc_bytes;
  double* sa = reinterpret_cast<double*>(base);
  double* sb = sa + M;
  uint32_t* bits = reinterpret_cast<uint32_t*>(sb + M);
  const int W = static_cast<int>(spew_words(M));
  for (int w = lane; w < W; w += 32) bits[w] = 0u;
  __syncwarp();
  const double bg = spew_op<OP>(0.0, 0.0);  // op(0, 0): 0, or NaN for divide
  const bool bg_kept = bg != 0.0;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kSpEwWarps;
  for (int64_t it = static_cast<int64_t>(blockIdx.x) * kSpEwWarps + warp; it < nitems; it += stride) {
    const SpEwPair& p = pairs[it / groups_per_pair];
    const int c0 = static_cast<int>(it % groups_per_pair) * 32;
    if (c0 >= p.cols) continue;
    const int rows = p.rows, words = (rows + 31) >> 5;
    double* tb = (OP == EW_ADD && p.native) ? sa : sb;  // case-1 add: one running sum, A's entries then B's
    int a0 = 0, a1 = 0, b0 = 0, b1 = 0;  // the column ranges of the group, one column per lane
    if (c0 + lane < p.cols) {
      a0 = p.ap[c0 + lane];
      a1 = p.ap[c0 + lane + 1];
      b0 = p.bp[c0 + lane];
      b1 = p.bp[c0 + lane + 1];
    }
    unsigned long long group_total = 0;
    const int ncol = min(32, p.cols - c0);
    for (int t = 0; t < ncol; ++t) {
      const int j = c0 + t;
      const int qa0 = __shfl_sync(0xffffffffu, a0, t), qa1 = __shfl_sync(0xffffffffu, a1, t);
      const int qb0 = __shfl_sync(0xffffffffu, b0, t), qb1 = __shfl_sync(0xffffffffu, b1, t);
      if (!bg_kept && qa0 == qa1 && qb0 == qb1) {  // nothing stored, nothing kept
        if (FILL && p.dense)
          for (int r = lane; r < rows; r += 32) p.dense[static_cast<int64_t>(j) * rows + r] = 0.0;
        else if (!FILL && lane == 0)
          p.colcnt[j] = 0;
        continue;
      }
      spew_scatter(p.ai, p.av, qa0, qa1, p.amode, sa, sb, sa, bits, lane);
      spew_scatter(p.bi, p.bv, qb0, qb1, p.bmode, sa, sb, tb, bits, lane);
      if (FILL && p.dense) {
        double* col = p.dense + static_cast<int64_t>(j) * rows;
        for (int r = lane; r < rows; r += 32) {
          double v = bg;
          if ((bits[r >> 5] >> (r & 31)) & 1u) v = spew_op<OP>(sa[r], sb[r]);
          if (p.native && !(v != 0.0)) v = 0.0;  // toDense of the CSC: unstored is +0.0
          col[r] = v;
        }
        __syncwarp();
        for (int w = lane; w < words; w += 32) bits[w] = 0u;
        __syncwarp();
        continue;
      }
      int out = FILL ? p.optr[j] : 0;
      for (int w0 = 0; w0 < words; w0 += 32) {
        const int w = w0 + lane;
        uint32_t word = 0, valid = 0;
        if (w < words) {
          word = bits[w];
          valid = (w == words - 1 && (rows & 31)) ? (1u << (rows & 31)) - 1u : 0xffffffffu;
        }
        // kept rows of this lane's word, ascending
        uint32_t kept = 0;
        for (uint32_t m = word; m; m &= m - 1) {
          const int b = __ffs(m) - 1;
          const int r = w * 32 + b;
          if (spew_op<OP>(sa[r], sb[r]) != 0.0) kept |= 1u << b;
        }
        if (bg_kept) kept |= ~word & valid;
        const int n = __popc(kept);
        int incl = n;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += y;
        }
        if (FILL) {
          int pos = out + incl - n;
          for (uint32_t m = kept; m; m &= m - 1) {
            const int b = __ffs(m) - 1;
            const int r = w * 32 + b;
            p.oidx[pos] = r;
            p.oval[pos] = ((word >> b) & 1u) ? spew_op<OP>(sa[r], sb[r]) : bg;
            ++pos;
          }
        }
        out += __shfl_sync(0xffffffffu, incl, 31);
        if (w < words) bits[w] = 0u;
      }
      __syncwarp();
      if (!FILL) {
        if (lane == 0) p.colcnt[j] = out;
        group_total += static_cast<unsigned long long>(out);
      }
    }
    if (!FILL && lane == 0 && group_total) atomicAdd(p.total, group_total);
  }
}

// One warp per stored line of a sparse block: C(r, c) = op(d, s) (op(s, d) when the sparse block is the left operand) at its
// stored positions, s the last stored value of the position.  A line whose indices strictly ascend is spread over the lanes;
// any other line is written by one lane in storage order, so the last write of a repeated position is its last stored entry.
template <int OP>
__global__ void __launch_bounds__(256) sparse_ew_scatter_kernel(const DsEwDesc* __restrict__ descs) {
  const DsEwDesc d = descs[blockIdx.y];
  const int line = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (line >= (d.sT ? d.rows : d.cols)) return;
  const int s0 = d.ptr[line], s1 = d.ptr[line + 1];
  if (s0 == s1) return;
  auto put = [&](int e) {
    const int minor = d.idx[e];
    const int r = d.sT ? line : minor, c = d.sT ? minor : line;
    const double x = d.D[d.dT ? static_cast<int64_t>(r) * d.cols + c : static_cast<int64_t>(c) * d.rows + r];
    const double s = d.val[e];
    d.C[static_cast<int64_t>(c) * d.rows + r] = d.sparse_left ? spew_op<OP>(s, x) : spew_op<OP>(x, s);
  };
  if (strictly_ascending(d.idx, s0, s1, lane)) {
    for (int e = s0 + lane; e < s1; e += 32) put(e);
  } else if (lane == 0) {
    for (int e = s0; e < s1; ++e) put(e);
  }
}

template <int OP>
cudaError_t set_smem_attrs() {
  cudaError_t r = cudaFuncSetAttribute(sparse_ew_kernel<OP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSpEwMaxSmem);
  if (r != cudaSuccess) return r;
  return cudaFuncSetAttribute(sparse_ew_kernel<OP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSpEwMaxSmem);
}

PerDeviceOnce g_spew_attr;

}  // namespace

SpEwLaunchShape sparse_ew_shape(int max_rows) {
  SpEwLaunchShape s{};
  const size_t smem = kSpEwWarps * spew_acc_bytes(max_rows);
  s.acc_in_smem = smem <= static_cast<size_t>(kSpEwMaxSmem);
  s.smem_bytes = s.acc_in_smem ? smem : 0;
  int dev = 0, sms = 132, smem_sm = 228 * 1024;
  if (cudaGetDevice(&dev) == cudaSuccess) {
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
  }
  // CTAs per SM: as many as the accumulators let fit (1 KB of shared memory per CTA is reserved by the driver), at most 8
  int per_sm = s.acc_in_smem ? static_cast<int>(smem_sm / (s.smem_bytes + 1024)) : 4;
  per_sm = per_sm < 1 ? 1 : per_sm > 8 ? 8 : per_sm;
  s.max_ctas = sms * per_sm;
  s.scratch_bytes = s.acc_in_smem ? 0 : static_cast<size_t>(s.max_ctas) * kSpEwWarps * spew_acc_bytes(max_rows);
  return s;
}

cudaError_t launch_sparse_ew(int op, bool fill, const SpEwPair* d_pairs, int npairs, int max_rows, int max_cols, void* d_scratch,
                             const SpEwLaunchShape& s, cudaStream_t stream) {
  if (npairs <= 0 || max_cols <= 0) return cudaSuccess;
  cudaError_t e = g_spew_attr.run([] {
    cudaError_t r = set_smem_attrs<EW_ADD>();
    if (r == cudaSuccess) r = set_smem_attrs<EW_MUL>();
    if (r == cudaSuccess) r = set_smem_attrs<EW_DIV>();
    return r;
  });
  if (e != cudaSuccess) return e;
  const int groups = (max_cols + 31) / 32;
  const int64_t nitems = static_cast<int64_t>(npairs) * groups;
  const int64_t need = (nitems + kSpEwWarps - 1) / kSpEwWarps;
  const int ctas = static_cast<int>(need < s.max_ctas ? need : s.max_ctas);
  char* scratch = s.acc_in_smem ? nullptr : static_cast<char*>(d_scratch);
  const int M = max_rows > 0 ? max_rows : 1;
#define MR_SPEW_LAUNCH(OPV)                                                                                                   \
  if (fill)                                                                                                                   \
    sparse_ew_kernel<OPV, true><<<ctas, kSpEwWarps * 32, s.smem_bytes, stream>>>(d_pairs, nitems, groups, scratch, M);       \
  else                                                                                                                        \
    sparse_ew_kernel<OPV, false><<<ctas, kSpEwWarps * 32, s.smem_bytes, stream>>>(d_pairs, nitems, groups, scratch, M);
  switch (op) {
    case EW_ADD: MR_SPEW_LAUNCH(EW_ADD) break;
    case EW_MUL: MR_SPEW_LAUNCH(EW_MUL) break;
    case EW_DIV: MR_SPEW_LAUNCH(EW_DIV) break;
    default: return cudaErrorInvalidValue;
  }
#undef MR_SPEW_LAUNCH
  return cudaGetLastError();
}

cudaError_t launch_sparse_ew_scatter(int op, const DsEwDesc* d_descs, int ndescs, int max_lines, cudaStream_t stream) {
  if (ndescs <= 0 || max_lines <= 0) return cudaSuccess;
  for (int off = 0; off < ndescs; off += 65535) {  // gridDim.y limit
    const dim3 grid((max_lines + 7) / 8, ndescs - off < 65535 ? ndescs - off : 65535);
    switch (op) {
      case EW_ADD: sparse_ew_scatter_kernel<EW_ADD><<<grid, 256, 0, stream>>>(d_descs + off); break;
      case EW_MUL: sparse_ew_scatter_kernel<EW_MUL><<<grid, 256, 0, stream>>>(d_descs + off); break;
      case EW_DIV: sparse_ew_scatter_kernel<EW_DIV><<<grid, 256, 0, stream>>>(d_descs + off); break;
      default: return cudaErrorInvalidValue;
    }
  }
  return cudaGetLastError();
}

}  // namespace matrel
