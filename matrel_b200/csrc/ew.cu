// HBM-bound sibling kernels of the block-multiply path, batched over the blocks of a dataset
// (one launch per operator call, not per block):
//   element-wise add / mul / div     LocalMatrix.addDense, elementWiseOpDenseDense (LocalMatrix.scala:56-63,493-505)
//   materialising transpose / copy   DenseMatrix.toArray (MLMatrix.scala:55-61) for isTransposed blocks
//   scalar add / mul / pow           LocalMatrix.scala:411-426, 931-980 (layout preserving maps)
//   rank-one update                  LocalMatrix.rankOneAdd (LocalMatrix.scala:1075-1093)
//   sparse -> dense                  SparseMatrix.toArray (MLMatrix.scala:637-663)
//   sparse x dense                   BLAS.gemmsdd (BLAS.scala:352-458)
//   java.util.Random U(0,1) fill     DenseMatrix.rand (MLMatrix.scala:453-457)
//   cross-GPU partial sum            reduceByKey(LocalMatrix.add) of matrixMultiplyGeneral (MatfastExecutionHelper.scala:255)
// Flat paths use 128-bit ld/st.global.v2.f64 with 4 independent vectors in flight per thread;
// layout-mixing paths stage a 32x32 tile through padded shared memory so both the row-major
// read and the column-major write are fully coalesced.
#include "kernels.h"

namespace matrel {
namespace {

template <int OP>
__device__ __forceinline__ double ew_apply(double a, double b) {
  if (OP == EW_ADD) return a + b;
  if (OP == EW_MUL) return a * b;
  if (OP == EW_DIV) return a / b;
  return a;  // EW_COPY
}

__device__ __forceinline__ double2 ld_stream(const double2* p) {
  double2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream(double2* p, double2 v) {
  asm volatile("st.global.L1::no_allocate.v2.f64 [%0], {%1,%2};" ::"l"(p), "d"(v.x), "d"(v.y) : "memory");
}

constexpr int FLAT_THREADS = 256;
constexpr int FLAT_UNROLL = 4;

// Both operands share C's layout: pure streaming.  A null A or B (EW_ADD/MUL/DIV) is an absent operand: 0.0.
template <int OP>
__global__ void __launch_bounds__(FLAT_THREADS) ew_flat_kernel(const EwDesc* __restrict__ descs) {
  const EwDesc d = descs[blockIdx.y];
  const int64_t n = static_cast<int64_t>(d.rows) * d.cols;
  const bool has_a = d.A != nullptr;
  const bool has_b = (OP != EW_COPY) && d.B != nullptr;
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(d.A) | reinterpret_cast<uintptr_t>(d.C) |
                        (has_b ? reinterpret_cast<uintptr_t>(d.B) : 0)) & 15) == 0;
  const int64_t nvec = vec_ok ? (n >> 1) : 0;
  const double2* A2 = reinterpret_cast<const double2*>(d.A);
  const double2* B2 = reinterpret_cast<const double2*>(d.B);
  double2* C2 = reinterpret_cast<double2*>(d.C);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * FLAT_THREADS;
  int64_t i = static_cast<int64_t>(blockIdx.x) * FLAT_THREADS + threadIdx.x;
  for (; i + (FLAT_UNROLL - 1) * stride < nvec; i += FLAT_UNROLL * stride) {
    double2 a[FLAT_UNROLL], b[FLAT_UNROLL];
#pragma unroll
    for (int u = 0; u < FLAT_UNROLL; ++u) a[u] = has_a ? ld_stream(A2 + i + u * stride) : make_double2(0.0, 0.0);
#pragma unroll
    for (int u = 0; u < FLAT_UNROLL; ++u) b[u] = has_b ? ld_stream(B2 + i + u * stride) : make_double2(0.0, 0.0);
#pragma unroll
    for (int u = 0; u < FLAT_UNROLL; ++u) {
      double2 c;
      c.x = ew_apply<OP>(a[u].x, b[u].x);
      c.y = ew_apply<OP>(a[u].y, b[u].y);
      st_stream(C2 + i + u * stride, c);
    }
  }
  for (; i < nvec; i += stride) {
    const double2 a = has_a ? ld_stream(A2 + i) : make_double2(0.0, 0.0);
    const double2 b = has_b ? ld_stream(B2 + i) : make_double2(0.0, 0.0);
    double2 c;
    c.x = ew_apply<OP>(a.x, b.x);
    c.y = ew_apply<OP>(a.y, b.y);
    st_stream(C2 + i, c);
  }
  // scalar tail (odd n, or unaligned borrowed pointers)
  for (int64_t j = 2 * nvec + static_cast<int64_t>(blockIdx.x) * FLAT_THREADS + threadIdx.x; j < n; j += stride)
    d.C[j] = ew_apply<OP>(has_a ? d.A[j] : 0.0, has_b ? d.B[j] : 0.0);
}

// Layout-mixing path: 32x32 tile, 32x8 threads; output (r = r0 + tx, c = c0 + ty + 8j).
__device__ __forceinline__ void load_tile(const double* __restrict__ X, bool xT, int rows, int cols, int r0, int c0,
                                          double (&sm)[32][33], double (&v)[4]) {
  const int tx = threadIdx.x, ty = threadIdx.y;
  if (!xT) {
    const int r = r0 + tx;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + ty + 8 * j;
      v[j] = (r < rows && c < cols) ? X[r + static_cast<size_t>(rows) * c] : 0.0;
    }
  } else {
    __syncthreads();  // protect sm against the previous operand's readers
    const int c = c0 + tx;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = r0 + ty + 8 * j;
      sm[ty + 8 * j][tx] = (r < rows && c < cols) ? X[c + static_cast<size_t>(cols) * r] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = sm[tx][ty + 8 * j];
  }
}

template <int OP>
__global__ void __launch_bounds__(256) ew_tiled_kernel(const EwDesc* __restrict__ descs, int tiles_c_max) {
  __shared__ double sm[32][33];
  const EwDesc d = descs[blockIdx.y];
  const int tr = blockIdx.x / tiles_c_max, tc = blockIdx.x % tiles_c_max;
  const int r0 = tr * 32, c0 = tc * 32;
  if (r0 >= d.rows || c0 >= d.cols) return;
  const int tx = threadIdx.x, ty = threadIdx.y;
  double a[4] = {0, 0, 0, 0}, b[4] = {0, 0, 0, 0};
  if (OP == EW_RANK1_COMPAT) {
    // flat C[k] = x_r * y_c with k = A's storage index; A itself is never read (defect B3).
    // aT: C_flat is row-major -> treat as the column-major (cols x rows) matrix y x^T.
    const double* x = d.B;
    const double* y = d.Y;
    if (!d.aT) {
      const int r = r0 + tx;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = c0 + ty + 8 * j;
        if (r < d.rows && c < d.cols) d.C[r + static_cast<size_t>(d.rows) * c] = x[r] * y[c];
      }
    } else {
      // iterate the same tile with roles swapped so writes stay coalesced along c
      const int c = c0 + tx;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int r = r0 + ty + 8 * j;
        if (r < d.rows && c < d.cols) d.C[c + static_cast<size_t>(d.cols) * r] = x[r] * y[c];
      }
    }
    return;
  }
  if (d.A != nullptr) load_tile(d.A, d.aT != 0, d.rows, d.cols, r0, c0, sm, a);
  if ((OP == EW_ADD || OP == EW_MUL || OP == EW_DIV) && d.B != nullptr) load_tile(d.B, d.bT != 0, d.rows, d.cols, r0, c0, sm, b);
  const int r = r0 + tx;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = c0 + ty + 8 * j;
    if (r < d.rows && c < d.cols) {
      double out;
      // a + (x y) with both operations rounded, as LocalMatrix.rankOneAdd: a contracted FMA would round once
      if (OP == EW_RANK1) out = __dadd_rn(a[j], __dmul_rn(d.B[r], d.Y[c]));
      else out = ew_apply<OP>(a[j], b[j]);
      d.C[r + static_cast<size_t>(d.rows) * c] = out;
    }
  }
}

template <int OP>
__device__ __forceinline__ double map_apply(double v, double alpha) {
  if (OP == MAP_ADD_SCALAR) return v + alpha;
  if (OP == MAP_MUL_SCALAR) return alpha * v;
  // math.pow (LocalMatrix.scala:931-946).  The common exponents take exact closed forms (the correctly rounded value
  // of x^2 is x*x, of x^0.5 is sqrt(x)) instead of the ~100-instruction general pow.
  if (alpha == 2.0) return v * v;
  if (alpha == 1.0) return v;
  if (alpha == 0.5) {
    if (v == 0.0) return 0.0;                       // pow(-0.0, 0.5) = +0.0
    if (isinf(v) && v < 0.0) return -v;             // pow(-inf, 0.5) = +inf
    return sqrt(v);
  }
  // java.lang.Math.pow, unlike C's pow, gives NaN for pow(+-1, +-inf) and pow(1, NaN)
  if (!isfinite(alpha) && fabs(v) == 1.0) return __longlong_as_double(0x7ff8000000000000LL);
  return pow(v, alpha);
}

template <int OP>
__global__ void __launch_bounds__(FLAT_THREADS) map_kernel(const MapDesc* __restrict__ descs, double alpha) {
  const MapDesc d = descs[blockIdx.y];
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(d.in) | reinterpret_cast<uintptr_t>(d.out)) & 15) == 0;
  const int64_t nvec = vec_ok ? (d.n >> 1) : 0;
  const double2* I2 = reinterpret_cast<const double2*>(d.in);
  double2* O2 = reinterpret_cast<double2*>(d.out);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * FLAT_THREADS;
  int64_t i = static_cast<int64_t>(blockIdx.x) * FLAT_THREADS + threadIdx.x;
  for (; i + (FLAT_UNROLL - 1) * stride < nvec; i += FLAT_UNROLL * stride) {
    double2 a[FLAT_UNROLL];
#pragma unroll
    for (int u = 0; u < FLAT_UNROLL; ++u) a[u] = ld_stream(I2 + i + u * stride);
#pragma unroll
    for (int u = 0; u < FLAT_UNROLL; ++u) {
      double2 c;
      c.x = map_apply<OP>(a[u].x, alpha);
      c.y = map_apply<OP>(a[u].y, alpha);
      st_stream(O2 + i + u * stride, c);
    }
  }
  for (; i < nvec; i += stride) {
    const double2 a = ld_stream(I2 + i);
    double2 c;
    c.x = map_apply<OP>(a.x, alpha);
    c.y = map_apply<OP>(a.y, alpha);
    st_stream(O2 + i, c);
  }
  for (int64_t j = 2 * nvec + static_cast<int64_t>(blockIdx.x) * FLAT_THREADS + threadIdx.x; j < d.n; j += stride)
    d.out[j] = map_apply<OP>(d.in[j], alpha);
}

// one warp per compressed line (column of CSC / row of CSR)
__global__ void sparse_to_dense_kernel(const int32_t* __restrict__ ptrs, const int32_t* __restrict__ idx,
                                       const double* __restrict__ vals, bool isT, double* __restrict__ out, int rows,
                                       int cols) {
  const int nlines = isT ? rows : cols;
  const int line = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (line >= nlines) return;
  const int beg = ptrs[line], end = ptrs[line + 1];
  for (int i = beg + lane; i < end; i += 32) {
    const int minor = idx[i];
    const size_t o = isT ? (static_cast<size_t>(line) + static_cast<size_t>(rows) * minor)
                         : (static_cast<size_t>(minor) + static_cast<size_t>(rows) * line);
    out[o] = vals[i];
  }
}

__device__ __forceinline__ double dense_at(const double* __restrict__ B, bool bT, int k, int n, int r, int c) {
  return bT ? B[c + static_cast<size_t>(n) * r] : B[r + static_cast<size_t>(k) * c];
}

// CSR x dense: thread per (row, column); rows fastest so C writes coalesce and the 32 lanes of a
// warp gather from one 8*k-byte column of B (L1/L2 resident).  BLAS.scala:375-413.
__global__ void __launch_bounds__(256) spmm_csr_kernel(const int32_t* __restrict__ ptrs, const int32_t* __restrict__ idx,
                                                       const double* __restrict__ vals, const double* __restrict__ B,
                                                       bool bT, double* __restrict__ C, int m, int k, int n,
                                                       bool accumulate) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (r >= m) return;
  const int beg = ptrs[r], end = ptrs[r + 1];
  double sum = 0.0;
  for (int i = beg; i < end; ++i) sum += vals[i] * dense_at(B, bT, k, n, idx[i], c);
  const size_t o = static_cast<size_t>(r) + static_cast<size_t>(m) * c;
  C[o] = accumulate ? C[o] + sum : sum;
}

// Fused CSR SpMM (see kernels.h): grid = (ceil(n_max / 8), output blocks), 512 threads.
// Thread = one (or two) row(s) of the output block x 8 columns held in registers across ALL block pairs; the B chunk
// (8 columns x kdim) is staged in shared memory per pair, so each CSR entry costs one index/value load and feeds 8 FMAs.
constexpr int SPMM_CW = 8;
constexpr int SPMM_THREADS = 512;
constexpr int SPMM_RPT = kSpmmMaxDim / SPMM_THREADS;  // rows per thread (2)
__global__ void __launch_bounds__(SPMM_THREADS) spmm_fused_kernel(const SpmmOut* __restrict__ outs, const SpmmPair* __restrict__ pairs) {
  extern __shared__ double spmm_smem[];
  const SpmmOut o = outs[blockIdx.y];
  const int c0 = blockIdx.x * SPMM_CW;
  if (c0 >= o.n) return;
  const int cw = min(SPMM_CW, o.n - c0);
  double* sB = spmm_smem;  // [SPMM_CW][kdim + 2]
  const int tid = threadIdx.x;
  double acc[SPMM_RPT][SPMM_CW];
#pragma unroll
  for (int u = 0; u < SPMM_RPT; ++u) {
    const int r = tid + u * SPMM_THREADS;
#pragma unroll
    for (int c = 0; c < SPMM_CW; ++c)
      acc[u][c] = (o.accumulate && r < o.m && c < cw) ? o.C[r + static_cast<size_t>(o.m) * (c0 + c)] : 0.0;
  }
  for (int p = 0; p < o.pair_count; ++p) {
    const SpmmPair pr = pairs[o.pair_begin + p];
    const int ldb = pr.kdim + 2;
    __syncthreads();  // previous pair's readers of sB are done
    if (!pr.bT) {
      for (int cc = 0; cc < SPMM_CW; ++cc) {
        const double* src = pr.B + static_cast<size_t>(pr.kdim) * (c0 + cc);
        for (int k = tid; k < pr.kdim; k += SPMM_THREADS) sB[cc * ldb + k] = cc < cw ? src[k] : 0.0;
      }
    } else {
      for (int idx = tid; idx < SPMM_CW * pr.kdim; idx += SPMM_THREADS) {
        const int k = idx / SPMM_CW, cc = idx % SPMM_CW;
        sB[cc * ldb + k] = cc < cw ? pr.B[c0 + cc + static_cast<size_t>(o.n) * k] : 0.0;
      }
    }
    __syncthreads();
    int beg[SPMM_RPT], len[SPMM_RPT], maxlen = 0;
#pragma unroll
    for (int u = 0; u < SPMM_RPT; ++u) {
      const int r = tid + u * SPMM_THREADS;
      beg[u] = r < o.m ? pr.ptrs[r] : 0;
      len[u] = r < o.m ? pr.ptrs[r + 1] - beg[u] : 0;
      maxlen = max(maxlen, len[u]);
    }
    for (int i = 0; i < maxlen; ++i) {  // ascending nonzero order within a row = the reference's summation order
#pragma unroll
      for (int u = 0; u < SPMM_RPT; ++u) {
        if (i < len[u]) {
          const double v = pr.vals[beg[u] + i];
          const double* b = sB + pr.idx[beg[u] + i];
#pragma unroll
          for (int c = 0; c < SPMM_CW; ++c) acc[u][c] += v * b[c * ldb];
        }
      }
    }
  }
#pragma unroll
  for (int u = 0; u < SPMM_RPT; ++u) {
    const int r = tid + u * SPMM_THREADS;
    if (r < o.m) {
#pragma unroll
      for (int c = 0; c < SPMM_CW; ++c)
        if (c < cw) o.C[r + static_cast<size_t>(o.m) * (c0 + c)] = acc[u][c];
    }
  }
}

// CSC x dense: scatter-AXPY (BLAS.scala:414-456).  Warp per (CSC column, output column); C must be
// initialised (zeros or the running sum) before launch.
__global__ void __launch_bounds__(256) spmm_csc_kernel(const int32_t* __restrict__ ptrs, const int32_t* __restrict__ idx,
                                                       const double* __restrict__ vals, const double* __restrict__ B,
                                                       bool bT, double* __restrict__ C, int m, int k, int n) {
  const int col = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.y;
  if (col >= k) return;
  const int beg = ptrs[col], end = ptrs[col + 1];
  if (beg == end) return;
  const double bval = dense_at(B, bT, k, n, col, c);
  for (int i = beg + lane; i < end; i += 32)
    atomicAdd(&C[static_cast<size_t>(idx[i]) + static_cast<size_t>(m) * c], vals[i] * bval);
}

// java.util.Random: s' = (s * 0x5DEECE66D + 0xB) mod 2^48; nextDouble = ((next(26) << 27) + next(27)) * 2^-53.
// Thread i jumps straight to draw i with an O(log i) affine-map power, so the fill is parallel and
// still bit-identical to the JVM's sequential stream.  Batched: blockIdx.y selects the block/stream.
__global__ void __launch_bounds__(256) java_rand_kernel(const RandDesc* __restrict__ descs) {
  const uint64_t MASK = (1ull << 48) - 1;
  const RandDesc d = descs[blockIdx.y];
  const uint64_t seed0 = (static_cast<uint64_t>(d.seed) ^ 0x5DEECE66Dull) & MASK;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < d.n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    // affine map x -> a*x + c applied (2*i) times
    uint64_t a_acc = 1, c_acc = 0;
    uint64_t a = 0x5DEECE66Dull, c = 0xBull;
    for (uint64_t e = 2ull * static_cast<uint64_t>(i); e != 0; e >>= 1) {
      if (e & 1) {
        a_acc = (a_acc * a) & MASK;
        c_acc = (c_acc * a + c) & MASK;
      }
      c = (c * a + c) & MASK;  // compose the map with itself: x -> a*(a*x + c) + c
      a = (a * a) & MASK;
    }
    uint64_t s = (a_acc * seed0 + c_acc) & MASK;
    s = (s * 0x5DEECE66Dull + 0xBull) & MASK;
    const uint64_t hi = s >> 22;  // next(26)
    s = (s * 0x5DEECE66Dull + 0xBull) & MASK;
    const uint64_t lo = s >> 21;  // next(27)
    d.out[i] = static_cast<double>((hi << 27) + lo) * (1.0 / 9007199254740992.0);
  }
}

// Row / column sums.  tx always runs along the block's contiguous ("fast") dimension so global reads are coalesced for both
// layouts.  Two CTA shapes, chosen per block:
//   kept index = fast (rowSum of a column-major block): a CTA reduces a 32 (fast) x 256 (slow) tile, one partial per thread,
//     8 partials per fast index folded through shared memory, one atomic per fast index;
//   kept index = slow (colSum of a column-major block): a warp owns ONE slow index and sweeps up to 1024 fast elements in
//     registers (32 independent 256-byte warp loads) before a single shuffle reduction and one atomic -- the first version
//     reduced every 32-element row separately and was shuffle/atomic-bound at 3.4 TB/s.
constexpr int AGG_SLOW = 256;      // slow extent of a "kept fast" tile
constexpr int AGG_SWEEP = 1024;    // fast extent one warp sweeps in a "kept slow" tile (8 slow indices per CTA)
__global__ void __launch_bounds__(256) axis_sum_kernel(const AggDesc* __restrict__ descs, int by_row, int tiles_slow_a,
                                                       int tiles_slow_b) {
  __shared__ double sm[8][33];
  const AggDesc d = descs[blockIdx.y];
  const int nfast = d.isT ? d.cols : d.rows, nslow = d.isT ? d.rows : d.cols;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const bool kept_is_fast = (by_row != 0) == (d.isT == 0);  // row sums of a column-major block keep the fast index
  if (kept_is_fast) {
    const int tf = blockIdx.x / tiles_slow_a, ts = blockIdx.x % tiles_slow_a;
    const int f0 = tf * 32, s0 = ts * AGG_SLOW;
    if (f0 >= nfast || s0 >= nslow) return;
    const int f = f0 + tx;
    double acc = 0.0;
    if (f < nfast)
      for (int s = s0 + ty; s < min(nslow, s0 + AGG_SLOW); s += 8) acc += d.v[f + static_cast<size_t>(nfast) * s];
    sm[ty][tx] = acc;
    __syncthreads();
    if (ty == 0 && f < nfast) {
#pragma unroll
      for (int k = 1; k < 8; ++k) acc += sm[k][tx];
      atomicAdd(&d.out[f], acc);
    }
  } else {
    const int tf = blockIdx.x / tiles_slow_b, ts = blockIdx.x % tiles_slow_b;
    const int f0 = tf * AGG_SWEEP, s = ts * 8 + ty;
    if (f0 >= nfast || s >= nslow) return;
    const double* __restrict__ line = d.v + static_cast<size_t>(nfast) * s;
    const int f1 = min(nfast, f0 + AGG_SWEEP);
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    int f = f0 + tx;
    for (; f + 96 < f1; f += 128) {  // four independent loads in flight per lane
      a0 += line[f];
      a1 += line[f + 32];
      a2 += line[f + 64];
      a3 += line[f + 96];
    }
    for (; f < f1; f += 32) a0 += line[f];
    double v = (a0 + a1) + (a2 + a3);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (tx == 0) atomicAdd(&d.out[s], v);
  }
}

// AGG_SUM: sum of every stored value; AGG_TRACE: sum of the diagonal (square blocks; same index for both layouts)
__global__ void __launch_bounds__(256) scalar_sum_kernel(const AggDesc* __restrict__ descs, int trace) {
  __shared__ double sm[8];
  const AggDesc d = descs[blockIdx.y];
  const int64_t n = trace ? min(d.rows, d.cols) : static_cast<int64_t>(d.rows) * d.cols;
  const int64_t stride = trace ? static_cast<int64_t>(d.isT ? d.cols : d.rows) + 1 : 1;
  double acc = 0.0;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * 256)
    acc += d.v[i * stride];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sm[k];
    atomicAdd(d.out, t);
  }
}

__global__ void __launch_bounds__(256) extract_lines_kernel(const LineDesc* __restrict__ descs) {
  const LineDesc d = descs[blockIdx.y];
  for (int i = blockIdx.x * 256 + threadIdx.x; i < d.len; i += gridDim.x * 256) {
    const int j = d.offset2 >= 0 ? d.offset2 : i;
    const int r = d.take_row ? d.offset : j, c = d.take_row ? j : d.offset;
    d.out[i] = d.isT ? d.v[c + static_cast<size_t>(d.cols) * r] : d.v[r + static_cast<size_t>(d.rows) * c];
  }
}

__global__ void __launch_bounds__(256) copy_words_kernel(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, size_t nwords) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x; i < nwords; i += static_cast<size_t>(gridDim.x) * 256) dst[i] = src[i];
}

// ---- K-split multiply: out = sum of the partial products of the contributing GPUs, in part order (kernels.h, KsplitDesc).
// Most parts live on peer GPUs, so every load is an NVLink round trip: each thread issues the loads of a group of parts before
// it adds any of them, and the adds then run strictly left to right (part 0's value, + part 1, + part 2, ...), which keeps the
// result bit-reproducible.  128-bit loads and stores when every window shares the output's 16-byte phase (with an odd blk a
// slot starts on an 8-byte boundary: one scalar element first), scalar ones otherwise.
constexpr int KSPLIT_THREADS = 256;
constexpr int KSPLIT_GROUP = 8;

__global__ void __launch_bounds__(KSPLIT_THREADS) ksplit_reduce_kernel(const KsplitDesc* __restrict__ descs,
                                                                      const double* const* __restrict__ parts, int nparts) {
  __shared__ const double* src[kKsplitMaxParts];
  const KsplitDesc d = descs[blockIdx.y];
  for (int q = threadIdx.x; q < nparts; q += KSPLIT_THREADS) src[q] = parts[q] + d.offset;
  __syncthreads();
  const uintptr_t phase = reinterpret_cast<uintptr_t>(d.out) & 15;
  bool same = true;
  for (int q = 0; q < nparts; ++q) same = same && (reinterpret_cast<uintptr_t>(src[q]) & 15) == phase;
  const int64_t head = same ? (phase != 0 && d.count > 0 ? 1 : 0) : d.count;  // scalar elements in front of the 128-bit body
  const int64_t nvec = (d.count - head) >> 1;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * KSPLIT_THREADS;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * KSPLIT_THREADS + threadIdx.x;
  for (int64_t i = t; i < nvec; i += stride) {
    double2 acc = make_double2(0.0, 0.0);
    for (int q0 = 0; q0 < nparts; q0 += KSPLIT_GROUP) {
      double2 v[KSPLIT_GROUP];
#pragma unroll
      for (int u = 0; u < KSPLIT_GROUP; ++u)
        if (q0 + u < nparts) v[u] = ld_stream(reinterpret_cast<const double2*>(src[q0 + u] + head) + i);
#pragma unroll
      for (int u = 0; u < KSPLIT_GROUP; ++u)
        if (q0 + u < nparts) {
          if (q0 + u == 0) {
            acc = v[0];
          } else {
            acc.x += v[u].x;
            acc.y += v[u].y;
          }
        }
    }
    st_stream(reinterpret_cast<double2*>(d.out + head) + i, acc);
  }
  auto scalar = [&](int64_t e) {
    double acc = __ldcs(src[0] + e);
    for (int q = 1; q < nparts; ++q) acc += __ldcs(src[q] + e);
    __stcs(d.out + e, acc);
  };
  for (int64_t e = t; e < head; e += stride) scalar(e);
  for (int64_t e = head + 2 * nvec + t; e < d.count; e += stride) scalar(e);
}

inline int flat_grid_x(int64_t max_n) {
  int64_t vec = (max_n + 1) / 2;
  int64_t gx = (vec + static_cast<int64_t>(FLAT_THREADS) * FLAT_UNROLL - 1) / (static_cast<int64_t>(FLAT_THREADS) * FLAT_UNROLL);
  if (gx < 1) gx = 1;
  if (gx > 65535) gx = 65535;
  return static_cast<int>(gx);
}

}  // namespace

cudaError_t launch_ew_batched(int op, const EwDesc* d_descs, int nblocks, int max_rows, int max_cols,
                              bool any_transposed, cudaStream_t stream) {
  if (nblocks <= 0) return cudaSuccess;
  const bool tiled = any_transposed || op == EW_RANK1 || op == EW_RANK1_COMPAT;
  if (nblocks > 65535) {  // gridDim.y limit
    for (int off = 0; off < nblocks; off += 65535) {
      cudaError_t e = launch_ew_batched(op, d_descs + off, nblocks - off < 65535 ? nblocks - off : 65535, max_rows, max_cols,
                                        any_transposed, stream);
      if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
  }
  if (!tiled) {
    dim3 grid(flat_grid_x(static_cast<int64_t>(max_rows) * max_cols), nblocks);
    switch (op) {
      case EW_ADD: ew_flat_kernel<EW_ADD><<<grid, FLAT_THREADS, 0, stream>>>(d_descs); break;
      case EW_MUL: ew_flat_kernel<EW_MUL><<<grid, FLAT_THREADS, 0, stream>>>(d_descs); break;
      case EW_DIV: ew_flat_kernel<EW_DIV><<<grid, FLAT_THREADS, 0, stream>>>(d_descs); break;
      case EW_COPY: ew_flat_kernel<EW_COPY><<<grid, FLAT_THREADS, 0, stream>>>(d_descs); break;
      default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
  }
  const int tiles_r = (max_rows + 31) / 32, tiles_c = (max_cols + 31) / 32;
  dim3 grid(tiles_r * tiles_c, nblocks), block(32, 8);
  switch (op) {
    case EW_ADD: ew_tiled_kernel<EW_ADD><<<grid, block, 0, stream>>>(d_descs, tiles_c); break;
    case EW_MUL: ew_tiled_kernel<EW_MUL><<<grid, block, 0, stream>>>(d_descs, tiles_c); break;
    case EW_DIV: ew_tiled_kernel<EW_DIV><<<grid, block, 0, stream>>>(d_descs, tiles_c); break;
    case EW_COPY: ew_tiled_kernel<EW_COPY><<<grid, block, 0, stream>>>(d_descs, tiles_c); break;
    case EW_RANK1: ew_tiled_kernel<EW_RANK1><<<grid, block, 0, stream>>>(d_descs, tiles_c); break;
    case EW_RANK1_COMPAT: ew_tiled_kernel<EW_RANK1_COMPAT><<<grid, block, 0, stream>>>(d_descs, tiles_c); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t launch_map_batched(int op, const MapDesc* d_descs, int nblocks, int64_t max_n, double alpha,
                               cudaStream_t stream) {
  if (nblocks <= 0) return cudaSuccess;
  if (nblocks > 65535) {  // gridDim.y limit
    for (int off = 0; off < nblocks; off += 65535) {
      cudaError_t e = launch_map_batched(op, d_descs + off, nblocks - off < 65535 ? nblocks - off : 65535, max_n, alpha, stream);
      if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
  }
  dim3 grid(flat_grid_x(max_n), nblocks);
  switch (op) {
    case MAP_ADD_SCALAR: map_kernel<MAP_ADD_SCALAR><<<grid, FLAT_THREADS, 0, stream>>>(d_descs, alpha); break;
    case MAP_MUL_SCALAR: map_kernel<MAP_MUL_SCALAR><<<grid, FLAT_THREADS, 0, stream>>>(d_descs, alpha); break;
    case MAP_POW: map_kernel<MAP_POW><<<grid, FLAT_THREADS, 0, stream>>>(d_descs, alpha); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t launch_sparse_to_dense(const int32_t* ptrs, const int32_t* idx, const double* vals, bool isT, double* out,
                                   int rows, int cols, cudaStream_t stream) {
  const int nlines = isT ? rows : cols;
  if (nlines <= 0) return cudaSuccess;
  const int warps_per_block = 8;
  const int grid = (nlines + warps_per_block - 1) / warps_per_block;
  sparse_to_dense_kernel<<<grid, warps_per_block * 32, 0, stream>>>(ptrs, idx, vals, isT, out, rows, cols);
  return cudaGetLastError();
}

cudaError_t launch_spmm(const int32_t* ptrs, const int32_t* idx, const double* vals, bool sT, const double* B, bool bT,
                        double* C, int m, int k, int n, bool accumulate, cudaStream_t stream) {
  if (m <= 0 || n <= 0) return cudaSuccess;
  if (sT) {
    dim3 grid((m + 255) / 256, n);
    spmm_csr_kernel<<<grid, 256, 0, stream>>>(ptrs, idx, vals, B, bT, C, m, k, n, accumulate);
  } else {
    if (!accumulate) {
      cudaError_t e = cudaMemsetAsync(C, 0, static_cast<size_t>(m) * n * sizeof(double), stream);
      if (e != cudaSuccess) return e;
    }
    if (k <= 0) return cudaSuccess;
    dim3 grid((k + 7) / 8, n);
    spmm_csc_kernel<<<grid, 256, 0, stream>>>(ptrs, idx, vals, B, bT, C, m, k, n);
  }
  return cudaGetLastError();
}

cudaError_t launch_spmm_fused(const SpmmOut* d_outs, int nouts, const SpmmPair* d_pairs, int max_n, cudaStream_t stream) {
  if (nouts <= 0 || max_n <= 0) return cudaSuccess;
  const size_t smem = static_cast<size_t>(SPMM_CW) * (kSpmmMaxDim + 2) * sizeof(double);
  static PerDeviceOnce configured;
  cudaError_t e = configured.run(
      [&] { return cudaFuncSetAttribute(spmm_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)); });
  if (e != cudaSuccess) return e;
  for (int off = 0; off < nouts; off += 65535) {
    const int nb = nouts - off < 65535 ? nouts - off : 65535;
    spmm_fused_kernel<<<dim3((max_n + SPMM_CW - 1) / SPMM_CW, nb), SPMM_THREADS, smem, stream>>>(d_outs + off, d_pairs);
  }
  return cudaGetLastError();
}

cudaError_t launch_aggregate(int op, const AggDesc* d_descs, int nblocks, int max_rows, int max_cols, cudaStream_t stream) {
  if (nblocks <= 0) return cudaSuccess;
  for (int off = 0; off < nblocks; off += 65535) {
    const int nb = nblocks - off < 65535 ? nblocks - off : 65535;
    if (op == AGG_ROW_SUM || op == AGG_COL_SUM) {
      const int mx = max_rows > max_cols ? max_rows : max_cols;
      // grid.x covers whichever of the two CTA shapes needs more tiles (a batch may mix layouts); extra CTAs return at once
      const int tiles_a = ((mx + 31) / 32) * ((mx + AGG_SLOW - 1) / AGG_SLOW);
      const int tiles_b = ((mx + AGG_SWEEP - 1) / AGG_SWEEP) * ((mx + 7) / 8);
      axis_sum_kernel<<<dim3(tiles_a > tiles_b ? tiles_a : tiles_b, nb), 256, 0, stream>>>(
          d_descs + off, op == AGG_ROW_SUM ? 1 : 0, (mx + AGG_SLOW - 1) / AGG_SLOW, (mx + 7) / 8);
    } else {
      const int64_t n = op == AGG_TRACE ? max_rows : static_cast<int64_t>(max_rows) * max_cols;
      int64_t gx = (n + 256 * 16 - 1) / (256 * 16);
      if (gx < 1) gx = 1;
      if (gx > 1024) gx = 1024;
      scalar_sum_kernel<<<dim3(static_cast<unsigned>(gx), nb), 256, 0, stream>>>(d_descs + off, op == AGG_TRACE ? 1 : 0);
    }
  }
  return cudaGetLastError();
}

cudaError_t launch_extract_lines(const LineDesc* d_descs, int nblocks, int max_len, cudaStream_t stream) {
  if (nblocks <= 0 || max_len <= 0) return cudaSuccess;
  for (int off = 0; off < nblocks; off += 65535) {
    const int nb = nblocks - off < 65535 ? nblocks - off : 65535;
    extract_lines_kernel<<<dim3((max_len + 255) / 256, nb), 256, 0, stream>>>(d_descs + off);
  }
  return cudaGetLastError();
}

cudaError_t launch_copy_words(void* dst, const void* src_mapped, size_t bytes, cudaStream_t stream) {
  const size_t nwords = (bytes + 3) / 4;
  if (nwords == 0) return cudaSuccess;
  size_t grid = (nwords + 255) / 256;
  if (grid > 64) grid = 64;
  copy_words_kernel<<<static_cast<unsigned>(grid), 256, 0, stream>>>(static_cast<uint32_t*>(dst), static_cast<const uint32_t*>(src_mapped), nwords);
  return cudaGetLastError();
}

cudaError_t launch_ksplit_reduce(const KsplitDesc* d_descs, int ndescs, const double* const* d_parts, int nparts, int64_t max_count,
                                 cudaStream_t stream) {
  if (ndescs <= 0 || max_count <= 0) return cudaSuccess;
  if (nparts < 1 || nparts > kKsplitMaxParts) return cudaErrorInvalidValue;
  int64_t gx = ((max_count + 1) / 2 + KSPLIT_THREADS - 1) / KSPLIT_THREADS;  // one 128-bit element per thread
  if (gx > 4096) gx = 4096;
  for (int off = 0; off < ndescs; off += 65535) {  // gridDim.y limit
    dim3 grid(static_cast<unsigned>(gx), static_cast<unsigned>(ndescs - off < 65535 ? ndescs - off : 65535));
    ksplit_reduce_kernel<<<grid, KSPLIT_THREADS, 0, stream>>>(d_descs + off, d_parts, nparts);
  }
  return cudaGetLastError();
}

cudaError_t launch_java_rand_batched(const RandDesc* d_descs, int nblocks, int64_t max_n, cudaStream_t stream) {
  if (nblocks <= 0 || max_n <= 0) return cudaSuccess;
  int64_t gx = (max_n + 255) / 256;
  if (gx > 65535) gx = 65535;
  for (int off = 0; off < nblocks; off += 65535) {  // gridDim.y limit
    dim3 grid(static_cast<unsigned>(gx), static_cast<unsigned>(nblocks - off < 65535 ? nblocks - off : 65535));
    java_rand_kernel<<<grid, 256, 0, stream>>>(d_descs + off);
  }
  return cudaGetLastError();
}

}  // namespace matrel
