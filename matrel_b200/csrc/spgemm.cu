// Sparse x sparse block products (LocalMatrix.multiplySparseSparse, LocalMatrix.scala:143-323) and their ascending-k partial sums
// (LocalMatrix.add, :74-139) on the device, without dense images of the operands or of the result.
//
// spgemm_chain_kernel: one warp per output column of a chain (an output block whose partials are all low-density sparse x sparse).
// The chain is computed in a CSC "frame": column j of P_l = sum over the stored entries b_kj of R_l(:, j) of L_l(:, k) * b_kj,
// accumulated in a dense per-warp column accP[m] (shared memory, or global scratch for tall blocks), then S(:, j) += P_l(:, j) in
// accS[m].  Arithmetic: every product and every sum rounded on its own (__dmul_rn / __dadd_rn), each P entry summed over the R
// column in stored order, lanes of one k step on distinct rows, partials added in ascending level; an entry is dropped iff it is
// == 0.0 (so accS == 0.0 means "absent": stored entries are never +-0).  Two passes with the same kernel: COUNT (per-column nnz
// of the final sum, per-level nnz(P) and nnz(S) transitions, scalar products) and FILL (the entries, at column pointers scanned
// from the counts, or a dense window).
//
// A triangular chain (SpgemmChain::tri: a diagonal block of a Gram product, whose every P_l is symmetric) accumulates only rows
// r <= c of output column c, and its count pass also counts, per level, the diagonal entries of P_l and the zero <-> nonzero
// transitions of S on the diagonal, so the host has the full block's counts (2 upper - diagonal).  Given an `unsorted` flag, the
// count pass raises it when a walked R column's row indices do not ascend (DESIGN section 4.1.2: when a mirrored result is exact).
//
// sptrans_*: stable CSR <-> CSC conversion (the compressed arrays of a block's transpose), indices ascending in every line.
#include <cub/block/block_scan.cuh>

#include "kernels.h"

namespace matrel {

namespace {

constexpr int kSpgemmWarps = 4;                       // warps per CTA
constexpr int kSpgemmCols = kSpgemmWarps * 32;        // output columns per work item
constexpr int kSpgemmSmemCounters = 4096;             // per-level counters kept in shared memory up to this many levels

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// Per-warp accumulator of one output column: accP / accS (m doubles each), mark (m ints: the level stamp that last touched the
// row), list (m ints: the rows the current level touched, in first-touch order).
struct ColAcc {
  double* accP;
  double* accS;
  int* mark;
  int* list;
};

__device__ __forceinline__ ColAcc acc_at(char* base, int M) {
  ColAcc a;
  a.accP = reinterpret_cast<double*>(base);
  a.accS = a.accP + M;
  a.mark = reinterpret_cast<int*>(a.accS + M);
  a.list = a.mark + M;
  return a;
}

// cnt_lines: per-level counter lines of the launch (2, or 4 when a chain is triangular); smem_counters: levels per line in shared
// memory (0: global atomics).  unsorted: nullptr, or the flag the count pass raises (see the file comment).
template <bool FILL>
__global__ void __launch_bounds__(kSpgemmWarps * 32, 1) spgemm_chain_kernel(const SpgemmItem* __restrict__ items, int nitems,
                                                                          const SpgemmChain* __restrict__ chains,
                                                                          const SpgemmPair* __restrict__ pairs, int* __restrict__ counts,
                                                                          unsigned long long* __restrict__ products, char* scratch,
                                                                          int M, int smem_counters, int cnt_lines, int* unsorted) {
  extern __shared__ __align__(16) char spgemm_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t acc_bytes = static_cast<size_t>(M) * (2 * sizeof(double) + 2 * sizeof(int));
  int* cnt_smem = reinterpret_cast<int*>(spgemm_smem);  // [cnt_lines * smem_counters] when smem_counters > 0
  char* acc_base = scratch ? scratch + (static_cast<size_t>(blockIdx.x) * kSpgemmWarps + warp) * acc_bytes
                           : spgemm_smem + static_cast<size_t>(cnt_lines * smem_counters) * sizeof(int) + warp * acc_bytes;
  const ColAcc acc = acc_at(acc_base, M);
  for (int r = lane; r < M; r += 32) {
    acc.accS[r] = 0.0;
    acc.mark[r] = -1;
  }
  if (!FILL)
    for (int t = threadIdx.x; t < cnt_lines * smem_counters; t += blockDim.x) cnt_smem[t] = 0;
  __syncthreads();
  int stamp = 0;
  unsigned long long prod_count = 0;  // per lane
  for (int it = blockIdx.x; it < nitems; it += gridDim.x) {
    const SpgemmItem item = items[it];
    const SpgemmChain& ch = chains[item.chain];
    const int L = ch.levels;
    const bool tri = ch.tri != 0;
    const bool cnt_in_smem = !FILL && L <= smem_counters;
    const int cstride = cnt_in_smem ? smem_counters : L;
    int* cntP = cnt_in_smem ? cnt_smem : counts + ch.count_off;  // then nnz(S) steps, [tri] diagonal nnz(P), diagonal S steps
    for (int jj = warp; jj < kSpgemmCols; jj += kSpgemmWarps) {
      const int j = item.col0 + jj;
      if (j >= ch.n) break;
      int q0_pref = 0, q1_pref = 0;
      for (int l = 0; l < L; ++l) {
        if ((l & 31) == 0 && l + lane < L) {  // the R column ranges of the next 32 levels, one per lane
          const int32_t* rp = pairs[ch.pair_begin + l + lane].rp;
          q0_pref = rp[j];
          q1_pref = rp[j + 1];
        }
        const int q0 = __shfl_sync(0xffffffffu, q0_pref, l & 31), q1 = __shfl_sync(0xffffffffu, q1_pref, l & 31);
        if (q0 == q1) continue;
        const int32_t* __restrict__ lp = pairs[ch.pair_begin + l].lp;
        const int32_t* __restrict__ li = pairs[ch.pair_begin + l].li;
        const double* __restrict__ lv = pairs[ch.pair_begin + l].lv;
        const int32_t* __restrict__ ri = pairs[ch.pair_begin + l].ri;
        const double* __restrict__ rv = pairs[ch.pair_begin + l].rv;
        ++stamp;
        int nlist = 0;
        int k_last = 0;  // the row index of the previous chunk's last entry
        for (int qc = q0; qc < q1; qc += 32) {
          // one stored R entry per lane: its row k, value b, and the range of L(:, k)
          int a0 = 0, a1 = 0, k = 0;
          double b = 0.0;
          if (qc + lane < q1) {
            k = ri[qc + lane];
            b = rv[qc + lane];
            a0 = lp[k];
            a1 = lp[k + 1];
          }
          if (!FILL && unsorted) {
            const int up = __shfl_up_sync(0xffffffffu, k, 1);
            const int prev = lane ? up : k_last;
            if (qc + lane < q1 && (lane || qc > q0) && prev >= k) *unsorted = 1;
            k_last = __shfl_sync(0xffffffffu, k, 31);
          }
          const int nq = min(32, q1 - qc);
          for (int t = 0; t < nq; ++t) {  // stored order of R(:, j)
            const int s0 = __shfl_sync(0xffffffffu, a0, t), s1 = __shfl_sync(0xffffffffu, a1, t);
            const double bb = __shfl_sync(0xffffffffu, b, t);
            for (int e0 = s0; e0 < s1; e0 += 32) {
              const int e = e0 + lane;
              bool first = false, take = false;
              int i = 0;
              double p = 0.0;
              if (e < s1) {
                i = li[e];
                take = !tri || i <= j;  // a triangular chain: rows on and above the diagonal only
              }
              if (take) {
                p = __dmul_rn(lv[e], bb);
                first = acc.mark[i] != stamp;
              }
              if (!FILL) prod_count += take;
              const unsigned fb = __ballot_sync(0xffffffffu, first);
              if (take) {
                if (first) {
                  acc.mark[i] = stamp;
                  acc.list[nlist + __popc(fb & lanemask_lt())] = i;
                  acc.accP[i] = __dadd_rn(0.0, p);
                } else {
                  acc.accP[i] = __dadd_rn(acc.accP[i], p);
                }
              }
              nlist += __popc(fb);
              __syncwarp();
            }
          }
        }
        // S(:, j) += P_l(:, j): each touched row once; count nnz(P_l) and the zero <-> nonzero transitions of S
        int pc = 0, sd = 0, pdg = 0, sdg = 0;
        for (int t = lane; t < nlist; t += 32) {
          const int i = acc.list[t];
          const double p = acc.accP[i];
          if (p != 0.0) {
            ++pc;
            const double s = acc.accS[i];
            const double ns = __dadd_rn(s, p);
            const int step = static_cast<int>(ns != 0.0) - static_cast<int>(s != 0.0);
            sd += step;
            if (i == j) {  // read only for triangular chains
              pdg = 1;
              sdg = step;
            }
            acc.accS[i] = ns;
          }
        }
        __syncwarp();
        if (!FILL) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            pc += __shfl_xor_sync(0xffffffffu, pc, o);
            sd += __shfl_xor_sync(0xffffffffu, sd, o);
          }
          if (tri) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              pdg += __shfl_xor_sync(0xffffffffu, pdg, o);
              sdg += __shfl_xor_sync(0xffffffffu, sdg, o);
            }
          }
          if (lane == 0) {
            if (pc) atomicAdd(cntP + l, pc);
            if (sd) atomicAdd(cntP + cstride + l, sd);
            if (tri && pdg) atomicAdd(cntP + 2 * cstride + l, pdg);
            if (tri && sdg) atomicAdd(cntP + 3 * cstride + l, sdg);
          }
        }
      }
      // the final column: rows ascending, entries != 0.0; accS is cleared for the next column.  A triangular chain ends at the
      // diagonal (nothing below it was accumulated, and a dense window's lower part is the mirror pass's).
      int out = 0;
      const int base = FILL && ch.oidx ? ch.optr[j] : 0;
      const int rows = tri ? min(ch.m, j + 1) : ch.m;
      for (int r0 = 0; r0 < rows; r0 += 32) {
        const int r = r0 + lane;
        double v = 0.0;
        if (r < rows) {
          v = acc.accS[r];
          acc.accS[r] = 0.0;
        }
        const bool nz = r < rows && v != 0.0;
        const unsigned nb = __ballot_sync(0xffffffffu, nz);
        if (FILL) {
          if (ch.dense) {
            if (r < rows) ch.dense[static_cast<int64_t>(r) * ch.drs + static_cast<int64_t>(j) * ch.dcs] = nz ? v : 0.0;
          } else if (nz) {
            const int pos = base + out + __popc(nb & lanemask_lt());
            ch.oidx[pos] = r;
            ch.oval[pos] = v;
          }
        }
        out += __popc(nb);
      }
      __syncwarp();
      if (!FILL && lane == 0) ch.colcnt[j] = out;
    }
    if (cnt_in_smem) {  // flush this item's per-level counters
      __syncthreads();
      const int lines = tri ? 4 : 2;
      for (int t = threadIdx.x; t < L; t += blockDim.x)
        for (int q = 0; q < lines; ++q) {
          if (cnt_smem[q * smem_counters + t]) atomicAdd(counts + ch.count_off + q * L + t, cnt_smem[q * smem_counters + t]);
          cnt_smem[q * smem_counters + t] = 0;
        }
      __syncthreads();
    }
  }
  if (!FILL) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) prod_count += __shfl_xor_sync(0xffffffffu, prod_count, o);
    if (lane == 0 && prod_count) atomicAdd(products, prod_count);
  }
}

// out[0] = 0, out[t + 1] = in[0] + ... + in[t]; one CTA per descriptor
constexpr int kScanThreads = 256;
__global__ void __launch_bounds__(kScanThreads) exclusive_scan_kernel(const ScanDesc* __restrict__ descs) {
  using BlockScan = cub::BlockScan<int, kScanThreads>;
  __shared__ typename BlockScan::TempStorage tmp;
  __shared__ int carry;
  const ScanDesc d = descs[blockIdx.x];
  if (threadIdx.x == 0) {
    carry = 0;
    d.out[0] = 0;
  }
  __syncthreads();
  for (int c0 = 0; c0 < d.n; c0 += kScanThreads) {
    const int t = c0 + threadIdx.x;
    const int v = t < d.n ? d.in[t] : 0;
    int incl = 0, total = 0;
    BlockScan(tmp).InclusiveSum(v, incl, total);
    if (t < d.n) d.out[t + 1] = carry + incl;
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
}

// entries per output line (grid-stride over the stored entries)
__global__ void __launch_bounds__(256) sptrans_count_kernel(const SpTransDesc* __restrict__ descs) {
  const SpTransDesc d = descs[blockIdx.y];
  const int nnz = d.nnz;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += gridDim.x * blockDim.x) atomicAdd(d.cur + d.idx[e], 1);
}

// thread per input line: its entries go to their output lines (in any order; sptrans_sort_kernel orders them).  `cur` still holds
// the counts of sptrans_count_kernel and ends at zero.
__global__ void __launch_bounds__(256) sptrans_fill_kernel(const SpTransDesc* __restrict__ descs) {
  const SpTransDesc d = descs[blockIdx.y];
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < d.nl; r += gridDim.x * blockDim.x)
    for (int e = d.ptr[r]; e < d.ptr[r + 1]; ++e) {
      const int c = d.idx[e];
      const int pos = d.optr[c] + atomicSub(d.cur + c, 1) - 1;  // counts down from the line's count
      d.oidx[pos] = r;
      d.oval[pos] = d.val[e];
    }
}

// thread per output line: insertion sort by index (an input line holds an index at most once, so the order is unique)
__global__ void __launch_bounds__(256) sptrans_sort_kernel(const SpTransDesc* __restrict__ descs) {
  const SpTransDesc d = descs[blockIdx.y];
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < d.no; c += gridDim.x * blockDim.x) {
    const int b = d.optr[c], e = d.optr[c + 1];
    for (int x = b + 1; x < e; ++x) {
      const int key = d.oidx[x];
      const double v = d.oval[x];
      int y = x - 1;
      while (y >= b && d.oidx[y] > key) {
        d.oidx[y + 1] = d.oidx[y];
        d.oval[y + 1] = d.oval[y];
        --y;
      }
      d.oidx[y + 1] = key;
      d.oval[y + 1] = v;
    }
  }
}

PerDeviceOnce g_spgemm_attr;
int g_sm_count[64] = {};

size_t spgemm_smem_bytes(int M, int smem_counters, int cnt_lines, bool acc_in_smem) {
  return static_cast<size_t>(cnt_lines * smem_counters) * sizeof(int) +
         (acc_in_smem ? static_cast<size_t>(kSpgemmWarps) * M * (2 * sizeof(double) + 2 * sizeof(int)) : 0);
}

}  // namespace

int spgemm_columns_per_item() { return kSpgemmCols; }

SpgemmLaunchShape spgemm_shape(int max_m, int max_levels, bool tri) {
  SpgemmLaunchShape s{};
  s.smem_counters = max_levels <= kSpgemmSmemCounters ? max_levels : 0;
  s.cnt_lines = tri ? 4 : 2;
  s.acc_in_smem = spgemm_smem_bytes(max_m, s.smem_counters, s.cnt_lines, true) <= kSpgemmMaxSmem;
  int dev = 0;
  cudaGetDevice(&dev);
  int sms = 132;
  if (dev >= 0 && dev < 64) {
    if (!g_sm_count[dev]) cudaDeviceGetAttribute(&g_sm_count[dev], cudaDevAttrMultiProcessorCount, dev);
    if (g_sm_count[dev] > 0) sms = g_sm_count[dev];
  }
  s.max_ctas = sms * (s.acc_in_smem ? 8 : 4);  // persistent grid; global accumulators: 4 CTAs (16 warps) per SM
  s.scratch_bytes = s.acc_in_smem ? 0 : static_cast<size_t>(s.max_ctas) * kSpgemmWarps * max_m * (2 * sizeof(double) + 2 * sizeof(int));
  return s;
}

cudaError_t launch_spgemm(bool fill, const SpgemmItem* d_items, int nitems, const SpgemmChain* d_chains, const SpgemmPair* d_pairs,
                          int* d_counts, unsigned long long* d_products, void* d_scratch, int max_m, const SpgemmLaunchShape& s,
                          int* d_unsorted, cudaStream_t stream) {
  if (nitems <= 0 || max_m <= 0) return cudaSuccess;
  cudaError_t e = g_spgemm_attr.run([&] {
    cudaError_t r = cudaFuncSetAttribute(spgemm_chain_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSpgemmMaxSmem);
    if (r != cudaSuccess) return r;
    return cudaFuncSetAttribute(spgemm_chain_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSpgemmMaxSmem);
  });
  if (e != cudaSuccess) return e;
  const int ctas = nitems < s.max_ctas ? nitems : s.max_ctas;
  const size_t smem = spgemm_smem_bytes(max_m, fill ? 0 : s.smem_counters, s.cnt_lines, s.acc_in_smem);
  char* scratch = s.acc_in_smem ? nullptr : static_cast<char*>(d_scratch);
  if (fill)
    spgemm_chain_kernel<true><<<ctas, kSpgemmWarps * 32, smem, stream>>>(d_items, nitems, d_chains, d_pairs, d_counts, d_products, scratch,
                                                                        max_m, 0, s.cnt_lines, nullptr);
  else
    spgemm_chain_kernel<false><<<ctas, kSpgemmWarps * 32, smem, stream>>>(d_items, nitems, d_chains, d_pairs, d_counts, d_products,
                                                                         scratch, max_m, s.smem_counters, s.cnt_lines, d_unsorted);
  return cudaGetLastError();
}

cudaError_t launch_exclusive_scan(const ScanDesc* d_descs, int ndescs, cudaStream_t stream) {
  if (ndescs <= 0) return cudaSuccess;
  exclusive_scan_kernel<<<ndescs, kScanThreads, 0, stream>>>(d_descs);
  return cudaGetLastError();
}

cudaError_t launch_sptrans(const SpTransDesc* d_descs, const ScanDesc* d_scans, int ndescs, int max_nnz, int max_nl, int max_no,
                           cudaStream_t stream) {
  if (ndescs <= 0) return cudaSuccess;
  auto blocks = [](int n) { return n <= 0 ? 1 : (n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024; };
  for (int off = 0; off < ndescs; off += 65535) {
    const int nb = ndescs - off < 65535 ? ndescs - off : 65535;
    sptrans_count_kernel<<<dim3(blocks(max_nnz), nb), 256, 0, stream>>>(d_descs + off);
  }
  cudaError_t e = launch_exclusive_scan(d_scans, ndescs, stream);
  if (e != cudaSuccess) return e;
  for (int off = 0; off < ndescs; off += 65535) {
    const int nb = ndescs - off < 65535 ? ndescs - off : 65535;
    sptrans_fill_kernel<<<dim3(blocks(max_nl), nb), 256, 0, stream>>>(d_descs + off);
  }
  for (int off = 0; off < ndescs; off += 65535) {
    const int nb = ndescs - off < 65535 ? ndescs - off : 65535;
    sptrans_sort_kernel<<<dim3(blocks(max_no), nb), 256, 0, stream>>>(d_descs + off);
  }
  return cudaGetLastError();
}

}  // namespace matrel
