// CSR-block x dense-block products for sm_90a: C(i,j) (+)= sum_k A(i,k) B(k,j) with A(i,k) sparse (CSR) and B(k,j) dense.
//
// Replaces BLAS.gemmsdd's CSR loop nests (M/matrix/BLAS.scala:375-413) and the reduceByKey(LocalMatrix.add) over k
// (M/execution/MatfastExecutionHelper.scala:255): one launch per multiply, the K loop over the block pairs of an output block is
// fused (the 32-column accumulators of a 512-row strip stay in registers across ALL k-blocks; C is written once).
//
// What bounds it: every multiply-add needs its own 8-byte B element at a data-dependent row, so the shared-memory port
// (128 B/clk/SM = 16 fp64 FMA/clk/SM, ~9 TFLOP/s) is the algorithmic roof, not the fp64 pipe.  The kernel is organised around
// spending as few shared-memory wavefronts AND as few issue slots per FMA as the format allows:
//   * B is staged ROW-major ([k][64 columns], 512-byte rows, TMA tensor copies of a {64, KC} box), and a whole WARP owns a row of
//     A: lane l accumulates columns 2l and 2l + 1, so one CSR entry costs one warp-uniform 16-byte read (value + byte offset of
//     its B row, packed by the preparation pass) and one 128-bit load per lane (four conflict-free wavefronts) for 64 FMAs.
//     No lane is ever predicated off: rows of different length cost different trip counts of a warp-uniform loop, not idle lanes.
//     (Column-major B blocks are transposed once per multiply by the host layer -- 2 x 8 bytes per element of HBM traffic against
//     ~10 uses per element.)
//   * the CSR entries of a (256-row strip, 128-wide k chunk) are re-packed by a preparation pass into one contiguous segment
//     that the producer warp brings in with ONE bulk copy per pipeline stage, together with its row-pointer table; a warp owns
//     16 CONSECUTIVE rows, reads their 17 row pointers with one load and hands them round by shuffles.
//   * producer warp + 16 consumer warps, 3-stage full/empty mbarrier ring (a fast warp runs up to two stages ahead of a slow
//     one); the 256 x 64 result tile is transposed through the (by then idle) stage buffers so that C is written as coalesced
//     column runs.
//
// The same two kernels, instantiated with kDs = true, compute dense x low-density sparse partials C = A S as C^T = S^T A^T:
// the CSC arrays of S are the CSR arrays of S^T, a column-major A is A^T row-major, and C^T row-major is C column-major.  That
// variant stages only the columns of A a (strip, chunk) segment references (one 64-row run per distinct k, found by the
// preparation pass), skips empty segments, keeps only the last of repeated (k, j) entries (SparseMatrix.toArray semantics),
// and writes C from registers: lane l holds rows 2l, 2l + 1 of one column, so a warp stores a 512-byte run per column.
// ds_flag_kernel / ds_fixup_kernel give C(i, j) the NaN the densified product gets from a non-finite A(i, k) meeting an
// implicit zero of column j of S.
#include <cuda.h>

#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

#include "kernels.h"

namespace matrel {
namespace {

constexpr int TM = kSpmm2StripRows;   // rows per CTA
constexpr int TN = kSpmm2TileCols;    // columns per CTA
constexpr int KC = kSpmm2ChunkK;      // k extent of one pipeline stage
constexpr int NSTAGE = 3;
constexpr int RP_PAD = TM + 4;        // row-pointer table entries per (strip, chunk): TM + 1, padded to a 16-byte multiple
constexpr int E_CAP = 664;            // entries per stage held in shared memory (larger segments are read from global memory)
constexpr int NCW = 16;               // consumer warps
constexpr int RPW = TM / NCW;         // rows per consumer warp
constexpr int THREADS = (NCW + 1) * 32;
constexpr int B_BYTES = KC * TN * 8;                 // 65536
constexpr int RP_BYTES = RP_PAD * 4;                 // 1040
constexpr int ENT_BYTES = E_CAP * 16;                // 10624
constexpr int STAGE_BYTES = B_BYTES + ENT_BYTES + RP_BYTES;
constexpr int STAGE_STRIDE = (STAGE_BYTES + 127) / 128 * 128;
constexpr int SMEM_BYTES = 128 + NSTAGE * STAGE_STRIDE + 64;
constexpr int CS_LD = TM + 1;                        // result tile in shared memory: [64 columns][TM + 1] doubles
static_assert(TN == 64 && RPW == 16, "lane <-> column pair and lane <-> row pointer mappings");
static_assert(CS_LD * TN * 8 <= NSTAGE * STAGE_STRIDE, "result tile must fit the stage buffers");
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");

struct __align__(16) Entry {
  double a;
  uint32_t boff;  // byte offset of B row k inside the stage's B tile: (k - chunk start) * TN * 8
  uint32_t pad;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"(bar), "r"(parity)
                 : "memory");
  } while (!ok);
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
               "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_2d(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
               "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
               : "memory");
}

// ------------------------------------------------------------------------------------------------
// preparation: CSR block -> per (strip, chunk) segments of packed entries + row-pointer tables
// ------------------------------------------------------------------------------------------------
// One CTA per sparse block (1024 threads: thread = row, two rows per thread above 1024 are not needed: m <= 1024).
// Order inside a segment: rows ascending, entries of a row in their CSR storage order (the reference's summation order within
// the chunk).  segoff[(s * nchunks + q)] = first entry of segment (s, q) in `ent`, segoff[nseg] = nnz.
// kDs (dense x sparse): the block is S^T (rows = columns of S); of entries repeating an index in a row only the one toArray keeps
// counts (kept_entry); every segment's distinct indices get slots in ascending order (kref, count at rp[TM + 1]) and boff
// addresses the slot.
constexpr int KW = KC / 32;  // words of a segment's index bitmap
static_assert(KC / 32 == 4, "kref stores an index inside its chunk as one byte; a producer lane reads its 4 slots as one word");
template <bool kDs>
using Spmm2PrepT = typename std::conditional<kDs, DspmmPrep, Spmm2Prep>::type;

template <bool kDs>
__global__ void __launch_bounds__(1024) spmm2_prep_kernel(const Spmm2PrepT<kDs>* __restrict__ preps) {
  extern __shared__ int32_t cnt[];  // [m_pad][nchunks] counters, then reused as write cursors (kDs: then [nseg][KW] index bitmaps)
  __shared__ int32_t warp_tot[32];
  const Spmm2PrepT<kDs> p = preps[blockIdx.x];
  const int m = p.m, nchunks = (p.kdim + KC - 1) / KC, nstrips = (m + TM - 1) / TM;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int total = nstrips * TM * nchunks;  // counters in (strip, chunk, row-in-strip) order
  uint32_t* kbits = reinterpret_cast<uint32_t*>(cnt + total);
  for (int i = tid; i < total; i += blockDim.x) cnt[i] = 0;
  if constexpr (kDs)
    for (int i = tid; i < nstrips * nchunks * KW; i += blockDim.x) kbits[i] = 0;
  __syncthreads();
  auto slot = [&](int row, int q) { return ((row / TM) * nchunks + q) * TM + (row % TM); };
  // kDs: is entry e of row [beg, end) the one its index keeps: the last with that index, or the first when p.repeats_reversed
  // (rows with strictly ascending indices have no repeats)
  auto kept_entry = [&](int e, int beg, int end, bool ascending) {
    if constexpr (kDs) {
      if (ascending) return true;
      const int c = p.idx[e];
      for (int f = p.repeats_reversed ? beg : e + 1; f < (p.repeats_reversed ? e : end); ++f)
        if (p.idx[f] == c) return false;
    }
    return true;
  };
  auto distinct = [&](int sg) {  // kDs: distinct indices of segment sg
    int n = 0;
    for (int w = 0; w < KW; ++w) n += __popc(kbits[sg * KW + w]);
    return n;
  };
  auto ascending_row = [&](int beg, int end) {
    for (int e = beg + 1; e < end; ++e)
      if (p.idx[e] <= p.idx[e - 1]) return false;
    return true;
  };
  for (int row = tid; row < m; row += blockDim.x) {
    const int beg = p.ptrs[row], end = p.ptrs[row + 1];
    if constexpr (kDs) {
      const bool asc = ascending_row(beg, end);
      for (int e = beg; e < end; ++e) {
        if (!kept_entry(e, beg, end, asc)) continue;
        const int col = p.idx[e], q = col / KC, kk = col - q * KC;
        atomicAdd(&cnt[slot(row, q)], 1);
        atomicOr(&kbits[((row / TM) * nchunks + q) * KW + (kk >> 5)], 1u << (kk & 31));
      }
    } else {
      for (int e = beg; e < end; ++e) atomicAdd(&cnt[slot(row, p.idx[e] / KC)], 1);  // own row only: no contention, plain RMW semantics
    }
  }
  __syncthreads();
  // exclusive scan of cnt[0 .. total) (block-wide, chunked by blockDim.x)
  int carry = 0;
  for (int base = 0; base < total; base += blockDim.x) {
    const int i = base + tid;
    const int v = i < total ? cnt[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = lane < (blockDim.x >> 5) ? warp_tot[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      warp_tot[lane] = w;  // inclusive scan of the warp totals
    }
    __syncthreads();
    const int warp_off = warp == 0 ? 0 : warp_tot[warp - 1];
    const int excl = carry + warp_off + x - v;
    if (i < total) cnt[i] = excl;
    const int chunk_total = warp_tot[(blockDim.x >> 5) - 1];
    __syncthreads();
    carry += chunk_total;
  }
  // row-pointer tables (relative to the segment start) and segment offsets
  const int nseg = nstrips * nchunks;
  for (int sg = tid; sg <= nseg; sg += blockDim.x) p.segoff[sg] = sg < nseg ? cnt[sg * TM] : carry;
  for (int i = tid; i < nseg * RP_PAD; i += blockDim.x) {
    const int sg = i / RP_PAD, r = i % RP_PAD;
    const int seg0 = cnt[sg * TM];
    int v;
    if (r < TM) v = cnt[sg * TM + r] - seg0;
    else v = (sg + 1 < nseg ? cnt[(sg + 1) * TM] : carry) - seg0;  // r == TM (and the padding): segment length
    if (kDs && r == TM + 1) v = distinct(sg);
    p.rp[i] = v;
  }
  // kDs: slot -> index inside the chunk
  auto slot_of = [&](int sg, int kk) {
    int n = __popc(kbits[sg * KW + (kk >> 5)] & ((1u << (kk & 31)) - 1u));
    for (int w = 0; w < (kk >> 5); ++w) n += __popc(kbits[sg * KW + w]);
    return n;
  };
  // kDs: the slot table of every segment, all KC bytes written (the producer reads it a word per lane; slots past the segment's
  // count are zero and never used)
  if constexpr (kDs)
    for (int i = tid; i < nseg * KC; i += blockDim.x) {
      const int sg = i / KC, kk = i % KC;
      if (kbits[sg * KW + (kk >> 5)] & (1u << (kk & 31))) p.kref[sg * KC + slot_of(sg, kk)] = static_cast<uint8_t>(kk);
      if (kk >= distinct(sg)) p.kref[sg * KC + kk] = 0;
    }
  __syncthreads();
  // scatter (cnt becomes the per (row, chunk) write cursor)
  Entry* ent = reinterpret_cast<Entry*>(p.ent);
  for (int row = tid; row < m; row += blockDim.x) {
    const int beg = p.ptrs[row], end = p.ptrs[row + 1];
    const bool asc = kDs ? ascending_row(beg, end) : true;
    for (int e = beg; e < end; ++e) {
      if (kDs && !kept_entry(e, beg, end, asc)) continue;
      const int col = p.idx[e];
      const int q = col / KC;
      const int pos = cnt[slot(row, q)]++;
      Entry en;
      en.a = p.vals[e];
      en.boff = static_cast<uint32_t>(kDs ? slot_of((row / TM) * nchunks + q, col - q * KC) : col - q * KC) * (TN * 8);
      en.pad = 0;
      ent[pos] = en;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// main kernel
// ------------------------------------------------------------------------------------------------
// shared-memory accesses by 32-bit shared address (plain C++ through the dynamically aligned base pointer compiles to generic loads)
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void lds_entry(uint32_t addr, double& a, uint32_t& boff) {
  uint32_t lo, hi, pad;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(lo), "=r"(hi), "=r"(boff), "=r"(pad) : "r"(addr));
  (void)pad;
  a = __hiloint2double(static_cast<int>(hi), static_cast<int>(lo));
}
__device__ __forceinline__ void lds_f64x2(uint32_t addr, double& x, double& y) {
  asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(x), "=d"(y) : "r"(addr));
}

template <bool kDs>
using Spmm2PairT = typename std::conditional<kDs, DspmmPair, Spmm2Pair>::type;

// kDs: out.m / out.n are the dims of C^T (columns of S / rows of A); element C^T(r, c) lives at out.C[r * out.n + c].
template <bool kDs>
__global__ void __launch_bounds__(THREADS, 1) spmm2_kernel(const Spmm2Item* __restrict__ items, const Spmm2Out* __restrict__ outs,
                                                           const Spmm2PairT<kDs>* __restrict__ pairs, const unsigned char* __restrict__ tmaps) {
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((128u - (smem_u32(smem_dyn) & 127u)) & 127u);
  const uint32_t smem_a = smem_u32(smem);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGE * STAGE_STRIDE);  // full[NSTAGE], empty[NSTAGE]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const Spmm2Item item = items[blockIdx.x];
  const Spmm2Out out = outs[item.out];
  const int row0 = item.strip * TM, col0 = item.ctile * TN;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE; ++s) {
      mbar_init(smem_u32(&bars[s]), 1);
      mbar_init(smem_u32(&bars[NSTAGE + s]), NCW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == NCW) {
    if constexpr (kDs) {
      // ===================== producer warp (kDs): one 64-row run of A per distinct k of a non-empty segment, issued by all lanes.
      // A pair's segment offsets and distinct-index counts are read once (lane q: chunk q), a stage's slot table (4 slots per lane)
      // before waiting for its buffer, so no dependent global read sits between the wait and the copies.
      const uint32_t run = static_cast<uint32_t>(min(TN, out.n - col0)) * 8u;  // out.n is even: a multiple of 16 bytes
      int s = 0;
      uint32_t ph = 0;
      for (int p = 0; p < out.pair_count; ++p) {
        const DspmmPair pr = pairs[out.pair_begin + p];
        const int nchunks = (pr.kdim + KC - 1) / KC, sg0 = item.strip * nchunks;
        const int so = lane <= nchunks ? __ldg(pr.segoff + sg0 + lane) : 0;
        const int nr = lane < nchunks ? __ldg(pr.rp + static_cast<size_t>(sg0 + lane) * RP_PAD + TM + 1) : 0;
        const int so_next = __shfl_down_sync(0xffffffffu, so, 1);
        for (uint32_t todo = __ballot_sync(0xffffffffu, lane < nchunks && so_next > so); todo; todo &= todo - 1) {
          const int q = __ffs(todo) - 1, sg = sg0 + q;
          const int e0 = __shfl_sync(0xffffffffu, so, q), len = __shfl_sync(0xffffffffu, so_next, q) - e0;
          const int nref = __shfl_sync(0xffffffffu, nr, q);
          const uint32_t kw = __ldg(reinterpret_cast<const uint32_t*>(pr.kref + static_cast<size_t>(sg) * KC) + lane);
          mbar_wait(smem_u32(&bars[NSTAGE + s]), ph ^ 1);
          const uint32_t st = smem_a + s * STAGE_STRIDE;
          const uint32_t full = smem_u32(&bars[s]);
          const uint32_t ent_bytes = len <= E_CAP ? static_cast<uint32_t>(len) * 16u : 0u;
          if (lane == 0) {
            mbar_arrive_expect_tx(full, static_cast<uint32_t>(nref) * run + RP_BYTES + ent_bytes);
            tma_bulk_g2s(st + B_BYTES + ENT_BYTES, pr.rp + static_cast<size_t>(sg) * RP_PAD, RP_BYTES, full);
            if (ent_bytes) tma_bulk_g2s(st + B_BYTES, pr.ent + static_cast<size_t>(e0) * 16, ent_bytes, full);
          }
          __syncwarp();
#pragma unroll
          for (int b = 0; b < KC / 32; ++b) {
            const int t = (KC / 32) * lane + b;
            if (t < nref) {
              const int k = q * KC + static_cast<int>((kw >> (8 * b)) & 255u);
              tma_bulk_g2s(st + t * (TN * 8), pr.A + static_cast<size_t>(k) * pr.lda + col0, run, full);
            }
          }
          if (++s == NSTAGE) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    } else if (lane == 0) {
      // ===================== producer warp (one elected lane) =====================
      int s = 0;
      uint32_t ph = 0;
      for (int p = 0; p < out.pair_count; ++p) {
        const Spmm2Pair pr = pairs[out.pair_begin + p];
        const int nchunks = (pr.kdim + KC - 1) / KC;
        const void* tm = tmaps + static_cast<size_t>(pr.tmB) * 128;
        for (int q = 0; q < nchunks; ++q) {
          mbar_wait(smem_u32(&bars[NSTAGE + s]), ph ^ 1);
          const uint32_t st = smem_a + s * STAGE_STRIDE;
          const int sg = item.strip * nchunks + q;
          const int e0 = pr.segoff[sg], len = pr.segoff[sg + 1] - e0;
          const uint32_t full = smem_u32(&bars[s]);
          const uint32_t ent_bytes = len <= E_CAP ? static_cast<uint32_t>(len) * 16u : 0u;
          mbar_arrive_expect_tx(full, B_BYTES + RP_BYTES + ent_bytes);
          tma_2d(st, tm, col0, q * KC, full);
          tma_bulk_g2s(st + B_BYTES + ENT_BYTES, pr.rp + static_cast<size_t>(sg) * RP_PAD, RP_BYTES, full);
          if (ent_bytes) tma_bulk_g2s(st + B_BYTES, pr.ent + static_cast<size_t>(e0) * 16, ent_bytes, full);
          if (++s == NSTAGE) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== consumer warps: warp w owns rows [16 w, 16 w + 16) of the strip, lane l columns 2l, 2l + 1 =====================
    double acc[RPW][2];
#pragma unroll
    for (int i = 0; i < RPW; ++i) acc[i][0] = acc[i][1] = 0.0;
    int s = 0;
    uint32_t ph = 0;
    for (int p = 0; p < out.pair_count; ++p) {
      const Spmm2PairT<kDs> pr = pairs[out.pair_begin + p];
      const int nchunks = (pr.kdim + KC - 1) / KC;
      uint32_t nonempty = 0;  // kDs: the chunks the producer stages (lane q reads chunk q's segment offsets)
      if constexpr (kDs) {
        const int so = lane <= nchunks ? __ldg(pr.segoff + item.strip * nchunks + lane) : 0;
        const int so_next = __shfl_down_sync(0xffffffffu, so, 1);
        nonempty = __ballot_sync(0xffffffffu, lane < nchunks && so_next > so);
      }
      for (int q = 0; q < nchunks; ++q) {
        if (kDs && !((nonempty >> q) & 1u)) continue;
        const uint32_t st = smem_a + s * STAGE_STRIDE;
        const uint32_t rp_a = st + B_BYTES + ENT_BYTES;
        const uint32_t bl = st + lane * 16;  // this lane's column pair inside a B row
        mbar_wait(smem_u32(&bars[s]), ph);
        const int rpv = static_cast<int>(lds_u32(rp_a + (warp * RPW + (lane < RPW ? lane : RPW)) * 4));  // lanes 0 .. 16: rp[16 w + lane]
        const int seglen = static_cast<int>(lds_u32(rp_a + TM * 4));
        if (seglen <= E_CAP) {
          int ev[RPW + 1];  // the 17 row pointers of this warp's rows, warp-uniform
#pragma unroll
          for (int r = 0; r <= RPW; ++r) ev[r] = __shfl_sync(0xffffffffu, rpv, r);
          const uint32_t ents = st + B_BYTES;
#pragma unroll
          for (int r = 0; r < RPW; ++r) {
            uint32_t ea = ents + static_cast<uint32_t>(ev[r]) * 16u;
            const uint32_t ee = ents + static_cast<uint32_t>(ev[r + 1]) * 16u;
#pragma unroll 1
            for (; ea < ee; ea += 16) {  // warp-uniform trip count, 1.3 on average at 1 % density: not worth unrolling
              double a, b0, b1;
              uint32_t boff;
              lds_entry(ea, a, boff);
              lds_f64x2(bl + boff, b0, b1);
              acc[r][0] = fma(a, b0, acc[r][0]);
              acc[r][1] = fma(a, b1, acc[r][1]);
            }
          }
        } else {
          // a segment larger than the stage buffer (denser blocks): the warp's entries (one contiguous run, rows ascending) are
          // fetched from global memory 32 at a time, one coalesced 16-byte load per lane, and handed round by shuffles
          const uint4* gents = reinterpret_cast<const uint4*>(pr.ent) + pr.segoff[item.strip * nchunks + q];
          const int eend = __shfl_sync(0xffffffffu, rpv, RPW);
          int e = __shfl_sync(0xffffffffu, rpv, 0), bb = e;
          uint4 mine = bb + lane < eend ? __ldg(gents + bb + lane) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
          for (int r = 0; r < RPW; ++r) {
            const int e1 = __shfl_sync(0xffffffffu, rpv, r + 1);
#pragma unroll 1
            for (; e < e1; ++e) {
              if (e - bb == 32) {
                bb = e;
                mine = bb + lane < eend ? __ldg(gents + bb + lane) : make_uint4(0u, 0u, 0u, 0u);
              }
              const int j = e - bb;
              const double a = __hiloint2double(static_cast<int>(__shfl_sync(0xffffffffu, mine.y, j)),
                                                static_cast<int>(__shfl_sync(0xffffffffu, mine.x, j)));
              const uint32_t boff = __shfl_sync(0xffffffffu, mine.z, j);
              double b0, b1;
              lds_f64x2(bl + boff, b0, b1);
              acc[r][0] = fma(a, b0, acc[r][0]);
              acc[r][1] = fma(a, b1, acc[r][1]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bars[NSTAGE + s]));
        if (++s == NSTAGE) {
          s = 0;
          ph ^= 1;
        }
      }
    }
    if constexpr (kDs) {
      // ---- epilogue: C^T row r = column row0 + r of C; this lane's two rows of C are adjacent, the warp's 64 a 512-byte run
      const int rows = min(TM, out.m - row0), c = col0 + 2 * lane;
#pragma unroll
      for (int i = 0; i < RPW; ++i) {
        const int r = warp * RPW + i;
        if (r < rows && c < out.n) {
          double2* dst = reinterpret_cast<double2*>(out.C + static_cast<size_t>(out.n) * (row0 + r) + c);
          double2 v = make_double2(acc[i][0], acc[i][1]);
          if (out.accumulate) {
            const double2 o = *dst;
            v.x = o.x + v.x;
            v.y = o.y + v.y;
          }
          *dst = v;
        }
      }
      return;
    }
    // ---- epilogue: registers -> shared memory [column][row] -> coalesced column runs of the column-major output block
    asm volatile("bar.sync 1, %0;" ::"r"(NCW * 32) : "memory");  // every consumer has finished reading the stage buffers
    double* Cs = reinterpret_cast<double*>(smem);
#pragma unroll
    for (int i = 0; i < RPW; ++i) {
      const int r = warp * RPW + i;
      Cs[(2 * lane) * CS_LD + r] = acc[i][0];
      Cs[(2 * lane + 1) * CS_LD + r] = acc[i][1];
    }
    asm volatile("bar.sync 1, %0;" ::"r"(NCW * 32) : "memory");
    const int rows = min(TM, out.m - row0), cols = min(TN, out.n - col0);
    for (int idx = threadIdx.x; idx < cols * TM; idx += NCW * 32) {
      const int c = idx / TM, r = idx % TM;
      if (r < rows) {
        double* dst = out.C + static_cast<size_t>(out.m) * (col0 + c) + row0 + r;
        const double v = Cs[c * CS_LD + r];
        *dst = out.accumulate ? *dst + v : v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// dense x sparse: the NaN of a non-finite A(i, k) times an implicit zero of column j of S (the densified product's Inf * 0)
// ------------------------------------------------------------------------------------------------
// Flag pass: one thread per row of a column-major A (one read of the block).  bits[i * 32 + w] bit b: A(i, 32 w + b) is not
// finite; rowflags bit i: row i has such an element; *any = 1 when the block has one (pre-zeroed by the caller).
__device__ __forceinline__ bool nonfinite(double v) { return (__double_as_longlong(v) & 0x7ff0000000000000ll) == 0x7ff0000000000000ll; }

// Grid: x = descriptor (no 65535 limit on the number of blocks), y = 256-row chunk of the block.
__global__ void __launch_bounds__(256) ds_flag_kernel(const DsFlagDesc* __restrict__ descs) {
  const DsFlagDesc d = descs[blockIdx.x];
  const int i = blockIdx.y * 256 + threadIdx.x;
  if (blockIdx.y * 256 >= d.m) return;
  bool row_nf = false;
  if (i < d.m) {
    for (int w = 0; w < DS_KW; ++w) {
      uint32_t bits = 0;
      if (w * 32 < d.kdim) {
#pragma unroll 8
        for (int b = 0; b < 32; ++b) {
          const int k = w * 32 + b;
          if (k < d.kdim && nonfinite(__ldg(d.A + static_cast<size_t>(k) * d.m + i))) bits |= 1u << b;
        }
      }
      d.bits[static_cast<size_t>(i) * DS_KW + w] = bits;
      row_nf = row_nf || bits != 0;
    }
  }
  const uint32_t flags = __ballot_sync(0xffffffffu, row_nf);
  if ((threadIdx.x & 31) == 0 && i < d.m) d.rowflags[i >> 5] = flags;
  if (row_nf) *d.any = 1;
}

// Fix-up, after every partial of the blocks: C(i, j) = NaN when some non-finite A(i, k) has no stored (k, j) in S.  Persistent
// CTAs over the pairs; a pair whose A block is all finite costs one read of its flag.  A warp per column j of S: its stored
// indices as a 1024-bit set (lane w holds word w), then every flagged row's non-finite set against it.
static_assert(DS_KW == 32, "lane w holds word w of a 1024-bit set");
__global__ void __launch_bounds__(256) ds_fixup_kernel(const DsFixPair* __restrict__ pairs, int npairs) {
  __shared__ uint32_t sb[8][DS_KW];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int p = blockIdx.x; p < npairs; p += gridDim.x) {
    const DsFixPair f = pairs[p];
    if (!*f.any) continue;
    for (int j = warp; j < f.n; j += 8) {
      sb[warp][lane] = 0;
      __syncwarp();
      for (int e = f.ptr[j] + lane; e < f.ptr[j + 1]; e += 32) atomicOr(&sb[warp][f.idx[e] >> 5], 1u << (f.idx[e] & 31));
      __syncwarp();
      const uint32_t stored = sb[warp][lane];
      __syncwarp();
      for (int i0 = 0; i0 < f.m; i0 += 32) {
        uint32_t rows = f.rowflags[i0 >> 5];
        while (rows) {
          const int i = i0 + __ffs(rows) - 1;
          rows &= rows - 1;
          if (__any_sync(0xffffffffu, (f.bits[static_cast<size_t>(i) * DS_KW + lane] & ~stored) != 0) && lane == 0)
            f.C[static_cast<size_t>(j) * f.m + i] = __longlong_as_double(0x7ff8000000000000ll);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// SparseMatrix.sprand on the device (M/matrix/MLMatrix.scala:791-856, the draw-by-draw branch, density < 0.34), bit-identical to
// the JVM: draws (rng.nextInt(numRows), rng.nextInt(numCols)) into a set until it holds nnz = ceil(rows * cols * density)
// distinct coordinates, sorts them column-major (fromCOO), then fills the values with rng.nextDouble() in storage order.
// The sequential loop is restated in parallel: draw t is computed by jumping the 48-bit LCG to step 2t (power-of-two bounds
// consume exactly one step per nextInt), duplicates are found by sorting (key, t), the cut t* is the draw at which the
// number of first occurrences reaches nnz, and value e of the sorted list comes from LCG steps 2 (t* + 1) + 2 e + {1, 2}.
// One CTA per block; everything lives in shared memory (up to 16384 draws).
// ------------------------------------------------------------------------------------------------
constexpr int SPR_MAX_T = 16384;
constexpr uint64_t LCG_A = 0x5DEECE66Dull, LCG_C = 0xBull, LCG_MASK = (1ull << 48) - 1;
__device__ __forceinline__ uint64_t lcg_jump(uint64_t s, uint64_t n) {
  uint64_t a = LCG_A, c = LCG_C, A = 1, C = 0;
  while (n) {
    if (n & 1) {
      A = (A * a) & LCG_MASK;
      C = (C * a + c) & LCG_MASK;
    }
    c = (c * (a + 1)) & LCG_MASK;
    a = (a * a) & LCG_MASK;
    n >>= 1;
  }
  return (A * s + C) & LCG_MASK;
}

__global__ void __launch_bounds__(1024) sprand_kernel(const SprandDesc* __restrict__ descs) {
  extern __shared__ unsigned char spr_smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(spr_smem);        // [SPR_MAX_T] (key << 32) | t
  int32_t* cnt = reinterpret_cast<int32_t*>(spr_smem + SPR_MAX_T * 8);               // [SPR_MAX_T] flags / prefix sums
  int32_t* colcnt = cnt + SPR_MAX_T;                                                  // [cols + 1]
  __shared__ int32_t warp_tot[32];
  __shared__ int32_t s_tstar;
  const SprandDesc d = descs[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int T = d.draws;                       // power of two >= nnz + slack, <= SPR_MAX_T
  const int rbits = 31 - __clz(d.rows), cbits = 31 - __clz(d.cols);
  const uint64_t s0 = (static_cast<uint64_t>(d.seed) ^ LCG_A) & LCG_MASK;
  if (tid == 0) s_tstar = -1;
  for (int t = tid; t < T; t += blockDim.x) {
    const uint64_t s1 = lcg_jump(s0, 2ull * t + 1);
    const uint64_t s2 = (s1 * LCG_A + LCG_C) & LCG_MASK;
    const uint32_t i = static_cast<uint32_t>(s1 >> 17) >> (31 - rbits);   // nextInt(rows), rows = 2^rbits
    const uint32_t j = static_cast<uint32_t>(s2 >> 17) >> (31 - cbits);   // nextInt(cols)
    keys[t] = (static_cast<unsigned long long>(j * static_cast<uint32_t>(d.rows) + i) << 32) | static_cast<unsigned>(t);
  }
  for (int c = tid; c <= d.cols; c += blockDim.x) colcnt[c] = 0;
  __syncthreads();
  // bitonic sort of (key, t)
  for (int k = 2; k <= T; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < T; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          const bool up = (i & k) == 0;
          if ((a > b) == up) {
            keys[i] = b;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  // dup[t] = 1 when draw t repeats an earlier coordinate
  for (int e = tid; e < T; e += blockDim.x) {
    const bool first = e == 0 || (keys[e] >> 32) != (keys[e - 1] >> 32);
    cnt[static_cast<uint32_t>(keys[e])] = first ? 1 : 0;   // indexed by draw number t
  }
  __syncthreads();
  // inclusive scan over t of the first-occurrence flags; t* = first t whose count reaches nnz
  auto block_scan = [&](int32_t* a, int n) {  // in place, inclusive
    int carry = 0;
    for (int base = 0; base < n; base += blockDim.x) {
      const int i = base + tid;
      int x = i < n ? a[i] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) warp_tot[warp] = x;
      __syncthreads();
      if (warp == 0) {
        int w = warp_tot[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, w, o);
          if (lane >= o) w += y;
        }
        warp_tot[lane] = w;
      }
      __syncthreads();
      x += carry + (warp ? warp_tot[warp - 1] : 0);
      if (i < n) a[i] = x;
      const int tot = warp_tot[31];
      __syncthreads();
      carry += tot;
    }
  };
  block_scan(cnt, T);
  for (int t = tid; t < T; t += blockDim.x)
    if (cnt[t] == d.nnz && (t == 0 || cnt[t - 1] < d.nnz)) s_tstar = t;
  __syncthreads();
  if (s_tstar < 0) {  // not enough distinct coordinates among T draws (cannot happen with the slack the host adds)
    if (tid == 0) *d.status = 1;
    return;
  }
  const int tstar = s_tstar;
  __syncthreads();
  // selected = first occurrence with t <= t*, in sorted (column-major) order
  for (int e = tid; e < T; e += blockDim.x) {
    const bool first = e == 0 || (keys[e] >> 32) != (keys[e - 1] >> 32);
    cnt[e] = (first && static_cast<int>(static_cast<uint32_t>(keys[e])) <= tstar) ? 1 : 0;
  }
  __syncthreads();
  block_scan(cnt, T);
  const uint64_t sv = lcg_jump(s0, 2ull * (static_cast<uint64_t>(tstar) + 1));
  for (int e = tid; e < T; e += blockDim.x) {
    const int sel = cnt[e] - (e ? cnt[e - 1] : 0);
    if (sel) {
      const int pos = cnt[e] - 1;
      const uint32_t key = static_cast<uint32_t>(keys[e] >> 32);
      const uint32_t col = key / static_cast<uint32_t>(d.rows), row = key - col * static_cast<uint32_t>(d.rows);
      d.rowIndices[pos] = static_cast<int32_t>(row);
      atomicAdd(&colcnt[col + 1], 1);
      const uint64_t a1 = lcg_jump(sv, 2ull * pos + 1);
      const uint64_t a2 = (a1 * LCG_A + LCG_C) & LCG_MASK;
      d.values[pos] = static_cast<double>(((a1 >> 22) << 27) + (a2 >> 21)) * (1.0 / 9007199254740992.0);
    }
  }
  __syncthreads();
  block_scan(colcnt, d.cols + 1);
  for (int c = tid; c <= d.cols; c += blockDim.x) d.colPtrs[c] = colcnt[c];
}

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn spmm_encode_fn() {
  static EncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeFn>(p);
  }();
  return fn;
}

}  // namespace

size_t spmm2_aux_bytes(int m, int kdim, int64_t nnz, size_t* ent_off, size_t* rp_off, size_t* seg_off) {
  const int nstrips = (m + TM - 1) / TM, nchunks = (kdim + KC - 1) / KC, nseg = nstrips * nchunks;
  size_t off = 0;
  *ent_off = off;
  off += (static_cast<size_t>(nnz) * 16 + 255) / 256 * 256;
  *rp_off = off;
  off += (static_cast<size_t>(nseg) * RP_PAD * 4 + 255) / 256 * 256;
  *seg_off = off;
  off += (static_cast<size_t>(nseg + 1) * 4 + 255) / 256 * 256;
  return off;
}

// Row-major dense operand (kdim rows x n columns, line stride ld doubles): box {TN columns, KC rows}, no swizzle.
bool spmm2_encode_b_tmap(void* out128, const double* base, int64_t kdim, int64_t n, int64_t ld) {
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld & 1) != 0 || kdim <= 0 || n <= 0) return false;
  EncodeFn fn = spmm_encode_fn();
  if (!fn) return false;
  alignas(64) CUtensorMap m;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(n), static_cast<cuuint64_t>(kdim)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld) * 8};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(TN), static_cast<cuuint32_t>(KC)};
  const cuuint32_t estr[2] = {1, 1};
  if (fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return false;
  memcpy(out128, &m, 128);
  return true;
}

cudaError_t launch_spmm2_prep(const Spmm2Prep* d_preps, int nblocks, int max_m, int max_kdim, cudaStream_t stream) {
  if (nblocks <= 0) return cudaSuccess;
  const int nstrips = (max_m + TM - 1) / TM, nchunks = (max_kdim + KC - 1) / KC;
  const size_t smem = static_cast<size_t>(nstrips) * TM * nchunks * sizeof(int32_t);
  static PerDeviceOnce once;
  cudaError_t e = once.run([&] { return cudaFuncSetAttribute(spmm2_prep_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024); });
  if (e != cudaSuccess) return e;
  if (smem > 64 * 1024) return cudaErrorInvalidValue;
  spmm2_prep_kernel<false><<<nblocks, 1024, smem, stream>>>(d_preps);
  return cudaGetLastError();
}

size_t dspmm_aux_bytes(int n, int kdim, int64_t nnz, size_t* ent_off, size_t* rp_off, size_t* seg_off, size_t* kref_off) {
  size_t off = spmm2_aux_bytes(n, kdim, nnz, ent_off, rp_off, seg_off);
  const int nseg = ((n + TM - 1) / TM) * ((kdim + KC - 1) / KC);
  *kref_off = off;
  return off + (static_cast<size_t>(nseg) * KC + 255) / 256 * 256;
}

cudaError_t launch_dspmm_prep(const DspmmPrep* d_preps, int nblocks, int max_n, int max_kdim, cudaStream_t stream) {
  if (nblocks <= 0) return cudaSuccess;
  const int nstrips = (max_n + TM - 1) / TM, nchunks = (max_kdim + KC - 1) / KC;
  const size_t smem = static_cast<size_t>(nstrips) * nchunks * (TM + KW) * sizeof(int32_t);
  static PerDeviceOnce once;
  cudaError_t e = once.run([&] { return cudaFuncSetAttribute(spmm2_prep_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024); });
  if (e != cudaSuccess) return e;
  if (smem > 64 * 1024) return cudaErrorInvalidValue;
  spmm2_prep_kernel<true><<<nblocks, 1024, smem, stream>>>(d_preps);
  return cudaGetLastError();
}

cudaError_t launch_dspmm(const Spmm2Item* d_items, int nitems, const Spmm2Out* d_outs, const DspmmPair* d_pairs, cudaStream_t stream) {
  if (nitems <= 0) return cudaSuccess;
  static PerDeviceOnce once;
  cudaError_t e = once.run([&] { return cudaFuncSetAttribute(spmm2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES); });
  if (e != cudaSuccess) return e;
  spmm2_kernel<true><<<nitems, THREADS, SMEM_BYTES, stream>>>(d_items, d_outs, d_pairs, nullptr);
  return cudaGetLastError();
}

cudaError_t launch_ds_flags(const DsFlagDesc* d_descs, int ndescs, int max_m, cudaStream_t stream) {
  if (ndescs <= 0) return cudaSuccess;
  ds_flag_kernel<<<dim3(ndescs, (max_m + 255) / 256), 256, 0, stream>>>(d_descs);
  return cudaGetLastError();
}

cudaError_t launch_ds_fixup(const DsFixPair* d_pairs, int npairs, cudaStream_t stream) {
  if (npairs <= 0) return cudaSuccess;
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  ds_fixup_kernel<<<std::min(npairs, std::max(sms, 1) * 8), 256, 0, stream>>>(d_pairs, npairs);
  return cudaGetLastError();
}

int sprand_draws(int64_t nnz) {  // power-of-two number of draws with room for the expected duplicates; 0 = too many for one CTA
  const int64_t need = nnz + std::max<int64_t>(512, nnz / 8);
  int T = 1024;
  while (T < need) T <<= 1;
  return T <= SPR_MAX_T ? T : 0;
}

cudaError_t launch_sprand(const SprandDesc* d_descs, int nblocks, int max_cols, cudaStream_t stream) {
  if (nblocks <= 0) return cudaSuccess;
  const size_t smem = static_cast<size_t>(SPR_MAX_T) * 12 + static_cast<size_t>(max_cols + 1) * 4 + 16;
  static PerDeviceOnce once;
  constexpr int kSprandSmemMax = 216 * 1024;  // dynamic part; the kernel's static shared variables come on top of it
  cudaError_t e = once.run([&] { return cudaFuncSetAttribute(sprand_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSprandSmemMax); });
  if (e != cudaSuccess) return e;
  if (smem > static_cast<size_t>(kSprandSmemMax)) return cudaErrorInvalidValue;
  sprand_kernel<<<nblocks, 1024, smem, stream>>>(d_descs);
  return cudaGetLastError();
}

cudaError_t launch_spmm2(const Spmm2Item* d_items, int nitems, const Spmm2Out* d_outs, const Spmm2Pair* d_pairs, const void* d_tmaps,
                         cudaStream_t stream) {
  if (nitems <= 0) return cudaSuccess;
  static PerDeviceOnce once;
  cudaError_t e = once.run([&] { return cudaFuncSetAttribute(spmm2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES); });
  if (e != cudaSuccess) return e;
  spmm2_kernel<false><<<nitems, THREADS, SMEM_BYTES, stream>>>(d_items, d_outs, d_pairs, static_cast<const unsigned char*>(d_tmaps));
  return cudaGetLastError();
}

}  // namespace matrel
