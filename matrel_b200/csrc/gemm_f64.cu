// fp64 block-GEMM for sm_90a: C(i,j) = sum_k A(i,k) * B(k,j) over the present k-blocks.
//
// Replaces, in one kernel launch per matrixMultiply call:
//   - BLAS.gemmddd -> nativeBLAS.dgemm per block pair   (M/matrix/BLAS.scala:327-346)
//   - MLMatrix.multiply's fresh zeroed C per pair       (M/matrix/MLMatrix.scala:100-104)
//   - reduceByKey(LocalMatrix.add) over k               (M/execution/MatfastExecutionHelper.scala:255)
//
// Design (wgmma has no fp64 kind; the fp64 tensor pipe is reached through
// mma.sync.m8n8k4.f64 = SASS DMMA):
//   - warp-specialised CTA: 1 producer warp + NCW consumer warps, STAGES-deep shared-memory ring,
//     full/empty mbarriers per stage; consumers keep the whole K reduction (all k-blocks of the
//     block row/column) in registers.
//   - each operand tile (TILE x BK) is staged in one of two layouts, chosen per k-block from the
//     block's isTransposed flag, so "T"/"N" cost nothing and no block is ever re-materialised:
//        MODE_K  (global lines contiguous along k): ONE TMA tensor copy per stage
//                (cp.async.bulk.tensor.2d, SASS UTMALDG), box {BK, TILE}, SWIZZLE_128B.
//        MODE_MN (global lines contiguous along m/n): BK TMA bulk copies (cp.async.bulk, SASS UBLKCP)
//                of TILE*8 bytes into rows padded to TILE+4 doubles.
//   - bank-conflict-free DMMA fragment loads (one 8-byte LDS per lane) in both layouts: the four k of
//     MMA step s are {2s, 2s+1, 2s+8, 2s+9}.  Under the 128-byte swizzle the 4 rows x 4 k of a
//     half-warp then hit 16 distinct 8-byte slots; in MODE_MN the producer places k-row k at padded
//     row pi(k) = 4*((k&7)>>1) + 2*(k>>3) + (k&1), which makes the same k-set four consecutive rows.
//   - ragged tiles: the tensor copy zero-fills out-of-bounds elements itself; for MODE_MN the
//     producer zero-fills what the bulk copies do not cover; blocks with an odd leading dimension
//     (TMA needs 16-byte strides) fall back to guarded element loads into the same layouts.
#include <cuda.h>

#include <cstring>

#include "kernels.h"

namespace matrel {
namespace {

constexpr int BK = 16;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// TMA bulk (1-D) global -> shared copy, completion signalled on an mbarrier.
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// TMA tensor (2-D tiled) global -> shared copy through a CUtensorMap resident in global memory.
__device__ __forceinline__ void tma_tensor_2d_g2s(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
               "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// ---- shared-memory layouts -------------------------------------------------------------------------
__host__ __device__ constexpr int kpos_of_k(int k) { return 4 * ((k & 7) >> 1) + 2 * (k >> 3) + (k & 1); }  // pi(k)
__host__ __device__ constexpr int k_of_kpos(int p) { return 2 * (p >> 2) + (p & 1) + 8 * ((p >> 1) & 1); }  // pi^-1

template <int TILE>
struct OperandLayout {
  static constexpr int LDS_MN = TILE + 4;  // (TILE mod 16 == 0) -> (LDS_MN mod 16) == 4
  static constexpr int BYTES_MN = BK * LDS_MN * 8;
  static constexpr int BYTES_K = TILE * BK * 8;  // dense 128-byte rows, SWIZZLE_128B
  static constexpr int BYTES = ((BYTES_MN > BYTES_K ? BYTES_MN : BYTES_K) + 1023) / 1024 * 1024;  // 1024-B aligned slots
};
// MODE_K element (row, k) -> double index inside the operand slot (128-byte swizzle: 16-byte chunk ^= row & 7)
__device__ __forceinline__ int swz_k_index(int row, int k) { return row * BK + ((((k >> 1) ^ (row & 7)) << 1) | (k & 1)); }

// Producer, MODE_MN operand (global lines contiguous along m / n).  Two passes: issue == false does
// the generic-proxy stores (zero fill / guarded loads) and returns this lane's share of the bytes the
// bulk copies will deliver; issue == true issues the bulk copies.
template <int TILE>
__device__ __forceinline__ uint32_t produce_mn(const double* __restrict__ g, int ld, int mv, int kv, double* s,
                                               uint32_t bar, int lane, bool issue) {
  using L = OperandLayout<TILE>;
  const bool fast = ((reinterpret_cast<uintptr_t>(g) & 15) == 0) && ((ld & 1) == 0) && ((mv & 1) == 0);
  if (fast) {
    uint32_t bytes = 0;
    if (lane < kv) {  // kv <= BK = 16 <= 32 lanes: one k-row per lane
      bytes = static_cast<uint32_t>(mv) * 8u;
      if (issue) tma_bulk_g2s(smem_u32(s + kpos_of_k(lane) * L::LDS_MN), g + static_cast<size_t>(lane) * ld, bytes, bar);
    }
    if (!issue && (mv < TILE || kv < BK)) {
      for (int idx = lane; idx < TILE * BK; idx += 32) {
        const int p = idx / TILE, mn = idx % TILE;
        if (mn >= mv || k_of_kpos(p) >= kv) s[p * L::LDS_MN + mn] = 0.0;
      }
    }
    return bytes;
  }
  if (!issue) {
#pragma unroll 4
    for (int idx = lane; idx < TILE * BK; idx += 32) {
      const int p = idx / TILE, mn = idx % TILE;
      const int k = k_of_kpos(p);
      double v = 0.0;
      if (mn < mv && k < kv) v = __ldg(g + static_cast<size_t>(k) * ld + mn);
      s[p * L::LDS_MN + mn] = v;
    }
  }
  return 0;
}

// Producer, MODE_K operand (global lines contiguous along k).  With a tensor map: one TMA tensor copy
// of the whole {BK, TILE} box (out-of-bounds rows / k are zero-filled by the TMA unit and still count
// towards the transaction bytes).  Without (odd leading dimension): guarded loads, same swizzle.
template <int TILE>
__device__ __forceinline__ uint32_t produce_k(const double* __restrict__ g, int ld, int mv, int kv, const void* tmap,
                                              int c_k, int c_row, double* s, uint32_t bar, int lane, bool issue) {
  using L = OperandLayout<TILE>;
  if (tmap != nullptr) {
    if (lane == 0) {
      if (issue) tma_tensor_2d_g2s(smem_u32(s), tmap, c_k, c_row, bar);
      return static_cast<uint32_t>(L::BYTES_K);
    }
    return 0;
  }
  if (!issue) {
#pragma unroll 4
    for (int idx = lane; idx < TILE * BK; idx += 32) {
      const int row = idx / BK, k = idx % BK;
      double v = 0.0;
      if (row < mv && k < kv) v = __ldg(g + static_cast<size_t>(row) * ld + k);
      s[swz_k_index(row, k)] = v;
    }
  }
  return 0;
}

// Consumer: one BK-deep stage for a warp tile of (MI*8) x (NJ*8).  Lane (g = lane/4, t = lane%4) holds
// A[row g][k_t] and B[k_t][col g] with k_t = 2s + (t&1) + 8*(t>>1) in MMA step s.
template <int BM, int BN, int MI, int NJ, bool A_K, bool B_K>
__device__ __forceinline__ void consume_stage(const double* __restrict__ sA, const double* __restrict__ sB, int m_base,
                                              int n_base, int g, int t, double (&acc)[MI][NJ][2]) {
  constexpr int LDA = OperandLayout<BM>::LDS_MN;
  constexpr int LDB = OperandLayout<BN>::LDS_MN;
  const int b = t & 1, h = t >> 1;
  // MODE_MN: s[(4s + t) * LD + row]            -> base + s*4*LD + i*8
  // MODE_K : s[row*16 + (((s + 4h) ^ g) << 1) + b], row = base + i*8 + g (row & 7 == g)
  const double* pa = A_K ? (sA + (m_base + g) * BK + b) : (sA + t * LDA + m_base + g);
  const double* pb = B_K ? (sB + (n_base + g) * BK + b) : (sB + t * LDB + n_base + g);
#pragma unroll
  for (int ks = 0; ks < BK / 4; ++ks) {
    const int swz = ((ks | (h << 2)) ^ g) << 1;  // chunk index (in doubles) of this lane's k under the swizzle
    double a[MI], bb[NJ];
#pragma unroll
    for (int i = 0; i < MI; ++i) a[i] = A_K ? pa[i * 8 * BK + swz] : pa[ks * 4 * LDA + i * 8];
#pragma unroll
    for (int j = 0; j < NJ; ++j) bb[j] = B_K ? pb[j * 8 * BK + swz] : pb[ks * 4 * LDB + j * 8];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) dmma(acc[i][j][0], acc[i][j][1], a[i], bb[j]);
  }
}

template <int BM, int BN, int WM, int WN, int STAGES>
struct GemmCfg {
  static constexpr int NCW = WM * WN;             // consumer warps
  static constexpr int THREADS = (NCW + 1) * 32;  // + 1 producer warp
  static constexpr int MI = BM / WM / 8;
  static constexpr int NJ = BN / WN / 8;
  static constexpr int A_BYTES = OperandLayout<BM>::BYTES;
  static constexpr int B_BYTES = OperandLayout<BN>::BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr size_t SMEM_BYTES = 1024 /* alignment slack */ + static_cast<size_t>(STAGES) * STAGE_BYTES + 2 * STAGES * 8;
};

template <int BM, int BN, int WM, int WN, int STAGES>
__global__ void __launch_bounds__(GemmCfg<BM, BN, WM, WN, STAGES>::THREADS, 1)
    gemm_f64_dmma_kernel(const GemmOut* __restrict__ outs, const GemmPair* __restrict__ pairs,
                         const GemmTile* __restrict__ tiles, const unsigned char* __restrict__ tmaps,
                         const int* __restrict__ run_if) {
  using Cfg = GemmCfg<BM, BN, WM, WN, STAGES>;
  extern __shared__ unsigned char smem_dyn[];
  if (run_if != nullptr && *run_if == 0) return;  // fallback launch behind an Ozaki-II job that did not need it
  // SWIZZLE_128B destinations must be 1024-byte aligned
  unsigned char* smem_raw = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + static_cast<size_t>(STAGES) * Cfg::STAGE_BYTES);
  // bars[0..STAGES) = full, bars[STAGES..2*STAGES) = empty

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const GemmTile tile = tiles[blockIdx.x];
  const GemmOut out = outs[tile.out];
  const int m0 = tile.tm * BM, n0 = tile.tn * BN;
  const int mv = min(BM, out.m - m0), nv = min(BN, out.n - n0);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bars[s]), 1);
      mbar_init(smem_u32(&bars[STAGES + s]), Cfg::NCW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == Cfg::NCW) {
    // ===================== producer warp =====================
    int it = 0;
    for (int p = 0; p < out.pair_count; ++p) {
      const GemmPair pr = pairs[out.pair_begin + p];
      const bool a_k = pr.aT != 0;  // row-major A block: lines contiguous along k
      const bool b_k = pr.bT == 0;  // column-major B block: lines contiguous along k
      const void* tmA = (a_k && pr.tmA >= 0) ? tmaps + static_cast<size_t>(pr.tmA) * 128 : nullptr;
      const void* tmB = (b_k && pr.tmB >= 0) ? tmaps + static_cast<size_t>(pr.tmB) * 128 : nullptr;
      for (int k0 = 0; k0 < pr.kdim; k0 += BK, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        const int kv = min(BK, pr.kdim - k0);
        mbar_wait(smem_u32(&bars[STAGES + s]), ph ^ 1);
        double* sA = reinterpret_cast<double*>(smem_raw + static_cast<size_t>(s) * Cfg::STAGE_BYTES);
        double* sB = reinterpret_cast<double*>(smem_raw + static_cast<size_t>(s) * Cfg::STAGE_BYTES + Cfg::A_BYTES);
        const double* gA = a_k ? pr.A + static_cast<size_t>(m0) * pr.lda + k0 : pr.A + static_cast<size_t>(k0) * pr.lda + m0;
        const double* gB = b_k ? pr.B + static_cast<size_t>(n0) * pr.ldb + k0 : pr.B + static_cast<size_t>(k0) * pr.ldb + n0;
        const uint32_t full = smem_u32(&bars[s]);
        uint32_t bytes = 0;
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
          const bool issue = pass == 1;
          uint32_t nb = a_k ? produce_k<BM>(gA, pr.lda, mv, kv, tmA, k0, m0, sA, full, lane, issue)
                            : produce_mn<BM>(gA, pr.lda, mv, kv, sA, full, lane, issue);
          nb += b_k ? produce_k<BN>(gB, pr.ldb, nv, kv, tmB, k0, n0, sB, full, lane, issue)
                    : produce_mn<BN>(gB, pr.ldb, nv, kv, sB, full, lane, issue);
          if (!issue) {
            bytes = nb;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
            __syncwarp();
            if (lane == 0) mbar_arrive_expect_tx(full, bytes);
            __syncwarp();
          }
        }
      }
    }
  } else {
    // ===================== consumer warps =====================
    const int wm = warp / WN, wn = warp % WN;
    const int g = lane >> 2, t = lane & 3;
    const int m_base = wm * (Cfg::MI * 8), n_base = wn * (Cfg::NJ * 8);
    double acc[Cfg::MI][Cfg::NJ][2];
#pragma unroll
    for (int i = 0; i < Cfg::MI; ++i)
#pragma unroll
      for (int j = 0; j < Cfg::NJ; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    int it = 0;
    for (int p = 0; p < out.pair_count; ++p) {
      const GemmPair pr = pairs[out.pair_begin + p];
      const bool a_k = pr.aT != 0;
      const bool b_k = pr.bT == 0;
      const int nchunks = (pr.kdim + BK - 1) / BK;
      for (int c = 0; c < nchunks; ++c, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        const double* sA = reinterpret_cast<const double*>(smem_raw + static_cast<size_t>(s) * Cfg::STAGE_BYTES);
        const double* sB = reinterpret_cast<const double*>(smem_raw + static_cast<size_t>(s) * Cfg::STAGE_BYTES + Cfg::A_BYTES);
        mbar_wait(smem_u32(&bars[s]), ph);
        if (a_k) {
          if (b_k) consume_stage<BM, BN, Cfg::MI, Cfg::NJ, true, true>(sA, sB, m_base, n_base, g, t, acc);
          else     consume_stage<BM, BN, Cfg::MI, Cfg::NJ, true, false>(sA, sB, m_base, n_base, g, t, acc);
        } else {
          if (b_k) consume_stage<BM, BN, Cfg::MI, Cfg::NJ, false, true>(sA, sB, m_base, n_base, g, t, acc);
          else     consume_stage<BM, BN, Cfg::MI, Cfg::NJ, false, false>(sA, sB, m_base, n_base, g, t, acc);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bars[STAGES + s]));
      }
    }

    // epilogue: C is column-major (ldc = out.m); lane holds rows g, columns 2t, 2t+1 of each 8x8
    double* C = out.C;
    const size_t ldc = static_cast<size_t>(out.m);
#pragma unroll
    for (int i = 0; i < Cfg::MI; ++i) {
      const int row = m0 + m_base + i * 8 + g;
      if (row < out.m) {
#pragma unroll
        for (int j = 0; j < Cfg::NJ; ++j) {
          const int col = n0 + n_base + j * 8 + 2 * t;
          if (col < out.n) C[row + ldc * col] = acc[i][j][0];
          if (col + 1 < out.n) C[row + ldc * (col + 1)] = acc[i][j][1];
        }
      }
    }
  }
}

template <int BM, int BN, int WM, int WN, int STAGES>
cudaError_t launch_variant(const GemmOut* d_outs, const GemmPair* d_pairs, const GemmTile* d_tiles, int ntiles,
                           const void* d_tmaps, cudaStream_t stream, const int* run_if) {
  using Cfg = GemmCfg<BM, BN, WM, WN, STAGES>;
  auto kern = gemm_f64_dmma_kernel<BM, BN, WM, WN, STAGES>;
  static PerDeviceOnce configured;
  cudaError_t e = configured.run(
      [&] { return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(Cfg::SMEM_BYTES)); });
  if (e != cudaSuccess) return e;
  kern<<<ntiles, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(d_outs, d_pairs, d_tiles, static_cast<const unsigned char*>(d_tmaps), run_if);
  return cudaGetLastError();
}

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode_fn() {
  static EncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeFn>(p);
  }();
  return fn;
}

}  // namespace

int gemm_tile_m(int variant) { return variant == GEMM_64x64 ? 64 : 128; }
int gemm_tile_n(int variant) { return variant == GEMM_64x64 ? 64 : 128; }

bool encode_kcontig_tmap(void* out128, const double* base, int64_t kdim, int64_t rows, int64_t ld, int tile_rows) {
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld & 1) != 0 || kdim <= 0 || rows <= 0) return false;
  EncodeFn fn = get_encode_fn();
  if (!fn) return false;
  static_assert(sizeof(CUtensorMap) == 128, "CUtensorMap is 128 bytes");
  alignas(64) CUtensorMap m;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(kdim), static_cast<cuuint64_t>(rows)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld) * 8};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>(tile_rows)};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double*>(base), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  memcpy(out128, &m, 128);
  return true;
}

cudaError_t launch_gemm_f64(const GemmOut* d_outs, const GemmPair* d_pairs, const GemmTile* d_tiles, int ntiles,
                            const void* d_tmaps, int variant, cudaStream_t stream, const int* run_if) {
  if (ntiles <= 0) return cudaSuccess;
  if (variant == GEMM_64x64) return launch_variant<64, 64, 2, 2, 4>(d_outs, d_pairs, d_tiles, ntiles, d_tmaps, stream, run_if);
  return launch_variant<128, 128, 2, 4, 5>(d_outs, d_pairs, d_tiles, ntiles, d_tmaps, stream, run_if);
}

}  // namespace matrel
