// fp64 block-GEMM on the Hopper tensor cores (wgmma, s8 x s8 -> s32) through Ozaki splitting.
//
// wgmma has no fp64 kind, so the north-star's "block multiply as tensor-core tiles" is only reachable for
// fp64 data by error-free integer slicing (Ozaki scheme I, the technique behind vendor "fp64 emulation"):
//   a_ik = 2^(e_i+2) * sum_{s=1..S} A_s[i,k] * 2^(-8s)      A_s in [-128,127]  (balanced base-256 digits, |a_ik| < 2^e_i)
//   b_kj = 2^(f_j+2) * sum_{t=1..S} B_t[k,j] * 2^(-8t)
//   c_ij ~= sum_{d=2..S+1} 2^(e_i+f_j+4-8d) * sum_{s+t=d} (A_s B_t)_ij     (products with s+t > S+1 dropped)
// e_i / f_j = exponent of the largest |a| in row i of A / column j of B (over ALL k-blocks), every slice
// product is an exact s32 GEMM on the tensor cores (|digit product| <= 2^14, K*|pairs| <= 2^17 per
// accumulator), and the only roundings are the final digit (2^-(8S-2) relative to the row/column maximum)
// and S fp64 additions per element.  S = 7 gives errors at the level of fp64 dgemm's own rounding for
// data of moderate dynamic range per row/column; the exact DMMA kernel (gemm_f64.cu) stays the default.
//
// Pipeline per multiply (replaces the same reference code as gemm_f64.cu: BLAS.scala:327-346,
// MLMatrix.scala:100-104, MatfastExecutionHelper.scala:255):
//   1. absmax pass over the blocks of A (per global row) and B (per global column)      -- HBM-bound
//   2. slice pass: S int8 matrices A_s [M x K] and B_t^T [N x K], K contiguous            -- HBM-bound
//   3. for each diagonal d: ONE GEMM launch: TMA (SWIZZLE_128B tensor maps) -> 4-stage smem ring ->
//      wgmma m64n256k32 s8 (two consumer warpgroups, 64 x 256 s32 accumulator in registers each) over all (s, d-s)
//      pairs and all k -> register epilogue: scale by 2^(e_i+f_j+4-8d) and accumulate into the fp64 output blocks.
#include <cuda.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <mutex>
#include <type_traits>
#include <vector>

#include "kernels.h"

namespace matrel {
namespace {

constexpr int BM = 128, BN = 256, BKB = 128 /* bytes (= int8 elements) of K per stage */, WGMMA_KB = 32 /* bytes of K per wgmma */, STAGES = 4;
constexpr int A_BYTES = BM * BKB, B_BYTES = BN * BKB, STAGE_BYTES = A_BYTES + B_BYTES;

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
__device__ __forceinline__ void tma_2d(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
               "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
               : "memory");
}
// wgmma shared-memory descriptor, K-major operand tile, SWIZZLE_128B: rows of 128 B, 8-row groups 1024 B apart
// (start >> 4 @ [0,14), LBO = 1 @ [16,30) (unused by swizzled K-major tiles), SBO = 1024 >> 4 @ [32,46), SWIZZLE_128B = 1 @ [62,64))
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t saddr) {
  return static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
#define WG_OPS16(c, a, o)                                                                                                          \
  c(a[o]), c(a[o + 1]), c(a[o + 2]), c(a[o + 3]), c(a[o + 4]), c(a[o + 5]), c(a[o + 6]), c(a[o + 7]), c(a[o + 8]), c(a[o + 9]),    \
      c(a[o + 10]), c(a[o + 11]), c(a[o + 12]), c(a[o + 13]), c(a[o + 14]), c(a[o + 15])
#define WG_OPS128(c, a)                                                                                                            \
  WG_OPS16(c, a, 0), WG_OPS16(c, a, 16), WG_OPS16(c, a, 32), WG_OPS16(c, a, 48), WG_OPS16(c, a, 64), WG_OPS16(c, a, 80),           \
      WG_OPS16(c, a, 96), WG_OPS16(c, a, 112)
#define WG_D128                                                                                                                    \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "     \
  "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, " \
  "%51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, " \
  "%76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, " \
  "%101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, "       \
  "%121, %122, %123, %124, %125, %126, %127}"
// D (64 x 256, this warpgroup's registers) (+)= A (64 x 32 bytes of K) * B (256 x 32 bytes of K), both from shared memory
__device__ __forceinline__ void wgmma_tile(int32_t (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 " WG_D128
               ", %128, %129, p;\n\t}"
               : WG_OPS128("+r", d)
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tile(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 " WG_D128
               ", %128, %129, p, 1, 1;\n\t}"
               : WG_OPS128("+f", d)
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

struct OzakiGemmParams {
  const unsigned char* tmaps;  // 2*S CUtensorMaps (128 B each): A_1..A_S then B_1..B_S
  const double* row_scale;     // 2^e_i per global row of A      (|a_ik| < 2^e_i)
  const double* col_scale;     // 2^f_j per global column of B   (|b_kj| < 2^f_j)
  double* const* ctab;         // [nbr * nbc] output block pointers (nullptr = block absent)
  int32_t M, N, Kpad;          // logical output dims, padded K (multiple of 128)
  int32_t blk, nbr, nbc;       // block size and block-grid extent of C
  int32_t S, d;                // slices, diagonal of this launch (pairs (s, d - s))
  int32_t accumulate;          // 0: C = term, 1: C += term
  int32_t tiles_m, tiles_n;    // tile grid (128 x 256 tiles)
  double diag_scale;           // 2^(4 - 8 d)
  // generalisation used by the fp32 path (tf32x3): explicit (A slice, B slice) tensor-map index pairs and the K extent of
  // one 128-byte stage row in elements (the accumulator type is the kernel's template parameter)
  int32_t npairs;
  int32_t pair_a[8], pair_b[8];
  int32_t kstep;               // elements of K per stage (128 int8 / 32 tf32)
  int32_t kc0, nkc;            // K range of this launch in stage units (the fp32 path re-accumulates K chunks in fp64)
  // CRT mode (Ozaki scheme II, gemm_algo 4): nmod > 0 makes ONE launch walk nmod x tiles work items; item (t, tile) multiplies
  // residue matrices A mod p_t (tensor map t) and B mod p_t (tensor map nmod + t) and stores (A_t B_t) mod p_t as int8.
  int32_t nmod;
  int32_t npad;                // row pitch of the residue planes (bytes)
  int8_t* planes;              // [nmod][Mpad][npad]
  size_t plane_stride;
  int32_t mod_p[16];
  double mod_inv[16];          // 1 / p_t
  // job mode (Ozaki-II engine): the tiles of this launch come from a list (any subset of the buffer's tile grid), the residue
  // planes are compact ([modulus][list index][128 x 256] bytes), and the whole launch is skipped when *gate != 0
  const int2* tile_list;       // (tm, tn) per tile, nullptr = the full tiles_m x tiles_n grid
  int32_t ntiles_list;
  const int* gate;
};

// warpgroup 0: TMA producer (one elected thread); warpgroups 1, 2: wgmma consumers, 64 of the tile's 128 rows each, and epilogue
constexpr int CONSUMER_WARPS = 8;
constexpr int GEMM_THREADS_P = 128 + CONSUMER_WARPS * 32;
constexpr size_t GEMM_SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 2 * STAGES * 8;  // alignment slack, ring, full[] + empty[] barriers
constexpr int TILE_BAND = 8;                       // n-tiles per rasterisation band (L2 reuse of A / B panels)

// 384 threads x 168 registers fill the register file: the producer warpgroup hands its share to the two accumulator holders
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int& tm, int& tn) {
  const int band_tiles = TILE_BAND * tiles_m;
  const int band = t / band_tiles;
  const int rem = t - band * band_tiles;
  const int bw = min(TILE_BAND, tiles_n - band * TILE_BAND);
  tm = rem / bw;
  tn = band * TILE_BAND + rem % bw;
}

// The wgmma accumulator fragment: thread (warp wq of the warpgroup, lane) holds, for every 8-column group j = 0..31,
// acc[4 j + e] = element (16 wq + lane / 4 + 8 (e >> 1), 8 j + 2 (lane % 4) + (e & 1)) of the warpgroup's 64 x 256 tile.

// K loop of one work item in a consumer warpgroup: `steps` ring stages accumulate into acc (the first overwrites it).  One
// stage's wgmmas stay in flight while the next stage is awaited; every warp hands a stage back once its wgmmas have retired.
template <class Acc, class Release>
__device__ __forceinline__ void consume_item(Acc (&acc)[128], unsigned char* smem, uint64_t* bars, int a_off, int steps, int& it, int lane,
                                             Release&& release) {
  wgmma_fence();
  for (int j = 0; j < steps; ++j, ++it) {
    const int st = it % STAGES;
    mbar_wait(smem_u32(&bars[st]), (it / STAGES) & 1);
    const uint32_t a0 = smem_u32(smem + st * STAGE_BYTES) + a_off, b0 = smem_u32(smem + st * STAGE_BYTES) + A_BYTES;
#pragma unroll
    for (int k = 0; k < BKB / WGMMA_KB; ++k)  // 4 wgmmas of 32 bytes of K each (32 int8 / 8 tf32)
      wgmma_tile(acc, wgmma_desc_k_sw128(a0 + k * WGMMA_KB), wgmma_desc_k_sw128(b0 + k * WGMMA_KB), (j | k) != 0);
    wgmma_commit();
    if (j > 0) {
      wgmma_wait<1>();
      if (lane == 0) release((it - 1) % STAGES);
    }
  }
  wgmma_wait<0>();
  if (lane == 0) release((it - 1) % STAGES);
}

// Residues of a warpgroup's exact s32 accumulator into the compact plane of its tile ([128 rows][256 columns] bytes).
// q = rint(c / p) is exact in fp64 (no integer c / p lies within 1/(2p) of a tie except the true ties of the even modulus 256,
// where either neighbour is a valid representative).  ADD: the residue byte this SAME thread stored for the lower K half joins
// the sum before the reduction: ((x mod p) + y) mod p = (x + y) mod p; |y| <= K/2 * 2^14 and x < 256 keep the sum inside int32.
template <bool ADD>
__device__ __forceinline__ void store_residues(const int32_t (&acc)[128], int8_t* tile, int row, int lane, int pm, double pinv) {
  int8_t* dst = tile + static_cast<size_t>(row) * BN + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint16_t* d2 = reinterpret_cast<uint16_t*>(dst + h * 8 * BN + 8 * j);
      const uint32_t prev = ADD ? *d2 : 0u;
      uint32_t wv = 0;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        int v = acc[4 * j + 2 * h + e];
        if (ADD) v += static_cast<int>((prev >> (8 * e)) & 0xffu);
        int res = v - __double2int_rn(static_cast<double>(v) * pinv) * pm;  // [-p/2, p/2]
        res += (res >> 31) & pm;                                          // [0, p): the CRT kernel reads unsigned bytes
        wv |= static_cast<uint32_t>(res) << (8 * e);
      }
      *d2 = static_cast<uint16_t>(wv);
    }
  }
}

// Persistent, warp-specialised: one CTA per SM loops over the output tiles of this launch.  F32 = false: s8 operands, exact s32
// accumulator (Ozaki slices or CRT residues); F32 = true: tf32 operands, fp32 accumulator written as is (tf32x3_gemm).
template <bool F32>
__global__ void __launch_bounds__(GEMM_THREADS_P, 1) ozaki_gemm_i8_kernel(const OzakiGemmParams p) {
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);  // full[STAGES], empty[STAGES]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (p.gate != nullptr && *p.gate != 0) return;  // uniform: non-finite / out-of-range operands take the exact DMMA kernel
  const int nk = p.nkc;
  const int per_tile = p.npairs * nk;
  const int ntiles = p.tile_list ? p.ntiles_list : p.tiles_m * p.tiles_n;
  const int nitems = ntiles * (p.nmod ? p.nmod : 1);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bars[s]), 1);                        // full: the producer's arrive.expect_tx
      mbar_init(smem_u32(&bars[STAGES + s]), CONSUMER_WARPS);  // empty: one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    producer_regs();
    // ===== TMA producer (one elected lane) =====
    if (warp == 0 && lane == 0) {
      int it = 0;
      for (int w = blockIdx.x; w < nitems; w += gridDim.x) {
        const int mi = w / ntiles, t = w - mi * ntiles;
        int tm, tn;
        if (p.tile_list) {
          const int2 tl = p.tile_list[t];
          tm = tl.x;
          tn = tl.y;
        } else {
          tile_coords(t, p.tiles_m, p.tiles_n, tm, tn);
        }
        const int m0 = tm * BM, n0 = tn * BN;
        for (int s = 0; s < p.npairs; ++s) {
          const void* tmA = p.tmaps + static_cast<size_t>(p.nmod ? mi : p.pair_a[s]) * 128;
          const void* tmB = p.tmaps + static_cast<size_t>(p.nmod ? p.nmod + mi : p.pair_b[s]) * 128;
          for (int kc = p.kc0; kc < p.kc0 + nk; ++kc, ++it) {
            const int st = it % STAGES;
            const uint32_t ph = (it / STAGES) & 1;
            mbar_wait(smem_u32(&bars[STAGES + st]), ph ^ 1);
            const uint32_t full = smem_u32(&bars[st]);
            mbar_arrive_expect_tx(full, STAGE_BYTES);
            tma_2d(smem_u32(smem + st * STAGE_BYTES), tmA, kc * p.kstep, m0, full);
            tma_2d(smem_u32(smem + st * STAGE_BYTES + A_BYTES), tmB, kc * p.kstep, n0, full);
          }
        }
      }
    }
  } else {
    consumer_regs();
    // ===== consumers: every (s, d-s) pair and every k accumulates into one register tile, then the epilogue =====
    const int cw = (warp - 4) >> 2, wq = warp & 3;  // consumer warpgroup, warp within it
    const int trow = 64 * cw + 16 * wq + (lane >> 2);  // first of this thread's two tile rows (the other is trow + 8)
    typename std::conditional<F32, float, int32_t>::type acc[128];
    int it = 0;
    for (int w = blockIdx.x; w < nitems; w += gridDim.x) {
      const int mi = w / ntiles, t = w - mi * ntiles;
      int tm, tn;
      if (p.tile_list) {
        const int2 tl = p.tile_list[t];
        tm = tl.x;
        tn = tl.y;
      } else {
        tile_coords(t, p.tiles_m, p.tiles_n, tm, tn);
      }
      consume_item(acc, smem, bars, cw * 64 * BKB, per_tile, it, lane, [&](int st) { mbar_arrive(smem_u32(&bars[STAGES + st])); });
      if constexpr (!F32) {
        if (p.nmod) {
          // compact planes: [modulus][tile of this launch][128 rows][256 columns], always whole tiles (no guards)
          store_residues<false>(acc, p.planes + static_cast<size_t>(mi) * p.plane_stride + static_cast<size_t>(t) * (BM * BN), trow, lane,
                                p.mod_p[mi], p.mod_inv[mi]);
          continue;
        }
      }
      // scale by 2^(e_i + f_j + 4 - 8d) (s32) or take as is (fp32) -> (+)= column-major fp64 output blocks
      // fp32 path: the fp64 mean corrections go in with the first K chunk (see slice_tf32_kernel)
      const bool f32_corr = F32 && !p.accumulate && p.row_scale != nullptr;
      bool row_ok[2];
      int rid[2], lr[2], brows[2];
      double rs[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = tm * BM + trow + 8 * h;
        row_ok[h] = row < p.M;
        rid[h] = row_ok[h] ? row / p.blk : 0;
        lr[h] = row - rid[h] * p.blk;
        brows[h] = min(p.blk, p.M - rid[h] * p.blk);
        rs[h] = !row_ok[h] ? 0.0 : (F32 ? (f32_corr ? p.row_scale[row] : 0.0) : p.row_scale[row] * p.diag_scale);
      }
      const int col0 = tn * BN + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int h = e >> 1, col = col0 + 8 * j + (e & 1);
          if (row_ok[h] && col < p.N) {
            const int cid = col / p.blk;
            double* blkp = p.ctab[rid[h] * p.nbc + cid];
            if (blkp != nullptr) {
              double* dst = blkp + lr[h] + static_cast<size_t>(brows[h]) * (col - cid * p.blk);
              double term;
              if constexpr (F32) term = static_cast<double>(acc[4 * j + e]) + (f32_corr ? rs[h] + __ldg(p.col_scale + col) : 0.0);
              else term = (static_cast<double>(acc[4 * j + e]) * rs[h]) * __ldg(p.col_scale + col);
              *dst = p.accumulate ? *dst + term : term;
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// The same residue GEMM on CTA PAIRS: a cluster of two CTAs computes a 256 x 256 tile, each CTA its own 128 rows.  Both need the
// same 256 columns (rows of the K-major B'), so each CTA fetches only HALF of them and multicasts that half into the shared
// memory of both (TMA .multicast::cluster): per stage a CTA requests 16 KB of A' and 16 KB of B' from L2 instead of 16 + 32,
// which is what the persistent kernel runs short of once the CTAs in flight have drifted apart in k.  Roles per CTA as in the
// single-CTA kernel; a stage is free for the pair's producers once the consumer warps of BOTH CTAs have released it, so the empty
// barriers count the arrivals of the whole pair.  Only used by the Ozaki-II engine: work item = (modulus, pair of vertically
// adjacent 128-row tiles); the tile list holds the two halves at positions 2 t and 2 t + 1.
// ------------------------------------------------------------------------------------------------
constexpr int B2_BYTES = (BN / 2) * BKB;

__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// the box lands at the same shared-memory offset, and completes the barrier at the same offset, in every CTA of the mask
__device__ __forceinline__ void tma_2d_multicast(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar, uint16_t cta_mask) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
               ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask)
               : "memory");
}

// The work items of ONE CTA pair in execution order; the producers and the consumer warps of both CTAs walk identical copies.
//   KSPLIT = false: item = (modulus, tile pair), flat index w = cl, cl + ncl, ... over nmod x npairs, the whole K per item.
//   KSPLIT = true : item = (modulus, K half, tile pair).  The pair that owns tile pair t2 of modulus mi runs BOTH halves (first
//                   the lower half of all its tiles of the modulus, then the upper half), so the thread that stored a residue byte
//                   of the lower half is the one that adds the upper half to it -- no cross-CTA ordering is needed.  The CTA pairs
//                   in flight then share panels of K / 2 residue bytes: half the L2 footprint of the unsplit order, which is what
//                   decides whether the panels survive in L2 once the pairs have drifted apart in k.  The leftover tile pairs of
//                   a sweep (npairs % ncl) rotate over the CTA pairs from one modulus to the next, so the load stays balanced
//                   over the launch.
template <bool KSPLIT>
struct Oz2Items {
  int npairs, ncl, cl, nmod, nk, rot, w, cur_mi, cur_kh, cur_t2;
  __device__ __forceinline__ int first_of(int mi) const { return (cl + ncl - (mi * rot) % ncl) % ncl; }
  __device__ __forceinline__ Oz2Items(int npairs_, int ncl_, int cl_, int nmod_, int nk_)
      : npairs(npairs_), ncl(ncl_), cl(cl_), nmod(nmod_), nk(nk_), rot(npairs_ % ncl_), w(cl_), cur_mi(0), cur_kh(0), cur_t2(0) {
    cur_t2 = first_of(0);
  }
  // next item: modulus mi, tile pair t2, k-chunks [kc0, kc0 + kcn), add = the epilogue adds the residue byte already stored
  __device__ __forceinline__ bool next(int& mi, int& t2, int& kc0, int& kcn, bool& add) {
    if constexpr (!KSPLIT) {
      if (w >= npairs * nmod) return false;
      mi = w / npairs;
      t2 = w - mi * npairs;
      kc0 = 0;
      kcn = nk;
      add = false;
      w += ncl;
      return true;
    } else {
      while (cur_mi < nmod) {
        if (cur_t2 < npairs) {
          mi = cur_mi;
          t2 = cur_t2;
          kcn = nk >> 1;
          kc0 = cur_kh * kcn;
          add = cur_kh != 0;
          cur_t2 += ncl;
          return true;
        }
        if (cur_kh == 0) {
          cur_kh = 1;
        } else {
          cur_kh = 0;
          ++cur_mi;
        }
        cur_t2 = first_of(cur_mi);
      }
      return false;
    }
  }
};

template <bool KSPLIT>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(GEMM_THREADS_P, 1) ozaki2_gemm_2sm_kernel(const OzakiGemmParams p) {
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);  // full[STAGES], empty[STAGES], per CTA
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t cta_rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(cta_rank));
  const bool gated = p.gate != nullptr && *p.gate != 0;  // uniform over the grid: both CTAs of a pair take the same path
  const int nk = p.nkc;
  const int npairs_list = p.ntiles_list >> 1;             // pairs of 128-row tiles
  const int nmod_run = gated ? 0 : p.nmod;
  const int ncl = gridDim.x >> 1, cl = blockIdx.x >> 1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bars[s]), 1);                            // full: own producer's arrive.expect_tx (A' + both halves of B')
      mbar_init(smem_u32(&bars[STAGES + s]), 2 * CONSUMER_WARPS);  // empty: every consumer warp of the pair
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");

  if (warp < 4) {
    producer_regs();
    // ===== TMA producer: this CTA's 128 rows of A', and 128 of the tile's 256 rows of B' for both CTAs =====
    if (warp == 0 && lane == 0) {
      int it = 0;
      Oz2Items<KSPLIT> items(npairs_list, ncl, cl, nmod_run, nk);
      int mi, t2, kc0, kcn;
      bool add;
      while (items.next(mi, t2, kc0, kcn, add)) {
        const int2 tl = p.tile_list[2 * t2 + static_cast<int>(cta_rank)];
        const int m0 = tl.x * BM, n0 = tl.y * BN + static_cast<int>(cta_rank) * (BN / 2);
        const void* tmA = p.tmaps + static_cast<size_t>(mi) * 128;
        const void* tmB = p.tmaps + static_cast<size_t>(2 * p.nmod + mi) * 128;  // the {128, 128}-box maps of B'
        for (int kc = kc0; kc < kc0 + kcn; ++kc, ++it) {
          const int st = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(smem_u32(&bars[STAGES + st]), ph ^ 1);  // released by both CTAs: the peer's copy of the stage is written too
          const uint32_t full = smem_u32(&bars[st]);
          mbar_arrive_expect_tx(full, STAGE_BYTES);
          tma_2d(smem_u32(smem + st * STAGE_BYTES), tmA, kc * BKB, m0, full);
          tma_2d_multicast(smem_u32(smem + st * STAGE_BYTES + A_BYTES) + cta_rank * B2_BYTES, tmB, kc * BKB, n0, full, 3);
        }
      }
    }
  } else {
    consumer_regs();
    // ===== consumers: own 128 rows x the pair's 256 columns -> residues -> compact plane of this CTA's tile =====
    const int cw = (warp - 4) >> 2, wq = warp & 3;
    const int trow = 64 * cw + 16 * wq + (lane >> 2);
    const uint32_t empty0 = mapa_u32(smem_u32(&bars[STAGES]), 0), empty1 = mapa_u32(smem_u32(&bars[STAGES]), 1);
    int32_t acc[128];
    int it = 0;
    Oz2Items<KSPLIT> items(npairs_list, ncl, cl, nmod_run, nk);
    int mi, t2, kc0, kcn;
    bool add;
    while (items.next(mi, t2, kc0, kcn, add)) {
      const int t = 2 * t2 + static_cast<int>(cta_rank);
      consume_item(acc, smem, bars, cw * 64 * BKB, kcn, it, lane, [&](int st) {
        mbar_arrive_cluster(empty0 + 8u * static_cast<uint32_t>(st));
        mbar_arrive_cluster(empty1 + 8u * static_cast<uint32_t>(st));
      });
      int8_t* tile = p.planes + static_cast<size_t>(mi) * p.plane_stride + static_cast<size_t>(t) * (BM * BN);
      if (KSPLIT && add) store_residues<true>(acc, tile, trow, lane, p.mod_p[mi], p.mod_inv[mi]);
      else store_residues<false>(acc, tile, trow, lane, p.mod_p[mi], p.mod_inv[mi]);
    }
  }
  __syncthreads();
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");  // nobody leaves while the peer may still signal / write
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- pass 1: per-row / per-column maximum magnitude (as the IEEE bit pattern, which orders like the value) -------
struct OzBlock {
  const double* v;
  int32_t rows, cols;  // logical dims of the block
  int32_t row0, col0;  // global offsets of its (0,0) element in the operand matrix
  uint8_t isT;
  uint8_t pad[7];
};

__device__ __forceinline__ double blk_at(const OzBlock& b, int r, int c) {
  return b.isT ? b.v[c + static_cast<size_t>(b.cols) * r] : b.v[r + static_cast<size_t>(b.rows) * c];
}

// by_row = true: out[row0 + r] = max_c |b(r,c)|; false: out[col0 + c] = max_r |b(r,c)|.  One CTA sweeps a tile of AM_FAST
// elements along the block's contiguous index (rows of a column-major block, columns of a row-major one) x AM_SLOW along the
// strided one: a warp reads eight 256-byte runs per strided index, so 8 x 8 independent loads are in flight per thread.
// minout (optional): the smallest NON-ZERO magnitude of the same line (initialised to all-ones by the caller); the Ozaki-II
// auto-selection uses it to bound the dynamic range inside a row / column.  grid.x = fast tiles x tiles_s_max.
constexpr int AM_FAST = 256, AM_SLOW = 64;
__global__ void __launch_bounds__(256) absmax_kernel(const OzBlock* __restrict__ blocks, unsigned long long* __restrict__ out,
                                                     unsigned long long* __restrict__ minout, int by_row, int tiles_s_max) {
  __shared__ unsigned long long sm[8][AM_FAST];
  __shared__ unsigned long long sn[8][AM_FAST];
  const OzBlock b = blocks[blockIdx.y];
  const int fastdim = b.isT ? b.cols : b.rows, slowdim = b.isT ? b.rows : b.cols;
  const int f0 = (blockIdx.x / tiles_s_max) * AM_FAST, s0 = (blockIdx.x % tiles_s_max) * AM_SLOW;
  if (f0 >= fastdim || s0 >= slowdim) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool kept_is_fast = (by_row != 0) == (b.isT == 0);  // the kept index is the contiguous one
  const int line0 = by_row ? b.row0 : b.col0;
  const bool want_min = minout != nullptr;
  if (kept_is_fast) {
    unsigned long long best[8], least[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      best[i] = 0ull;
      least[i] = ~0ull;
    }
#pragma unroll 2
    for (int j = 0; j < AM_SLOW / 8; ++j) {
      const int sidx = s0 + warp + 8 * j;
      if (sidx >= slowdim) break;
      const double* src = b.v + static_cast<size_t>(fastdim) * sidx + f0 + lane;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        unsigned long long bits = 0ull;
        if (f0 + lane + 32 * i < fastdim) bits = static_cast<unsigned long long>(__double_as_longlong(fabs(src[32 * i])));
        best[i] = max(best[i], bits);
        least[i] = min(least[i], bits ? bits : ~0ull);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      sm[warp][lane + 32 * i] = best[i];
      sn[warp][lane + 32 * i] = least[i];
    }
    __syncthreads();
    const int f = f0 + threadIdx.x;
    if (f < fastdim) {
      unsigned long long m = sm[0][threadIdx.x], n = sn[0][threadIdx.x];
#pragma unroll
      for (int k = 1; k < 8; ++k) {
        m = max(m, sm[k][threadIdx.x]);
        n = min(n, sn[k][threadIdx.x]);
      }
      if (m != 0ull) atomicMax(&out[line0 + f], m);
      if (want_min && n != ~0ull) atomicMin(&minout[line0 + f], n);
    }
  } else {
#pragma unroll 2
    for (int j = 0; j < AM_SLOW / 8; ++j) {
      const int sidx = s0 + warp + 8 * j;
      if (sidx >= slowdim) break;  // warp-uniform
      const double* src = b.v + static_cast<size_t>(fastdim) * sidx + f0 + lane;
      unsigned long long m = 0ull, n = ~0ull;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        unsigned long long bits = 0ull;
        if (f0 + lane + 32 * i < fastdim) bits = static_cast<unsigned long long>(__double_as_longlong(fabs(src[32 * i])));
        m = max(m, bits);
        n = min(n, bits ? bits : ~0ull);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (want_min) n = min(n, __shfl_xor_sync(0xffffffffu, n, o));
      }
      if (lane == 0) {
        if (m != 0ull) atomicMax(&out[line0 + sidx], m);
        if (want_min && n != ~0ull) atomicMin(&minout[line0 + sidx], n);
      }
    }
  }
}

// grid of absmax_kernel for blocks of at most max_rows x max_cols (either orientation)
struct AbsmaxGrid {
  int ts, tiles;
  AbsmaxGrid(int max_rows, int max_cols) {
    const int d = max_rows > max_cols ? max_rows : max_cols;
    ts = (d + AM_SLOW - 1) / AM_SLOW;
    tiles = ((d + AM_FAST - 1) / AM_FAST) * ts;
  }
};

// exponent table: e = ilogb(max) + 1 (so |x| * 2^-e < 1), 0 for all-zero lines; flags non-finite input.
// range_bits > 0 (Ozaki-II auto-selection): also flags a line whose smallest non-zero magnitude lies more than range_bits
// binary orders below its maximum -- such an element would keep too few of its significand bits after the per-line scaling.
__global__ void exp_kernel(const unsigned long long* __restrict__ maxbits, const unsigned long long* __restrict__ minbits,
                           int32_t* __restrict__ e, double* __restrict__ scale, int n, int range_bits, int* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double m = __longlong_as_double(static_cast<long long>(maxbits[i]));
  int ex = 0;
  if (!isfinite(m)) {
    *bad = 1;
  } else if (m != 0.0) {
    ex = ilogb(m) + 1;
    if (range_bits > 0 && minbits != nullptr && minbits[i] != ~0ull) {
      const double lo = __longlong_as_double(static_cast<long long>(minbits[i]));
      if (ex - 1 - ilogb(lo) > range_bits) *bad = 1;
    }
  }
  e[i] = ex;
  if (scale != nullptr) scale[i] = scalbn(1.0, ex);
}

// ---- pass 2: balanced base-256 digits.  out_s[line * Kpad + k], line = row of A (transpose_out = 0) or column of B --
// One CTA = 32 lines x 128 k of one block, staged through shared memory so global reads follow the block's
// contiguous dimension and the int8 writes are 128-byte rows.
__global__ void __launch_bounds__(256) slice_kernel(const OzBlock* __restrict__ blocks, const int32_t* __restrict__ line_exp,
                                                    int8_t* __restrict__ out, size_t slice_stride, int Kpad, int S,
                                                    int lines_are_rows, int tiles_k_max) {
  __shared__ double sm[32][129];
  const OzBlock b = blocks[blockIdx.y];
  const int tl = blockIdx.x / tiles_k_max, tk = blockIdx.x % tiles_k_max;
  // "line" = kept index (row of A / column of B), "k" = reduction index (column of A / row of B)
  const int nlines = lines_are_rows ? b.rows : b.cols;
  const int nks = lines_are_rows ? b.cols : b.rows;
  const int l0 = tl * 32, k0 = tk * 128;
  if (l0 >= nlines || k0 >= nks) return;
  const int tid = threadIdx.x;
  // element (line l, k) lives at: lines_are_rows ? blk(l, k) : blk(k, l).  Memory-contiguous index:
  //   column-major block (isT = 0): row index fastest;  row-major (isT = 1): column index fastest.
  const bool k_fast = lines_are_rows ? (b.isT != 0) : (b.isT == 0);
  if (k_fast) {
    for (int idx = tid; idx < 32 * 128; idx += 256) {
      const int l = idx / 128, k = idx % 128;
      double v = 0.0;
      if (l0 + l < nlines && k0 + k < nks) v = lines_are_rows ? blk_at(b, l0 + l, k0 + k) : blk_at(b, k0 + k, l0 + l);
      sm[l][k] = v;
    }
  } else {
    for (int idx = tid; idx < 32 * 128; idx += 256) {
      const int k = idx / 32, l = idx % 32;
      double v = 0.0;
      if (l0 + l < nlines && k0 + k < nks) v = lines_are_rows ? blk_at(b, l0 + l, k0 + k) : blk_at(b, k0 + k, l0 + l);
      sm[l][k] = v;
    }
  }
  __syncthreads();
  const int gl_base = (lines_are_rows ? b.row0 : b.col0) + l0;
  const int gk_base = (lines_are_rows ? b.col0 : b.row0) + k0;
  const int warp = tid >> 5, lane = tid & 31;
  for (int l = warp; l < 32; l += 8) {
    if (l0 + l >= nlines) continue;
    const int e = line_exp[gl_base + l];
    long long X[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double x = scalbn(sm[l][lane * 4 + j], 8 * S - 2 - e);  // |x| < 2^(8S-2): exact power-of-two scaling
      X[j] = __double2ll_rn(x);
    }
    // least-significant digit first; digit in [-128, 127], carry folded into the next one
    for (int s = S; s >= 1; --s) {
      uint32_t packed = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long dgt = ((X[j] + 128) & 255) - 128;
        X[j] = (X[j] - dgt) >> 8;
        packed |= (static_cast<uint32_t>(dgt) & 0xffu) << (8 * j);
      }
      const int kq = k0 + lane * 4;  // first k of this quad inside the block
      const int gk = gk_base + lane * 4;
      int8_t* dst = out + static_cast<size_t>(s - 1) * slice_stride + static_cast<size_t>(gl_base + l) * Kpad + gk;
      if (kq + 3 < nks && (gk & 3) == 0) {
        *reinterpret_cast<uint32_t*>(dst) = packed;
      } else {  // block edge / unaligned block offset: never touch a neighbouring block's bytes
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (kq + j < nks) dst[j] = static_cast<int8_t>((packed >> (8 * j)) & 0xffu);
      }
    }
  }
}

// ---- Ozaki scheme II (gemm_algo 4): residues of the scaled integer operands modulo T pairwise-coprime p_t <= 256 ------
// A' = rint(A * 2^(alpha - e_i)) (|a'| <= 2^alpha <= 2^62), B' likewise per column; C' = A' B' is an exact integer with
// |c'| < P / 2 (P = prod p_t) by the choice of alpha, so it is recovered from the T int8 GEMMs (A' mod p_t)(B' mod p_t) by the
// Chinese remainder theorem: T tensor-core GEMMs instead of the S (S + 1) / 2 of the digit-slicing scheme.
constexpr int CRT_MAX_T = 16;
constexpr int CRT_MIN_T = 6;
struct CrtConst {
  uint32_t p[CRT_MAX_T];       // moduli
  uint32_t clo[CRT_MAX_T];     // bytes (256^0, 256^1, 256^2, 256^3) mod p
  uint32_t chi[CRT_MAX_T];     // bytes (256^4, 256^5, 256^6, 256^7) mod p
  float invpf[CRT_MAX_T];      // 1 / p
  int32_t T, pad;
};
__constant__ CrtConst c_crt[CRT_MAX_T + 1];  // indexed by T, filled once on first use
// the same CRT weights and P as exact fp64 chunks of CRT_CHUNK_BITS bits (little-endian; the top chunk takes the rest)
constexpr int CRT_CHUNK_BITS = 40;
struct CrtF {
  double w[CRT_MAX_T][4];
  double P[4];
  double invP;
  int32_t nch, pad;
  // three chunks cover P < 2^120 (top chunk < 2^40); four are needed above (T = 16: P ~ 2^125.4, top chunk < 2^6)
  static int nch_for(unsigned __int128 P) { return (P >> (3 * CRT_CHUNK_BITS)) == 0 ? 3 : 4; }
  static double chunk(unsigned __int128 x, int i, int nch) {
    const unsigned __int128 sh = x >> (CRT_CHUNK_BITS * i);
    return static_cast<double>(static_cast<uint64_t>(i + 1 < nch ? sh & ((static_cast<unsigned __int128>(1) << CRT_CHUNK_BITS) - 1) : sh));
  }
};
__constant__ CrtF c_crtf[CRT_MAX_T + 1];

// An element too far below the maximum of its line to keep enough significand bits after the per-line scaling.  It is left out
// of the residues (treated as zero) and its products are added exactly, in fp64, by oz2_fixup_kernel after the CRT pass.
struct OutlierRec {
  int32_t line;  // buffer line (row of A' / row of B') of the side it belongs to
  int32_t k;     // inner index
  double v;      // the element
};
constexpr int OZ2_REC_CAP = 64;  // records per slot (block row / block column); more than that raises the fallback flag
__device__ __forceinline__ int exponent_of(double x) { return ((__double2hiint(x) >> 20) & 0x7ff) - 1023; }  // ilogb for normal x

// out_t[line * Kpad + k] = symmetric residue of a'(line, k) mod p_t, same tiling / staging as slice_kernel.
// range_bits > 0: non-zero elements more than range_bits binary orders below their line maximum become OutlierRecs of their
// slot (recs / rec_cnt are the tables of this side, sstride lines per slot); a full slot table raises *gate.
__global__ void __launch_bounds__(256) residue_kernel(const OzBlock* __restrict__ blocks, const int32_t* __restrict__ line_exp,
                                                      int8_t* __restrict__ out, size_t slice_stride, int Kpad, int T, int alpha,
                                                      int lines_are_rows, int tiles_k_max, int* __restrict__ gate, int range_bits,
                                                      OutlierRec* __restrict__ recs, int* __restrict__ rec_cnt, int sstride) {
  __shared__ double sm[32][129];
  if (gate != nullptr && *gate != 0) return;
  const OzBlock b = blocks[blockIdx.y];
  const int tl = blockIdx.x / tiles_k_max, tk = blockIdx.x % tiles_k_max;
  const int nlines = lines_are_rows ? b.rows : b.cols;
  const int nks = lines_are_rows ? b.cols : b.rows;
  const int l0 = tl * 32, k0 = tk * 128;
  if (l0 >= nlines || k0 >= nks) return;
  const int tid = threadIdx.x;
  const bool k_fast = lines_are_rows ? (b.isT != 0) : (b.isT == 0);
  for (int idx = tid; idx < 32 * 128; idx += 256) {
    const int l = k_fast ? idx / 128 : idx % 32, k = k_fast ? idx % 128 : idx / 32;
    double v = 0.0;
    if (l0 + l < nlines && k0 + k < nks) v = lines_are_rows ? blk_at(b, l0 + l, k0 + k) : blk_at(b, k0 + k, l0 + l);
    sm[l][k] = v;
  }
  __syncthreads();
  const CrtConst& cc = c_crt[T];
  const int gl_base = (lines_are_rows ? b.row0 : b.col0) + l0;
  const int gk_base = (lines_are_rows ? b.col0 : b.row0) + k0;
  const int warp = tid >> 5, lane = tid & 31;
  for (int l = warp; l < 32; l += 8) {
    if (l0 + l >= nlines) continue;
    const int e = line_exp[gl_base + l];
    const double line_scale = scalbn(1.0, alpha - e);  // exact power of two
    uint32_t hi[4], lo[4];
    float sgn[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double xv = sm[l][lane * 4 + j];
      if (range_bits > 0 && xv != 0.0 && exponent_of(xv) < e - 1 - range_bits) {
        const int slot = (gl_base + l) / sstride;
        const int at = atomicAdd(&rec_cnt[slot], 1);
        if (at < OZ2_REC_CAP) recs[static_cast<size_t>(slot) * OZ2_REC_CAP + at] = OutlierRec{gl_base + l, gk_base + lane * 4 + j, xv};
        else *gate = 1;
        xv = 0.0;
      }
      const long long X = __double2ll_rn(xv * line_scale);  // exact scaling, |X| <= 2^alpha
      sgn[j] = X < 0 ? -1.0f : 1.0f;
      const unsigned long long U = static_cast<unsigned long long>(X < 0 ? -X : X);
      hi[j] = static_cast<uint32_t>(U >> 32);
      lo[j] = static_cast<uint32_t>(U);
    }
    const int kq = k0 + lane * 4;
    const int gk = gk_base + lane * 4;
    const bool whole = kq + 3 < nks && (gk & 3) == 0;
    // All arithmetic below stays on the FMA / ALU pipes (no int<->float conversion instructions, which run at a quarter rate):
    //   x = sum_i byte_i (256^i mod p) < 2^19 (two dp4a), congruent to |X|;
    //   float(x) by the exponent trick (x < 2^23): as_float(0x4B000000 | x) - 2^23;
    //   q = rint(x / p) by the 1.5 * 2^23 magic add (the fp32 quotient is off by < 4e-4; for odd p a fractional part is never closer
    //   than 1 / (2 p) >= 2e-3 to one half, so the rounding decision is exact; p = 256 has true ties, either neighbour is congruent);
    //   r = x - q p exactly (|r| <= 128), signed, and its low byte read out of the mantissa of r * sgn + 1.5 * 2^23.
    const float kMagic = 12582912.0f;
    for (int t = 0; t < T; ++t) {
      const float pf = static_cast<float>(cc.p[t]);
      const uint32_t wl = cc.clo[t], wh = cc.chi[t];
      const float ip = cc.invpf[t];
      uint32_t bytes[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t x = __dp4a(lo[j], wl, __dp4a(hi[j], wh, 0u));
        const float f = __uint_as_float(0x4B000000u | x) - 8388608.0f;
        const float q = __fadd_rn(__fmaf_rn(f, ip, kMagic), -kMagic);
        const float r = __fmaf_rn(-q, pf, f);
        bytes[j] = __float_as_uint(__fmaf_rn(r, sgn[j], kMagic));   // low byte = r * sgn in two's complement (+-128 wrap to -128: p = 256 only)
      }
      const uint32_t packed = __byte_perm(__byte_perm(bytes[0], bytes[1], 0x0040), __byte_perm(bytes[2], bytes[3], 0x0040), 0x5410);
      int8_t* dst = out + static_cast<size_t>(t) * slice_stride + static_cast<size_t>(gl_base + l) * Kpad + gk;
      if (whole) {
        *reinterpret_cast<uint32_t*>(dst) = packed;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (kq + j < nks) dst[j] = static_cast<int8_t>((packed >> (8 * j)) & 0xffu);
      }
    }
  }
}

// CRT reconstruction: one CTA = 32 rows x 128 columns of one 128 x 256 tile of the job (8 CTAs per tile).  Thread (row, 4 columns)
// reads its T residue quads (coalesced along the compact plane rows) and accumulates S = sum_t r_t w_t in fp64, EXACTLY: every
// weight is split into 40-bit chunks (c_crtf), so each chunk sum stays an integer below 2^52 (r < 2^8, T <= 2^4).  With
// q = rint(S / P) the chunk differences D_i = S_i - q P_i are again exact (one FMA each, |q P_i| < 2^52) and represent the
// symmetric residue C' = S - q P, |C'| <= P / 2; a carry pass makes the chunks non-overlapping signed digits, so the top-down
// Horner sum rounds once per step and is exact whenever C' fits 53 bits (integer data give the exact integer product).  The
// scaling by 2^(e_i + f_j - 2 alpha) is a multiplication by a constructed power of two.  The tile is transposed through shared
// memory so the stores follow the column-major output blocks.  Buffer rows / columns are organised in slots of `sstride` lines
// (one block row / block column each); ctab[rslot * ncslots + cslot] is the output block or nullptr.
__device__ __forceinline__ double pow2_double(int n) {  // 2^n, -1022 <= n <= 1023
  return __hiloint2double((n + 1023) << 20, 0);
}
__device__ __forceinline__ double scale_by_pow2(double x, int n) {
  const int n1 = max(-1022, min(1023, n));
  x *= pow2_double(n1);
  n -= n1;
  while (n != 0) {  // beyond the normal exponent range (sub-normal or overflowing results): continue in steps
    const int n2 = max(-1022, min(1023, n));
    x *= pow2_double(n2);
    n -= n2;
  }
  return x;
}

template <int NCH>
__global__ void __launch_bounds__(256) crt_kernel(const int8_t* __restrict__ planes, size_t plane_stride, int T,
                                                  const int2* __restrict__ tiles, const int32_t* __restrict__ row_exp,
                                                  const int32_t* __restrict__ col_exp, int two_alpha, double* const* __restrict__ ctab,
                                                  const int32_t* __restrict__ rdims, const int32_t* __restrict__ cdims, int sstride,
                                                  int ncslots, const int* __restrict__ gate) {
  __shared__ double tile[128][33];
  if (gate != nullptr && *gate != 0) return;
  const CrtF& cf = c_crtf[T];
  const int t_idx = blockIdx.x >> 3, sub = blockIdx.x & 7;
  const int2 tl = tiles[t_idx];
  const int r0t = (sub >> 1) * 32, c0t = (sub & 1) * 128;  // inside the tile
  const int r0 = tl.x * BM + r0t, c0 = tl.y * BN + c0t;     // buffer coordinates
  const int tid = threadIdx.x;
  const int lr = tid >> 5, lc = (tid & 31) * 4;  // 8 rows per pass, 4 passes
  const int8_t* tbase = planes + static_cast<size_t>(t_idx) * (BM * BN);
  constexpr double kTwo52 = 4503599627370496.0, kMagic = 6755399441055744.0;  // 2^52, 1.5 * 2^52
  constexpr double kUp = 1099511627776.0, kDown = 1.0 / 1099511627776.0;        // 2^40, 2^-40
#pragma unroll 1
  for (int pass = 0; pass < 4; ++pass) {
    const int row = r0 + pass * 8 + lr;
    double S[4][NCH];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int i = 0; i < NCH; ++i) S[j][i] = 0.0;
    const int8_t* src = tbase + static_cast<size_t>(r0t + pass * 8 + lr) * BN + c0t + lc;
#pragma unroll 4
    for (int t = 0; t < T; ++t) {
      const uint32_t quad = *reinterpret_cast<const uint32_t*>(src + static_cast<size_t>(t) * plane_stride);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        // byte j as a double: 2^52 + r has r in its low mantissa bits
        const double x = __hiloint2double(0x43300000, static_cast<int>(__byte_perm(quad, 0u, 0x4440u + j))) - kTwo52;
#pragma unroll
        for (int i = 0; i < NCH; ++i) S[j][i] = fma(x, cf.w[t][i], S[j][i]);
      }
    }
    const int er = row_exp[row];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double v = S[j][NCH - 1];
#pragma unroll
      for (int i = NCH - 2; i >= 0; --i) v = fma(v, kUp, S[j][i]);
      const double q = fma(v, cf.invP, kMagic) - kMagic;  // rint(S / P), < 2^12
      double D[NCH];
#pragma unroll
      for (int i = 0; i < NCH; ++i) D[i] = fma(-q, cf.P[i], S[j][i]);
#pragma unroll
      for (int i = 0; i + 1 < NCH; ++i) {
        const double c = fma(D[i], kDown, kMagic) - kMagic;  // nearest multiple of 2^40 carried upwards
        D[i] = fma(-c, kUp, D[i]);
        D[i + 1] += c;
      }
      double x = D[NCH - 1];
#pragma unroll
      for (int i = NCH - 2; i >= 0; --i) x = fma(x, kUp, D[i]);
      const int ec = col_exp[c0 + lc + j];
      tile[lc + j][pass * 8 + lr] = scale_by_pow2(x, er + ec - two_alpha);
    }
  }
  __syncthreads();
  // store: warp w writes columns w, w + 8, ...; lanes run along the 32 rows (contiguous in the column-major block)
  const int warp = tid >> 5, lane = tid & 31;
  const int row = r0 + lane;
  const int rslot = row / sstride;
  const int lrow = row - rslot * sstride;
  const int brows = rdims[rslot];
  if (lrow >= brows) return;
  for (int cidx = warp; cidx < 128; cidx += 8) {
    const int col = c0 + cidx;
    const int cslot = col / sstride;
    if (cslot >= ncslots) break;
    const int lcol = col - cslot * sstride;
    if (lcol >= cdims[cslot]) continue;
    double* blkp = ctab[static_cast<size_t>(rslot) * ncslots + cslot];
    if (blkp != nullptr) blkp[lrow + static_cast<size_t>(brows) * lcol] = tile[cidx][lane];
  }
}

// Exact products of the outlier elements (see OutlierRec), added to the C blocks of a job after its CRT pass.  One CTA per output
// block: first the outliers of its block row of A (C(i, :) += a_ik B(k, :), thread = column), then those of its block column of
// B (C(:, j) += A(:, k) b_kj, thread = row; an a_ik that is an outlier itself was already paired with the original b_kj in the
// first phase and is skipped).  Operand values come from the original fp64 blocks.
__global__ void __launch_bounds__(256) oz2_fixup_kernel(const Oz2FixOut* __restrict__ outs, const Oz2FixSrc* __restrict__ srcs,
                                                        const OutlierRec* __restrict__ recs, const int* __restrict__ rec_cnt, int cap_r,
                                                        int sstride, const int32_t* __restrict__ row_exp, int range_bits,
                                                        const int* __restrict__ gate) {
  if (*gate != 0) return;
  const Oz2FixOut o = outs[blockIdx.x];
  const int nA = min(rec_cnt[o.rslot], OZ2_REC_CAP), nB = min(rec_cnt[cap_r + o.cslot], OZ2_REC_CAP);
  if (nA == 0 && nB == 0) return;
  const OutlierRec* ra = recs + static_cast<size_t>(o.rslot) * OZ2_REC_CAP;
  const OutlierRec* rb = recs + static_cast<size_t>(cap_r + o.cslot) * OZ2_REC_CAP;
  for (int q = 0; q < nA; ++q) {
    const OutlierRec r = ra[q];
    const int i = r.line - o.rslot * sstride;
    if (i < 0 || i >= o.m) continue;
    for (int t = 0; t < o.src_count; ++t) {
      const Oz2FixSrc sc = srcs[o.src_begin + t];
      if (r.k < sc.k0 || r.k >= sc.k0 + sc.kdim) continue;
      const int kk = r.k - sc.k0;
      for (int j = threadIdx.x; j < o.n; j += blockDim.x) {
        const double b = sc.bT ? sc.B[static_cast<size_t>(kk) * sc.b_cols + j] : sc.B[kk + static_cast<size_t>(sc.kdim) * j];
        o.C[i + static_cast<size_t>(o.m) * j] += r.v * b;
      }
      break;
    }
  }
  __syncthreads();
  for (int q = 0; q < nB; ++q) {
    const OutlierRec r = rb[q];
    const int j = r.line - o.cslot * sstride;
    if (j < 0 || j >= o.n) continue;
    for (int t = 0; t < o.src_count; ++t) {
      const Oz2FixSrc sc = srcs[o.src_begin + t];
      if (r.k < sc.k0 || r.k >= sc.k0 + sc.kdim) continue;
      const int kk = r.k - sc.k0;
      for (int i = threadIdx.x; i < o.m; i += blockDim.x) {
        const double a = sc.aT ? sc.A[static_cast<size_t>(i) * sc.kdim + kk] : sc.A[i + static_cast<size_t>(sc.a_rows) * kk];
        if (a == 0.0 || exponent_of(a) < row_exp[o.rslot * sstride + i] - 1 - range_bits) continue;
        o.C[i + static_cast<size_t>(o.m) * j] += a * r.v;
      }
      break;
    }
  }
}

// ---- fp32 path (BASELINE configs[3]): 3xTF32 split.  hi = tf32(a), lo = tf32(a - hi); A B ~= hi hi' + hi lo' + lo hi'
// with fp32 accumulation in the tensor core.  out_hi/out_lo[line * Kpad + k] (fp32, K contiguous), same staging as slice_kernel.
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
// Sum of all elements of the blocks (for the operand mean): the value arrays are summed in storage order (coalesced whatever
// the block's orientation); blockIdx.x strides over 4096-element pieces, blockIdx.y = block.
__global__ void __launch_bounds__(256) block_sum_kernel(const OzBlock* __restrict__ blocks, double* __restrict__ total) {
  __shared__ double part[8];
  const OzBlock b = blocks[blockIdx.y];
  const size_t count = static_cast<size_t>(b.rows) * b.cols;
  double acc = 0.0;
  for (size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x; i < count; i += static_cast<size_t>(gridDim.x) * 256) acc += b.v[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += part[w];
    atomicAdd(total, t);
  }
}

// hi = tf32(a'), lo = tf32(a' - hi) of the CENTRED fp32 value a' = fl32(a - mean): the tensor core's fp32 accumulation truncates,
// which for same-signed data is a bias that grows with the number of accumulation steps (measured ~1e-4 at K = 16384 for U(0,1)
// data); on centred data the same truncation errors have random signs.  The mean is put back in fp64 by the epilogue through
//   (A' + muA 11^T)(B' + muB 11^T) = A'B' + muB (A'1) 1^T + muA 1 (1^T B') + K muA muB 11^T,
// for which this pass also accumulates the line sums A'1 / 1^T B' (line_sum, fp64 atomics).
__global__ void __launch_bounds__(256) slice_tf32_kernel(const OzBlock* __restrict__ blocks, float* __restrict__ out_hi,
                                                         float* __restrict__ out_lo, int Kpad, int lines_are_rows, int tiles_k_max,
                                                         const double* __restrict__ total, double inv_count, double* __restrict__ line_sum) {
  __shared__ double sm[32][129];
  const OzBlock b = blocks[blockIdx.y];
  const int tl = blockIdx.x / tiles_k_max, tk = blockIdx.x % tiles_k_max;
  const int nlines = lines_are_rows ? b.rows : b.cols;
  const int nks = lines_are_rows ? b.cols : b.rows;
  const int l0 = tl * 32, k0 = tk * 128;
  if (l0 >= nlines || k0 >= nks) return;
  const int tid = threadIdx.x;
  const double mu = total != nullptr ? total[0] * inv_count : 0.0;
  const bool k_fast = lines_are_rows ? (b.isT != 0) : (b.isT == 0);
  for (int idx = tid; idx < 32 * 128; idx += 256) {
    const int l = k_fast ? idx / 128 : idx % 32, k = k_fast ? idx % 128 : idx / 32;
    double v = 0.0;
    if (l0 + l < nlines && k0 + k < nks) v = lines_are_rows ? blk_at(b, l0 + l, k0 + k) : blk_at(b, k0 + k, l0 + l);
    sm[l][k] = v;
  }
  __syncthreads();
  const int gl_base = (lines_are_rows ? b.row0 : b.col0) + l0;
  const int gk_base = (lines_are_rows ? b.col0 : b.row0) + k0;
  for (int idx = tid; idx < 32 * 128; idx += 256) {   // a warp covers 32 consecutive k of ONE line per pass
    const int l = idx / 128, k = idx % 128;
    double contrib = 0.0;
    if (l0 + l < nlines && k0 + k < nks) {
      const float a = static_cast<float>(sm[l][k] - mu);
      const float hi = to_tf32(a);
      const float lo = to_tf32(a - hi);
      const size_t o = static_cast<size_t>(gl_base + l) * Kpad + gk_base + k;
      out_hi[o] = hi;
      out_lo[o] = lo;
      contrib = static_cast<double>(a);
    }
    if (line_sum != nullptr) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
      if ((tid & 31) == 0 && l0 + l < nlines) atomicAdd(&line_sum[gl_base + l], contrib);
    }
  }
}

// additive fp64 corrections of the centred product: row_corr[i] = muB * (A'1)_i + K muA muB, col_corr[j] = muA * (1^T B')_j
__global__ void tf32_corr_kernel(const double* __restrict__ totals, double inv_a, double inv_b, double K, double* __restrict__ row_corr, int m,
                                 double* __restrict__ col_corr, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double muA = totals[0] * inv_a, muB = totals[1] * inv_b;
  if (i < m) row_corr[i] = muB * row_corr[i] + K * muA * muB;
  if (i < n) col_corr[i] = muA * col_corr[i];
}

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn encode_fn() {
  static EncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeFn>(p);
  }();
  return fn;
}

bool make_i8_map(unsigned char* out128, void* base, uint64_t Kpad, uint64_t rows, uint32_t box_rows) {
  EncodeFn fn = encode_fn();
  if (!fn) return false;
  alignas(64) CUtensorMap m;
  const cuuint64_t gdim[2] = {Kpad, rows};
  const cuuint64_t gstr[1] = {Kpad};
  const cuuint32_t box[2] = {BKB, box_rows};
  const cuuint32_t est[2] = {1, 1};
  if (fn(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, gdim, gstr, box, est, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return false;
  memcpy(out128, &m, 128);
  return true;
}

bool make_f32_map(unsigned char* out128, void* base, uint64_t Kpad, uint64_t rows, uint32_t box_rows) {
  EncodeFn fn = encode_fn();
  if (!fn) return false;
  alignas(64) CUtensorMap m;
  const cuuint64_t gdim[2] = {Kpad, rows};
  const cuuint64_t gstr[1] = {Kpad * 4};
  const cuuint32_t box[2] = {32, box_rows};  // 32 fp32 = one 128-byte swizzle row
  const cuuint32_t est[2] = {1, 1};
  if (fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, gdim, gstr, box, est, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return false;
  memcpy(out128, &m, 128);
  return true;
}

#define OZ_CHECK(x)                      \
  do {                                   \
    cudaError_t e_ = (x);                \
    if (e_ != cudaSuccess) return e_;    \
  } while (0)

// The slice / residue matrices only need zero-filling where no block writes: K padding (garbage there would enter every dot
// product) and absent blocks.  Row padding beyond M / N may hold garbage: those accumulator rows are never stored.
bool covers_operand(const OzakiOperand* blocks, int n, int64_t lines, int64_t K, int64_t Kpad) {
  if (K != Kpad) return false;
  int64_t area = 0;
  for (int i = 0; i < n; ++i) area += static_cast<int64_t>(blocks[i].rows) * blocks[i].cols;
  return area == lines * K;  // block ids are unique, so equal area means full coverage
}
// gridDim.y carries the block index of the batched passes: split lists longer than its 65535 limit
constexpr int kMaxGridY = 65535;
template <class Launch>
cudaError_t for_block_chunks(int nblocks, Launch&& launch) {
  for (int off = 0; off < nblocks; off += kMaxGridY) {
    launch(off, std::min(kMaxGridY, nblocks - off));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t configure_gemm_kernels() {
  static PerDeviceOnce once;
  return once.run([&] {
    const int bytes = static_cast<int>(GEMM_SMEM_BYTES);
    cudaError_t e = cudaFuncSetAttribute(ozaki_gemm_i8_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ozaki_gemm_i8_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ozaki2_gemm_2sm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ozaki2_gemm_2sm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    return e;
  });
}

struct AsyncBuf {  // stream-ordered scratch
  void* p = nullptr;
  cudaStream_t s;
  explicit AsyncBuf(cudaStream_t st) : s(st) {}
  cudaError_t alloc(size_t n) { return cudaMallocAsync(&p, n ? n : 16, s); }
  ~AsyncBuf() {
    if (p) cudaFreeAsync(p, s);
  }
};

}  // namespace

cudaError_t ozaki_gemm_f64(const OzakiOperand* a_blocks, int na, const OzakiOperand* b_blocks, int nb, int64_t M, int64_t K,
                           int64_t N, int slices, double* const* h_ctab, int blk, int nbr, int nbc, bool accumulate,
                           int* launches, int* nonfinite, cudaStream_t stream) {
  *nonfinite = 0;
  if (M <= 0 || N <= 0 || K <= 0) return cudaSuccess;
  const int S = slices < 2 ? 2 : (slices > 7 ? 7 : slices);
  const int64_t Mpad = (M + BM - 1) / BM * BM, Npad = (N + BN - 1) / BN * BN, Kpad = (K + BKB - 1) / BKB * BKB;
  OZ_CHECK(configure_gemm_kernels());
  // block descriptor tables
  std::vector<OzBlock> ha(na), hb(nb);
  int max_ar = 1, max_ac = 1, max_br = 1, max_bc = 1;
  for (int i = 0; i < na; ++i) {
    ha[i] = OzBlock{a_blocks[i].v, a_blocks[i].rows, a_blocks[i].cols, a_blocks[i].row0, a_blocks[i].col0, a_blocks[i].isT, {0}};
    max_ar = std::max(max_ar, a_blocks[i].rows);
    max_ac = std::max(max_ac, a_blocks[i].cols);
  }
  for (int i = 0; i < nb; ++i) {
    hb[i] = OzBlock{b_blocks[i].v, b_blocks[i].rows, b_blocks[i].cols, b_blocks[i].row0, b_blocks[i].col0, b_blocks[i].isT, {0}};
    max_br = std::max(max_br, b_blocks[i].rows);
    max_bc = std::max(max_bc, b_blocks[i].cols);
  }
  AsyncBuf d_ab(stream), d_bb(stream), d_max(stream), d_exp(stream), d_scale(stream), d_bad(stream), d_As(stream), d_Bs(stream), d_maps(stream), d_ctab(stream);
  OZ_CHECK(d_ab.alloc(sizeof(OzBlock) * na));
  OZ_CHECK(d_bb.alloc(sizeof(OzBlock) * nb));
  OZ_CHECK(cudaMemcpyAsync(d_ab.p, ha.data(), sizeof(OzBlock) * na, cudaMemcpyHostToDevice, stream));
  OZ_CHECK(cudaMemcpyAsync(d_bb.p, hb.data(), sizeof(OzBlock) * nb, cudaMemcpyHostToDevice, stream));
  OZ_CHECK(d_max.alloc(sizeof(unsigned long long) * (Mpad + Npad)));
  OZ_CHECK(d_exp.alloc(sizeof(int32_t) * (Mpad + Npad)));
  OZ_CHECK(d_scale.alloc(sizeof(double) * (Mpad + Npad)));
  OZ_CHECK(d_bad.alloc(sizeof(int)));
  OZ_CHECK(cudaMemsetAsync(d_max.p, 0, sizeof(unsigned long long) * (Mpad + Npad), stream));
  OZ_CHECK(cudaMemsetAsync(d_bad.p, 0, sizeof(int), stream));
  unsigned long long* rowmax = static_cast<unsigned long long*>(d_max.p);
  unsigned long long* colmax = rowmax + Mpad;
  int32_t* row_exp = static_cast<int32_t*>(d_exp.p);
  int32_t* col_exp = row_exp + Mpad;
  // pass 1
  {
    const AbsmaxGrid ga(max_ar, max_ac), gb(max_br, max_bc);
    OZ_CHECK(for_block_chunks(na, [&](int off, int cnt) {
      absmax_kernel<<<dim3(ga.tiles, cnt), 256, 0, stream>>>(static_cast<const OzBlock*>(d_ab.p) + off, rowmax, nullptr, 1, ga.ts);
    }));
    OZ_CHECK(for_block_chunks(nb, [&](int off, int cnt) {
      absmax_kernel<<<dim3(gb.tiles, cnt), 256, 0, stream>>>(static_cast<const OzBlock*>(d_bb.p) + off, colmax, nullptr, 0, gb.ts);
    }));
    exp_kernel<<<static_cast<unsigned>((Mpad + Npad + 255) / 256), 256, 0, stream>>>(rowmax, nullptr, row_exp, static_cast<double*>(d_scale.p),
                                                                                      static_cast<int>(Mpad + Npad), 0, static_cast<int*>(d_bad.p));
    *launches += 3;
  }
  int h_bad = 0;
  OZ_CHECK(cudaMemcpyAsync(&h_bad, d_bad.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
  OZ_CHECK(cudaStreamSynchronize(stream));
  if (h_bad) {
    *nonfinite = 1;  // Inf/NaN input: integer slicing is undefined; the caller falls back to the exact DMMA kernel
    return cudaSuccess;
  }
  // pass 2
  const size_t a_stride = static_cast<size_t>(Mpad) * Kpad, b_stride = static_cast<size_t>(Npad) * Kpad;
  OZ_CHECK(d_As.alloc(a_stride * S));
  OZ_CHECK(d_Bs.alloc(b_stride * S));
  if (!covers_operand(a_blocks, na, M, K, Kpad)) OZ_CHECK(cudaMemsetAsync(d_As.p, 0, a_stride * S, stream));
  if (!covers_operand(b_blocks, nb, N, K, Kpad)) OZ_CHECK(cudaMemsetAsync(d_Bs.p, 0, b_stride * S, stream));
  {
    const int tk = (max_ac + 127) / 128, tl = (max_ar + 31) / 32;
    OZ_CHECK(for_block_chunks(na, [&](int off, int cnt) {
      slice_kernel<<<dim3(tl * tk, cnt), 256, 0, stream>>>(static_cast<const OzBlock*>(d_ab.p) + off, row_exp, static_cast<int8_t*>(d_As.p),
                                                           a_stride, static_cast<int>(Kpad), S, 1, tk);
    }));
    const int tkb = (max_br + 127) / 128, tlb = (max_bc + 31) / 32;
    OZ_CHECK(for_block_chunks(nb, [&](int off, int cnt) {
      slice_kernel<<<dim3(tlb * tkb, cnt), 256, 0, stream>>>(static_cast<const OzBlock*>(d_bb.p) + off, col_exp, static_cast<int8_t*>(d_Bs.p),
                                                             b_stride, static_cast<int>(Kpad), S, 0, tkb);
    }));
    *launches += 2;
  }
  // tensor maps + output block table
  std::vector<unsigned char> hmaps(static_cast<size_t>(2 * S) * 128);
  for (int s = 0; s < S; ++s) {
    if (!make_i8_map(&hmaps[static_cast<size_t>(s) * 128], static_cast<int8_t*>(d_As.p) + a_stride * s, Kpad, Mpad, BM) ||
        !make_i8_map(&hmaps[static_cast<size_t>(S + s) * 128], static_cast<int8_t*>(d_Bs.p) + b_stride * s, Kpad, Npad, BN))
      return cudaErrorInvalidValue;
  }
  OZ_CHECK(d_maps.alloc(hmaps.size()));
  OZ_CHECK(cudaMemcpyAsync(d_maps.p, hmaps.data(), hmaps.size(), cudaMemcpyHostToDevice, stream));
  OZ_CHECK(d_ctab.alloc(sizeof(double*) * nbr * nbc));
  OZ_CHECK(cudaMemcpyAsync(d_ctab.p, h_ctab, sizeof(double*) * nbr * nbc, cudaMemcpyHostToDevice, stream));
  // pass 3: smallest terms first (diagonal S+1 down to 2)
  OzakiGemmParams p{};
  p.tmaps = static_cast<const unsigned char*>(d_maps.p);
  p.row_scale = static_cast<const double*>(d_scale.p);
  p.col_scale = p.row_scale + Mpad;
  p.ctab = static_cast<double* const*>(d_ctab.p);
  p.M = static_cast<int32_t>(M);
  p.N = static_cast<int32_t>(N);
  p.Kpad = static_cast<int32_t>(Kpad);
  p.blk = blk;
  p.nbr = nbr;
  p.nbc = nbc;
  p.S = S;
  p.kstep = BKB;
  p.kc0 = 0;
  p.nkc = static_cast<int32_t>(Kpad / BKB);
  p.tiles_m = static_cast<int32_t>(Mpad / BM);
  p.tiles_n = static_cast<int32_t>(Npad / BN);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t ntiles = static_cast<int64_t>(p.tiles_m) * p.tiles_n;
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(ntiles, sms));
  bool first = !accumulate;
  for (int d = S + 1; d >= 2; --d) {
    p.d = d;
    p.accumulate = first ? 0 : 1;
    p.diag_scale = std::ldexp(1.0, 4 - 8 * d);
    p.npairs = 0;
    for (int sl = std::max(1, d - S); sl <= std::min(S, d - 1); ++sl) {  // pairs (s, d - s)
      p.pair_a[p.npairs] = sl - 1;
      p.pair_b[p.npairs] = S + (d - sl) - 1;
      ++p.npairs;
    }
    first = false;
    ozaki_gemm_i8_kernel<false><<<grid, GEMM_THREADS_P, GEMM_SMEM_BYTES, stream>>>(p);
    OZ_CHECK(cudaGetLastError());
    *launches += 1;
  }
  // scratch is freed stream-ordered by the AsyncBuf destructors; pageable staging vectors were consumed synchronously
  return cudaSuccess;
}

namespace {
const int kCrtModuli[CRT_MAX_T] = {256, 255, 253, 251, 247, 241, 239, 233, 229, 227, 223, 217, 211, 199, 197, 193};  // pairwise coprime

// fills c_crt[T] for every supported T once; returns floor(log2 P) per T through log2P
cudaError_t crt_constants(int* log2P, bool upload = true) {
  static PerDeviceOnce uploaded;
  static std::once_flag built;
  static int l2[CRT_MAX_T + 1];
  static std::vector<CrtConst> all(CRT_MAX_T + 1);
  static std::vector<CrtF> allf(CRT_MAX_T + 1);
  std::call_once(built, [&] {
    for (int T = CRT_MIN_T; T <= CRT_MAX_T; ++T) {
      CrtConst& c = all[T];
      CrtF& f = allf[T];
      memset(&c, 0, sizeof(c));
      memset(&f, 0, sizeof(f));
      unsigned __int128 P = 1;
      for (int t = 0; t < T; ++t) P *= static_cast<unsigned>(kCrtModuli[t]);
      for (int t = 0; t < T; ++t) {
        const unsigned pm = static_cast<unsigned>(kCrtModuli[t]);
        c.p[t] = pm;
        uint32_t pw = 1;
        for (int i = 0; i < 8; ++i) {  // 256^i mod p, one byte each
          if (i < 4) c.clo[t] |= pw << (8 * i);
          else c.chi[t] |= pw << (8 * (i - 4));
          pw = (pw * 256u) % pm;
        }
        c.invpf[t] = 1.0f / static_cast<float>(pm);
        const unsigned __int128 Mt = P / pm;
        const unsigned mr = static_cast<unsigned>(Mt % pm);
        unsigned inv = 1;
        while ((mr * inv) % pm != 1u) ++inv;  // Mt is coprime to pm, the inverse exists below pm
        const unsigned __int128 w = Mt * inv;  // CRT weight (P / p_t) * ((P / p_t)^-1 mod p_t) < P
        for (int i = 0; i < f.nch_for(P); ++i) f.w[t][i] = CrtF::chunk(w, i, f.nch_for(P));
      }
      f.nch = f.nch_for(P);
      for (int i = 0; i < f.nch; ++i) f.P[i] = CrtF::chunk(P, i, f.nch);
      f.invP = 1.0 / static_cast<double>(P);
      c.T = T;
      int lg = 0;
      while ((P >> (lg + 1)) != 0) ++lg;
      l2[T] = lg;
    }
  });
  for (int T = 0; T <= CRT_MAX_T; ++T) log2P[T] = l2[T];
  if (!upload) return cudaSuccess;
  return uploaded.run([&] {
    const cudaError_t e1 = cudaMemcpyToSymbol(c_crt, all.data(), sizeof(CrtConst) * (CRT_MAX_T + 1));
    return e1 != cudaSuccess ? e1 : cudaMemcpyToSymbol(c_crtf, allf.data(), sizeof(CrtF) * (CRT_MAX_T + 1));
  });
}
}  // namespace

// ------------------------------------------------------------------------------------------------
// gemm_algo 4 / auto: Ozaki scheme II as a job engine.
//
// The scaled-integer residue matrices A' mod p_t [T][Mpad][Kpad] and B' mod p_t [T][Npad][Kpad] live in slot-organised buffers:
// slot s of A' holds one block row of A (rows [s * sstride, s * sstride + rows)), slot s of B' one block column of B.  A block
// row / column is PREPARED (absmax -> exponents -> residues) as soon as all of its blocks have landed, independently of the
// others, and a JOB multiplies any set of output blocks whose row and column slots are prepared: one persistent wgmma launch
// over (modulus x tile list) work items writing compact residue planes, then the CRT kernel over the same tile list.  That is
// what lets the multiply run chunk by chunk behind the host->device ingest, and what panels the scratch for operands whose
// residues do not fit the budget.  Nothing here synchronises with the host: non-finite input (and, in auto mode, a dynamic range
// inside a line that the per-line scaling cannot carry) raises a device flag that turns the remaining engine kernels into no-ops
// and un-gates the exact DMMA launch the caller enqueues behind every job.
// ------------------------------------------------------------------------------------------------
struct Oz2Engine {
  int T = 0, alpha = 0, crt_chunks = 4, blk = 0, sstride = 0, cap_r = 0, cap_c = 0, max_tiles = 0, range_bits = 0;
  int ksplit = 0;  // CTA-pair kernel walks (modulus, K half, tile pair) items (half the L2 footprint of the panels in flight): 1 = for
                   // long tile lists and deep K only, 2 = whenever K has an even number of chunks (tests)
  bool paired = false;   // tile lists hold vertically adjacent 128-row tiles in pairs: the CTA-pair kernel runs them
  int64_t K = 0, Kpad = 0, Mpad = 0, Npad = 0;
  size_t a_stride = 0, b_stride = 0, plane_stride = 0;
  int8_t *As = nullptr, *Bs = nullptr, *planes = nullptr;
  unsigned long long* maxb = nullptr;
  int32_t *exps = nullptr, *dims = nullptr;   // exps: [Mpad + Npad]; dims: rows per row slot [cap_r] then columns per column slot [cap_c]
  int* bad = nullptr;
  OutlierRec* recs = nullptr;                 // [cap_r + cap_c][OZ2_REC_CAP]: A slots first, then B slots
  int* rec_cnt = nullptr;                     // [cap_r + cap_c]
  const unsigned char* d_maps = nullptr;      // uploaded by the caller (oz2_host_maps)
  std::vector<unsigned char> h_maps;
  int sms = 132;
  int launches = 0;
};

// K * (2^alpha)^2 <= 2^(floor(log2 P) - 1) < P / 2: the exact integer product is recovered from its residues
static int crt_alpha(int log2P, int64_t K) {
  int lgK = 0;
  while ((1ll << lgK) < K) ++lgK;
  const int alpha = (log2P - 1 - lgK) / 2;
  return alpha > 62 ? 62 : alpha;
}

// Number of moduli for an inner dimension K.  requested > 0: that many (clamped to the supported range).  requested <= 0: the
// smallest count whose operand truncation 2^-alpha (relative to the line maxima), grown by sqrt(K) over a dot product of
// length K, stays below half the classical fp64 rounding bound K 2^-53 of the same dot product: alpha >= 54 - ceil(lg K / 2).
int oz2_moduli_for(int64_t K, int requested) {
  if (requested > 0) return requested < CRT_MIN_T ? CRT_MIN_T : (requested > CRT_MAX_T ? CRT_MAX_T : requested);
  int log2P[CRT_MAX_T + 1];
  crt_constants(log2P, false);
  int lgK = 0;
  while ((1ll << lgK) < K) ++lgK;
  const int want = 54 - (lgK + 1) / 2;
  for (int T = CRT_MIN_T; T <= CRT_MAX_T; ++T)
    if (crt_alpha(log2P[T], K) >= want) return T;
  return CRT_MAX_T;
}

size_t oz2_scratch_bytes(int blk, int64_t K, int T, int cap_r, int cap_c, int max_tiles) {
  const int64_t sstride = (blk + BM - 1) / BM * BM;
  const int64_t Kpad = (K + BKB - 1) / BKB * BKB;
  const int64_t Mpad = sstride * cap_r, Npad = (sstride * cap_c + BN - 1) / BN * BN;
  return static_cast<size_t>(T) * (Mpad + Npad) * Kpad + static_cast<size_t>(T) * max_tiles * (BM * BN);
}

int oz2_tiles_per_block(int blk) {
  const int s = (blk + BM - 1) / BM * BM;
  return (s / BM) * ((s + BN - 1) / BN);
}

// Creates the engine and its scratch (stream-ordered allocations).  cap_r / cap_c = row / column slots held at once.
cudaError_t oz2_create(Oz2Engine** out, int blk, int64_t K, int moduli, int cap_r, int cap_c, int max_tiles, int guard_range,
                       cudaStream_t stream) {
  *out = nullptr;
  const int T = oz2_moduli_for(K, moduli);
  int log2P[CRT_MAX_T + 1];
  OZ_CHECK(crt_constants(log2P));
  int alpha = crt_alpha(log2P[T], K);
  if (alpha < 8 || K >= (1 << 17) || cap_r <= 0 || cap_c <= 0 || max_tiles <= 0) return cudaErrorInvalidValue;
  std::unique_ptr<Oz2Engine> e(new Oz2Engine);
  e->T = T;
  e->alpha = alpha;
  e->crt_chunks = log2P[T] < 3 * CRT_CHUNK_BITS ? 3 : 4;
  e->blk = blk;
  e->sstride = (blk + BM - 1) / BM * BM;
  e->cap_r = cap_r;
  e->cap_c = cap_c;
  e->max_tiles = max_tiles;
  // auto mode: every non-zero element must keep >= 18 bits after the per-line scaling, which bounds the error of every product
  // term by 2^-17 of the term itself, i.e. the result by 2^-17 |A||B| element-wise (north-star tolerance 1e-5) in the worst
  // case; data of ordinary dynamic range sees the full alpha bits (1e-14 .. 1e-16)
  e->range_bits = guard_range ? std::max(1, alpha - 18) : 0;
  e->K = K;
  e->Kpad = (K + BKB - 1) / BKB * BKB;
  e->Mpad = static_cast<int64_t>(e->sstride) * cap_r;
  e->Npad = (static_cast<int64_t>(e->sstride) * cap_c + BN - 1) / BN * BN;
  e->a_stride = static_cast<size_t>(e->Mpad) * e->Kpad;
  e->b_stride = static_cast<size_t>(e->Npad) * e->Kpad;
  e->plane_stride = static_cast<size_t>(max_tiles) * (BM * BN);
  OZ_CHECK(configure_gemm_kernels());
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&e->sms, cudaDevAttrMultiProcessorCount, dev);
  auto alloc = [&](void** p, size_t n) { return cudaMallocAsync(p, n ? n : 16, stream); };
  cudaError_t err = cudaSuccess;
  const size_t lines = static_cast<size_t>(e->Mpad + e->Npad);
  if ((err = alloc(reinterpret_cast<void**>(&e->As), e->a_stride * T)) != cudaSuccess ||
      (err = alloc(reinterpret_cast<void**>(&e->Bs), e->b_stride * T)) != cudaSuccess ||
      (err = alloc(reinterpret_cast<void**>(&e->planes), e->plane_stride * T)) != cudaSuccess ||
      (err = alloc(reinterpret_cast<void**>(&e->maxb), lines * 8)) != cudaSuccess ||
      (err = alloc(reinterpret_cast<void**>(&e->exps), lines * 4)) != cudaSuccess ||
      (err = alloc(reinterpret_cast<void**>(&e->dims), static_cast<size_t>(cap_r + cap_c) * 4)) != cudaSuccess ||
      (err = alloc(reinterpret_cast<void**>(&e->recs), static_cast<size_t>(cap_r + cap_c) * OZ2_REC_CAP * sizeof(OutlierRec))) != cudaSuccess ||
      (err = alloc(reinterpret_cast<void**>(&e->rec_cnt), static_cast<size_t>(cap_r + cap_c) * sizeof(int))) != cudaSuccess ||
      (err = alloc(reinterpret_cast<void**>(&e->bad), sizeof(int))) != cudaSuccess) {
    Oz2Engine* raw = e.release();
    oz2_destroy(raw, stream);
    return err;
  }
  OZ_CHECK(cudaMemsetAsync(e->bad, 0, sizeof(int), stream));
  OZ_CHECK(cudaMemsetAsync(e->rec_cnt, 0, static_cast<size_t>(cap_r + cap_c) * sizeof(int), stream));
  // B' rows beyond the last column slot (Npad rounding to the 256-wide tile) are read by the last tile: keep them defined
  if (e->Npad > static_cast<int64_t>(e->sstride) * cap_c)
    for (int t = 0; t < T; ++t)
      OZ_CHECK(cudaMemsetAsync(e->Bs + e->b_stride * t + static_cast<size_t>(e->sstride) * cap_c * e->Kpad, 0,
                               static_cast<size_t>(e->Npad - static_cast<int64_t>(e->sstride) * cap_c) * e->Kpad, stream));
  // tensor maps: A' (box 128 rows), B' (box 256 rows: single-CTA kernel), B' (box 128 rows: each CTA of a pair loads half)
  e->h_maps.resize(static_cast<size_t>(3 * T) * 128);
  for (int t = 0; t < T; ++t) {
    if (!make_i8_map(&e->h_maps[static_cast<size_t>(t) * 128], e->As + e->a_stride * t, e->Kpad, e->Mpad, BM) ||
        !make_i8_map(&e->h_maps[static_cast<size_t>(T + t) * 128], e->Bs + e->b_stride * t, e->Kpad, e->Npad, BN) ||
        !make_i8_map(&e->h_maps[static_cast<size_t>(2 * T + t) * 128], e->Bs + e->b_stride * t, e->Kpad, e->Npad, BN / 2)) {
      Oz2Engine* raw = e.release();
      oz2_destroy(raw, stream);
      return cudaErrorInvalidValue;
    }
  }
  *out = e.release();
  return cudaSuccess;
}

void oz2_destroy(Oz2Engine* e, cudaStream_t stream) {
  if (!e) return;
  void* ptrs[] = {e->As, e->Bs, e->planes, e->maxb, e->exps, e->dims, e->bad, e->recs, e->rec_cnt};
  for (void* p : ptrs)
    if (p) cudaFreeAsync(p, stream);
  delete e;
}

const void* oz2_host_maps(const Oz2Engine* e, size_t* bytes) {
  *bytes = e->h_maps.size();
  return e->h_maps.data();
}
void oz2_set_device_maps(Oz2Engine* e, const void* d_maps) { e->d_maps = static_cast<const unsigned char*>(d_maps); }
const int* oz2_flag(const Oz2Engine* e) { return e->bad; }
int oz2_alpha(const Oz2Engine* e) { return e->alpha; }
int oz2_moduli(const Oz2Engine* e) { return e->T; }
int oz2_slot_stride(const Oz2Engine* e) { return e->sstride; }
int oz2_launches(Oz2Engine* e) {
  const int n = e->launches;
  e->launches = 0;
  return n;
}

// Prepares slots [slot0, slot0 + nslots) of the A side (is_a) or B side from `nblocks` device-resident block descriptors whose
// row0 (A) / col0 (B) already point into those slots.  d_dims = the slots' line counts (device, nslots ints).  need_zero: the
// blocks do not cover every (line, k) of the slots (absent k-blocks, K padding): the residue rows are cleared first.
cudaError_t oz2_prepare(Oz2Engine* e, bool is_a, const OzakiOperand* d_blocks, int nblocks, int max_rows, int max_cols, int slot0,
                        int nslots, const int32_t* d_dims, bool need_zero, cudaStream_t stream) {
  if (nslots <= 0) return cudaSuccess;
  if (slot0 < 0 || slot0 + nslots > (is_a ? e->cap_r : e->cap_c)) return cudaErrorInvalidValue;
  static_assert(sizeof(OzakiOperand) == sizeof(OzBlock), "OzakiOperand is the device block descriptor");
  const OzBlock* blocks = reinterpret_cast<const OzBlock*>(d_blocks);
  const size_t line0 = (is_a ? 0 : static_cast<size_t>(e->Mpad)) + static_cast<size_t>(slot0) * e->sstride;
  const size_t nlines = static_cast<size_t>(nslots) * e->sstride;
  // the tables are indexed by buffer line: A lines first, then B lines
  unsigned long long* maxb = e->maxb + (is_a ? 0 : e->Mpad);
  int32_t* exps = e->exps + (is_a ? 0 : e->Mpad);
  OZ_CHECK(cudaMemsetAsync(e->maxb + line0, 0, nlines * 8, stream));
  OZ_CHECK(cudaMemsetAsync(e->rec_cnt + (is_a ? 0 : e->cap_r) + slot0, 0, static_cast<size_t>(nslots) * sizeof(int), stream));
  OZ_CHECK(cudaMemcpyAsync(e->dims + (is_a ? 0 : e->cap_r) + slot0, d_dims, static_cast<size_t>(nslots) * 4, cudaMemcpyDeviceToDevice, stream));
  int8_t* res = is_a ? e->As : e->Bs;
  const size_t stride = is_a ? e->a_stride : e->b_stride;
  if (need_zero)
    for (int t = 0; t < e->T; ++t)
      OZ_CHECK(cudaMemsetAsync(res + stride * t + static_cast<size_t>(slot0) * e->sstride * e->Kpad, 0, nlines * e->Kpad, stream));
  if (nblocks > 0) {
    const AbsmaxGrid g(max_rows, max_cols);
    OZ_CHECK(for_block_chunks(nblocks, [&](int off, int cnt) {
      absmax_kernel<<<dim3(g.tiles, cnt), 256, 0, stream>>>(blocks + off, maxb, nullptr, is_a ? 1 : 0, g.ts);
    }));
    e->launches += 1;
  }
  // the exponent pass flags non-finite lines only; elements too far below their line maximum are handled one by one (OutlierRec)
  exp_kernel<<<static_cast<unsigned>((nlines + 255) / 256), 256, 0, stream>>>(e->maxb + line0, nullptr, e->exps + line0, nullptr,
                                                                               static_cast<int>(nlines), 0, e->bad);
  OZ_CHECK(cudaGetLastError());
  e->launches += 1;
  if (nblocks > 0) {
    // "line" = row of A / column of B, "k" = the other index
    const int max_l = is_a ? max_rows : max_cols, max_k = is_a ? max_cols : max_rows;
    const int tk = (max_k + 127) / 128, tl = (max_l + 31) / 32;
    OZ_CHECK(for_block_chunks(nblocks, [&](int off, int cnt) {
      residue_kernel<<<dim3(tl * tk, cnt), 256, 0, stream>>>(blocks + off, exps, res, stride, static_cast<int>(e->Kpad), e->T, e->alpha,
                                                             is_a ? 1 : 0, tk, e->bad, e->range_bits,
                                                             e->recs + static_cast<size_t>(is_a ? 0 : e->cap_r) * OZ2_REC_CAP,
                                                             e->rec_cnt + (is_a ? 0 : e->cap_r), e->sstride);
    }));
    e->launches += 1;
  }
  return cudaSuccess;
}

// One job: C blocks (+)= A' B' over the tiles of d_tiles (buffer tile coordinates (tm, tn), device array; the order is the
// execution order, so the caller bands it for L2 reuse), written through d_ctab[rslot * cap_c + cslot] (nullptr = not part of
// this job).  Lists longer than the plane capacity are processed in consecutive pieces.  ms_gemm (optional) accumulates the
// residue GEMM launch time (events, synchronises): used for the roofline figure only.
void oz2_set_ksplit(Oz2Engine* e, int level) { e->ksplit = level; }
void oz2_set_paired(Oz2Engine* e, bool paired) { e->paired = paired && (e->max_tiles % 2 == 0) && (e->Mpad % (2 * BM) == 0); }
bool oz2_paired(const Oz2Engine* e) { return e->paired; }

cudaError_t oz2_multiply(Oz2Engine* e, const int2* d_tiles, int ntiles, double* const* d_ctab, cudaStream_t stream, double* ms_gemm,
                         cudaEvent_t ev0, cudaEvent_t ev1) {
  if (ntiles <= 0) return cudaSuccess;
  if (e->d_maps == nullptr) return cudaErrorInvalidValue;
  if (e->paired && (ntiles & 1)) return cudaErrorInvalidValue;
  OzakiGemmParams p{};
  p.tmaps = e->d_maps;
  p.Kpad = static_cast<int32_t>(e->Kpad);
  p.kstep = BKB;
  p.kc0 = 0;
  p.nkc = static_cast<int32_t>(e->Kpad / BKB);
  p.npairs = 1;
  p.tiles_m = static_cast<int32_t>(e->Mpad / BM);
  p.tiles_n = static_cast<int32_t>(e->Npad / BN);
  p.nmod = e->T;
  p.planes = e->planes;
  p.plane_stride = e->plane_stride;
  p.gate = e->bad;
  for (int t = 0; t < e->T; ++t) {
    p.mod_p[t] = kCrtModuli[t];
    p.mod_inv[t] = 1.0 / kCrtModuli[t];
  }
  for (int off = 0; off < ntiles; off += e->max_tiles) {
    const int cnt = std::min(e->max_tiles, ntiles - off);
    p.tile_list = d_tiles + off;
    p.ntiles_list = cnt;
    const int64_t nitems = static_cast<int64_t>(cnt) * e->T;
    if (ms_gemm) OZ_CHECK(cudaEventRecord(ev0, stream));
    if (e->paired) {  // one cluster of two CTAs per (modulus, tile pair) work item
      const int64_t npair_items = nitems / 2;
      const unsigned clusters = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(npair_items, e->sms / 2)));
      // K-split order (opt-in, oz2_set_ksplit): only for lists long enough that every CTA pair sweeps several tiles per (modulus, half)
      const bool ks = (p.nkc % 2 == 0) && (e->ksplit >= 2 || (e->ksplit == 1 && p.nkc >= 64 && (cnt / 2) >= 4 * static_cast<int>(clusters)));
      if (ks) ozaki2_gemm_2sm_kernel<true><<<2 * clusters, GEMM_THREADS_P, GEMM_SMEM_BYTES, stream>>>(p);
      else ozaki2_gemm_2sm_kernel<false><<<2 * clusters, GEMM_THREADS_P, GEMM_SMEM_BYTES, stream>>>(p);
    } else {
      ozaki_gemm_i8_kernel<false><<<static_cast<unsigned>(std::min<int64_t>(nitems, e->sms)), GEMM_THREADS_P, GEMM_SMEM_BYTES, stream>>>(p);
    }
    OZ_CHECK(cudaGetLastError());
    if (ms_gemm) {
      OZ_CHECK(cudaEventRecord(ev1, stream));
      OZ_CHECK(cudaEventSynchronize(ev1));
      float ms = 0.f;
      OZ_CHECK(cudaEventElapsedTime(&ms, ev0, ev1));
      *ms_gemm += ms;
    }
    auto crt = e->crt_chunks == 3 ? crt_kernel<3> : crt_kernel<4>;
    crt<<<static_cast<unsigned>(cnt) * 8u, 256, 0, stream>>>(e->planes, e->plane_stride, e->T, d_tiles + off, e->exps, e->exps + e->Mpad,
                                                              2 * e->alpha, d_ctab, e->dims, e->dims + e->cap_r, e->sstride, e->cap_c,
                                                              e->bad);
    OZ_CHECK(cudaGetLastError());
    e->launches += 2;
  }
  return cudaSuccess;
}

// Adds the exact products of the outlier elements recorded while the slots were prepared to the output blocks of a job (to be
// called behind oz2_multiply of the same job, on the same stream).  No-op for an engine without the range guard.
cudaError_t oz2_fixup(Oz2Engine* e, const Oz2FixOut* d_outs, int nouts, const Oz2FixSrc* d_srcs, cudaStream_t stream) {
  if (nouts <= 0 || e->range_bits <= 0) return cudaSuccess;
  oz2_fixup_kernel<<<nouts, 256, 0, stream>>>(d_outs, d_srcs, e->recs, e->rec_cnt, e->cap_r, e->sstride, e->exps, e->range_bits, e->bad);
  OZ_CHECK(cudaGetLastError());
  e->launches += 1;
  return cudaSuccess;
}

// fp32 multiply on wgmma tf32 with the 3xTF32 split (gemm_algo = 3).  Inputs are rounded to fp32, products are
// accumulated in fp32 by the tensor cores, the result is stored into the fp64 output blocks.
cudaError_t tf32x3_gemm(const OzakiOperand* a_blocks, int na, const OzakiOperand* b_blocks, int nb, int64_t M, int64_t K, int64_t N,
                        double* const* h_ctab, int blk, int nbr, int nbc, int* launches, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return cudaSuccess;
  const int64_t Mpad = (M + BM - 1) / BM * BM, Npad = (N + BN - 1) / BN * BN, Kpad = (K + 31) / 32 * 32;
  OZ_CHECK(configure_gemm_kernels());
  std::vector<OzBlock> ha(na), hb(nb);
  int max_ar = 1, max_ac = 1, max_br = 1, max_bc = 1;
  for (int i = 0; i < na; ++i) {
    ha[i] = OzBlock{a_blocks[i].v, a_blocks[i].rows, a_blocks[i].cols, a_blocks[i].row0, a_blocks[i].col0, a_blocks[i].isT, {0}};
    max_ar = std::max(max_ar, a_blocks[i].rows);
    max_ac = std::max(max_ac, a_blocks[i].cols);
  }
  for (int i = 0; i < nb; ++i) {
    hb[i] = OzBlock{b_blocks[i].v, b_blocks[i].rows, b_blocks[i].cols, b_blocks[i].row0, b_blocks[i].col0, b_blocks[i].isT, {0}};
    max_br = std::max(max_br, b_blocks[i].rows);
    max_bc = std::max(max_bc, b_blocks[i].cols);
  }
  AsyncBuf d_ab(stream), d_bb(stream), d_A(stream), d_B(stream), d_maps(stream), d_ctab(stream), d_corr(stream);
  OZ_CHECK(d_ab.alloc(sizeof(OzBlock) * na));
  OZ_CHECK(d_bb.alloc(sizeof(OzBlock) * nb));
  OZ_CHECK(cudaMemcpyAsync(d_ab.p, ha.data(), sizeof(OzBlock) * na, cudaMemcpyHostToDevice, stream));
  OZ_CHECK(cudaMemcpyAsync(d_bb.p, hb.data(), sizeof(OzBlock) * nb, cudaMemcpyHostToDevice, stream));
  // operand means (absent blocks count as zeros: the mean is over the full M x K / K x N extent) and the correction vectors
  OZ_CHECK(d_corr.alloc(sizeof(double) * (2 + Mpad + Npad)));
  OZ_CHECK(cudaMemsetAsync(d_corr.p, 0, sizeof(double) * (2 + Mpad + Npad), stream));
  double* totals = static_cast<double*>(d_corr.p);
  double* row_corr = totals + 2;
  double* col_corr = row_corr + Mpad;
  const double inv_a = 1.0 / (static_cast<double>(M) * static_cast<double>(K)), inv_b = 1.0 / (static_cast<double>(K) * static_cast<double>(N));
  // centring needs A = A' + muA 11^T element for element, absent blocks (implicit zeros) included: it is applied when the
  // blocks cover both operands completely (the dense case the fp32 configuration is about); otherwise the means stay 0
  int64_t area_a = 0, area_b = 0;
  for (int i = 0; i < na; ++i) area_a += static_cast<int64_t>(a_blocks[i].rows) * a_blocks[i].cols;
  for (int i = 0; i < nb; ++i) area_b += static_cast<int64_t>(b_blocks[i].rows) * b_blocks[i].cols;
  const bool centre = area_a == M * K && area_b == K * N;
  if (centre) {
    const unsigned pieces_a = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(64, (static_cast<int64_t>(max_ar) * max_ac + 4095) / 4096)));
    OZ_CHECK(for_block_chunks(na, [&](int off, int cnt) {
      block_sum_kernel<<<dim3(pieces_a, cnt), 256, 0, stream>>>(static_cast<const OzBlock*>(d_ab.p) + off, totals);
    }));
    const unsigned pieces_b = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(64, (static_cast<int64_t>(max_br) * max_bc + 4095) / 4096)));
    OZ_CHECK(for_block_chunks(nb, [&](int off, int cnt) {
      block_sum_kernel<<<dim3(pieces_b, cnt), 256, 0, stream>>>(static_cast<const OzBlock*>(d_bb.p) + off, totals + 1);
    }));
    *launches += 2;
  }
  const size_t a_elems = static_cast<size_t>(Mpad) * Kpad, b_elems = static_cast<size_t>(Npad) * Kpad;
  OZ_CHECK(d_A.alloc(a_elems * 2 * sizeof(float)));
  OZ_CHECK(d_B.alloc(b_elems * 2 * sizeof(float)));
  OZ_CHECK(cudaMemsetAsync(d_A.p, 0, a_elems * 2 * sizeof(float), stream));
  OZ_CHECK(cudaMemsetAsync(d_B.p, 0, b_elems * 2 * sizeof(float), stream));
  float* Ahi = static_cast<float*>(d_A.p);
  float* Alo = Ahi + a_elems;
  float* Bhi = static_cast<float*>(d_B.p);
  float* Blo = Bhi + b_elems;
  {
    const int tk = (max_ac + 127) / 128, tl = (max_ar + 31) / 32;
    OZ_CHECK(for_block_chunks(na, [&](int off, int cnt) {
      slice_tf32_kernel<<<dim3(tl * tk, cnt), 256, 0, stream>>>(static_cast<const OzBlock*>(d_ab.p) + off, Ahi, Alo, static_cast<int>(Kpad), 1, tk,
                                                                centre ? totals : nullptr, inv_a, row_corr);
    }));
    const int tkb = (max_br + 127) / 128, tlb = (max_bc + 31) / 32;
    OZ_CHECK(for_block_chunks(nb, [&](int off, int cnt) {
      slice_tf32_kernel<<<dim3(tlb * tkb, cnt), 256, 0, stream>>>(static_cast<const OzBlock*>(d_bb.p) + off, Bhi, Blo, static_cast<int>(Kpad), 0, tkb,
                                                                  centre ? totals + 1 : nullptr, inv_b, col_corr);
    }));
    const int mx = static_cast<int>(std::max(Mpad, Npad));
    tf32_corr_kernel<<<(mx + 255) / 256, 256, 0, stream>>>(totals, inv_a, inv_b, static_cast<double>(K), row_corr, static_cast<int>(Mpad), col_corr,
                                                           static_cast<int>(Npad));
    OZ_CHECK(cudaGetLastError());
    *launches += 3;
  }
  std::vector<unsigned char> hmaps(4 * 128);
  if (!make_f32_map(&hmaps[0], Ahi, Kpad, Mpad, BM) || !make_f32_map(&hmaps[128], Alo, Kpad, Mpad, BM) ||
      !make_f32_map(&hmaps[256], Bhi, Kpad, Npad, BN) || !make_f32_map(&hmaps[384], Blo, Kpad, Npad, BN))
    return cudaErrorInvalidValue;
  OZ_CHECK(d_maps.alloc(hmaps.size()));
  OZ_CHECK(cudaMemcpyAsync(d_maps.p, hmaps.data(), hmaps.size(), cudaMemcpyHostToDevice, stream));
  OZ_CHECK(d_ctab.alloc(sizeof(double*) * nbr * nbc));
  OZ_CHECK(cudaMemcpyAsync(d_ctab.p, h_ctab, sizeof(double*) * nbr * nbc, cudaMemcpyHostToDevice, stream));
  OzakiGemmParams p{};
  p.tmaps = static_cast<const unsigned char*>(d_maps.p);
  p.ctab = static_cast<double* const*>(d_ctab.p);
  p.M = static_cast<int32_t>(M);
  p.N = static_cast<int32_t>(N);
  p.Kpad = static_cast<int32_t>(Kpad);
  p.blk = blk;
  p.nbr = nbr;
  p.nbc = nbc;
  p.kstep = 32;
  p.accumulate = 0;
  p.diag_scale = 1.0;
  p.row_scale = row_corr;   // fp32 path: additive mean corrections, applied with the first K chunk
  p.col_scale = col_corr;
  // small terms first: lo*hi, hi*lo, then hi*hi
  p.npairs = 3;
  p.pair_a[0] = 1; p.pair_b[0] = 2;
  p.pair_a[1] = 0; p.pair_b[1] = 3;
  p.pair_a[2] = 0; p.pair_b[2] = 2;
  p.tiles_m = static_cast<int32_t>(Mpad / BM);
  p.tiles_n = static_cast<int32_t>(Npad / BN);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t ntiles = static_cast<int64_t>(p.tiles_m) * p.tiles_n;
  // fp32 accumulation in the tensor core truncates: besides the centring above (which removes the bias for same-signed data), K
  // is cut into chunks of 2048 whose fp32 tile sums are re-accumulated in fp64 by the epilogue (read-modify-write of C), which
  // keeps the random-walk part of the truncation error below 1e-5 of max|C| even for heavily cancelling data.
  const int stages_total = static_cast<int>(Kpad / 32);
  const int chunk = 2048 / 32;
  for (int kc = 0; kc < stages_total; kc += chunk) {
    p.kc0 = kc;
    p.nkc = std::min(chunk, stages_total - kc);
    p.accumulate = kc == 0 ? 0 : 1;
    ozaki_gemm_i8_kernel<true><<<static_cast<unsigned>(std::min<int64_t>(ntiles, sms)), GEMM_THREADS_P, GEMM_SMEM_BYTES, stream>>>(p);
    OZ_CHECK(cudaGetLastError());
    *launches += 1;
  }
  return cudaSuccess;
}

}  // namespace matrel
