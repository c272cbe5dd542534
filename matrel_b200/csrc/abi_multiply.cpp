// Block multiply: planning (LocalMatrix.matrixMultiplication dispatch), the fused DMMA launch incl. the pipelined chunks,
// the wgmma paths, sparse x dense and sparse x sparse partial products, and the mr_matrix_multiply entry point.
#include "host.h"

using namespace matrel;
using namespace mrhost;

namespace {

// ------------------------------------------------------------------------------------------------
// block product planning (LocalMatrix.matrixMultiplication, LocalMatrix.scala:889-914)
// ------------------------------------------------------------------------------------------------
// How LocalMatrix.matrixMultiplication computes one partial product a x b (LocalMatrix.scala:889-914)
enum PairKind { PAIR_GEMM = 0, PAIR_SPMM = 1, PAIR_SPSP = 2 };
int pair_kind(const Block& a, const Block& b) {
  if (a.dense()) return PAIR_GEMM;  // dense x dense, dense x sparse.toDense (:891-892)
  if (b.dense()) return PAIR_SPMM;  // sparse x dense (:893-899)
  const double s1 = a.valuesLen * 1.0 / (static_cast<double>(a.numRows) * a.numCols);
  const double s2 = b.valuesLen * 1.0 / (static_cast<double>(b.numRows) * b.numCols);
  if (s1 > 0.1) return PAIR_GEMM;   // :903-904
  if (s2 > 0.1) return PAIR_SPMM;   // :906-907
  return PAIR_SPSP;                 // :909-911
}

// Dense x sparse pairs whose right block is at most this dense are computed from its stored entries (run_dense_sparse) instead of
// its dense image, when their output block has no pair on the dense engines (DESIGN section 4.5.2: where the value comes from).
constexpr double kDspmmMaxDensity = 0.02;

// Metadata-only part of the rule: the density and the dims the dense x sparse kernel takes.
bool dspmm_candidate(const Block& a, const Block& b) {
  if (!a.dense() || b.dense()) return false;
  if (b.numRows <= 0 || b.numRows > kSpmmMaxDim || b.numCols < 128 || b.numCols > kSpmmMaxDim) return false;
  if (a.numRows < 16 || a.numRows > kSpmmMaxDim || (a.numRows % 2) != 0) return false;
  return b.valuesLen * 1.0 / (static_cast<double>(b.numRows) * b.numCols) <= kDspmmMaxDensity;
}

// Where one partial product of an output block is computed
enum Route : uint8_t {
  ROUTE_GEMM,       // the dense engines; a sparse operand through its dense image
  ROUTE_SPMM,       // sparse x dense (the n == 1 SpMV case is the same kernel); a sparse right operand through its dense image
  ROUTE_SPSP,       // low-density sparse x sparse in a block made of such pairs only (run_sparse_chains)
  ROUTE_SPSP_SPMM,  // low-density sparse x sparse next to other partials: sparse x the dense image of the right operand
  ROUTE_DSPMM,      // dense x low-density sparse from the stored entries (run_dense_sparse)
  ROUTE_MV,         // matrix x thin matrix (run_matvec)
};

struct PlanPair {
  const Block* a;
  const Block* b;
  int32_t k, kb;  // the blocks are a = (rid, k) and b = (kb, cid); k == kb except in the outer product
  Route route;
};

struct OutPlan {
  int32_t rid, cid;
  int32_t m = -1, n = -1;
  std::vector<PlanPair> pairs;  // ascending k
  bool has(Route r) const {
    return std::any_of(pairs.begin(), pairs.end(), [r](const PlanPair& p) { return p.route == r; });
  }
  bool only(Route r) const {
    return std::all_of(pairs.begin(), pairs.end(), [r](const PlanPair& p) { return p.route == r; });
  }
  bool has_spmm() const { return has(ROUTE_SPMM) || has(ROUTE_SPSP_SPMM); }
};

// The output blocks of left x right and the route of every partial product, from block metadata only (the blocks may be
// host-resident).  outer: the outer-product paths (MatfastExecution.scala:714-721 -> helper :175-221), every left block x every
// right block with no reduce, the last duplicate key winning as when collected into a map (reference defect B1, DuplicateLeft
// throws, is not reproduced: both branches return what DuplicateRight returns).  Else matrixMultiplyGeneral (helper :235-263):
// join on k, then reduce by (i, j) in ascending k.
std::vector<OutPlan> plan_multiply(const mr_matrix* left, const mr_matrix* right, bool outer, bool mv) {
  std::vector<OutPlan> plans;
  std::map<std::pair<int32_t, int32_t>, size_t> index;
  auto add_pair = [&](int32_t rid, int32_t cid, const Block& a, const Block& b, int32_t k, int32_t kb) {
    // shape checks: BLAS.gemmddd / gemmsdd `require`s (BLAS.scala:338-343, 363-366)
    MR_REQUIRE(a.numCols == b.numRows, MR_EDIM, "The columns of A don't match the rows of B. A: %d, B: %d", a.numCols,
               b.numRows);
    auto it = index.find({rid, cid});
    if (it == index.end()) {
      it = index.emplace(std::make_pair(rid, cid), plans.size()).first;
      plans.emplace_back();
    } else if (outer) {
      plans[it->second] = OutPlan();
    }
    OutPlan& o = plans[it->second];
    o.rid = rid;
    o.cid = cid;
    if (o.m < 0) {
      o.m = a.numRows;
      o.n = b.numCols;
    } else {
      // LocalMatrix.add `require`s on the partial products (LocalMatrix.scala:36-41)
      MR_REQUIRE(o.m == a.numRows, MR_EDIM,
                 "Matrix A and B must have the same number of rows. But found A.numRows = %d, B.numRows = %d", o.m,
                 a.numRows);
      MR_REQUIRE(o.n == b.numCols, MR_EDIM,
                 "Matrix A and B must have the same number of cols. But found A.numCols = %d, B.numCols = %d", o.n,
                 b.numCols);
    }
    Route r = ROUTE_MV;  // the matrix x vector route keeps every pair as it is
    if (!mv) {
      const int kind = pair_kind(a, b);
      r = kind == PAIR_SPMM ? ROUTE_SPMM : kind == PAIR_SPSP ? ROUTE_SPSP : dspmm_candidate(a, b) ? ROUTE_DSPMM : ROUTE_GEMM;
    }
    o.pairs.push_back(PlanPair{&a, &b, k, kb, r});
  };
  if (outer) {
    for (auto& l : left->blocks)
      for (auto& r : right->blocks) add_pair(l.first.first, r.first.second, l.second, r.second, l.first.second, r.first.first);
  } else {
    std::map<int32_t, std::vector<std::pair<int32_t, const Block*>>> rights;  // k -> (j, B(k,j))
    for (auto& r : right->blocks) rights[r.first.first].push_back({r.first.second, &r.second});
    // left->blocks is ordered by (i, k): iterating it visits k ascending within each i
    for (auto& l : left->blocks) {
      auto rit = rights.find(l.first.second);
      if (rit == rights.end()) continue;
      for (auto& jb : rit->second) add_pair(l.first.first, jb.first, l.second, *jb.second, l.first.second, l.first.second);
    }
  }
  // Dense x sparse candidates take the stored-entry route only in a block with no pair on the dense engines, else they are
  // densified in their places among its GEMM pairs (the summation order of the product without the route).  Low-density sparse x
  // sparse pairs next to any other partial make a dense block sum whatever the partial's own format (LocalMatrix.add), so there
  // they are sparse x dense products of the densified right operand; a block made of such pairs ONLY replays the reference's
  // format rules (run_sparse_chains).
  for (OutPlan& o : plans) {
    const bool gemm = o.has(ROUTE_GEMM);
    for (PlanPair& p : o.pairs)
      if (gemm && p.route == ROUTE_DSPMM) p.route = ROUTE_GEMM;
    if (!o.only(ROUTE_SPSP))
      for (PlanPair& p : o.pairs)
        if (p.route == ROUTE_SPSP) p.route = ROUTE_SPSP_SPMM;
  }
  return plans;
}

// What the plans decide for the whole product: the DMMA tile variant (large tiles unless they cannot fill the 132 SMs), and
// whether to try the Ozaki-II engine (gemm_algo 4, or auto with >= 2^33 flop; a block with sparse partials next to dense ones
// keeps the whole product off it).
MultiplyDecisions decide(const mr_context* ctx, const std::vector<OutPlan>& plans, int mv) {
  MultiplyDecisions d;
  d.mv = mv;
  int64_t flops = 0, tiles128 = 0;
  bool mixed = false;
  for (const OutPlan& o : plans) {
    if (!o.has(ROUTE_GEMM) || o.m == 0 || o.n == 0) continue;
    for (const PlanPair& p : o.pairs)
      if (p.route == ROUTE_GEMM) flops += 2ll * p.a->numRows * p.b->numCols * p.a->numCols;
    tiles128 += static_cast<int64_t>((o.m + 127) / 128) * ((o.n + 127) / 128);
    mixed = mixed || !o.only(ROUTE_GEMM);
  }
  d.variant = tiles128 >= 2 * 132 ? GEMM_128x128 : GEMM_64x64;
  d.oz2 = !mixed && (ctx->gemm_algo == 4 || (ctx->gemm_algo == 0 && flops >= (1ll << 33)));
  return d;
}

// The dense images the routes read (GEMM operands, right operands of sparse x dense pairs), made once per sparse block; the pairs
// then point at them.  `temps` keeps them alive until the launches are enqueued (a deque: growth must not move them).
void densify_operands(mr_context* ctx, std::vector<OutPlan>& plans, std::deque<Block>& temps) {
  std::map<const Block*, const Block*> densified;
  auto dense_of = [&](const Block* b) {
    if (b->dense()) return b;
    auto it = densified.find(b);
    if (it == densified.end()) {
      temps.push_back(densify(ctx, *b));
      it = densified.emplace(b, &temps.back()).first;
    }
    return it->second;
  };
  for (OutPlan& o : plans)
    for (PlanPair& p : o.pairs)
      if (p.route == ROUTE_GEMM) {
        p.a = dense_of(p.a);
        p.b = dense_of(p.b);
      } else if (p.route == ROUTE_SPMM || p.route == ROUTE_SPSP_SPMM) {
        p.b = dense_of(p.b);
      }
}

// Times the launches enqueued between its construction and stop() when the time_kernels option is on: last_gemm_ms is that time,
// gemm_ms_total accumulates it.
struct KernelTimer {
  mr_context* ctx;
  explicit KernelTimer(mr_context* c) : ctx(c) {
    if (ctx->time_kernels) CUDA_CHECK(cudaEventRecord(ctx->ev0, ctx->stream));
  }
  void stop() {
    if (!ctx->time_kernels) return;
    CUDA_CHECK(cudaEventRecord(ctx->ev1, ctx->stream));
    CUDA_CHECK(cudaEventSynchronize(ctx->ev1));
    float ms = 0.f;
    CUDA_CHECK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    ctx->stats.last_gemm_ms = ms;
    ctx->stats.gemm_ms_total += ms;
  }
};

// Consecutive slots 0, 1, ... of the block rows and the block columns that hold the output blocks plans[i], i in `outs` (a rank
// of the process grid owns every pr-th block row and pc-th block column: slicing and multiplying the absent ones would only
// produce zeros).
void compact_slots(const std::vector<OutPlan>& plans, const std::vector<size_t>& outs, std::map<int32_t, int>& crow,
                   std::map<int32_t, int>& ccol) {
  for (size_t i : outs) {
    crow.emplace(plans[i].rid, 0);
    ccol.emplace(plans[i].cid, 0);
  }
  int s = 0;
  for (auto& kv : crow) kv.second = s++;
  s = 0;
  for (auto& kv : ccol) kv.second = s++;
}

// gemm_algo 2: the dense pairs of every output block through the wgmma int8 Ozaki pipeline (gemm_ozaki.cu).
// gemm_algo 3: the same through the 3xTF32 fp32 pipeline.
// Returns false when the problem does not fit its regular-grid assumptions or holds Inf/NaN (caller uses DMMA).
bool try_ozaki(mr_context* ctx, const std::vector<OutPlan>& plans, const std::vector<double*>& cptr, int32_t blkSize, int64_t M,
               int64_t K, int64_t N, bool outer) {
  const bool tf32 = ctx->gemm_algo == 3;
  const int S_eff = std::min(7, std::max(2, ctx->ozaki_slices > 0 ? ctx->ozaki_slices : 7));
  // s32 accumulator bound: up to S pairs x K terms of |digit product| <= 2^14 land in one accumulator
  if (M <= 0 || K <= 0 || N <= 0 || M > INT32_MAX || N > INT32_MAX || K > INT32_MAX / 2) return false;
  if (!tf32 && K * S_eff >= (1 << 17)) return false;
  std::vector<size_t> outs;
  for (size_t i = 0; i < plans.size(); ++i)
    if (plans[i].has(ROUTE_GEMM)) outs.push_back(i);
  std::map<int32_t, int> crow, ccol;
  compact_slots(plans, outs, crow, ccol);
  if (crow.empty()) return false;
  const int64_t nbr = static_cast<int64_t>(crow.size()), nbc = static_cast<int64_t>(ccol.size());
  if (nbr * nbc > (1 << 24)) return false;
  const int64_t last_r = crow.rbegin()->first, last_c = ccol.rbegin()->first;
  if (last_r * static_cast<int64_t>(blkSize) >= M || last_c * static_cast<int64_t>(blkSize) >= N) return false;
  const int64_t Mc = (nbr - 1) * blkSize + std::min<int64_t>(blkSize, M - last_r * blkSize);
  const int64_t Nc = (nbc - 1) * blkSize + std::min<int64_t>(blkSize, N - last_c * blkSize);
  std::vector<double*> ctab(static_cast<size_t>(nbr * nbc), nullptr);
  std::map<const Block*, int> ia, ib;
  std::vector<OzakiOperand> va, vb;
  for (size_t i : outs) {
    const OutPlan& o = plans[i];
    const int32_t cr = crow[o.rid], cc = ccol[o.cid];
    // every block row / column but the last must be a full blkSize tall / wide (the kernel finds blocks by division)
    if (o.m != ((o.rid == last_r) ? Mc - (nbr - 1) * blkSize : blkSize) || o.n != ((o.cid == last_c) ? Nc - (nbc - 1) * blkSize : blkSize))
      return false;
    if (o.has_spmm()) return false;  // mixed dense / sparse partial sums stay on the exact path
    ctab[static_cast<size_t>(cr) * nbc + cc] = cptr[i];
    for (const PlanPair& g : o.pairs) {
      const int64_t k0 = outer ? 0 : static_cast<int64_t>(g.k) * blkSize;
      if (k0 + g.a->numCols > K || g.a->numCols != g.b->numRows) return false;
      if (!ia.count(g.a)) {
        ia[g.a] = 1;
        va.push_back(OzakiOperand{g.a->values.ptr<double>(), g.a->numRows, g.a->numCols, cr * blkSize, static_cast<int32_t>(k0),
                                  static_cast<uint8_t>(g.a->isT), {0}});
      }
      if (!ib.count(g.b)) {
        ib[g.b] = 1;
        vb.push_back(OzakiOperand{g.b->values.ptr<double>(), g.b->numRows, g.b->numCols, static_cast<int32_t>(k0), cc * blkSize,
                                  static_cast<uint8_t>(g.b->isT), {0}});
      }
    }
  }
  if (va.empty() || vb.empty()) return false;
  int launches = 0, nonfinite = 0;
  KernelTimer timer(ctx);
  if (tf32)
    CUDA_CHECK(tf32x3_gemm(va.data(), static_cast<int>(va.size()), vb.data(), static_cast<int>(vb.size()), Mc, K, Nc, ctab.data(),
                           blkSize, static_cast<int>(nbr), static_cast<int>(nbc), &launches, &nonfinite, ctx->stream));
  else
    CUDA_CHECK(ozaki_gemm_f64(va.data(), static_cast<int>(va.size()), vb.data(), static_cast<int>(vb.size()), Mc, K, Nc,
                              ctx->ozaki_slices > 0 ? ctx->ozaki_slices : 7, ctab.data(), blkSize, static_cast<int>(nbr),
                              static_cast<int>(nbc), &launches, &nonfinite, ctx->stream));
  note_launch(ctx, launches);
  if (nonfinite) return false;
  ctx->stats.gemm_launches += 1;
  timer.stop();
  return true;
}

// The largest (row panel x column panel) job grid cap_r x cap_c of an nr x nc grid of output blocks whose residue scratch fits the
// ozaki_scratch_mb budget (0 = 16 GiB), halving the longer side first.  Returns false when not even 1 x 1 fits.  `bytes`: that
// scratch (an upper bound of what oz2_create allocates).  share_ab: the residues of one operand (a Gram product, nr == nc).
bool oz2_capacity(const mr_context* ctx, int32_t blk, int64_t K, int T, int nr, int nc, int& cap_r, int& cap_c, size_t* bytes = nullptr,
                  bool share_ab = false) {
  const int ss = (blk + kOz2TileM - 1) / kOz2TileM * kOz2TileM;
  auto panel_tiles = [&](int ncr, int ncc) {  // upper bound of a panel's tile count
    const int64_t tm = static_cast<int64_t>(ncr) * (ss / kOz2TileM);
    const int64_t tn = (static_cast<int64_t>(ncc) * ss + kOz2TileN - 1) / kOz2TileN;
    return tm * tn;
  };
  const int64_t plane_cap_tiles = std::max<int64_t>(64, (2ll << 30) / (static_cast<int64_t>(T) * kOz2TileM * kOz2TileN));
  const size_t budget = static_cast<size_t>(ctx->ozaki_scratch_mb > 0 ? ctx->ozaki_scratch_mb : 16384) << 20;
  cap_r = nr;
  cap_c = nc;
  auto max_tiles_for = [&](int r, int cc_) { return static_cast<int>(std::min<int64_t>(plane_cap_tiles, panel_tiles(r, cc_))); };
  size_t need;
  while ((need = oz2_scratch_bytes(blk, K, T, cap_r, cap_c, max_tiles_for(cap_r, cap_c), share_ab)) > budget) {
    if (cap_r == 1 && cap_c == 1) return false;
    if (cap_r >= cap_c) cap_r = (cap_r + 1) / 2;
    else cap_c = (cap_c + 1) / 2;
  }
  if (bytes) *bytes = need;
  return true;
}

// The triangular tile rule of a diagonal block of a Gram product (DESIGN section 4.1.2): keep the Ozaki-II tile (a, b) of a job's
// buffer when it holds an element (r, c) of the block with r <= c.  The block starts at buffer row row0 and column col0 and has
// n columns.  Tiles run across slot boundaries when the slot stride is not a multiple of kOz2TileN, so the rule is applied per
// element, block by block, and the union is kept.  With the CTA-pair kernel the caller asks for the first tile of a vertical pair,
// so that pairs stay whole.
bool gram_tile_kept(int a, int b, int64_t row0, int64_t col0, int n) {
  const int64_t r_min = std::max<int64_t>(0, static_cast<int64_t>(a) * kOz2TileM - row0);
  const int64_t c_max = std::min<int64_t>(n, static_cast<int64_t>(b + 1) * kOz2TileN - col0) - 1;
  return r_min <= c_max;
}

// ------------------------------------------------------------------------------------------------
// gemm_algo 0 (auto) / 4: the dense pairs through the Ozaki-II job engine (gemm_ozaki.cu), group by group.
//
// plan():    checks that the product fits the engine's regular-grid assumptions, assigns one residue slot per block row of A /
//            block column of B that has output blocks, and turns every launch group (the chunks of a pipelined multiply, or the
//            single group of a resident one) into jobs: which slots to prepare first, the tile list, the output-block table.
//            Operands whose residues exceed the scratch budget are cut into (row panel x column panel) jobs that re-prepare.
//            gram: a Gram product's blocks on and above the diagonal (gram_tile_kept); resident, its slots share their residues.
// upload_tables(): every table goes to the device up front (before the side streams fork).
// run_group():     enqueues the jobs of one group on a stream.  No host synchronisation anywhere: see oz2_flag().
// ------------------------------------------------------------------------------------------------
struct Oz2Run {
  struct Prep {
    bool is_a = true;
    int slot0 = 0, nslots = 0;
    std::vector<OzakiOperand> blocks;
    std::vector<int32_t> dims;
    int max_rows = 1, max_cols = 1;
    bool need_zero = true;
    Buf d_blocks, d_dims;
  };
  struct Job {
    int group = 0;
    std::vector<Prep> preps;
    std::vector<int2> tiles;
    std::vector<double*> ctab;
    std::vector<Oz2FixOut> fouts;   // auto mode: the job's output blocks and their operand pairs, for the exact products of
    std::vector<Oz2FixSrc> fsrcs;   // elements the residue scheme leaves out (oz2_fixup)
    Buf d_tiles, d_ctab, d_fouts, d_fsrcs;
  };
  mr_context* ctx = nullptr;
  Oz2Engine* eng = nullptr;
  std::vector<Job> jobs;
  Buf d_maps;
  int cap_r = 0, cap_c = 0;
  int64_t int8_ops = 0;
  bool strassen = false;  // the single job runs one Strassen level (DESIGN section 4.1.3)

  Oz2Run() = default;
  Oz2Run(const Oz2Run&) = delete;
  Oz2Run& operator=(const Oz2Run&) = delete;
  ~Oz2Run() {
    if (eng) oz2_destroy(eng, ctx->stream);
  }
  const int* flag() const { return eng ? oz2_flag(eng) : nullptr; }

  // Returns false when the multiply must stay on the exact kernel.  `group_of` may be rewritten to a single group (operands too
  // large to keep every residue resident cannot be pipelined chunk by chunk).  pipelined: operands are still arriving.
  bool plan(mr_context* c, const std::vector<OutPlan>& plans, const std::vector<size_t>& out_plan, const std::vector<double*>& cptr,
            std::vector<int>& group_of, int& ngroups, int32_t blk, int64_t M, int64_t K, int64_t N, bool outer, bool guard, bool gram,
            bool pipelined) {
    ctx = c;
    if (M <= 0 || K <= 0 || N <= 0 || K >= (1 << 17) || out_plan.empty()) return false;
    const int T = oz2_moduli_for(K, ctx->crt_moduli);
    const int ss = (blk + kOz2TileM - 1) / kOz2TileM * kOz2TileM;
    std::map<int32_t, int> crow, ccol;
    compact_slots(plans, out_plan, crow, ccol);
    const int nr = static_cast<int>(crow.size()), nc = static_cast<int>(ccol.size());
    if (static_cast<int64_t>(nr) * ss > INT32_MAX / 2 || static_cast<int64_t>(nc) * ss > INT32_MAX / 2) return false;
    std::vector<int32_t> rdim(nr, -1), cdim(nc, -1);
    std::vector<std::vector<const PlanPair*>> asrc(nr), bsrc(nc);  // unique blocks per block row / column
    std::map<const Block*, int> seen_a, seen_b;
    for (size_t oi : out_plan) {
      const OutPlan& o = plans[oi];
      if (!o.only(ROUTE_GEMM) || o.m <= 0 || o.n <= 0 || o.m > blk || o.n > blk) return false;
      const int cr = crow[o.rid], cc = ccol[o.cid];
      if (rdim[cr] < 0) rdim[cr] = o.m;
      if (cdim[cc] < 0) cdim[cc] = o.n;
      if (rdim[cr] != o.m || cdim[cc] != o.n) return false;
      for (const PlanPair& g : o.pairs) {
        const int64_t k0 = outer ? 0 : static_cast<int64_t>(g.k) * blk;
        if (g.a->numCols != g.b->numRows || g.a->numCols > blk || k0 + g.a->numCols > K) return false;
        if (g.a->numRows != o.m || g.b->numCols != o.n) return false;
        auto ia = seen_a.find(g.a);
        if (ia == seen_a.end()) {
          seen_a[g.a] = cr;
          asrc[cr].push_back(&g);
        } else if (ia->second != cr) {
          return false;  // one block feeding two block rows: not a regular grid
        }
        auto ib = seen_b.find(g.b);
        if (ib == seen_b.end()) {
          seen_b[g.b] = cc;
          bsrc[cc].push_back(&g);
        } else if (ib->second != cc) {
          return false;
        }
      }
    }
    // ---- capacity: everything resident, or (row panel x column panel) jobs within the scratch budget
    const int64_t plane_cap_tiles = std::max<int64_t>(64, (2ll << 30) / (static_cast<int64_t>(T) * kOz2TileM * kOz2TileN));
    // Gram product: row slot s and column slot s hold the same block index and the same data, so they share one set of residues
    // when every slot fits at once
    const bool share = gram && crow == ccol && rdim == cdim && oz2_capacity(ctx, blk, K, T, nr, nc, cap_r, cap_c, nullptr, true) &&
                       cap_r == nr && cap_c == nc;
    if (!share && !oz2_capacity(ctx, blk, K, T, nr, nc, cap_r, cap_c)) return false;
    const bool resident = cap_r == nr && cap_c == nc;
    if (!resident) {  // panels re-prepare their slots: one group, after every operand has landed
      std::fill(group_of.begin(), group_of.end(), 0);
      ngroups = 1;
    }
    const int64_t Kpad = (K + 127) / 128 * 128;
    auto make_prep = [&](bool is_a, const std::vector<int>& ids /* compact ids, ascending */, int slot0) {
      Prep p;
      p.is_a = is_a;
      p.slot0 = slot0;
      p.nslots = static_cast<int>(ids.size());
      int64_t area = 0, want = 0;
      for (size_t s_ = 0; s_ < ids.size(); ++s_) {
        const int id = ids[s_];
        const int32_t base = static_cast<int32_t>((slot0 + static_cast<int>(s_)) * ss);
        p.dims.push_back(is_a ? rdim[id] : cdim[id]);
        want += static_cast<int64_t>(is_a ? rdim[id] : cdim[id]) * K;
        for (const PlanPair* g : (is_a ? asrc[id] : bsrc[id])) {
          const Block* b = is_a ? g->a : g->b;
          const int32_t k0 = outer ? 0 : g->k * blk;
          p.blocks.push_back(OzakiOperand{b->values.ptr<double>(), b->numRows, b->numCols, is_a ? base : k0, is_a ? k0 : base,
                                          static_cast<uint8_t>(b->isT), {0}});
          p.max_rows = std::max(p.max_rows, b->numRows);
          p.max_cols = std::max(p.max_cols, b->numCols);
          area += static_cast<int64_t>(b->numRows) * b->numCols;
        }
      }
      p.need_zero = !(area == want && K == Kpad);
      return p;
    };
    auto runs_of = [](std::vector<int> ids) {  // ids -> maximal runs of consecutive values
      std::sort(ids.begin(), ids.end());
      std::vector<std::vector<int>> runs;
      for (int id : ids) {
        if (runs.empty() || runs.back().back() + 1 != id) runs.emplace_back();
        runs.back().push_back(id);
      }
      return runs;
    };
    // slots that start on even 128-row tiles let the CTA-pair kernel run the tiles in vertically adjacent pairs
    const bool paired = (ss % (2 * kOz2TileM)) == 0 && ctx->force_variant != 2;
    // diag: a diagonal block of a Gram product, whose tiles are kept only where they hold an element on or above its diagonal
    auto add_tiles = [&](Job& j, int rslot, int cslot, int m, int n, bool diag) {
      const int tm0 = rslot * ss / kOz2TileM;
      int tm1 = (rslot * ss + m + kOz2TileM - 1) / kOz2TileM;
      if (paired && ((tm1 - tm0) & 1)) ++tm1;  // the padding tile lies inside the slot: garbage rows, never stored
      const int tn0 = cslot * ss / kOz2TileN, tn1 = (cslot * ss + n + kOz2TileN - 1) / kOz2TileN;
      for (int a = tm0; a < tm1; ++a)
        for (int b = tn0; b < tn1; ++b)
          if (!diag || gram_tile_kept(paired ? a & ~1 : a, b, rslot * ss, cslot * ss, n)) j.tiles.push_back(make_int2(a, b));
    };
    auto finish_tiles = [&](Job& j) {
      std::sort(j.tiles.begin(), j.tiles.end(), [&](const int2& x, const int2& y) {
        const int bx = x.y / 8, by = y.y / 8;  // bands of 8 n-tiles: the resident CTAs share A row- and B column-panels in L2
        if (bx != by) return bx < by;
        if (paired) {                          // (2a, b) directly followed by (2a + 1, b)
          if ((x.x >> 1) != (y.x >> 1)) return x.x < y.x;
          if (x.y != y.y) return x.y < y.y;
          return x.x < y.x;
        }
        if (x.x != y.x) return x.x < y.x;
        return x.y < y.y;
      });
      j.tiles.erase(std::unique(j.tiles.begin(), j.tiles.end(), [](const int2& x, const int2& y) { return x.x == y.x && x.y == y.y; }),
                    j.tiles.end());
      int8_ops += static_cast<int64_t>(j.tiles.size()) * T * 2ll * kOz2TileM * kOz2TileN * Kpad;
    };
    auto add_fix = [&](Job& j, const OutPlan& o, double* C, int rslot, int cslot) {
      if (!guard) return;
      Oz2FixOut fo{C, o.m, o.n, rslot, cslot, static_cast<int32_t>(j.fsrcs.size()), static_cast<int32_t>(o.pairs.size()),
                   gram && o.rid == o.cid ? 1 : 0, 0};
      for (const PlanPair& g : o.pairs)
        j.fsrcs.push_back(Oz2FixSrc{g.a->values.ptr<double>(), g.b->values.ptr<double>(), outer ? 0 : g.k * blk, g.a->numCols, g.a->numRows,
                                    g.b->numCols, static_cast<uint8_t>(g.a->isT), static_cast<uint8_t>(g.b->isT), {0}});
      j.fouts.push_back(fo);
    };
    // ---- one Strassen level (DESIGN section 4.1.3): a resident single-group product of an even grid of whole blocks, whose
    // quadrants are whole 256-row tile pairs and 128-byte k-chunks, within the scratch budget at 7/4 of the plain residues.
    // oz2_strassen = 1 takes it from M, N, K >= 16384 on (measured faster there; 4096^3 measured slower: the extra residue and CRT
    // traffic outweighs an eighth of a short GEMM), 2 whenever it is eligible.
    int max_tiles = 1;
    const int nkb = static_cast<int>(K / blk);
    constexpr int64_t kStrassenMinDim = 16384;
    const bool big = M >= kStrassenMinDim && N >= kStrassenMinDim && K >= kStrassenMinDim;
    strassen = (ctx->oz2_strassen >= 2 || (ctx->oz2_strassen == 1 && big)) && !outer && !gram && !share && resident && !pipelined && ngroups == 1 && blk % kOz2TileM == 0 &&
               K % blk == 0 && nr % 2 == 0 && nc % 2 == 0 && nkb % 2 == 0 && M == static_cast<int64_t>(nr) * blk &&
               N == static_cast<int64_t>(nc) * blk && (M / 2) % (2 * kOz2TileM) == 0 && (N / 2) % kOz2TileN == 0 && (K / 2) % 128 == 0 &&
               out_plan.size() == static_cast<size_t>(nr) * nc;
    std::vector<int2> pos;  // positions: tiles of a quadrant of C, in the banded order of finish_tiles
    int pp = 0;             // positions per piece
    if (strassen) {
      std::set<std::pair<int, int>> ablk, bblk;  // (row, k) of A / (k, column) of B with a whole block
      for (size_t oi : out_plan) {
        const OutPlan& o = plans[oi];
        if (o.m != blk || o.n != blk || o.pairs.size() != static_cast<size_t>(nkb)) strassen = false;
        for (const PlanPair& g : o.pairs)
          if (g.a->numRows == blk && g.a->numCols == blk && g.b->numCols == blk) {
            ablk.insert({crow[o.rid], g.k});
            bblk.insert({g.k, ccol[o.cid]});
          }
      }
      strassen = strassen && ablk.size() == static_cast<size_t>(nr) * nkb && bblk.size() == static_cast<size_t>(nkb) * nc;
    }
    if (strassen) {
      const int qtm = static_cast<int>(M / 2 / kOz2TileM), qtn = static_cast<int>(N / 2 / kOz2TileN);
      for (int a = 0; a < qtm; ++a)
        for (int b = 0; b < qtn; ++b) pos.push_back(make_int2(a, b));
      std::sort(pos.begin(), pos.end(), [](const int2& x, const int2& y) {  // bands of 8 n-tiles, (2a, b) followed by (2a + 1, b)
        if (x.y / 8 != y.y / 8) return x.y / 8 < y.y / 8;
        if ((x.x >> 1) != (y.x >> 1)) return x.x < y.x;
        if (x.y != y.y) return x.y < y.y;
        return x.x < y.x;
      });
      // pieces of equal size: each holds the 7 sub-product tiles of its positions within the 2 GiB residue planes
      const int npos = static_cast<int>(pos.size());
      const int ppmax = static_cast<int>(std::min<int64_t>(npos, plane_cap_tiles / 7)) & ~1;
      const int npieces = (npos + ppmax - 1) / ppmax;
      pp = (npos + npieces - 1) / npieces;
      pp += pp & 1;
      size_t need = oz2_scratch_bytes(blk, K, T, nr, nc, 7 * pp, false, true);
      const size_t budget = static_cast<size_t>(ctx->ozaki_scratch_mb > 0 ? ctx->ozaki_scratch_mb : 16384) << 20;
      strassen = need <= budget;
    }
    if (strassen) {
      Job j;
      j.group = 0;
      j.ctab.assign(static_cast<size_t>(cap_r) * cap_c, nullptr);
      for (size_t t = 0; t < out_plan.size(); ++t) {
        const OutPlan& o = plans[out_plan[t]];
        const int cr = crow[o.rid], cc = ccol[o.cid];
        j.ctab[static_cast<size_t>(cr) * cap_c + cc] = cptr[out_plan[t]];
        add_fix(j, o, cptr[out_plan[t]], cr, cc);
      }
      // every slot at once, the blocks in quads of (line half, k half): (0, 0), (0, 1), (1, 0), (1, 1)
      for (bool is_a : {true, false}) {
        const int nl = is_a ? nr : nc;
        std::vector<int> ids(nl);
        for (int i = 0; i < nl; ++i) ids[i] = i;
        Prep p = make_prep(is_a, ids, 0);
        std::vector<const OzakiOperand*> at(static_cast<size_t>(nl) * nkb, nullptr);
        for (const OzakiOperand& b : p.blocks) {
          const int lb = (is_a ? b.row0 : b.col0) / blk, kb = (is_a ? b.col0 : b.row0) / blk;
          at[static_cast<size_t>(lb) * nkb + kb] = &b;
        }
        std::vector<OzakiOperand> quads;
        for (int lb = 0; lb < nl / 2; ++lb)
          for (int kb = 0; kb < nkb / 2; ++kb)
            for (int q = 0; q < 4; ++q) quads.push_back(*at[static_cast<size_t>(lb + (q >> 1) * (nl / 2)) * nkb + kb + (q & 1) * (nkb / 2)]);
        p.blocks = std::move(quads);
        j.preps.push_back(std::move(p));
      }
      // piece by piece, the 7 sub-products product-major
      const int qtm = static_cast<int>(M / 2 / kOz2TileM), qtn = static_cast<int>(N / 2 / kOz2TileN);
      for (size_t p0 = 0; p0 < pos.size(); p0 += pp)
        for (int i = 0; i < 7; ++i)
          for (size_t u = p0; u < std::min(pos.size(), p0 + pp); ++u) j.tiles.push_back(make_int2(i * qtm + pos[u].x, i * qtn + pos[u].y));
      int8_ops += static_cast<int64_t>(j.tiles.size()) * T * 2ll * kOz2TileM * kOz2TileN * (Kpad / 2);
      max_tiles = 7 * pp;
      jobs.push_back(std::move(j));
    } else if (resident) {
      std::vector<char> rprep(nr, 0), cprep(nc, 0);
      for (int gi = 0; gi < ngroups; ++gi) {
        Job j;
        j.group = gi;
        j.ctab.assign(static_cast<size_t>(cap_r) * cap_c, nullptr);
        std::vector<int> newr, newc;
        for (size_t t = 0; t < out_plan.size(); ++t) {
          if (group_of[t] != gi) continue;
          const OutPlan& o = plans[out_plan[t]];
          const int cr = crow[o.rid], cc = ccol[o.cid];
          if (!rprep[cr]) {
            rprep[cr] = 1;
            newr.push_back(cr);
          }
          if (!cprep[cc]) {
            cprep[cc] = 1;
            newc.push_back(cc);
          }
          j.ctab[static_cast<size_t>(cr) * cap_c + cc] = cptr[out_plan[t]];
          add_tiles(j, cr, cc, o.m, o.n, gram && o.rid == o.cid);
          add_fix(j, o, cptr[out_plan[t]], cr, cc);
        }
        if (j.tiles.empty()) continue;
        if (share) {  // a slot prepared on the B side is also the A slot of the same index
          std::vector<int> ids;
          for (int id : newr) ids.push_back(id);
          for (int id : newc) ids.push_back(id);
          std::sort(ids.begin(), ids.end());
          ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
          for (int id : ids) rprep[id] = cprep[id] = 1;
          newr.clear();
          newc = ids;
        }
        for (auto& run : runs_of(newr)) j.preps.push_back(make_prep(true, run, run.front()));
        for (auto& run : runs_of(newc)) j.preps.push_back(make_prep(false, run, run.front()));
        finish_tiles(j);
        max_tiles = std::max<int>(max_tiles, static_cast<int>(j.tiles.size()));
        jobs.push_back(std::move(j));
      }
    } else {
      std::map<std::pair<int, int>, size_t> at;  // (cr, cc) -> index into out_plan
      for (size_t t = 0; t < out_plan.size(); ++t) at[{crow[plans[out_plan[t]].rid], ccol[plans[out_plan[t]].cid]}] = t;
      for (int r0 = 0; r0 < nr; r0 += cap_r) {
        const int r1 = std::min(nr, r0 + cap_r);
        bool row_prepared = false;
        for (int c0 = 0; c0 < nc; c0 += cap_c) {
          const int c1 = std::min(nc, c0 + cap_c);
          Job j;
          j.group = 0;
          j.ctab.assign(static_cast<size_t>(cap_r) * cap_c, nullptr);
          for (int cr = r0; cr < r1; ++cr)
            for (int cc = c0; cc < c1; ++cc) {
              auto it = at.find({cr, cc});
              if (it == at.end()) continue;
              const OutPlan& o = plans[out_plan[it->second]];
              j.ctab[static_cast<size_t>(cr - r0) * cap_c + (cc - c0)] = cptr[out_plan[it->second]];
              add_tiles(j, cr - r0, cc - c0, o.m, o.n, gram && o.rid == o.cid);
              add_fix(j, o, cptr[out_plan[it->second]], cr - r0, cc - c0);
            }
          if (j.tiles.empty()) continue;
          if (!row_prepared) {
            std::vector<int> ids;
            for (int cr = r0; cr < r1; ++cr) ids.push_back(cr);
            j.preps.push_back(make_prep(true, ids, 0));
            row_prepared = true;
          }
          std::vector<int> ids;
          for (int cc = c0; cc < c1; ++cc) ids.push_back(cc);
          j.preps.push_back(make_prep(false, ids, 0));
          finish_tiles(j);
          max_tiles = std::max<int>(max_tiles, static_cast<int>(j.tiles.size()));
          jobs.push_back(std::move(j));
        }
      }
    }
    if (jobs.empty()) return false;
    if (!strassen) {
      max_tiles = static_cast<int>(std::min<int64_t>(max_tiles, plane_cap_tiles));
      max_tiles += max_tiles & 1;
    }
    cudaError_t e = oz2_create(&eng, blk, K, T, cap_r, cap_c, max_tiles, guard ? 1 : 0, share, strassen, ctx->stream);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      eng = nullptr;
      jobs.clear();
      return false;  // e.g. out of memory for the scratch: the exact kernel needs none
    }
    oz2_set_paired(eng, paired);
    oz2_set_ksplit(eng, ctx->oz2_ksplit);
    if (paired && !oz2_paired(eng)) {  // cannot happen (ss % 256 == 0 makes Mpad a multiple of 256); stay on the safe side
      oz2_destroy(eng, ctx->stream);
      eng = nullptr;
      jobs.clear();
      return false;
    }
    return true;
  }

  void upload_tables() {
    size_t bytes = 0;
    const void* hm = oz2_host_maps(eng, &bytes);
    d_maps = upload_bytes(ctx, hm, bytes);
    oz2_set_device_maps(eng, d_maps->p);
    for (Job& j : jobs) {
      for (Prep& p : j.preps) {
        p.d_blocks = upload(ctx, p.blocks);
        p.d_dims = upload(ctx, p.dims);
      }
      j.d_tiles = upload(ctx, j.tiles);
      j.d_ctab = upload(ctx, j.ctab);
      if (!j.fouts.empty()) {
        j.d_fouts = upload(ctx, j.fouts);
        j.d_fsrcs = upload(ctx, j.fsrcs);
      }
    }
  }

  void run_group(int gi, cudaStream_t cs) {
    const bool timed = ctx->time_kernels != 0;
    double ms = 0.0;
    for (Job& j : jobs) {
      if (j.group != gi) continue;
      for (Prep& p : j.preps)
        CUDA_CHECK(oz2_prepare(eng, p.is_a, static_cast<const OzakiOperand*>(p.d_blocks->p), static_cast<int>(p.blocks.size()),
                               p.max_rows, p.max_cols, p.slot0, p.nslots, static_cast<const int32_t*>(p.d_dims->p), p.need_zero, cs));
      CUDA_CHECK(oz2_multiply(eng, static_cast<const int2*>(j.d_tiles->p), static_cast<int>(j.tiles.size()),
                              static_cast<double* const*>(j.d_ctab->p), cs, timed ? &ms : nullptr, ctx->ev2, ctx->ev3));
      if (!j.fouts.empty())
        CUDA_CHECK(oz2_fixup(eng, static_cast<const Oz2FixOut*>(j.d_fouts->p), static_cast<int>(j.fouts.size()),
                             static_cast<const Oz2FixSrc*>(j.d_fsrcs->p), cs));
    }
    note_launch(ctx, oz2_launches(eng));
    if (timed) ctx->stats.tc_gemm_ms_total += ms;
  }
};

// ------------------------------------------------------------------------------------------------
// Output blocks whose partial products are ALL low-density sparse x sparse (LocalMatrix.multiplySparseSparse,
// LocalMatrix.scala:143-323), computed natively on the stored entries by spgemm.cu.  Storage format: the reference's four loop
// nests end in four different rules, and `reduceByKey(LocalMatrix.add)` re-decides the format at every sparse + sparse step, so
// the chain is replayed partial by partial in ascending k (Spark's own reduce order is arbitrary; ascending k is the
// deterministic choice):
//   CSC x CSC (:155-196): CSC iff rows*cols > 2 nnz + cols + 1, else dense      CSR x CSR (:198-239): CSR iff ... + rows + 1
//   CSR x CSC (:241-286): always CSC (both branches build a SparseMatrix)       CSC x CSR (:288-323): dense iff rows*cols <= 2 nnz + cols
//   sparse + sparse (:74-139): CSC iff rows*cols > 2 nnz + cols + 1, else dense; anything + dense: dense.
// The values do not depend on these formats (every product and sum is rounded on its own and zeros are dropped after each, so a
// dense partial sum holds exactly the sparse one's entries), so the device computes every chain sparsely and the rules only need
// nnz(P_l) and nnz(S_l) of each level: a count pass returns them in ONE read-back, the host replays the rules, and a fill pass
// writes each result in its final format (a dense window only for chains that end dense).
// ------------------------------------------------------------------------------------------------
enum ChainFmt { FMT_DENSE = 0, FMT_CSC = 1, FMT_CSR = 2 };

int partial_format(bool aT, bool bT, int64_t m, int64_t n, int64_t nnz) {
  const int64_t cells = m * n;
  if (!aT && !bT) return cells > 2 * nnz + n + 1 ? FMT_CSC : FMT_DENSE;
  if (aT && bT) return cells > 2 * nnz + m + 1 ? FMT_CSR : FMT_DENSE;
  if (aT && !bT) return FMT_CSC;
  return cells <= 2 * nnz + n ? FMT_DENSE : FMT_CSC;
}

// The format a chain ends in, from its per-level counts: the rules above, level by level with the layouts of o's pairs.  *nnz: the
// entries of the final sum.
int chain_format(const OutPlan& o, const int64_t* cp, const int64_t* cs, int64_t* nnz) {
  int fmt = FMT_DENSE;
  int64_t s_nnz = 0;
  for (size_t l = 0; l < o.pairs.size(); ++l) {
    s_nnz += cs[l];
    const int pf = partial_format(o.pairs[l].a->isT, o.pairs[l].b->isT, o.m, o.n, cp[l]);
    if (l == 0) fmt = pf;
    else if (fmt == FMT_DENSE || pf == FMT_DENSE) fmt = FMT_DENSE;
    else fmt = static_cast<int64_t>(o.m) * o.n > 2 * s_nnz + o.n + 1 ? FMT_CSC : FMT_DENSE;
  }
  *nnz = s_nnz;
  return fmt;
}

// gram: the product is a sparse Gram product (gram_route, DESIGN section 4.1.2).  The chains of square blocks below the diagonal
// are not run: each such block is its upper mirror's transpose, written after the fill (a dense window by gram_mirror_kernel,
// sparse arrays shared with or converted from the mirror's).  Diagonal chains are triangular, and gram_sym_kernel completes their
// sparse results.  When the count pass finds a walked line whose indices do not ascend, the mirror is not exact: every chain is
// then run as without `gram`.
void run_sparse_chains(mr_context* ctx, const std::vector<OutPlan>& plans, const std::vector<double*>& cptr, mr_matrix* result,
                       bool gram) {
  std::vector<size_t> chains;  // empty output blocks keep the (empty) dense block allocate_outputs gave them
  std::vector<std::pair<size_t, size_t>> mirrored;  // gram: (lower plan, its chain)
  {
    std::map<std::pair<int32_t, int32_t>, size_t> at;
    for (size_t i = 0; i < plans.size(); ++i) at[{plans[i].rid, plans[i].cid}] = i;
    std::map<size_t, size_t> chain_of;
    for (size_t i = 0; i < plans.size(); ++i) {
      const OutPlan& o = plans[i];
      if (!o.has(ROUTE_SPSP) || o.m <= 0 || o.n <= 0) continue;
      if (gram && o.rid > o.cid && o.m == o.n) continue;
      chain_of[i] = chains.size();
      chains.push_back(i);
    }
    if (gram)
      for (size_t i = 0; i < plans.size(); ++i) {
        const OutPlan& o = plans[i];
        if (o.has(ROUTE_SPSP) && o.m > 0 && o.rid > o.cid && o.m == o.n) mirrored.push_back({i, chain_of.at(at.at({o.cid, o.rid}))});
      }
  }
  if (chains.empty()) return;
  const size_t nc = chains.size();
  // ---- frames: an all-CSR chain runs as C^T = B^T A^T on the CSR arrays; any other chain in CSC, its CSR operands converted once
  std::vector<char> csr_frame(nc, 1);
  for (size_t c = 0; c < nc; ++c)
    for (const PlanPair& pr : plans[chains[c]].pairs) {
      wait_ready(ctx, *pr.a);
      wait_ready(ctx, *pr.b);
      if (!pr.a->isT || !pr.b->isT) csr_frame[c] = 0;
    }
  std::map<const Block*, size_t> conv;  // CSR operand -> offset of its CSC copy in the conversion buffer
  size_t conv_bytes = 0;
  for (size_t c = 0; c < nc; ++c)
    if (!csr_frame[c])
      for (const PlanPair& pr : plans[chains[c]].pairs)
        for (const Block* b : {pr.a, pr.b})
          if (b->isT && !conv.count(b)) {
            conv.emplace(b, conv_bytes);
            conv_bytes += CscLayout(b->numCols, b->valuesLen).bytes;
          }
  Buf cbuf;
  if (!conv.empty()) {
    cbuf = std::make_shared<DevBuf>(ctx, conv_bytes);
    std::vector<CsrToCsc> cv;
    for (auto& kv : conv) {
      const Block* b = kv.first;
      cv.push_back(CsrToCsc{b->colPtrs.ptr<int32_t>(), b->rowIndices.ptr<int32_t>(), b->values.ptr<double>(), b->numRows, b->numCols,
                            b->valuesLen, static_cast<char*>(cbuf->p) + kv.second});
    }
    csr_to_csc(ctx, cv);
  }
  // ---- the chains and their pairs in the frame
  std::vector<SpgemmChain> ch(nc);
  std::vector<SpgemmPair> pairs;
  std::vector<SpgemmItem> items;
  const int per_item = spgemm_columns_per_item();
  int32_t count_total = 0;
  int64_t col_total = 0;
  int max_m = 0, max_levels = 0;
  bool any_tri = false;
  for (size_t c = 0; c < nc; ++c) {
    const OutPlan& o = plans[chains[c]];
    SpgemmChain& h = ch[c];
    h.m = csr_frame[c] ? o.n : o.m;
    h.n = csr_frame[c] ? o.m : o.n;
    h.pair_begin = static_cast<int32_t>(pairs.size());
    h.levels = static_cast<int32_t>(o.pairs.size());
    h.tri = gram && o.rid == o.cid ? 1 : 0;  // its pairs are A(i, k) x A(i, k)^T, one CSR side and one CSC side: a CSC frame
    MR_REQUIRE(!h.tri || !csr_frame[c], MR_EINVAL, "internal: a diagonal Gram chain in the CSR frame");
    any_tri = any_tri || h.tri;
    h.count_off = count_total;
    count_total += (h.tri ? 4 : 2) * h.levels;
    col_total += h.n;
    max_m = std::max(max_m, h.m);
    max_levels = std::max(max_levels, h.levels);
    auto csc_of = [&](const Block* b, const int32_t*& p, const int32_t*& i, const double*& v) {
      if (b->isT && !csr_frame[c]) {
        const char* w = static_cast<const char*>(cbuf->p) + conv.at(b);
        const CscLayout L(b->numCols, b->valuesLen);
        p = reinterpret_cast<const int32_t*>(w + L.ptr);
        i = reinterpret_cast<const int32_t*>(w + L.idx);
        v = reinterpret_cast<const double*>(w + L.val);
      } else {  // CSC, or (CSR frame) the CSC arrays of the block's transpose
        p = b->colPtrs.ptr<int32_t>();
        i = b->rowIndices.ptr<int32_t>();
        v = b->values.ptr<double>();
      }
    };
    for (const PlanPair& pr : o.pairs) {
      SpgemmPair q{};
      const Block* lb = csr_frame[c] ? pr.b : pr.a;
      const Block* rb = csr_frame[c] ? pr.a : pr.b;
      csc_of(lb, q.lp, q.li, q.lv);
      csc_of(rb, q.rp, q.ri, q.rv);
      pairs.push_back(q);
    }
    for (int32_t c0 = 0; c0 < h.n; c0 += per_item) items.push_back(SpgemmItem{static_cast<int32_t>(c), c0});
  }
  // ---- count pass: per-level counters, scalar products, per-column counts of the final sums
  const size_t counts_off = 0, prod_off = align_up(static_cast<size_t>(count_total) * sizeof(int32_t)),
               flag_off = prod_off + align_up(sizeof(unsigned long long)), colcnt_off = flag_off + align_up(sizeof(int32_t));
  Buf meta = std::make_shared<DevBuf>(ctx, colcnt_off + static_cast<size_t>(col_total) * sizeof(int32_t));
  CUDA_CHECK(cudaMemsetAsync(meta->p, 0, colcnt_off, ctx->stream));
  char* mbase = static_cast<char*>(meta->p);
  int32_t* d_counts = reinterpret_cast<int32_t*>(mbase + counts_off);
  auto* d_products = reinterpret_cast<unsigned long long*>(mbase + prod_off);
  int32_t* d_unsorted = reinterpret_cast<int32_t*>(mbase + flag_off);
  {
    int64_t off = 0;
    for (size_t c = 0; c < nc; ++c) {
      ch[c].colcnt = reinterpret_cast<int32_t*>(mbase + colcnt_off) + off;
      off += ch[c].n;
    }
  }
  const SpgemmLaunchShape shape = spgemm_shape(max_m, max_levels, any_tri);
  Buf scratch = shape.scratch_bytes ? std::make_shared<DevBuf>(ctx, shape.scratch_bytes) : nullptr;
  Buf d_pairs = upload(ctx, pairs), d_items = upload(ctx, items), d_ch = upload(ctx, ch);
  CUDA_CHECK(launch_spgemm(false, static_cast<const SpgemmItem*>(d_items->p), static_cast<int>(items.size()),
                           static_cast<const SpgemmChain*>(d_ch->p), static_cast<const SpgemmPair*>(d_pairs->p), d_counts, d_products,
                           scratch ? scratch->p : nullptr, max_m, shape, gram ? d_unsorted : nullptr, ctx->stream));
  note_launch(ctx);
  std::vector<int32_t> h_counts_v(static_cast<size_t>(count_total));
  unsigned long long h_products = 0;
  int32_t h_unsorted = 0;
  CUDA_CHECK(cudaMemcpyAsync(h_counts_v.data(), d_counts, h_counts_v.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaMemcpyAsync(&h_products, d_products, sizeof(h_products), cudaMemcpyDeviceToHost, ctx->stream));
  ctx->stats.d2h_bytes += static_cast<int64_t>(h_counts_v.size() * sizeof(int32_t) + sizeof(h_products));
  if (gram) {
    CUDA_CHECK(cudaMemcpyAsync(&h_unsorted, d_unsorted, sizeof(h_unsorted), cudaMemcpyDeviceToHost, ctx->stream));
    ctx->stats.d2h_bytes += static_cast<int64_t>(sizeof(h_unsorted));
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  const int32_t* h_counts = h_counts_v.data();
  ctx->stats.spgemm_pairs += static_cast<int64_t>(pairs.size());
  ctx->stats.spgemm_products += static_cast<int64_t>(h_products);
  if (h_unsorted) {  // the mirror would not be exact: the general route
    run_sparse_chains(ctx, plans, cptr, result, false);
    return;
  }
  // ---- the reference's format rules, level by level; a triangular chain's full counts are 2 upper - diagonal
  std::vector<int> fmt(nc);
  std::vector<int64_t> nnz(nc), nnz_up(nc);
  std::vector<std::vector<int64_t>> cnt_p(nc), cnt_s(nc);
  for (size_t c = 0; c < nc; ++c) {
    const int32_t L = ch[c].levels;
    const int32_t* cu = h_counts + ch[c].count_off;
    cnt_p[c].resize(L);
    cnt_s[c].resize(L);
    int64_t up = 0;
    for (int32_t l = 0; l < L; ++l) {
      up += cu[L + l];
      cnt_p[c][l] = ch[c].tri ? 2ll * cu[l] - cu[2 * L + l] : cu[l];
      cnt_s[c][l] = ch[c].tri ? 2ll * cu[L + l] - cu[3 * L + l] : cu[L + l];
    }
    nnz_up[c] = up;
    fmt[c] = chain_format(plans[chains[c]], cnt_p[c].data(), cnt_s[c].data(), &nnz[c]);
    MR_REQUIRE(!ch[c].tri || fmt[c] != FMT_CSR, MR_EINVAL, "internal: a diagonal Gram chain ending CSR");
  }
  // a mirrored block: its own pairs' layouts and its mirror's counts (nnz(P_l), nnz(S_l) do not change under transposition).  The
  // rules' thresholds of a square block pair up, so both end dense or both sparse; a CSR result only comes from a CSC frame.
  std::vector<int> mfmt(mirrored.size());
  for (size_t t = 0; t < mirrored.size(); ++t) {
    const size_t c = mirrored[t].second;
    int64_t e = 0;
    mfmt[t] = chain_format(plans[mirrored[t].first], cnt_p[c].data(), cnt_s[c].data(), &e);
    MR_REQUIRE((mfmt[t] == FMT_DENSE) == (fmt[c] == FMT_DENSE) && e == nnz[c] && !(mfmt[t] == FMT_CSR && csr_frame[c]), MR_EINVAL,
               "internal: a Gram block and its mirror disagree on their format");
  }
  // ---- outputs: a dense window (the caller's, or from a slab of the dense-ending chains), or exactly sized sparse arrays.  A
  // triangular chain's sparse upper triangle and its transpose go to `tmp`, freed behind the launches.
  size_t dense_total = 0, sparse_total = 0, tmp_total = 0;
  auto sparse_bytes = [](int32_t lines, int64_t e) {
    return align_up((static_cast<size_t>(lines) + 1) * sizeof(int32_t)) + align_up(static_cast<size_t>(e) * sizeof(int32_t)) +
           align_up(static_cast<size_t>(e) * sizeof(double));
  };
  for (size_t c = 0; c < nc; ++c) {
    const OutPlan& o = plans[chains[c]];
    if (fmt[c] == FMT_DENSE) {
      if (!cptr[chains[c]]) dense_total += align_up(static_cast<size_t>(o.m) * o.n * sizeof(double));
    } else {
      sparse_total += sparse_bytes(ch[c].n, nnz[c]);
      if (csr_frame[c] && fmt[c] == FMT_CSC) sparse_total += CscLayout(o.n, nnz[c]).bytes;  // S in the CSR frame, then CSC
      if (ch[c].tri) tmp_total += sparse_bytes(ch[c].n, nnz_up[c]) + CscLayout(o.n, nnz_up[c]).bytes + align_up(o.n * sizeof(int32_t));
    }
  }
  for (size_t t = 0; t < mirrored.size(); ++t) {
    const OutPlan& o = plans[mirrored[t].first];
    const size_t c = mirrored[t].second;
    if (mfmt[t] == FMT_DENSE) {
      if (!cptr[mirrored[t].first]) dense_total += align_up(static_cast<size_t>(o.m) * o.n * sizeof(double));
    } else if (mfmt[t] == FMT_CSC && !csr_frame[c]) {
      sparse_total += CscLayout(o.n, nnz[c]).bytes;
    }
  }
  std::unique_ptr<Slab> dslab, sslab, tslab;
  if (dense_total) dslab.reset(new Slab(ctx, dense_total));
  if (sparse_total) sslab.reset(new Slab(ctx, sparse_total));
  if (tmp_total) tslab.reset(new Slab(ctx, tmp_total));
  std::vector<ScanDesc> scans;
  std::vector<CsrToCsc> finals;
  std::vector<GramMirror> mirrors;
  std::vector<GramSym> syms;
  std::vector<ScanDesc> sym_scans;
  std::vector<Span> frame_ptr(nc), frame_idx(nc), frame_val(nc);  // a sparse chain's arrays in its frame
  int mir_m = 0, mir_n = 0, sym_n = 0;
  auto sparse_block = [](int32_t m, int32_t n, int64_t e, bool isT, Span ptr, Span idx, Span val) {
    Block b;
    b.type = 0;
    b.numRows = m;
    b.numCols = n;
    b.valuesLen = e;
    b.colPtrs = ptr;
    b.rowIndices = idx;
    b.values = val;
    b.colPtrsLen = (isT ? m : n) + 1;
    b.isT = isT;
    return b;
  };
  auto csc_window = [](const Span& w, int32_t cols, int64_t e, Span& ptr, Span& idx, Span& val) {
    const CscLayout L(cols, e);
    ptr = Span{w.buf, w.off + L.ptr};
    idx = Span{w.buf, w.off + L.idx};
    val = Span{w.buf, w.off + L.val};
  };
  for (size_t c = 0; c < nc; ++c) {
    const OutPlan& o = plans[chains[c]];
    SpgemmChain& h = ch[c];
    Block& out = result->blocks[{o.rid, o.cid}];
    if (fmt[c] == FMT_DENSE) {
      if (cptr[chains[c]]) {
        h.dense = cptr[chains[c]];
      } else {
        Span s = dslab->take(static_cast<size_t>(o.m) * o.n * sizeof(double));
        h.dense = s.ptr<double>();
        out = dense_block(o.m, o.n, s, false);
      }
      h.drs = csr_frame[c] ? o.m : 1;
      h.dcs = csr_frame[c] ? 1 : o.m;
      if (h.tri) {
        mirrors.push_back(GramMirror{h.dense, h.dense, o.m, o.n, 1, 0});
        mir_m = std::max(mir_m, o.m);
        mir_n = std::max(mir_n, o.n);
      }
      continue;
    }
    const size_t e = static_cast<size_t>(nnz[c]);
    Span ptr = sslab->take((static_cast<size_t>(h.n) + 1) * sizeof(int32_t)), idx = sslab->take(e * sizeof(int32_t)),
         val = sslab->take(e * sizeof(double));
    frame_ptr[c] = ptr;
    frame_idx[c] = idx;
    frame_val[c] = val;
    if (h.tri) {  // the fill writes U to tmp; U^T, then the full columns into ptr / idx / val
      const size_t eu = static_cast<size_t>(nnz_up[c]);
      Span uptr = tslab->take((static_cast<size_t>(h.n) + 1) * sizeof(int32_t)), uidx = tslab->take(eu * sizeof(int32_t)),
           uval = tslab->take(eu * sizeof(double)), tw = tslab->take(CscLayout(h.n, nnz_up[c]).bytes),
           cnt = tslab->take(static_cast<size_t>(h.n) * sizeof(int32_t));
      h.optr = uptr.ptr<int32_t>();
      h.oidx = uidx.ptr<int32_t>();
      h.oval = uval.ptr<double>();
      scans.push_back(ScanDesc{h.colcnt, uptr.ptr<int32_t>(), h.n, 0});
      // U's CSC arrays are the CSR arrays of U^T: their CSC copy is U^T's CSC
      finals.push_back(CsrToCsc{uptr.ptr<int32_t>(), uidx.ptr<int32_t>(), uval.ptr<double>(), h.n, h.m, nnz_up[c], tw.ptr<char>()});
      Span tp, ti, tv;
      csc_window(tw, h.m, nnz_up[c], tp, ti, tv);
      syms.push_back(GramSym{uptr.ptr<int32_t>(), uidx.ptr<int32_t>(), uval.ptr<double>(), tp.ptr<int32_t>(), ti.ptr<int32_t>(),
                             tv.ptr<double>(), cnt.ptr<int32_t>(), ptr.ptr<int32_t>(), idx.ptr<int32_t>(), val.ptr<double>(), h.n, 0});
      sym_scans.push_back(ScanDesc{cnt.ptr<int32_t>(), ptr.ptr<int32_t>(), h.n, 0});
      sym_n = std::max(sym_n, h.n);
      out = sparse_block(o.m, o.n, static_cast<int64_t>(e), false, ptr, idx, val);
      continue;
    }
    h.optr = ptr.ptr<int32_t>();
    h.oidx = idx.ptr<int32_t>();
    h.oval = val.ptr<double>();
    scans.push_back(ScanDesc{h.colcnt, ptr.ptr<int32_t>(), h.n, 0});
    if (csr_frame[c] && fmt[c] == FMT_CSC) {  // CSR arrays of C -> CSC
      const Span w = sslab->take(CscLayout(o.n, nnz[c]).bytes);
      finals.push_back(CsrToCsc{ptr.ptr<int32_t>(), idx.ptr<int32_t>(), val.ptr<double>(), o.m, o.n, nnz[c], w.ptr<char>()});
      Span p2, i2, v2;
      csc_window(w, o.n, nnz[c], p2, i2, v2);
      out = sparse_block(o.m, o.n, nnz[c], false, p2, i2, v2);
    } else {  // the frame's arrays are the result's: CSC (CSC frame) or CSR (CSR frame)
      out = sparse_block(o.m, o.n, nnz[c], csr_frame[c] != 0, ptr, idx, val);
    }
  }
  // ---- mirrored blocks.  The frame arrays of the mirror are the CSR (CSC frame) or CSC (CSR frame) arrays of this block: its
  // result when that is its format (the arrays are shared, as A.t() shares A's), else converted to CSC.
  for (size_t t = 0; t < mirrored.size(); ++t) {
    const OutPlan& o = plans[mirrored[t].first];
    const size_t c = mirrored[t].second;
    Block& out = result->blocks[{o.rid, o.cid}];
    if (mfmt[t] == FMT_DENSE) {
      double* dst = cptr[mirrored[t].first];
      if (!dst) {
        Span s = dslab->take(static_cast<size_t>(o.m) * o.n * sizeof(double));
        dst = s.ptr<double>();
        out = dense_block(o.m, o.n, s, false);
      }
      mirrors.push_back(GramMirror{ch[c].dense, dst, o.m, o.n, 0, 0});
      mir_m = std::max(mir_m, o.m);
      mir_n = std::max(mir_n, o.n);
    } else if (mfmt[t] == FMT_CSC && !csr_frame[c]) {
      const Span w = sslab->take(CscLayout(o.n, nnz[c]).bytes);
      finals.push_back(CsrToCsc{frame_ptr[c].ptr<int32_t>(), frame_idx[c].ptr<int32_t>(), frame_val[c].ptr<double>(), o.m, o.n, nnz[c],
                                w.ptr<char>()});
      Span p2, i2, v2;
      csc_window(w, o.n, nnz[c], p2, i2, v2);
      out = sparse_block(o.m, o.n, nnz[c], false, p2, i2, v2);
    } else {
      out = sparse_block(o.m, o.n, nnz[c], mfmt[t] == FMT_CSR, frame_ptr[c], frame_idx[c], frame_val[c]);
    }
  }
  if (gram) {
    ctx->stats.gram_blocks += static_cast<int64_t>(nc);
    ctx->stats.gram_mirrored_blocks += static_cast<int64_t>(mirrored.size());
  }
  // ---- fill pass
  if (!scans.empty()) {
    Buf d_scans = upload(ctx, scans);
    CUDA_CHECK(launch_exclusive_scan(static_cast<const ScanDesc*>(d_scans->p), static_cast<int>(scans.size()), ctx->stream));
    note_launch(ctx);
  }
  Buf d_ch2 = upload(ctx, ch);
  CUDA_CHECK(launch_spgemm(true, static_cast<const SpgemmItem*>(d_items->p), static_cast<int>(items.size()),
                           static_cast<const SpgemmChain*>(d_ch2->p), static_cast<const SpgemmPair*>(d_pairs->p), d_counts, d_products,
                           scratch ? scratch->p : nullptr, max_m, shape, nullptr, ctx->stream));
  note_launch(ctx);
  csr_to_csc(ctx, finals);
  if (!syms.empty()) {
    Buf d_syms = upload(ctx, syms), d_sym_scans = upload(ctx, sym_scans);
    CUDA_CHECK(launch_gram_sym(false, static_cast<const GramSym*>(d_syms->p), static_cast<int>(syms.size()), sym_n, ctx->stream));
    CUDA_CHECK(launch_exclusive_scan(static_cast<const ScanDesc*>(d_sym_scans->p), static_cast<int>(sym_scans.size()), ctx->stream));
    CUDA_CHECK(launch_gram_sym(true, static_cast<const GramSym*>(d_syms->p), static_cast<int>(syms.size()), sym_n, ctx->stream));
    note_launch(ctx, 3);
  }
  if (!mirrors.empty()) {
    Buf d_mirrors = upload(ctx, mirrors);
    CUDA_CHECK(launch_gram_mirror(static_cast<const GramMirror*>(d_mirrors->p), static_cast<int>(mirrors.size()), mir_m, mir_n,
                                  ctx->stream));
    note_launch(ctx);
  }
}

// ------------------------------------------------------------------------------------------------
// Dense x low-density sparse partials (LocalMatrix.scala:892, dm.multiply(sp.toDense)) from the stored entries of S, after every
// sparse x dense partial of the same blocks: C (+)= A S as C^T = S^T A^T on spmm2_kernel's dense x sparse variant (spmm.cu).
// S goes in as its CSC arrays (a CSR block through sptrans), A as a column-major image (row-major or unaligned blocks through an
// EW_COPY into the scratch).  A flag pass over the A images and a fix-up after the partials give the NaN of a non-finite A(i, k)
// meeting an implicit zero of S, as the dense image does.  No host synchronisation.
// ------------------------------------------------------------------------------------------------
void run_dense_sparse(mr_context* ctx, const std::vector<OutPlan>& plans, const std::vector<double*>& cptr) {
  std::vector<size_t> routed;
  for (size_t i = 0; i < plans.size(); ++i)
    if (plans[i].has(ROUTE_DSPMM) && plans[i].m > 0 && plans[i].n > 0) routed.push_back(i);
  if (routed.empty()) return;
  // ---- scratch: one buffer (CSC copies of CSR blocks, prepared segments, column-major images, non-finite sets), and one small
  // zero-filled one (the per-block "any non-finite" flags)
  size_t bytes = 0, zbytes = 0;
  auto take = [](size_t& total, size_t n) {
    const size_t off = total;
    total += align_up(std::max<size_t>(n, 1));
    return off;
  };
  struct SInfo {
    size_t csc = 0;  // CSC copy of a CSR block
    size_t ent = 0, rp = 0, seg = 0, kref = 0;
  };
  struct AInfo {
    bool copy = false;
    size_t img = 0, bits = 0, rowflags = 0, any = 0;
  };
  std::map<const Block*, SInfo> sinfo;
  std::map<const Block*, AInfo> ainfo;
  std::vector<const Block*> sorder, aorder;
  for (size_t i : routed)
    for (const PlanPair& pr : plans[i].pairs) {
      if (pr.route != ROUTE_DSPMM) continue;
      const Block &a = *pr.a, &sb = *pr.b;
      wait_ready(ctx, a);
      wait_ready(ctx, sb);
      if (!sinfo.count(&sb)) {
        SInfo v;
        if (sb.isT) v.csc = take(bytes, CscLayout(sb.numCols, sb.valuesLen).bytes);
        size_t eo, ro, so, ko;
        const size_t aux = take(bytes, dspmm_aux_bytes(sb.numCols, sb.numRows, sb.valuesLen, &eo, &ro, &so, &ko));
        v.ent = aux + eo;
        v.rp = aux + ro;
        v.seg = aux + so;
        v.kref = aux + ko;
        sinfo.emplace(&sb, v);
        sorder.push_back(&sb);
      }
      if (!ainfo.count(&a)) {
        AInfo v;
        v.copy = a.isT || (reinterpret_cast<uintptr_t>(a.values.ptr<double>()) & 15) != 0;
        if (v.copy) v.img = take(bytes, static_cast<size_t>(a.numRows) * a.numCols * sizeof(double));
        v.bits = take(bytes, static_cast<size_t>(a.numRows) * DS_KW * sizeof(uint32_t));
        v.rowflags = take(bytes, static_cast<size_t>((a.numRows + 31) / 32) * sizeof(uint32_t));
        v.any = take(zbytes, sizeof(int32_t));
        ainfo.emplace(&a, v);
        aorder.push_back(&a);
      }
    }
  Buf scratch = std::make_shared<DevBuf>(ctx, bytes), zero = std::make_shared<DevBuf>(ctx, zbytes);
  CUDA_CHECK(cudaMemsetAsync(zero->p, 0, zbytes, ctx->stream));
  char* const base = static_cast<char*>(scratch->p);
  char* const zbase = static_cast<char*>(zero->p);
  auto csc_of = [&](const Block* sb, const int32_t*& ptr, const int32_t*& idx, const double*& val) {
    if (sb->isT) {
      const char* w = base + sinfo.at(sb).csc;
      const CscLayout L(sb->numCols, sb->valuesLen);
      ptr = reinterpret_cast<const int32_t*>(w + L.ptr);
      idx = reinterpret_cast<const int32_t*>(w + L.idx);
      val = reinterpret_cast<const double*>(w + L.val);
    } else {
      ptr = sb->colPtrs.ptr<int32_t>();
      idx = sb->rowIndices.ptr<int32_t>();
      val = sb->values.ptr<double>();
    }
  };
  auto image_of = [&](const Block* a) {
    const AInfo& v = ainfo.at(a);
    return v.copy ? reinterpret_cast<const double*>(base + v.img) : a->values.ptr<double>();
  };
  // ---- CSR right blocks -> CSC
  {
    std::vector<CsrToCsc> cv;
    for (const Block* sb : sorder)
      if (sb->isT)
        cv.push_back(CsrToCsc{sb->colPtrs.ptr<int32_t>(), sb->rowIndices.ptr<int32_t>(), sb->values.ptr<double>(), sb->numRows,
                              sb->numCols, sb->valuesLen, base + sinfo.at(sb).csc});
    csr_to_csc(ctx, cv);
  }
  // ---- segments of S^T (one prepared copy per right block)
  {
    std::vector<DspmmPrep> preps;
    int max_n = 0, max_k = 0;
    for (const Block* sb : sorder) {
      const SInfo& v = sinfo.at(sb);
      DspmmPrep pp{};
      const double* val;
      csc_of(sb, pp.ptrs, pp.idx, val);
      pp.vals = val;
      pp.m = sb->numCols;
      pp.kdim = sb->numRows;
      pp.ent = reinterpret_cast<unsigned char*>(base + v.ent);
      pp.rp = reinterpret_cast<int32_t*>(base + v.rp);
      pp.segoff = reinterpret_cast<int32_t*>(base + v.seg);
      pp.kref = reinterpret_cast<uint8_t*>(base + v.kref);
      pp.repeats_reversed = sb->isT ? 1 : 0;  // sptrans_fill_kernel places a row's entries of one column counting down
      preps.push_back(pp);
      max_n = std::max(max_n, pp.m);
      max_k = std::max(max_k, pp.kdim);
    }
    Buf d_preps = upload(ctx, preps);
    CUDA_CHECK(launch_dspmm_prep(static_cast<const DspmmPrep*>(d_preps->p), static_cast<int>(preps.size()), max_n, max_k, ctx->stream));
    note_launch(ctx);
  }
  // ---- column-major images of row-major or unaligned left blocks, and their non-finite sets
  {
    std::vector<EwDesc> copies;
    std::vector<DsFlagDesc> flags;
    int max_r = 0, max_c = 0, max_m = 0;
    bool any_t = false;
    for (const Block* a : aorder) {
      const AInfo& v = ainfo.at(a);
      if (v.copy) {
        EwDesc d{};
        d.A = a->values.ptr<double>();
        d.C = reinterpret_cast<double*>(base + v.img);
        d.rows = a->numRows;
        d.cols = a->numCols;
        d.aT = a->isT ? 1 : 0;
        any_t = any_t || a->isT;
        max_r = std::max(max_r, d.rows);
        max_c = std::max(max_c, d.cols);
        copies.push_back(d);
      }
      flags.push_back(DsFlagDesc{image_of(a), a->numRows, a->numCols, reinterpret_cast<uint32_t*>(base + v.bits),
                                 reinterpret_cast<uint32_t*>(base + v.rowflags), reinterpret_cast<int32_t*>(zbase + v.any)});
      max_m = std::max(max_m, a->numRows);
    }
    if (!copies.empty()) {
      Buf d_cp = upload(ctx, copies);
      CUDA_CHECK(launch_ew_batched(EW_COPY, static_cast<const EwDesc*>(d_cp->p), static_cast<int>(copies.size()), max_r, max_c, any_t,
                                   ctx->stream));
      note_launch(ctx);
    }
    Buf d_fl = upload(ctx, flags);
    CUDA_CHECK(launch_ds_flags(static_cast<const DsFlagDesc*>(d_fl->p), static_cast<int>(flags.size()), max_m, ctx->stream));
    note_launch(ctx);
  }
  // ---- the partials: one CTA per (256 columns, 64 rows) of an output block, over all of its routed pairs; then the fix-up
  std::vector<Spmm2Out> outs;
  std::vector<DspmmPair> pairs;
  std::vector<DsFixPair> fixes;
  struct Keyed {
    int32_t rid, ctile, cid, strip;
    Spmm2Item it;
  };
  std::vector<Keyed> items;
  for (size_t i : routed) {
    const OutPlan& o = plans[i];
    Spmm2Out fo{};
    fo.C = cptr[i];
    fo.m = o.n;
    fo.n = o.m;
    fo.pair_begin = static_cast<int32_t>(pairs.size());
    fo.accumulate = o.has_spmm() ? 1 : 0;  // the block's sparse x dense partials ran before
    for (const PlanPair& pr : o.pairs) {
      if (pr.route != ROUTE_DSPMM) continue;
      const Block &a = *pr.a, &sb = *pr.b;
      const SInfo& v = sinfo.at(&sb);
      const AInfo& av = ainfo.at(&a);
      DspmmPair dp{};
      dp.ent = reinterpret_cast<const unsigned char*>(base + v.ent);
      dp.rp = reinterpret_cast<const int32_t*>(base + v.rp);
      dp.segoff = reinterpret_cast<const int32_t*>(base + v.seg);
      dp.kref = reinterpret_cast<const uint8_t*>(base + v.kref);
      dp.A = image_of(&a);
      dp.kdim = sb.numRows;
      dp.lda = a.numRows;
      pairs.push_back(dp);
      DsFixPair fx{};
      const double* val;
      csc_of(&sb, fx.ptr, fx.idx, val);
      fx.bits = reinterpret_cast<const uint32_t*>(base + av.bits);
      fx.rowflags = reinterpret_cast<const uint32_t*>(base + av.rowflags);
      fx.any = reinterpret_cast<const int32_t*>(zbase + av.any);
      fx.C = cptr[i];
      fx.m = o.m;
      fx.n = o.n;
      fixes.push_back(fx);
      ctx->stats.dspmm_pairs += 1;
      ctx->stats.dspmm_products += sb.valuesLen * a.numRows;
    }
    fo.pair_count = static_cast<int32_t>(pairs.size()) - fo.pair_begin;
    const int32_t oi = static_cast<int32_t>(outs.size());
    outs.push_back(fo);
    for (int st = 0; st * kSpmm2StripRows < o.n; ++st)
      for (int ct = 0; ct * kSpmm2TileCols < o.m; ++ct) items.push_back(Keyed{o.rid, ct, o.cid, st, Spmm2Item{oi, st, ct, 0}});
  }
  // CTAs resident together read the same 64-row panel of a block row of A: order by (block row, tile, block column, strip)
  std::sort(items.begin(), items.end(), [](const Keyed& x, const Keyed& y) {
    return std::tie(x.rid, x.ctile, x.cid, x.strip) < std::tie(y.rid, y.ctile, y.cid, y.strip);
  });
  std::vector<Spmm2Item> sorted(items.size());
  for (size_t t = 0; t < items.size(); ++t) sorted[t] = items[t].it;
  Buf d_outs = upload(ctx, outs), d_pairs = upload(ctx, pairs), d_items = upload(ctx, sorted), d_fix = upload(ctx, fixes);
  KernelTimer timer(ctx);
  CUDA_CHECK(launch_dspmm(static_cast<const Spmm2Item*>(d_items->p), static_cast<int>(sorted.size()), static_cast<const Spmm2Out*>(d_outs->p),
                          static_cast<const DspmmPair*>(d_pairs->p), ctx->stream));
  note_launch(ctx);
  timer.stop();
  CUDA_CHECK(launch_ds_fixup(static_cast<const DsFixPair*>(d_fix->p), static_cast<int>(fixes.size()), ctx->stream));
  note_launch(ctx);
}

// ------------------------------------------------------------------------------------------------
// Matrix x thin-matrix products (DESIGN section 4.5.5): C = A X (rightColNum <= kMvMaxCols) or C = X A (leftRowNum <= kMvMaxCols)
// whose thin side is all dense, over matrix blocks of any kind, computed by matvec.cu as C = M X with M = A or A^T.  The pairs whose terms of an output are
// scattered over the stored lines (CSC blocks of A x, CSR blocks of x A) and the x A pairs of CSC blocks get their partials from
// the pre-pass; everything else, and the sum over k, is ONE launch.  No host synchronisation.
// ------------------------------------------------------------------------------------------------
int matvec_route(const mr_context* ctx, const mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, const mr_matrix* right,
                 int64_t rightRowNum, int64_t rightColNum, int32_t blkSize) {
  auto all_dense = [](const mr_matrix* m) {
    for (auto& kv : m->blocks)
      if (!kv.second.dense()) return false;
    return true;
  };
  int side = MV_NONE;
  if (rightColNum >= 1 && rightColNum <= kMvMaxCols && all_dense(right)) side = MV_AX;
  else if (leftRowNum >= 1 && leftRowNum <= kMvMaxCols && all_dense(left)) side = MV_XA;
  if (side == MV_NONE || ctx->gemm_algo == 0) return side;
  // gemm_algo 1-4 request an engine for the dense x dense pairs: a product with one keeps the engines
  const mr_matrix* mat = side == MV_AX ? left : right;
  const mr_matrix* vec = side == MV_AX ? right : left;
  const bool outer = ceil_div(leftColNum, blkSize) == 1 && ceil_div(rightRowNum, blkSize) == 1;  // every block meets every block
  std::set<int32_t> ks;
  for (auto& kv : vec->blocks) ks.insert(side == MV_AX ? kv.first.first : kv.first.second);
  for (auto& kv : mat->blocks)
    if (kv.second.dense() && (outer ? !ks.empty() : ks.count(side == MV_AX ? kv.first.second : kv.first.first) != 0)) return MV_NONE;
  return side;
}

// A Gram product C = A^T A or A A^T (DESIGN section 4.1.2), from block metadata: every block (k, j) of right has a block (j, k) in
// left over the same device arrays, with swapped dims and the opposite layout flag (what mr_transpose makes), both have the same
// number of blocks, C is square, and the product is not on the matrix x vector route.  Then GRAM_DENSE when every block is dense
// and gemm_algo is 0, 1 or 4 (2 and 3 keep the general route); GRAM_SPARSE when every block is sparse, under any gemm_algo (the
// sparse x sparse chains do not depend on it), and multiply_impl keeps it only when every output block is a chain.
GramKind gram_route(const mr_context* ctx, const mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, const mr_matrix* right,
                    int64_t rightRowNum, int64_t rightColNum, int32_t blkSize) {
  if (leftRowNum != rightColNum || leftColNum != rightRowNum || left->blocks.size() != right->blocks.size()) return GRAM_NONE;
  size_t ndense = 0;
  for (auto& kv : right->blocks) {
    auto it = left->blocks.find({kv.first.second, kv.first.first});
    if (it == left->blocks.end()) return GRAM_NONE;
    const Block &a = it->second, &b = kv.second;
    if (a.dense() != b.dense() || a.numRows != b.numCols || a.numCols != b.numRows || a.isT == b.isT) return GRAM_NONE;
    if (a.values.ptr<double>() != b.values.ptr<double>() || a.colPtrs.ptr<int32_t>() != b.colPtrs.ptr<int32_t>() ||
        a.rowIndices.ptr<int32_t>() != b.rowIndices.ptr<int32_t>())
      return GRAM_NONE;
    ndense += a.dense() ? 1 : 0;
  }
  if (matvec_route(ctx, left, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize) != MV_NONE) return GRAM_NONE;
  if (ndense == 0) return GRAM_SPARSE;
  if (ndense < right->blocks.size()) return GRAM_NONE;  // mixed: pairs (i, j) and (j, i) take different kernels
  return ctx->gemm_algo == 0 || ctx->gemm_algo == 1 || ctx->gemm_algo == 4 ? GRAM_DENSE : GRAM_NONE;
}

void run_matvec(mr_context* ctx, const std::vector<OutPlan>& plans, const std::vector<double*>& cptr, bool xa) {
  std::vector<MvOut> outs;
  std::vector<MvPair> pairs;
  std::vector<MvItem> items;
  std::vector<MvPartDesc> parts;
  std::vector<MvXLayout> pair_xl, part_xl;   // the X block strides of each pair / pre-pass partial
  std::vector<size_t> part_pair, part_off;  // per pre-pass partial: its pair, its offset (elements) in the scratch
  size_t part_elems = 0;
  int max_nlines = 0, max_across = 0, max_cols = 1;
  for (size_t i = 0; i < plans.size(); ++i) {
    const OutPlan& o = plans[i];
    if (o.m <= 0 || o.n <= 0) continue;
    const int32_t len = xa ? o.n : o.m, cols = xa ? o.m : o.n;
    max_cols = std::max(max_cols, static_cast<int>(cols));
    MvOut mo{};
    mo.C = cptr[i];
    mo.len = len;
    mo.cols = cols;
    mo.pair_begin = static_cast<int32_t>(pairs.size());
    mo.pair_count = static_cast<int32_t>(o.pairs.size());
    for (const PlanPair& g : o.pairs) {
      const Block& a = xa ? *g.b : *g.a;  // the matrix block
      const Block& x = xa ? *g.a : *g.b;  // the thin block: kdim x cols (A X) or cols x kdim (X A), in either layout
      wait_ready(ctx, a);
      wait_ready(ctx, x);
      // x(c, j) = X(c, j) for A X, X(j, c) for X A; the inner index c is contiguous when the block's layout runs along it
      const int32_t ld = x.isT ? x.numCols : x.numRows;
      const MvXLayout xl = xa == x.isT ? MvXLayout{1, ld} : MvXLayout{ld, 1};
      pair_xl.push_back(xl);
      MvPair p{};
      p.x = x.values.ptr<double>();
      p.kdim = xa ? a.numRows : a.numCols;
      ctx->stats.mv_pairs += 1;
      if (a.dense()) {
        p.A = a.values.ptr<double>();
        // M(i, c) = A(i, c) for A x, A(c, i) for x A; column-major A(r, c) at r + c numRows, row-major at r numCols + c
        const int64_t rs = a.isT ? a.numCols : 1, cs = a.isT ? 1 : a.numRows;
        p.si = xa ? cs : rs;
        p.sc = xa ? rs : cs;
        p.kind = p.sc == 1 ? MV_DENSE_KCONT : MV_DENSE_ICONT;
      } else {
        ctx->stats.mv_sparse_entries += a.valuesLen;
        const bool csr = a.isT;
        if (!xa && csr) {
          p.kind = MV_CSR;
          p.ptr = a.colPtrs.ptr<int32_t>();
          p.idx = a.rowIndices.ptr<int32_t>();
          p.val = a.values.ptr<double>();
        } else {
          MvPartDesc d{};
          d.ptr = a.colPtrs.ptr<int32_t>();
          d.idx = a.rowIndices.ptr<int32_t>();
          d.val = a.values.ptr<double>();
          d.x = p.x;
          d.nlines = csr ? a.numRows : a.numCols;
          d.len = len;
          d.xlen = p.kdim;
          d.mode = (xa && !csr) ? MV_ALONG : MV_ACROSS;
          d.image = xa ? 1 : 0;
          d.cols = cols;
          max_nlines = std::max(max_nlines, d.mode == MV_ALONG ? d.nlines : 1);
          if (d.mode == MV_ACROSS) max_across = std::max(max_across, len);
          p.kind = MV_PART;
          part_pair.push_back(pairs.size());
          part_off.push_back(part_elems);
          part_elems += align_up(static_cast<size_t>(len) * cols * sizeof(double)) / sizeof(double);
          parts.push_back(d);
          part_xl.push_back(xl);
        }
      }
      pairs.push_back(p);
    }
    const int32_t oi = static_cast<int32_t>(outs.size());
    outs.push_back(mo);
    for (int32_t t = 0; t * kMvTile < len; ++t) items.push_back(MvItem{oi, t});
  }
  if (items.empty()) return;
  Buf scratch;
  // The strides are only read above width 1
  const auto xls = [&](const std::vector<MvXLayout>& v) { return max_cols > 1 ? upload(ctx, v) : Buf(); };
  if (!parts.empty()) {  // the partials: at most one output block per pair
    scratch = std::make_shared<DevBuf>(ctx, part_elems * sizeof(double));
    double* base = static_cast<double*>(scratch->p);
    for (size_t t = 0; t < parts.size(); ++t) {
      parts[t].part = base + part_off[t];
      pairs[part_pair[t]].part = base + part_off[t];
    }
    Buf d_parts = upload(ctx, parts), d_part_xl = xls(part_xl);
    CUDA_CHECK(launch_matvec_parts(static_cast<const MvPartDesc*>(d_parts->p), static_cast<int>(parts.size()), max_nlines, max_across,
                                   max_cols, d_part_xl ? static_cast<const MvXLayout*>(d_part_xl->p) : nullptr, ctx->stream));
    note_launch(ctx);
  }
  Buf d_outs = upload(ctx, outs), d_pairs = upload(ctx, pairs), d_items = upload(ctx, items), d_pair_xl = xls(pair_xl);
  CUDA_CHECK(launch_matvec(static_cast<const MvOut*>(d_outs->p), static_cast<const MvPair*>(d_pairs->p),
                           static_cast<const MvItem*>(d_items->p), static_cast<int>(items.size()), max_cols,
                           d_pair_xl ? static_cast<const MvXLayout*>(d_pair_xl->p) : nullptr, xa, ctx->stream));
  note_launch(ctx);
}

// Allocates all output blocks from one slab (packed in plan order, or at their slots when the result is a sharded dataset), or takes
// them from the caller's windows.  Returns where each plan's block is written.
std::vector<double*> allocate_outputs(mr_context* ctx, const std::vector<OutPlan>& plans, mr_matrix* result,
                                      const OutWindowFn* out_windows) {
  const ShardInfo* out_shard = result->shard.get();
  std::vector<double*> cptr(plans.size());
  if (out_windows) {
    for (size_t i = 0; i < plans.size(); ++i) {
      auto& o = plans[i];
      Span s = (*out_windows)(o.rid, o.cid);
      cptr[i] = s.ptr<double>();
      result->blocks[{o.rid, o.cid}] = dense_block(o.m, o.n, s, false);
    }
  } else if (out_shard) {
    const ShardLayout& L = out_shard->L;
    // absent output blocks must read as zeros for whoever pulls this slab later (a sharded dataset is dense over its grid)
    if (static_cast<int64_t>(plans.size()) < L.slots_r_of(L.r) * ((L.nbc > L.c ? (L.nbc - L.c + L.pc - 1) / L.pc : 0)))
      CUDA_CHECK(cudaMemsetAsync(out_shard->slab->p, 0, out_shard->slab->bytes, ctx->stream));
    for (size_t i = 0; i < plans.size(); ++i) {
      auto& o = plans[i];
      MR_REQUIRE(o.rid % L.pr == L.r && o.cid % L.pc == L.c && o.rid < L.nbr && o.cid < L.nbc, MR_EINVAL,
                 "output block (%d, %d) does not belong to rank (%d, %d)", o.rid, o.cid, L.r, L.c);
      Span s{out_shard->slab, static_cast<size_t>(L.slot(o.rid, o.cid)) * L.slot_elems * sizeof(double)};
      cptr[i] = s.ptr<double>();
      result->blocks[{o.rid, o.cid}] = dense_block(o.m, o.n, s, false);
    }
  } else {
    // chain outputs (run_sparse_chains) get their arrays once their format is known: a dense window only if they end dense
    auto chain_out = [&](const OutPlan& o) { return o.has(ROUTE_SPSP) && o.m > 0 && o.n > 0; };
    size_t total = 0;
    for (auto& o : plans)
      if (!chain_out(o)) total += align_up(static_cast<size_t>(o.m) * o.n * sizeof(double));
    Slab slab(ctx, total);
    for (size_t i = 0; i < plans.size(); ++i) {
      auto& o = plans[i];
      if (chain_out(o)) continue;  // cptr[i] stays null
      Span s = slab.take(static_cast<size_t>(o.m) * o.n * sizeof(double));
      cptr[i] = s.ptr<double>();
      result->blocks[{o.rid, o.cid}] = dense_block(o.m, o.n, s, false);  // product is never transposed (MLMatrix.scala:101)
    }
  }
  return cptr;
}

// A Gram product's strictly-lower elements, from their transposes (gram_mirror_kernel), behind everything that writes the blocks
// on and above the diagonal.
void run_gram_mirror(mr_context* ctx, const std::vector<OutPlan>& plans, const std::vector<double*>& cptr) {
  std::map<std::pair<int32_t, int32_t>, size_t> at;
  for (size_t i = 0; i < plans.size(); ++i) at[{plans[i].rid, plans[i].cid}] = i;
  std::vector<GramMirror> items;
  int max_m = 0, max_n = 0;
  for (size_t i = 0; i < plans.size(); ++i) {
    const OutPlan& o = plans[i];
    if (o.rid < o.cid || o.m == 0 || o.n == 0) continue;
    const size_t up = at.at({o.cid, o.rid});
    items.push_back(GramMirror{cptr[up], cptr[i], o.m, o.n, o.rid == o.cid ? 1 : 0, 0});
    max_m = std::max(max_m, o.m);
    max_n = std::max(max_n, o.n);
    if (o.rid > o.cid) ctx->stats.gram_mirrored_blocks += 1;
  }
  if (items.empty()) return;
  Buf d_items = upload(ctx, items);
  CUDA_CHECK(launch_gram_mirror(static_cast<const GramMirror*>(d_items->p), static_cast<int>(items.size()), max_m, max_n, ctx->stream));
  note_launch(ctx);
}

// The GEMM pairs of every output block on the dense engines: Ozaki-I / 3xTF32 (gemm_algo 2 / 3) when they fit, else ONE fused
// DMMA launch (chunked while operands are still arriving from the host), behind the Ozaki-II engine when `dec` says to try it.
// gram: a Gram product (DESIGN section 4.1.2), whose engines compute the blocks on and above the diagonal only; the mirror pass
// writes the rest.
void run_dense_engines(mr_context* ctx, const std::vector<OutPlan>& plans, const std::vector<double*>& cptr, const MultiplyDecisions& dec,
                       int32_t blkSize, mr_matrix* result, int64_t M, int64_t K, int64_t N, bool outer, bool gram) {
  std::vector<GemmOut> outs;
  std::vector<GemmPair> pairs;
  std::vector<size_t> out_plan;
  int64_t flops = 0;
  for (size_t i = 0; i < plans.size(); ++i) {
    const OutPlan& o = plans[i];
    if (!o.has(ROUTE_GEMM) || o.m == 0 || o.n == 0 || (gram && o.rid > o.cid)) continue;
    GemmOut go{};
    go.C = cptr[i];
    go.m = o.m;
    go.n = o.n;
    go.pair_begin = static_cast<int32_t>(pairs.size());
    for (const PlanPair& g : o.pairs) {
      if (g.route != ROUTE_GEMM) continue;
      GemmPair p{};
      p.A = g.a->values.ptr<double>();
      p.B = g.b->values.ptr<double>();
      p.aT = g.a->isT;
      p.bT = g.b->isT;
      p.lda = g.a->isT ? g.a->numCols : g.a->numRows;  // BLAS.scala:335
      p.ldb = g.b->isT ? g.b->numCols : g.b->numRows;  // BLAS.scala:336
      p.kdim = g.a->numCols;
      p.tmA = p.tmB = -1;
      pairs.push_back(p);
      flops += 2ll * o.m * o.n * p.kdim;
    }
    go.pair_count = static_cast<int32_t>(pairs.size()) - go.pair_begin;
    outs.push_back(go);
    out_plan.push_back(i);
  }
  if (outs.empty()) return;
  if (gram) ctx->stats.gram_blocks = static_cast<int64_t>(outs.size());
  // which dense operands are still being produced on another stream (ingest copies)?
  bool pending = false;
  for (size_t i = 0; i < plans.size() && !pending; ++i)
    for (const PlanPair& g : plans[i].pairs)
      if (g.route == ROUTE_GEMM && ((g.a->ready && !block_done(*g.a)) || (g.b->ready && !block_done(*g.b)))) {
        pending = true;
        break;
      }
  (void)cudaGetLastError();
  // gemm_algo: 0 = auto (Ozaki-II on wgmma with the range guard when the product is large and regular, else DMMA), 1 = DMMA,
  // 2 = Ozaki-I, 3 = 3xTF32, 4 = Ozaki-II without the range guard
  const int algo = ctx->gemm_algo;
  if (algo == 2 || algo == 3) {
    for (const OutPlan& o : plans)
      for (const PlanPair& g : o.pairs)
        if (g.route == ROUTE_GEMM) {
          wait_ready(ctx, *g.a);
          wait_ready(ctx, *g.b);
        }
    if (try_ozaki(ctx, plans, cptr, blkSize, M, K, N, outer)) {
      ctx->stats.last_gemm_flops = flops;
      return;
    }
  }
  const int variant = ctx->force_variant >= 0 ? ctx->force_variant : dec.variant;
  const int BM = gemm_tile_m(variant), BN = gemm_tile_n(variant);
  const int tpbm = std::max(1, (blkSize + BM - 1) / BM), tpbn = std::max(1, (blkSize + BN - 1) / BN);
  struct Keyed {
    int64_t band, gm, gn;
    GemmTile t;
  };
  std::vector<Keyed> keyed;
  constexpr int kBand = 12;  // the ~132 resident tiles (12 columns x 11 rows) share A row- and B column-panels in L2; carried over, not re-tuned for H100
  for (size_t oi = 0; oi < outs.size(); ++oi) {
    const OutPlan& o = plans[out_plan[oi]];
    const int tm = (outs[oi].m + BM - 1) / BM, tn = (outs[oi].n + BN - 1) / BN;
    for (int a = 0; a < tm; ++a)
      for (int b = 0; b < tn; ++b) {
        const int64_t gm = static_cast<int64_t>(o.rid) * tpbm + a, gn = static_cast<int64_t>(o.cid) * tpbn + b;
        keyed.push_back({gn / kBand, gm, gn, GemmTile{static_cast<int32_t>(oi), a, b, 0}});
      }
  }
  // Chunked launch when operands are still arriving from the host: one launch per block row of C, each waiting
  // only for the A row panel it reads (and all of B), so compute overlaps the remaining ingest and the egress of
  // finished rows.  With resident operands it is ONE launch.
  // Chunk key of an output block = ingest sequence number of the LAST operand block it needs that is still in flight
  // (the ingest stream is in order, so waiting for that one copy implies all earlier ones).  Output blocks are
  // launched in key order, in chunks of >= ~8 waves of tiles, so whatever has landed is multiplied while the rest of
  // A and B is still on the wire -- row panels, column panels or an interleaving of both, whatever order the caller
  // uploaded them in.
  const bool chunked = pending && ctx->pipeline != 0;
  std::vector<int> group_of(outs.size(), 0);
  int ngroups_dyn = 1;
  if (chunked) {
    std::vector<std::pair<uint64_t, size_t>> order(outs.size());
    for (size_t oi = 0; oi < outs.size(); ++oi) {
      uint64_t key = 0;
      for (const PlanPair& g : plans[out_plan[oi]].pairs) {
        if (g.route != ROUTE_GEMM) continue;
        if (g.a->ready) key = std::max(key, g.a->seq);
        if (g.b->ready) key = std::max(key, g.b->seq);
      }
      order[oi] = {key, oi};
    }
    std::sort(order.begin(), order.end());
    const int64_t min_tiles = 132;  // >= one wave; the launches overlap on the side streams, so small chunks cost nothing
    int64_t acc_tiles = 0;
    int gcur = 0;
    for (size_t r = 0; r < order.size(); ++r) {
      const size_t oi = order[r].second;
      // close the chunk when it is big enough AND the next block waits for a later copy
      if (acc_tiles >= min_tiles && r > 0 && order[r].first != order[r - 1].first) {
        ++gcur;
        acc_tiles = 0;
      }
      group_of[oi] = gcur;
      acc_tiles += static_cast<int64_t>((outs[oi].m + BM - 1) / BM) * ((outs[oi].n + BN - 1) / BN);
    }
    ngroups_dyn = gcur + 1;
  }
  // The int8 tensor-core path (Ozaki-II residues + CRT) runs group by group in front of the DMMA launches, which then only execute
  // when the engine's device flag reports operands it cannot represent.  Small products stay on the exact kernel in auto mode.
  Oz2Run oz2;
  const bool use_oz2 = dec.oz2 && oz2.plan(ctx, plans, out_plan, cptr, group_of, ngroups_dyn, blkSize, M, K, N, outer, algo == 0, gram, chunked);
  auto grp = [&](const Keyed& k) { return group_of[k.t.out]; };
  std::sort(keyed.begin(), keyed.end(), [&](const Keyed& x, const Keyed& y) {
    const int gx = grp(x), gy = grp(y);
    if (gx != gy) return gx < gy;
    if (x.band != y.band) return x.band < y.band;
    if (x.gm != y.gm) return x.gm < y.gm;
    return x.gn < y.gn;
  });
  std::vector<GemmTile> tiles(keyed.size());
  for (size_t i = 0; i < keyed.size(); ++i) tiles[i] = keyed[i].t;
  // TMA descriptors of the K-contiguous operand blocks (row-major A blocks, column-major B blocks)
  struct TmapBytes { unsigned char b[128]; };
  std::vector<TmapBytes> tmaps;
  std::map<std::tuple<const double*, int64_t, int64_t, int64_t>, int32_t> tmap_index;
  auto tmap_of = [&](const double* base, int64_t kdim, int64_t rows, int64_t ld, int tile) -> int32_t {
    auto key = std::make_tuple(base, kdim, rows, ld);
    auto it = tmap_index.find(key);
    if (it != tmap_index.end()) return it->second;
    TmapBytes t;
    int32_t idx = -1;
    if (encode_kcontig_tmap(t.b, base, kdim, rows, ld, tile)) {
      idx = static_cast<int32_t>(tmaps.size());
      tmaps.push_back(t);
    }
    tmap_index.emplace(key, idx);
    return idx;
  };
  for (auto& go : outs)
    for (int p = go.pair_begin; p < go.pair_begin + go.pair_count; ++p) {
      GemmPair& pr = pairs[p];
      if (pr.aT) pr.tmA = tmap_of(pr.A, pr.kdim, go.m, pr.lda, BM);
      if (!pr.bT) pr.tmB = tmap_of(pr.B, pr.kdim, go.n, pr.ldb, BN);
    }
  Buf d_outs = upload(ctx, outs), d_pairs = upload(ctx, pairs), d_tiles = upload(ctx, tiles), d_tmaps = upload(ctx, tmaps);
  if (use_oz2) {
    oz2.upload_tables();
    ctx->stats.tc_int8_ops = oz2.int8_ops;
    ctx->stats.tc_moduli = oz2_moduli(oz2.eng);
    ctx->stats.tc_strassen_jobs = oz2.strassen ? static_cast<int64_t>(oz2.jobs.size()) : 0;
    ctx->stats.tc_gemm_launches += 1;
  }
  KernelTimer timer(ctx);
  const int ngroups = ngroups_dyn;
  const bool side = chunked && ngroups > 1;
  if (side) {  // fork: the side streams start after everything enqueued so far (output slab, descriptor tables)
    CUDA_CHECK(cudaEventRecord(ctx->ev_order, ctx->stream));
    for (int i = 0; i < mr_context::kChunkStreams; ++i) CUDA_CHECK(cudaStreamWaitEvent(ctx->chunk_stream[i], ctx->ev_order, 0));
  }
  size_t t0 = 0;
  for (int gi = 0; gi < ngroups; ++gi) {
    size_t t1 = t0;
    while (t1 < keyed.size() && grp(keyed[t1]) == gi) ++t1;
    // DMMA chunks are independent launches: round-robin over the side streams so that tails overlap.  The Ozaki-II engine's
    // jobs share its residue planes and each fills the machine by itself (persistent kernel): one side stream, in order.
    cudaStream_t cs = side ? ctx->chunk_stream[use_oz2 ? 0 : gi % mr_context::kChunkStreams] : ctx->stream;
    // wait for exactly the operand blocks this chunk reads
    std::vector<char> seen(outs.size(), 0);
    for (size_t t = t0; t < t1; ++t) {
      const int oi = keyed[t].t.out;
      if (seen[oi]) continue;
      seen[oi] = 1;
      for (const PlanPair& g : plans[out_plan[oi]].pairs) {
        if (g.route != ROUTE_GEMM) continue;
        wait_ready_on(cs, *g.a);
        wait_ready_on(cs, *g.b);
      }
    }
    if (use_oz2) oz2.run_group(gi, cs);
    CUDA_CHECK(launch_gemm_f64(static_cast<const GemmOut*>(d_outs->p), static_cast<const GemmPair*>(d_pairs->p),
                               static_cast<const GemmTile*>(d_tiles->p) + t0, static_cast<int>(t1 - t0), d_tmaps->p, variant,
                               cs, use_oz2 ? oz2.flag() : nullptr));
    note_launch(ctx);
    if (chunked) {  // consumers on the egress stream wait for this chunk only
      ReadyPtr r = std::make_shared<Ready>();
      CUDA_CHECK(cudaEventRecord(r->ev, cs));
      for (size_t oi = 0; oi < outs.size(); ++oi)
        if (seen[oi]) {
          const OutPlan& o = plans[out_plan[oi]];
          // blocks with sparse partials finish later, and a Gram product's diagonal blocks with the mirror pass
          if (!o.has_spmm() && !(gram && o.rid == o.cid)) result->blocks[{o.rid, o.cid}].ready = r;
        }
    }
    t0 = t1;
  }
  if (side) {  // join: later work on the context stream (and the release of the descriptor tables) follows every chunk
    for (int i = 0; i < mr_context::kChunkStreams; ++i) {
      CUDA_CHECK(cudaEventRecord(ctx->chunk_join[i], ctx->chunk_stream[i]));
      CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->chunk_join[i], 0));
    }
  }
  if (gram) run_gram_mirror(ctx, plans, cptr);
  ctx->stats.gemm_launches += 1;
  ctx->stats.last_gemm_flops = flops;
  timer.stop();
}

// ------------------------------------------------------------------------------------------------
// Sparse x dense partial products, accumulated onto the GEMM result (LocalMatrix.add of partials).  CSR pairs with block dims
// <= 1024 go through ONE fused launch (K loop over the pairs inside the kernel): the pipelined TMA kernel of spmm.cu when the
// output block is large enough to fill its 512 x 32 tiles and B can be addressed by a tensor map, else the simple shared-memory
// kernel of ew.cu; CSC pairs and oversized blocks use the per-pair kernels.  In a block, its own sparse x dense pairs come first
// in ascending k, then its low-density sparse x sparse ones (the summation order of the densifying reference).
// ------------------------------------------------------------------------------------------------
void run_sparse_dense(mr_context* ctx, const std::vector<OutPlan>& plans, const std::vector<double*>& cptr) {
  std::vector<SpmmOut> fouts;
  std::vector<SpmmPair> fpairs;
  int fused_max_n = 0;
  std::vector<Spmm2Out> outs2;
  std::vector<std::pair<const Block*, const Block*>> pairs2;  // (S, B) of each pair of the pipelined kernel
  std::vector<Spmm2Item> items2;
  struct Key2 {
    int32_t cid, ctile, rid, strip;
  };
  std::vector<Key2> keys2;
  // scratch offsets: re-packed CSR segments of every sparse block, row-major copies of the column-major dense blocks
  struct SegOff {
    size_t ent, rp, seg;
  };
  std::map<const Block*, SegOff> seg_of;
  std::vector<const Block*> sorder, torder;
  std::map<const Block*, size_t> trans_of;  // column-major dense block -> offset of its row-major copy
  std::map<const Block*, int32_t> tmap_of_b;  // dense block -> tensor map index
  size_t aux_total = 0, trans_total = 0;
  for (size_t i = 0; i < plans.size(); ++i) {
    const OutPlan& o = plans[i];
    bool have = o.has(ROUTE_GEMM);
    if (o.m == 0 || o.n == 0 || o.has(ROUTE_SPSP)) continue;
    std::vector<std::pair<const Block*, const Block*>> slow, fused;
    for (Route r : {ROUTE_SPMM, ROUTE_SPSP_SPMM})
      for (const PlanPair& p : o.pairs) {
        if (p.route != r) continue;
        wait_ready(ctx, *p.a);
        wait_ready(ctx, *p.b);
        if (p.a->isT && o.m <= kSpmmMaxDim && p.a->numCols <= kSpmmMaxDim) fused.emplace_back(p.a, p.b);
        else slow.emplace_back(p.a, p.b);
      }
    for (auto& sp : slow) {  // per-pair kernels first so the fused launch can simply accumulate on top
      const Block& s = *sp.first;
      const Block& b = *sp.second;
      CUDA_CHECK(launch_spmm(s.colPtrs.ptr<int32_t>(), s.rowIndices.ptr<int32_t>(), s.values.ptr<double>(), s.isT,
                             b.values.ptr<double>(), b.isT, cptr[i], s.numRows, s.numCols, b.numCols, have, ctx->stream));
      note_launch(ctx);
      have = true;
    }
    bool use2 = ctx->spmm_algo != 1 && !fused.empty() && o.m >= 128 && o.n >= 16 && (o.n % 2) == 0;
    if (use2)
      for (auto& sp : fused)
        if ((reinterpret_cast<uintptr_t>(sp.second->values.ptr<double>()) & 15) != 0) use2 = false;
    if (use2) {
      Spmm2Out fo{};
      fo.C = cptr[i];
      fo.m = o.m;
      fo.n = o.n;
      fo.pair_begin = static_cast<int32_t>(pairs2.size());
      fo.pair_count = static_cast<int32_t>(fused.size());
      fo.accumulate = have ? 1 : 0;
      for (auto& sp : fused) {
        const Block& sblk = *sp.first;
        const Block& bblk = *sp.second;
        if (!seg_of.count(&sblk)) {
          size_t eo, ro, so;
          const size_t bytes = spmm2_aux_bytes(sblk.numRows, sblk.numCols, sblk.valuesLen, &eo, &ro, &so);
          seg_of.emplace(&sblk, SegOff{aux_total + eo, aux_total + ro, aux_total + so});
          aux_total += bytes;
          sorder.push_back(&sblk);
        }
        if (!tmap_of_b.count(&bblk)) {
          if (!bblk.isT) {  // column-major: row-major copy in the scratch buffer (one transposing pass per multiply)
            trans_of.emplace(&bblk, trans_total);
            trans_total += align_up(static_cast<size_t>(bblk.numRows) * bblk.numCols * sizeof(double));
            torder.push_back(&bblk);
          }
          tmap_of_b.emplace(&bblk, static_cast<int32_t>(tmap_of_b.size()));
        }
        pairs2.push_back(sp);
      }
      const int32_t oi = static_cast<int32_t>(outs2.size());
      outs2.push_back(fo);
      for (int st = 0; st * kSpmm2StripRows < o.m; ++st)
        for (int ct = 0; ct * kSpmm2TileCols < o.n; ++ct) {
          items2.push_back(Spmm2Item{oi, st, ct, 0});
          keys2.push_back(Key2{o.cid, ct, o.rid, st});
        }
      have = true;
    } else if (!fused.empty()) {
      SpmmOut fo{};
      fo.C = cptr[i];
      fo.m = o.m;
      fo.n = o.n;
      fo.pair_begin = static_cast<int32_t>(fpairs.size());
      for (auto& sp : fused) {
        SpmmPair pr{};
        pr.ptrs = sp.first->colPtrs.ptr<int32_t>();
        pr.idx = sp.first->rowIndices.ptr<int32_t>();
        pr.vals = sp.first->values.ptr<double>();
        pr.B = sp.second->values.ptr<double>();
        pr.kdim = sp.first->numCols;
        pr.bT = sp.second->isT;
        fpairs.push_back(pr);
      }
      fo.pair_count = static_cast<int32_t>(fpairs.size()) - fo.pair_begin;
      fo.accumulate = have ? 1 : 0;
      fouts.push_back(fo);
      fused_max_n = std::max(fused_max_n, o.n);
      have = true;
    }
    if (!have && !o.has(ROUTE_DSPMM)) CUDA_CHECK(cudaMemsetAsync(cptr[i], 0, static_cast<size_t>(o.m) * o.n * sizeof(double), ctx->stream));
  }
  if (!fouts.empty()) {
    Buf d_fo = upload(ctx, fouts), d_fp = upload(ctx, fpairs);
    KernelTimer timer(ctx);
    CUDA_CHECK(launch_spmm_fused(static_cast<const SpmmOut*>(d_fo->p), static_cast<int>(fouts.size()),
                                 static_cast<const SpmmPair*>(d_fp->p), fused_max_n, ctx->stream));
    note_launch(ctx);
    timer.stop();
  }
  if (outs2.empty()) return;
  Buf aux = std::make_shared<DevBuf>(ctx, std::max<size_t>(aux_total, 16));
  Buf trans = std::make_shared<DevBuf>(ctx, std::max<size_t>(trans_total, 16));
  char* const aux_base = static_cast<char*>(aux->p);
  char* const trans_base = static_cast<char*>(trans->p);
  std::vector<Spmm2Prep> preps;
  int prep_max_m = 0, prep_max_k = 0;
  for (const Block* s : sorder) {
    const SegOff& so = seg_of.at(s);
    Spmm2Prep pp{};
    pp.ptrs = s->colPtrs.ptr<int32_t>();
    pp.idx = s->rowIndices.ptr<int32_t>();
    pp.vals = s->values.ptr<double>();
    pp.m = s->numRows;
    pp.kdim = s->numCols;
    pp.ent = reinterpret_cast<unsigned char*>(aux_base + so.ent);
    pp.rp = reinterpret_cast<int32_t*>(aux_base + so.rp);
    pp.segoff = reinterpret_cast<int32_t*>(aux_base + so.seg);
    prep_max_m = std::max(prep_max_m, pp.m);
    prep_max_k = std::max(prep_max_k, pp.kdim);
    preps.push_back(pp);
  }
  std::vector<Spmm2Pair> spairs;
  for (auto& sp : pairs2) {
    const SegOff& so = seg_of.at(sp.first);
    Spmm2Pair pr{};
    pr.ent = reinterpret_cast<const unsigned char*>(aux_base + so.ent);
    pr.rp = reinterpret_cast<const int32_t*>(aux_base + so.rp);
    pr.segoff = reinterpret_cast<const int32_t*>(aux_base + so.seg);
    pr.kdim = sp.first->numCols;
    pr.tmB = tmap_of_b.at(sp.second);
    spairs.push_back(pr);
  }
  std::vector<EwDesc> transposes;
  int trans_max_r = 0, trans_max_c = 0;
  for (const Block* b : torder) {
    EwDesc d{};
    d.A = b->values.ptr<double>();
    d.C = reinterpret_cast<double*>(trans_base + trans_of.at(b));
    d.rows = b->numCols;  // the k x n block read as its n x k transpose, stored row-major (aT): see run_sparse_chains
    d.cols = b->numRows;
    d.aT = 1;
    trans_max_r = std::max(trans_max_r, d.rows);
    trans_max_c = std::max(trans_max_c, d.cols);
    transposes.push_back(d);
  }
  struct TmapBytes {
    unsigned char b[128];
  };
  std::vector<TmapBytes> tmaps(tmap_of_b.size());
  bool maps_ok = true;
  for (auto& kv : tmap_of_b) {
    const Block* bb = kv.first;
    const double* base = bb->isT ? bb->values.ptr<double>() : reinterpret_cast<const double*>(trans_base + trans_of.at(bb));
    maps_ok = maps_ok && spmm2_encode_b_tmap(tmaps[kv.second].b, base, bb->numRows, bb->numCols, bb->numCols);
  }
  if (!maps_ok) fail(MR_ECUDA, "cuTensorMapEncodeTiled failed for a dense operand of the sparse x dense multiply");
  // concurrently resident CTAs share the B panel of one 32-column tile: order by (block column, tile, block row, strip)
  std::vector<size_t> ord(items2.size());
  for (size_t t = 0; t < ord.size(); ++t) ord[t] = t;
  std::sort(ord.begin(), ord.end(), [&](size_t x, size_t y) {
    const Key2 &a = keys2[x], &b2 = keys2[y];
    return std::tie(a.cid, a.ctile, a.rid, a.strip) < std::tie(b2.cid, b2.ctile, b2.rid, b2.strip);
  });
  std::vector<Spmm2Item> sorted_items(items2.size());
  for (size_t t = 0; t < ord.size(); ++t) sorted_items[t] = items2[ord[t]];
  Buf d_preps = upload(ctx, preps), d_outs2 = upload(ctx, outs2), d_pairs2 = upload(ctx, spairs), d_items = upload(ctx, sorted_items),
      d_tmaps = upload(ctx, tmaps);
  CUDA_CHECK(launch_spmm2_prep(static_cast<const Spmm2Prep*>(d_preps->p), static_cast<int>(preps.size()), prep_max_m, prep_max_k, ctx->stream));
  note_launch(ctx);
  if (!transposes.empty()) {
    Buf d_tr = upload(ctx, transposes);
    CUDA_CHECK(launch_ew_batched(EW_COPY, static_cast<const EwDesc*>(d_tr->p), static_cast<int>(transposes.size()), trans_max_r,
                                 trans_max_c, true, ctx->stream));
    note_launch(ctx);
  }
  KernelTimer timer(ctx);
  CUDA_CHECK(launch_spmm2(static_cast<const Spmm2Item*>(d_items->p), static_cast<int>(sorted_items.size()),
                          static_cast<const Spmm2Out*>(d_outs2->p), static_cast<const Spmm2Pair*>(d_pairs2->p), d_tmaps->p, ctx->stream));
  note_launch(ctx);
  timer.stop();
  ctx->stats.gemm_launches += 1;
}

void run_multiply(mr_context* ctx, const std::vector<OutPlan>& plans, const MultiplyDecisions& dec, int32_t blkSize, mr_matrix* result,
                  int64_t M, int64_t K, int64_t N, bool outer, const OutWindowFn* out_windows, GramKind gram) {
  const std::vector<double*> cptr = allocate_outputs(ctx, plans, result, out_windows);
  if (dec.mv != MV_NONE) {
    run_matvec(ctx, plans, cptr, dec.mv == MV_XA);
    return;
  }
  run_dense_engines(ctx, plans, cptr, dec, blkSize, result, M, K, N, outer, gram == GRAM_DENSE);
  run_sparse_dense(ctx, plans, cptr);
  run_dense_sparse(ctx, plans, cptr);
  run_sparse_chains(ctx, plans, cptr, result, gram == GRAM_SPARSE);
}

}  // namespace

namespace mrhost {

mr_matrix* multiply_impl(mr_context* ctx, mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right, int64_t rightRowNum,
                         int64_t rightColNum, int32_t blkSize, const ShardLayout* out_layout, const OutWindowFn* out_windows,
                         const MultiplyDecisions* decisions, GramKind gram) {
  for (auto& kv : left->blocks)
    if (!kv.second.dense()) wait_ready(ctx, kv.second);
  for (auto& kv : right->blocks)
    if (!kv.second.dense()) wait_ready(ctx, kv.second);
  const int mv = decisions ? decisions->mv : matvec_route(ctx, left, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize);
  // MatfastExecution.scala:712-713: a single block column of A and block row of B take the outer-product paths
  const bool outer = ceil_div(leftColNum, blkSize) == 1 && ceil_div(rightRowNum, blkSize) == 1;
  std::vector<OutPlan> plans = plan_multiply(left, right, outer, mv != MV_NONE);
  // a sparse Gram product whose output blocks are all chains (every pair at density <= 0.1 on both sides)
  if (gram == GRAM_SPARSE && !std::all_of(plans.begin(), plans.end(), [](const OutPlan& o) { return o.only(ROUTE_SPSP); }))
    gram = GRAM_NONE;
  MultiplyDecisions own;
  if (!decisions) {
    own = decide(ctx, plans, mv);
    decisions = &own;
  }
  std::deque<Block> temps;
  densify_operands(ctx, plans, temps);
  std::unique_ptr<mr_matrix> result(out_layout ? new_sharded(ctx, *out_layout, false, false) : new_matrix(ctx));
  if (out_layout) result->blocks.clear();  // only the blocks the product has are present (join semantics); absent ones stay absent
  run_multiply(ctx, plans, *decisions, blkSize, result.get(), leftRowNum, leftColNum, rightColNum, outer, out_windows, gram);
  return result.release();
}

MultiplyDecisions multiply_decisions(const mr_context* ctx, const mr_matrix* left, int64_t leftRowNum, int64_t leftColNum,
                                     const mr_matrix* right, int64_t rightRowNum, int64_t rightColNum, int32_t blkSize) {
  const int mv = matvec_route(ctx, left, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize);
  MultiplyDecisions d;
  d.mv = mv;
  if (mv != MV_NONE) return d;
  const bool outer = ceil_div(leftColNum, blkSize) == 1 && ceil_div(rightRowNum, blkSize) == 1;
  std::vector<OutPlan> plans;
  try {
    plans = plan_multiply(left, right, outer, false);
  } catch (const MrError&) {
    // plan_multiply raises nothing but its shape checks.  A streamed multiply reports a shape error from the tile that holds the
    // mismatched pair, with the status and message the resident multiply of that tile gives; until then its tiles run with these
    // default decisions (no dense x sparse scratch in the tiling bound) and their results are dropped with the error.
    return d;
  }
  d = decide(ctx, plans, mv);
  // the blocks of the dense x sparse pairs, for the scratch bound of the tiles
  for (const OutPlan& o : plans)
    for (const PlanPair& p : o.pairs)
      if (p.route == ROUTE_DSPMM) {
        d.ds_left.insert({o.rid, p.k});
        d.ds_right.insert({p.kb, o.cid});
      } else if (p.route == ROUTE_GEMM && dspmm_candidate(*p.a, *p.b)) {
        d.ds_dense_right.insert({p.kb, o.cid});
      }
  return d;
}

// Upper bounds of run_dense_sparse's scratch per left block (column-major copy, non-finite sets) and right block (CSC copy of a
// CSR block and its csr_to_csc cursors, prepared segments).
size_t dspmm_left_scratch(const Block& a) {
  return align_up(static_cast<size_t>(a.numRows) * a.numCols * sizeof(double)) +
         align_up(static_cast<size_t>(a.numRows) * DS_KW * sizeof(uint32_t)) +
         align_up(static_cast<size_t>((a.numRows + 31) / 32) * sizeof(uint32_t)) + align_up(sizeof(int32_t));
}
size_t dspmm_right_scratch(const Block& b) {
  size_t eo, ro, so, ko, n = align_up(dspmm_aux_bytes(b.numCols, b.numRows, b.valuesLen, &eo, &ro, &so, &ko));
  if (b.isT) n += CscLayout(b.numCols, b.valuesLen).bytes + align_up(static_cast<size_t>(b.numCols) * sizeof(int32_t));
  return n;
}

size_t oz2_scratch_for(const mr_context* ctx, int32_t blk, int64_t K, int nr, int nc) {
  if (K <= 0 || K >= (1 << 17) || nr <= 0 || nc <= 0) return 0;
  int cap_r = 0, cap_c = 0;
  size_t bytes = 0;
  return oz2_capacity(ctx, blk, K, oz2_moduli_for(K, ctx->crt_moduli), nr, nc, cap_r, cap_c, &bytes) ? bytes : 0;
}

}  // namespace mrhost

extern "C" {

// ------------------------------------------------------------------------------------------------
// ABI: operators
// ------------------------------------------------------------------------------------------------
mr_status mr_matrix_multiply(mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right,
                             int64_t rightRowNum, int64_t rightColNum, int32_t blkSize, mr_matrix** out) {
  return guarded([&] {
    MR_REQUIRE(left && right && out, MR_EINVAL, "null argument");
    MR_REQUIRE(left->ctx == right->ctx, MR_EINVAL, "operands belong to different contexts");
    MR_REQUIRE(blkSize > 0, MR_EINVAL, "blkSize must be positive, got %d", blkSize);
    // MatfastExecution.scala:702-703
    MR_REQUIRE(leftColNum == rightRowNum, MR_EDIM, "Matrix dimension not match, leftColNum = %lld, rightRowNum = %lld",
               (long long)leftColNum, (long long)rightRowNum);
    mr_context* ctx = left->ctx;
    DeviceScope dev(ctx);
    std::lock_guard<std::mutex> lock(ctx->mu);
    ctx->stats.spgemm_pairs = 0;
    ctx->stats.spgemm_products = 0;
    ctx->stats.dspmm_pairs = 0;
    ctx->stats.dspmm_products = 0;
    ctx->stats.mv_pairs = 0;
    ctx->stats.mv_sparse_entries = 0;
    ctx->stats.gram_blocks = 0;
    ctx->stats.gram_mirrored_blocks = 0;
    ctx->stats.tc_strassen_jobs = 0;
    if (left->host || right->host)  // C tile by C tile through the device, into a host-resident result (abi_stream.cpp)
      *out = multiply_streamed(ctx, left, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize);
    else
      *out = multiply_impl(ctx, left, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize, nullptr, nullptr, nullptr,
                           gram_route(ctx, left, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize));
  });
}


}  // extern "C"
