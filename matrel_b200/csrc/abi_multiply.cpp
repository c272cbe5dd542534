// Block multiply: planning (LocalMatrix.matrixMultiplication dispatch), the fused DMMA launch incl. the pipelined chunks,
// the wgmma paths, sparse x dense and sparse x sparse partial products, and the mr_matrix_multiply entry point.
#include "host.h"

using namespace matrel;
using namespace mrhost;

namespace {

// ------------------------------------------------------------------------------------------------
// block product planning (LocalMatrix.matrixMultiplication, LocalMatrix.scala:889-914)
// ------------------------------------------------------------------------------------------------
struct GemmSrc {
  const Block* a;
  const Block* b;
  int32_t k;
};

struct OutPlan {
  int32_t rid, cid;
  int32_t m = -1, n = -1;
  std::vector<GemmPair> gemm;                            // dense x dense (possibly densified) pairs
  std::vector<GemmSrc> src;                              // the blocks behind each gemm pair (+ its k-block id)
  std::vector<std::pair<const Block*, const Block*>> spmm;  // sparse x dense pairs
  std::vector<std::pair<const Block*, const Block*>> spsp;  // sparse x sparse, both densities <= 0.1 (ascending k)
};

struct MultiplyPlanner {
  mr_context* ctx;
  std::deque<Block> temps;   // densified sparse operands kept alive until the launches are enqueued (deque: the
                             // plans hold pointers to these blocks, so growth must not move them)
  std::map<const Block*, size_t> densified;

  const Block& dense_of(const Block& b) {
    if (b.dense()) return b;
    auto it = densified.find(&b);
    if (it == densified.end()) {
      temps.push_back(densify(ctx, b));
      it = densified.emplace(&b, temps.size() - 1).first;
    }
    return temps[it->second];
  }

  void add_pair(OutPlan& o, const Block& a, const Block& b, int32_t k) {
    // shape checks: BLAS.gemmddd / gemmsdd `require`s (BLAS.scala:338-343, 363-366)
    MR_REQUIRE(a.numCols == b.numRows, MR_EDIM, "The columns of A don't match the rows of B. A: %d, B: %d", a.numCols,
               b.numRows);
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
    if (a.dense()) {
      push_gemm(o, a, dense_of(b), k);  // dense x dense, dense x sparse.toDense (:891-892)
    } else if (b.dense()) {
      o.spmm.emplace_back(&a, &b);   // sparse x dense (:893-899; the n == 1 SpMV case is the same kernel)
    } else {
      const double s1 = a.valuesLen * 1.0 / (static_cast<double>(a.numRows) * a.numCols);
      const double s2 = b.valuesLen * 1.0 / (static_cast<double>(b.numRows) * b.numCols);
      if (s1 > 0.1) {
        push_gemm(o, dense_of(a), dense_of(b), k);  // :903-904
      } else if (s2 > 0.1) {
        o.spmm.emplace_back(&a, &dense_of(b));   // :906-907
      } else {
        o.spsp.emplace_back(&a, &b);  // LocalMatrix.multiplySparseSparse (:909-911, :143-323): see run_sparse_chains
      }
    }
  }

  void push_gemm(OutPlan& o, const Block& a, const Block& b, int32_t k) {
    GemmPair p{};
    p.A = a.values.ptr<double>();
    p.B = b.values.ptr<double>();
    p.aT = a.isT;
    p.bT = b.isT;
    p.lda = a.isT ? a.numCols : a.numRows;  // BLAS.scala:335
    p.ldb = b.isT ? b.numCols : b.numRows;  // BLAS.scala:336
    p.kdim = a.numCols;
    p.tmA = p.tmB = -1;
    o.gemm.push_back(p);
    o.src.push_back(GemmSrc{&a, &b, k});
  }
};

// gemm_algo 2: the dense pairs of every output block through the wgmma int8 Ozaki pipeline (gemm_ozaki.cu).
// Returns false when the problem does not fit its regular-grid assumptions or holds Inf/NaN (caller uses DMMA).
bool try_ozaki(mr_context* ctx, std::vector<OutPlan>& plans, const std::vector<double*>& cptr, int32_t blkSize, int64_t M,
               int64_t K, int64_t N, bool outer) {
  const bool tf32 = ctx->gemm_algo == 3;
  const int S_eff = std::min(7, std::max(2, ctx->ozaki_slices > 0 ? ctx->ozaki_slices : 7));
  // s32 accumulator bound: up to S pairs x K terms of |digit product| <= 2^14 land in one accumulator
  if (M <= 0 || K <= 0 || N <= 0 || M > INT32_MAX || N > INT32_MAX || K > INT32_MAX / 2) return false;
  if (!tf32 && K * S_eff >= (1 << 17)) return false;
  // Compact the block rows / columns that actually have output blocks (a rank of the process grid owns every pr-th
  // block row and pc-th block column: slicing and multiplying the absent ones would only produce zeros).
  std::map<int32_t, int32_t> crow, ccol;
  for (const OutPlan& o : plans)
    if (!o.gemm.empty()) {
      crow.emplace(o.rid, 0);
      ccol.emplace(o.cid, 0);
    }
  if (crow.empty()) return false;
  {
    int32_t i = 0;
    for (auto& kv : crow) kv.second = i++;
    i = 0;
    for (auto& kv : ccol) kv.second = i++;
  }
  const int64_t nbr = static_cast<int64_t>(crow.size()), nbc = static_cast<int64_t>(ccol.size());
  if (nbr * nbc > (1 << 24)) return false;
  const int64_t last_r = crow.rbegin()->first, last_c = ccol.rbegin()->first;
  if (last_r * static_cast<int64_t>(blkSize) >= M || last_c * static_cast<int64_t>(blkSize) >= N) return false;
  const int64_t Mc = (nbr - 1) * blkSize + std::min<int64_t>(blkSize, M - last_r * blkSize);
  const int64_t Nc = (nbc - 1) * blkSize + std::min<int64_t>(blkSize, N - last_c * blkSize);
  std::vector<double*> ctab(static_cast<size_t>(nbr * nbc), nullptr);
  std::map<const Block*, int> ia, ib;
  std::vector<OzakiOperand> va, vb;
  for (size_t i = 0; i < plans.size(); ++i) {
    const OutPlan& o = plans[i];
    if (o.gemm.empty()) continue;
    const int32_t cr = crow[o.rid], cc = ccol[o.cid];
    // every block row / column but the last must be a full blkSize tall / wide (the kernel finds blocks by division)
    if (o.m != ((o.rid == last_r) ? Mc - (nbr - 1) * blkSize : blkSize) || o.n != ((o.cid == last_c) ? Nc - (nbc - 1) * blkSize : blkSize))
      return false;
    if (!o.spmm.empty()) return false;  // mixed dense / sparse partial sums stay on the exact path
    ctab[static_cast<size_t>(cr) * nbc + cc] = cptr[i];
    for (const GemmSrc& g : o.src) {
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
  if (ctx->time_kernels) CUDA_CHECK(cudaEventRecord(ctx->ev0, ctx->stream));
  if (tf32)
    CUDA_CHECK(tf32x3_gemm(va.data(), static_cast<int>(va.size()), vb.data(), static_cast<int>(vb.size()), Mc, K, Nc, ctab.data(),
                           blkSize, static_cast<int>(nbr), static_cast<int>(nbc), &launches, ctx->stream));
  else
    CUDA_CHECK(ozaki_gemm_f64(va.data(), static_cast<int>(va.size()), vb.data(), static_cast<int>(vb.size()), Mc, K, Nc,
                              ctx->ozaki_slices > 0 ? ctx->ozaki_slices : 7, ctab.data(), blkSize, static_cast<int>(nbr),
                              static_cast<int>(nbc), false, &launches, &nonfinite, ctx->stream));
  note_launch(ctx, launches);
  if (nonfinite) return false;
  ctx->stats.gemm_launches += 1;
  if (ctx->time_kernels) {
    CUDA_CHECK(cudaEventRecord(ctx->ev1, ctx->stream));
    CUDA_CHECK(cudaEventSynchronize(ctx->ev1));
    float ms = 0.f;
    CUDA_CHECK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    ctx->stats.last_gemm_ms = ms;
    ctx->stats.gemm_ms_total += ms;
  }
  return true;
}

// ------------------------------------------------------------------------------------------------
// gemm_algo 0 (auto) / 4: the dense pairs through the Ozaki-II job engine (gemm_ozaki.cu), group by group.
//
// plan():    checks that the product fits the engine's regular-grid assumptions, assigns one residue slot per block row of A /
//            block column of B that has output blocks, and turns every launch group (the chunks of a pipelined multiply, or the
//            single group of a resident one) into jobs: which slots to prepare first, the tile list, the output-block table.
//            Operands whose residues exceed the scratch budget are cut into (row panel x column panel) jobs that re-prepare.
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

  Oz2Run() = default;
  Oz2Run(const Oz2Run&) = delete;
  Oz2Run& operator=(const Oz2Run&) = delete;
  ~Oz2Run() {
    if (eng) oz2_destroy(eng, ctx->stream);
  }
  const int* flag() const { return eng ? oz2_flag(eng) : nullptr; }

  // Returns false when the multiply must stay on the exact kernel.  `group_of` may be rewritten to a single group (operands too
  // large to keep every residue resident cannot be pipelined chunk by chunk).
  bool plan(mr_context* c, const std::vector<OutPlan>& plans, const std::vector<size_t>& out_plan, const std::vector<double*>& cptr,
            std::vector<int>& group_of, int& ngroups, int32_t blk, int64_t M, int64_t K, int64_t N, bool outer, bool guard) {
    ctx = c;
    if (M <= 0 || K <= 0 || N <= 0 || K >= (1 << 17) || out_plan.empty()) return false;
    const int T = oz2_moduli_for(K, ctx->crt_moduli);
    const int ss = (blk + kOz2TileM - 1) / kOz2TileM * kOz2TileM;
    std::map<int32_t, int> crow, ccol;
    for (size_t oi : out_plan) {
      crow.emplace(plans[oi].rid, 0);
      ccol.emplace(plans[oi].cid, 0);
    }
    int i = 0;
    for (auto& kv : crow) kv.second = i++;
    i = 0;
    for (auto& kv : ccol) kv.second = i++;
    const int nr = static_cast<int>(crow.size()), nc = static_cast<int>(ccol.size());
    if (static_cast<int64_t>(nr) * ss > INT32_MAX / 2 || static_cast<int64_t>(nc) * ss > INT32_MAX / 2) return false;
    std::vector<int32_t> rdim(nr, -1), cdim(nc, -1);
    std::vector<std::vector<const GemmSrc*>> asrc(nr), bsrc(nc);  // unique blocks per block row / column
    std::map<const Block*, int> seen_a, seen_b;
    for (size_t oi : out_plan) {
      const OutPlan& o = plans[oi];
      if (!o.spmm.empty() || !o.spsp.empty() || o.m <= 0 || o.n <= 0 || o.m > blk || o.n > blk) return false;
      const int cr = crow[o.rid], cc = ccol[o.cid];
      if (rdim[cr] < 0) rdim[cr] = o.m;
      if (cdim[cc] < 0) cdim[cc] = o.n;
      if (rdim[cr] != o.m || cdim[cc] != o.n) return false;
      for (const GemmSrc& g : o.src) {
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
    while (oz2_scratch_bytes(blk, K, T, cap_r, cap_c, max_tiles_for(cap_r, cap_c)) > budget) {
      if (cap_r == 1 && cap_c == 1) return false;
      if (cap_r >= cap_c) cap_r = (cap_r + 1) / 2;
      else cap_c = (cap_c + 1) / 2;
    }
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
        for (const GemmSrc* g : (is_a ? asrc[id] : bsrc[id])) {
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
    auto add_tiles = [&](Job& j, int rslot, int cslot, int m, int n) {
      const int tm0 = rslot * ss / kOz2TileM;
      int tm1 = (rslot * ss + m + kOz2TileM - 1) / kOz2TileM;
      if (paired && ((tm1 - tm0) & 1)) ++tm1;  // the padding tile lies inside the slot: garbage rows, never stored
      const int tn0 = cslot * ss / kOz2TileN, tn1 = (cslot * ss + n + kOz2TileN - 1) / kOz2TileN;
      for (int a = tm0; a < tm1; ++a)
        for (int b = tn0; b < tn1; ++b) j.tiles.push_back(make_int2(a, b));
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
      Oz2FixOut fo{C, o.m, o.n, rslot, cslot, static_cast<int32_t>(j.fsrcs.size()), static_cast<int32_t>(o.src.size())};
      for (const GemmSrc& g : o.src)
        j.fsrcs.push_back(Oz2FixSrc{g.a->values.ptr<double>(), g.b->values.ptr<double>(), outer ? 0 : g.k * blk, g.a->numCols, g.a->numRows,
                                    g.b->numCols, static_cast<uint8_t>(g.a->isT), static_cast<uint8_t>(g.b->isT), {0}});
      j.fouts.push_back(fo);
    };
    int max_tiles = 1;
    if (resident) {
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
          add_tiles(j, cr, cc, o.m, o.n);
          add_fix(j, o, cptr[out_plan[t]], cr, cc);
        }
        if (j.tiles.empty()) continue;
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
              add_tiles(j, cr - r0, cc - c0, o.m, o.n);
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
    max_tiles = static_cast<int>(std::min<int64_t>(max_tiles, plane_cap_tiles));
    max_tiles += max_tiles & 1;
    cudaError_t e = oz2_create(&eng, blk, K, T, cap_r, cap_c, max_tiles, guard ? 1 : 0, ctx->stream);
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
// LocalMatrix.scala:143-323).  Values: each partial is computed as sparse A x densified B (the same sums in a different
// order).  Storage format: the reference's four loop nests end in four different rules, and `reduceByKey(LocalMatrix.add)`
// re-decides the format at every sparse + sparse step, so the chain is replayed partial by partial in ascending k (Spark's
// own reduce order is arbitrary; ascending k is the deterministic choice):
//   CSC x CSC (:155-196): CSC iff rows*cols > 2 nnz + cols + 1, else dense      CSR x CSR (:198-239): CSR iff ... + rows + 1
//   CSR x CSC (:241-286): always CSC (both branches build a SparseMatrix)       CSC x CSR (:288-323): dense iff rows*cols <= 2 nnz + cols
//   sparse + sparse (:74-139): CSC iff rows*cols > 2 nnz + cols + 1, else dense; anything + dense: dense.
// ------------------------------------------------------------------------------------------------
enum ChainFmt { FMT_DENSE = 0, FMT_CSC = 1, FMT_CSR = 2 };

void run_sparse_chains(mr_context* ctx, std::vector<OutPlan>& plans, const std::vector<size_t>& chains,
                       const std::vector<double*>& cptr, MultiplyPlanner& planner, mr_matrix* result) {
  if (chains.empty()) return;
  size_t levels = 0;
  for (size_t i : chains) levels = std::max(levels, plans[i].spsp.size());
  std::vector<int> fmt(chains.size(), FMT_DENSE);
  std::vector<Buf> scratch(chains.size());
  for (size_t lv = 0; lv < levels; ++lv) {
    std::vector<size_t> act;  // chains that have a partial at this level
    std::vector<DenseWin> pw;
    for (size_t c = 0; c < chains.size(); ++c) {
      OutPlan& o = plans[chains[c]];
      if (lv >= o.spsp.size() || o.m == 0 || o.n == 0) continue;
      const Block& a = *o.spsp[lv].first;
      const Block& b = planner.dense_of(*o.spsp[lv].second);
      wait_ready(ctx, a);
      wait_ready(ctx, *o.spsp[lv].second);
      const size_t bytes = static_cast<size_t>(o.m) * o.n * sizeof(double);
      double* target = cptr[chains[c]];
      if (lv > 0) {
        if (!scratch[c]) scratch[c] = std::make_shared<DevBuf>(ctx, bytes);
        target = static_cast<double*>(scratch[c]->p);
      }
      if (!a.isT) CUDA_CHECK(cudaMemsetAsync(target, 0, bytes, ctx->stream));  // the CSC kernel scatters into zeros
      CUDA_CHECK(launch_spmm(a.colPtrs.ptr<int32_t>(), a.rowIndices.ptr<int32_t>(), a.values.ptr<double>(), a.isT,
                             b.values.ptr<double>(), b.isT, target, a.numRows, a.numCols, b.numCols, false, ctx->stream));
      note_launch(ctx);
      act.push_back(c);
      pw.push_back(DenseWin{target, o.m, o.n});
    }
    if (act.empty()) continue;
    const auto pcounts = column_counts(ctx, pw);
    std::vector<size_t> recount;  // chains whose running sum is sparse + sparse at this level
    std::vector<EwDesc> adds;
    int max_rows = 0, max_cols = 0;
    for (size_t t = 0; t < act.size(); ++t) {
      const size_t c = act[t];
      OutPlan& o = plans[chains[c]];
      const bool aT = o.spsp[lv].first->isT, bT = o.spsp[lv].second->isT;
      const int64_t cells = static_cast<int64_t>(o.m) * o.n, nnz = total_count(pcounts[t]);
      int pf;
      if (!aT && !bT) pf = cells > 2 * nnz + o.n + 1 ? FMT_CSC : FMT_DENSE;
      else if (aT && bT) pf = cells > 2 * nnz + o.m + 1 ? FMT_CSR : FMT_DENSE;
      else if (aT && !bT) pf = FMT_CSC;
      else pf = cells <= 2 * nnz + o.n ? FMT_DENSE : FMT_CSC;
      if (lv == 0) {
        fmt[c] = pf;
        continue;
      }
      EwDesc d{};
      d.A = cptr[chains[c]];
      d.B = pw[t].p;
      d.C = cptr[chains[c]];  // in place: every element is read and written by the same thread
      d.rows = o.m;
      d.cols = o.n;
      adds.push_back(d);
      max_rows = std::max(max_rows, o.m);
      max_cols = std::max(max_cols, o.n);
      if (fmt[c] == FMT_DENSE || pf == FMT_DENSE) fmt[c] = FMT_DENSE;
      else recount.push_back(c);
    }
    if (!adds.empty()) {
      Buf d = upload(ctx, adds);
      CUDA_CHECK(launch_ew_batched(EW_ADD, static_cast<const EwDesc*>(d->p), static_cast<int>(adds.size()), max_rows, max_cols,
                                   false, ctx->stream));
      note_launch(ctx);
    }
    if (!recount.empty()) {
      std::vector<DenseWin> sw;
      for (size_t c : recount) sw.push_back(DenseWin{cptr[chains[c]], plans[chains[c]].m, plans[chains[c]].n});
      const auto scounts = column_counts(ctx, sw);
      for (size_t t = 0; t < recount.size(); ++t) {
        const OutPlan& o = plans[chains[recount[t]]];
        fmt[recount[t]] = static_cast<int64_t>(o.m) * o.n > 2 * total_count(scounts[t]) + o.n + 1 ? FMT_CSC : FMT_DENSE;
      }
    }
  }
  // final storage: dense results stay in their slab window; CSC / CSR results are compacted out of it
  std::vector<DenseWin> cw;
  std::vector<size_t> cw_chain;
  std::vector<Buf> keep;
  for (size_t c = 0; c < chains.size(); ++c) {
    const OutPlan& o = plans[chains[c]];
    if (o.m == 0 || o.n == 0 || fmt[c] == FMT_DENSE) continue;
    if (fmt[c] == FMT_CSC) {
      cw.push_back(DenseWin{cptr[chains[c]], o.m, o.n});
    } else {  // CSR of C = CSC of C^T: materialise the row-major copy (= column-major n x m) first
      Buf t = std::make_shared<DevBuf>(ctx, static_cast<size_t>(o.m) * o.n * sizeof(double));
      EwDesc d{};
      d.A = cptr[chains[c]];
      d.C = static_cast<double*>(t->p);
      d.rows = o.n;
      d.cols = o.m;
      d.aT = 1;
      std::vector<EwDesc> one{d};
      Buf dd = upload(ctx, one);
      CUDA_CHECK(launch_ew_batched(EW_COPY, static_cast<const EwDesc*>(dd->p), 1, o.n, o.m, true, ctx->stream));
      note_launch(ctx);
      cw.push_back(DenseWin{static_cast<const double*>(t->p), o.n, o.m});
      keep.push_back(t);
    }
    cw_chain.push_back(c);
  }
  if (!cw.empty()) {
    const auto counts = column_counts(ctx, cw);
    std::vector<Block> blocks = compact_csc(ctx, cw, counts);
    for (size_t t = 0; t < blocks.size(); ++t) {
      const size_t c = cw_chain[t];
      const OutPlan& o = plans[chains[c]];
      Block& b = blocks[t];
      if (fmt[c] == FMT_CSR) {  // the CSC arrays of C^T are the CSR arrays of C
        b.numRows = o.m;
        b.numCols = o.n;
        b.isT = true;
      }
      result->blocks[{o.rid, o.cid}] = std::move(b);
    }
  }
}

void run_multiply(mr_context* ctx, std::vector<OutPlan>& plans, MultiplyPlanner& planner, int32_t blkSize,
                  mr_matrix* result, int64_t M, int64_t K, int64_t N, bool outer) {
  const ShardInfo* out_shard = result->shard.get();
  // Low-density sparse x sparse pairs: next to any dense partial the block sum is dense whatever the partial's own format
  // (LocalMatrix.add), so there they are ordinary sparse x dense products of the densified right operand; an output block
  // made of such pairs ONLY replays the reference's format rules (run_sparse_chains).
  std::vector<size_t> chains;
  for (size_t i = 0; i < plans.size(); ++i) {
    OutPlan& o = plans[i];
    if (o.spsp.empty()) continue;
    if (o.gemm.empty() && o.spmm.empty()) {
      chains.push_back(i);
    } else {
      for (auto& pr : o.spsp) o.spmm.emplace_back(pr.first, &planner.dense_of(*pr.second));
      o.spsp.clear();
    }
  }
  // allocate all output blocks from one slab (packed in plan order, or at their slots when the result is a sharded dataset)
  std::vector<double*> cptr(plans.size());
  if (out_shard) {
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
    size_t total = 0;
    for (auto& o : plans) total += align_up(static_cast<size_t>(o.m) * o.n * sizeof(double));
    Slab slab(ctx, total);
    for (size_t i = 0; i < plans.size(); ++i) {
      auto& o = plans[i];
      Span s = slab.take(static_cast<size_t>(o.m) * o.n * sizeof(double));
      cptr[i] = s.ptr<double>();
      result->blocks[{o.rid, o.cid}] = dense_block(o.m, o.n, s, false);  // product is never transposed (MLMatrix.scala:101)
    }
  }

  // ---- fused GEMM launch over every output block that has dense pairs
  std::vector<GemmOut> outs;
  std::vector<GemmPair> pairs;
  std::vector<size_t> out_plan;
  int64_t flops = 0;
  for (size_t i = 0; i < plans.size(); ++i) {
    auto& o = plans[i];
    if (o.gemm.empty() || o.m == 0 || o.n == 0) continue;
    GemmOut go{};
    go.C = cptr[i];
    go.m = o.m;
    go.n = o.n;
    go.pair_begin = static_cast<int32_t>(pairs.size());
    go.pair_count = static_cast<int32_t>(o.gemm.size());
    for (auto& p : o.gemm) {
      pairs.push_back(p);
      flops += 2ll * o.m * o.n * p.kdim;
    }
    outs.push_back(go);
    out_plan.push_back(i);
  }
  // which dense operands are still being produced on another stream (ingest copies)?
  bool pending = false;
  for (size_t i = 0; i < plans.size() && !pending; ++i)
    for (const GemmSrc& g : plans[i].src)
      if ((g.a->ready && !block_done(*g.a)) || (g.b->ready && !block_done(*g.b))) {
        pending = true;
        break;
      }
  (void)cudaGetLastError();
  auto wait_all_sources = [&] {
    for (auto& o : plans)
      for (const GemmSrc& g : o.src) {
        wait_ready(ctx, *g.a);
        wait_ready(ctx, *g.b);
      }
  };
  // gemm_algo: 0 = auto (Ozaki-II on wgmma with the range guard when the product is large and regular, else DMMA), 1 = DMMA,
  // 2 = Ozaki-I, 3 = 3xTF32, 4 = Ozaki-II without the range guard
  const int algo = ctx->gemm_algo;
  bool ozaki_done = false;
  if (!outs.empty() && (algo == 2 || algo == 3)) {
    wait_all_sources();
    ozaki_done = try_ozaki(ctx, plans, cptr, blkSize, M, K, N, outer);
    if (ozaki_done) ctx->stats.last_gemm_flops = flops;
  }
  if (!outs.empty() && !ozaki_done) {
    // tile shape: large tiles unless they cannot fill the 132 SMs
    int64_t tiles128 = 0;
    for (auto& go : outs) tiles128 += static_cast<int64_t>((go.m + 127) / 128) * ((go.n + 127) / 128);
    int variant = tiles128 >= 2 * 132 ? GEMM_128x128 : GEMM_64x64;
    if (ctx->force_variant >= 0) variant = ctx->force_variant;
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
        for (const GemmSrc& g : plans[out_plan[oi]].src) {
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
    bool use_oz2 = false;
    if (algo == 4 || (algo == 0 && flops >= (1ll << 33)))
      use_oz2 = oz2.plan(ctx, plans, out_plan, cptr, group_of, ngroups_dyn, blkSize, M, K, N, outer, algo == 0);
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
      ctx->stats.tc_gemm_launches += 1;
    }
    if (ctx->time_kernels) CUDA_CHECK(cudaEventRecord(ctx->ev0, ctx->stream));
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
        for (const GemmSrc& g : plans[out_plan[oi]].src) {
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
            if (o.spmm.empty()) result->blocks[{o.rid, o.cid}].ready = r;  // blocks with sparse partials finish later
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
    ctx->stats.gemm_launches += 1;
    ctx->stats.last_gemm_flops = flops;
    if (ctx->time_kernels) {
      CUDA_CHECK(cudaEventRecord(ctx->ev1, ctx->stream));
      CUDA_CHECK(cudaEventSynchronize(ctx->ev1));
      float ms = 0.f;
      CUDA_CHECK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
      ctx->stats.last_gemm_ms = ms;
      ctx->stats.gemm_ms_total += ms;
    }
  }

  // ---- sparse x dense partial products accumulate onto the GEMM result (LocalMatrix.add of partials).
  // CSR pairs with block dims <= 1024 go through ONE fused launch (K loop over the pairs inside the kernel): the pipelined
  // TMA kernel of spmm.cu when the output block is large enough to fill its 512 x 32 tiles and B can be addressed by a tensor
  // map, else the simple shared-memory kernel of ew.cu; CSC pairs and oversized blocks use the per-pair kernels.
  std::vector<SpmmOut> fouts;
  std::vector<SpmmPair> fpairs;
  int fused_max_n = 0;
  std::vector<Spmm2Out> outs2;
  std::vector<Spmm2Pair> pairs2;
  std::vector<Spmm2Prep> preps2;
  std::vector<Spmm2Item> items2;
  struct Key2 {
    int32_t cid, ctile, rid, strip;
  };
  std::vector<Key2> keys2;
  std::map<const Block*, int> prep_of;                     // sparse block -> index into preps2
  std::map<const Block*, int32_t> tmap_of_b;               // dense block -> tensor map index
  struct TmapBytes2 { unsigned char b[128]; };
  std::vector<TmapBytes2> tmaps2;
  std::vector<EwDesc> transposes;                          // column-major B blocks -> row-major scratch
  std::vector<std::pair<const Block*, size_t>> trans_of;   // (block, offset in the scratch buffer)
  std::vector<size_t> aux_off;                             // per prep: offset of its aux region
  size_t aux_total = 0, trans_total = 0;
  int prep_max_m = 0, prep_max_k = 0, trans_max_r = 0, trans_max_c = 0;
  for (size_t i = 0; i < plans.size(); ++i) {
    auto& o = plans[i];
    bool have = !o.gemm.empty();
    if (o.m == 0 || o.n == 0 || !o.spsp.empty()) continue;
    std::vector<std::pair<const Block*, const Block*>> slow, fused;
    for (auto& sp : o.spmm) {
      const Block& s = *sp.first;
      const Block& b = *sp.second;
      wait_ready(ctx, s);
      wait_ready(ctx, b);
      if (s.isT && o.m <= kSpmmMaxDim && s.numCols <= kSpmmMaxDim) fused.push_back(sp);
      else slow.push_back(sp);
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
        auto pit = prep_of.find(&sblk);
        if (pit == prep_of.end()) {
          size_t eo, ro, so;
          const size_t bytes = spmm2_aux_bytes(sblk.numRows, sblk.numCols, sblk.valuesLen, &eo, &ro, &so);
          Spmm2Prep pp{};
          pp.ptrs = sblk.colPtrs.ptr<int32_t>();
          pp.idx = sblk.rowIndices.ptr<int32_t>();
          pp.vals = sblk.values.ptr<double>();
          pp.m = sblk.numRows;
          pp.kdim = sblk.numCols;
          // offsets for now; rebased on the aux allocation below
          pp.ent = reinterpret_cast<unsigned char*>(aux_total + eo);
          pp.rp = reinterpret_cast<int32_t*>(aux_total + ro);
          pp.segoff = reinterpret_cast<int32_t*>(aux_total + so);
          aux_off.push_back(aux_total);
          aux_total += bytes;
          prep_max_m = std::max(prep_max_m, pp.m);
          prep_max_k = std::max(prep_max_k, pp.kdim);
          pit = prep_of.emplace(&sblk, static_cast<int>(preps2.size())).first;
          preps2.push_back(pp);
        }
        if (!tmap_of_b.count(&bblk)) {
          if (!bblk.isT) {  // column-major: row-major copy in the scratch buffer (one transposing pass per multiply)
            EwDesc d{};
            d.A = bblk.values.ptr<double>();
            d.C = reinterpret_cast<double*>(trans_total);  // offset for now
            d.rows = bblk.numCols;  // the k x n block read as its n x k transpose, stored row-major (aT): see run_sparse_chains
            d.cols = bblk.numRows;
            d.aT = 1;
            trans_of.emplace_back(&bblk, trans_total);
            trans_total += align_up(static_cast<size_t>(bblk.numRows) * bblk.numCols * sizeof(double));
            trans_max_r = std::max(trans_max_r, d.rows);
            trans_max_c = std::max(trans_max_c, d.cols);
            transposes.push_back(d);
          }
          tmap_of_b.emplace(&bblk, static_cast<int32_t>(tmap_of_b.size()));
        }
        Spmm2Pair pr{};
        pr.ent = reinterpret_cast<const unsigned char*>(static_cast<uintptr_t>(pit->second));  // prep index for now
        pr.kdim = sblk.numCols;
        pr.tmB = tmap_of_b[&bblk];
        pairs2.push_back(pr);
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
    if (!have) CUDA_CHECK(cudaMemsetAsync(cptr[i], 0, static_cast<size_t>(o.m) * o.n * sizeof(double), ctx->stream));
  }
  if (!fouts.empty()) {
    Buf d_fo = upload(ctx, fouts), d_fp = upload(ctx, fpairs);
    if (ctx->time_kernels) CUDA_CHECK(cudaEventRecord(ctx->ev0, ctx->stream));
    CUDA_CHECK(launch_spmm_fused(static_cast<const SpmmOut*>(d_fo->p), static_cast<int>(fouts.size()),
                                 static_cast<const SpmmPair*>(d_fp->p), fused_max_n, ctx->stream));
    note_launch(ctx);
    if (ctx->time_kernels) {
      CUDA_CHECK(cudaEventRecord(ctx->ev1, ctx->stream));
      CUDA_CHECK(cudaEventSynchronize(ctx->ev1));
      float ms = 0.f;
      CUDA_CHECK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
      ctx->stats.last_gemm_ms = ms;
      ctx->stats.gemm_ms_total += ms;
    }
  }
  if (!outs2.empty()) {
    // scratch: re-packed CSR segments of every sparse block, row-major copies of the column-major dense blocks
    Buf aux = std::make_shared<DevBuf>(ctx, std::max<size_t>(aux_total, 16));
    Buf trans = std::make_shared<DevBuf>(ctx, std::max<size_t>(trans_total, 16));
    char* aux_base = static_cast<char*>(aux->p);
    for (Spmm2Prep& pp : preps2) {
      pp.ent = reinterpret_cast<unsigned char*>(aux_base + reinterpret_cast<uintptr_t>(pp.ent));
      pp.rp = reinterpret_cast<int32_t*>(aux_base + reinterpret_cast<uintptr_t>(pp.rp));
      pp.segoff = reinterpret_cast<int32_t*>(aux_base + reinterpret_cast<uintptr_t>(pp.segoff));
    }
    for (Spmm2Pair& pr : pairs2) {
      const Spmm2Prep& pp = preps2[static_cast<size_t>(reinterpret_cast<uintptr_t>(pr.ent))];
      pr.ent = pp.ent;
      pr.rp = pp.rp;
      pr.segoff = pp.segoff;
    }
    std::map<const Block*, const double*> rowmajor;  // dense block -> its row-major image
    for (size_t t = 0; t < transposes.size(); ++t) {
      transposes[t].C = reinterpret_cast<double*>(static_cast<char*>(trans->p) + reinterpret_cast<uintptr_t>(transposes[t].C));
      rowmajor[trans_of[t].first] = transposes[t].C;
    }
    tmaps2.resize(tmap_of_b.size());
    bool maps_ok = true;
    for (auto& kv : tmap_of_b) {
      const Block* bb = kv.first;
      const double* base = bb->isT ? bb->values.ptr<double>() : rowmajor[bb];
      maps_ok = maps_ok && spmm2_encode_b_tmap(tmaps2[kv.second].b, base, bb->numRows, bb->numCols, bb->numCols);
    }
    if (!maps_ok) fail(MR_ECUDA, "cuTensorMapEncodeTiled failed for a dense operand of the sparse x dense multiply");
    // concurrently resident CTAs share the B panel of one 32-column tile: order by (block column, tile, block row, strip)
    std::vector<size_t> ord(items2.size());
    for (size_t t = 0; t < ord.size(); ++t) ord[t] = t;
    std::sort(ord.begin(), ord.end(), [&](size_t x, size_t y) {
      const Key2 &a = keys2[x], &b2 = keys2[y];
      if (a.cid != b2.cid) return a.cid < b2.cid;
      if (a.ctile != b2.ctile) return a.ctile < b2.ctile;
      if (a.rid != b2.rid) return a.rid < b2.rid;
      return a.strip < b2.strip;
    });
    std::vector<Spmm2Item> sorted_items(items2.size());
    for (size_t t = 0; t < ord.size(); ++t) sorted_items[t] = items2[ord[t]];
    Buf d_preps = upload(ctx, preps2), d_outs2 = upload(ctx, outs2), d_pairs2 = upload(ctx, pairs2), d_items = upload(ctx, sorted_items),
        d_tmaps2 = upload(ctx, tmaps2);
    CUDA_CHECK(launch_spmm2_prep(static_cast<const Spmm2Prep*>(d_preps->p), static_cast<int>(preps2.size()), prep_max_m, prep_max_k, ctx->stream));
    note_launch(ctx);
    if (!transposes.empty()) {
      Buf d_tr = upload(ctx, transposes);
      CUDA_CHECK(launch_ew_batched(EW_COPY, static_cast<const EwDesc*>(d_tr->p), static_cast<int>(transposes.size()), trans_max_r,
                                   trans_max_c, true, ctx->stream));
      note_launch(ctx);
    }
    if (ctx->time_kernels) CUDA_CHECK(cudaEventRecord(ctx->ev0, ctx->stream));
    CUDA_CHECK(launch_spmm2(static_cast<const Spmm2Item*>(d_items->p), static_cast<int>(sorted_items.size()),
                            static_cast<const Spmm2Out*>(d_outs2->p), static_cast<const Spmm2Pair*>(d_pairs2->p), d_tmaps2->p, ctx->stream));
    note_launch(ctx);
    if (ctx->time_kernels) {
      CUDA_CHECK(cudaEventRecord(ctx->ev1, ctx->stream));
      CUDA_CHECK(cudaEventSynchronize(ctx->ev1));
      float ms = 0.f;
      CUDA_CHECK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
      ctx->stats.last_gemm_ms = ms;
      ctx->stats.gemm_ms_total += ms;
    }
    ctx->stats.gemm_launches += 1;
  }
  run_sparse_chains(ctx, plans, chains, cptr, planner, result);
}


}  // namespace

namespace mrhost {

mr_matrix* multiply_impl(mr_context* ctx, mr_matrix* left, int64_t leftRowNum, int64_t leftColNum, mr_matrix* right, int64_t rightRowNum,
                         int64_t rightColNum, int32_t blkSize, const ShardLayout* out_layout) {
  for (auto& kv : left->blocks)
    if (!kv.second.dense()) wait_ready(ctx, kv.second);
  for (auto& kv : right->blocks)
    if (!kv.second.dense()) wait_ready(ctx, kv.second);
  MultiplyPlanner planner{ctx};
  std::vector<OutPlan> plans;
  const int64_t leftColBlkNum = ceil_div(leftColNum, blkSize);    // MatfastExecution.scala:712
  const int64_t rightRowBlkNum = ceil_div(rightRowNum, blkSize);  // :713
  if (leftColBlkNum == 1 && rightRowBlkNum == 1) {
    // outer-product paths (:714-721 -> helper :175-221): every left block x every right block, no
    // reduce.  Reference defect B1 (DuplicateLeft throws) is not reproduced; both branches return
    // what DuplicateRight returns.
    std::map<std::pair<int32_t, int32_t>, size_t> seen;
    for (auto& l : left->blocks)
      for (auto& r : right->blocks) {
        OutPlan o;
        o.rid = l.first.first;
        o.cid = r.first.second;
        planner.add_pair(o, l.second, r.second, 0);
        auto key = std::make_pair(o.rid, o.cid);
        auto it = seen.find(key);
        if (it == seen.end()) {
          seen[key] = plans.size();
          plans.push_back(std::move(o));
        } else {
          plans[it->second] = std::move(o);  // duplicate keys: the last row wins when collected into a map
        }
      }
  } else {
    // matrixMultiplyGeneral (helper :235-263): join on k, then reduce by (i, j) in ascending k.
    std::map<int32_t, std::vector<std::pair<int32_t, const Block*>>> rights;  // k -> (j, B(k,j))
    for (auto& r : right->blocks) rights[r.first.first].push_back({r.first.second, &r.second});
    std::map<std::pair<int32_t, int32_t>, size_t> index;
    // left->blocks is ordered by (i, k): iterating it visits k ascending within each i
    for (auto& l : left->blocks) {
      const int32_t i = l.first.first, k = l.first.second;
      auto rit = rights.find(k);
      if (rit == rights.end()) continue;
      for (auto& jb : rit->second) {
        auto key = std::make_pair(i, jb.first);
        auto it = index.find(key);
        if (it == index.end()) {
          OutPlan o;
          o.rid = i;
          o.cid = jb.first;
          it = index.emplace(key, plans.size()).first;
          plans.push_back(std::move(o));
        }
        planner.add_pair(plans[it->second], l.second, *jb.second, k);
      }
    }
  }
  std::unique_ptr<mr_matrix> result(out_layout ? new_sharded(ctx, *out_layout, false, false) : new_matrix(ctx));
  if (out_layout) result->blocks.clear();  // only the blocks the product has are present (join semantics); absent ones stay absent
  run_multiply(ctx, plans, planner, blkSize, result.get(), leftRowNum, leftColNum, rightColNum, leftColBlkNum == 1 && rightRowBlkNum == 1);
  return result.release();
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
    *out = multiply_impl(ctx, left, leftRowNum, leftColNum, right, rightRowNum, rightColNum, blkSize, nullptr);
  });
}


}  // extern "C"
