// plan.h -- host-side work planner for the persistent fused ABFT-SGEMM kernel.
//
// The reference launches one CTA per output tile and lets the hardware scheduler deal them out
// (kernel/ft_sgemm/sgemm.cu:110-199 of the reference: grid = (M/ms, N/ns)).  A persistent kernel with one CTA per SM has
// to do that job itself, and with 256x256 tiles a 3072^3 problem is only 144 tiles on 66 two-CTA units: dealing whole
// tiles round-robin leaves the machine 27 % idle in the last of 3 waves.  The planner therefore cuts the last H data
// tiles of the raster along K into pieces and levels the units with a list scheduler.
//
// A cut tile is computed as a CHAIN: the unit that owns piece p+1 first loads the raw accumulator its predecessor
// parked ("seeds" its accumulator with it) and then keeps accumulating, so the sum is formed in exactly the k order of an
// uncut tile -- bit-identical results, and (what matters for ABFT) the tensor core's accumulation bias stays the same
// as in the checksum tile-columns.  (Adding independently accumulated partial sums, the usual split-K, raises the
// fault-free ABFT residual.)
//
// Global item order:  [early first pieces][checksum tiles][whole data tiles, raster order]
//                     [late first pieces][2nd pieces][3rd pieces]...
//   * early first pieces run at the very start: their epilogue only parks the accumulator (no checksum needed); made as
//     long as a checksum item they keep all units in step (the units that share A / B panels then stream the same k range);
//   * late first pieces and all later pieces run at the end, longest first, and level the finishing times.
// Every unit's list is increasing in that order and every wait (piece -> previous piece, data tile -> checksum tiles)
// points to an earlier item, which makes the in-kernel waits deadlock-free (tests/test_schedule.py simulates it).
#pragma once
#include <algorithm>
#include <cstdint>
#include <queue>
#include <vector>

namespace ftsgemm {

struct PlanItem {
  int tile;        // decode order: checksum tiles first, then data tiles
  int kb_begin, kb_end;
  int kind;        // 0 whole tile, 1 first piece (park), 3 middle piece (seed + park), 2 last piece (seed + finish)
  int slice;       // piece index within its tile
  int split_idx;   // index among the cut tiles (workspace slot), -1 otherwise
};

struct Plan {
  int units = 0;
  int sk_tiles = 0;   // H: number of cut data tiles (the last H of the raster)
  int sk_slices = 1;  // largest number of pieces of any tile
  double makespan = 0.0;
  std::vector<int> offsets;          // units + 1
  std::vector<PlanItem> items;       // grouped by unit, in execution order
};

struct PlanInput {
  int units;            // work units of CG CTAs
  int n_chk_tiles;      // checksum tile-columns x tiles_m x chk_slices (first tiles in decode order)
  int chk_slices = 1;   // K-slices per checksum tile (tile t belongs to slice t / (n_chk_tiles / chk_slices))
  int n_data_tiles;
  int num_kb;           // k-blocks per tile
  int tiles_m;          // checksum tile t belongs to checksum tile-column t / tiles_m
  std::vector<double> chk_col_cost;  // tile-times of one tile of each checksum tile-column
  double chk_release = 0.0;          // tile-times before checksum items can start (their operand comes from the pre-pass)
  double item_overhead = 0.0;        // tile-times per item (pipeline fill + drain)
  double park_latency = 0.0;         // tile-times between the end of a piece's main loop and its successor's start
  double seed_overhead = 0.0;        // extra tile-times of a seeded piece (its accumulator is loaded before the first MMA)
  int max_slices = 2;   // 1 disables cutting
  int force_slices = 0; // > 1: cut into exactly this many equal pieces (tests)
  int full_search = 0;  // 1: always try the full candidate menu (default: a reduced menu from 8 waves up, where a cut
                        //    can only buy a few per cent and the simulation of thousands of items is what costs)
  int lockstep = 0;     // 1: the operands do not fit in L2, so the units must keep streaming the SAME k range of the
                        //    panels they share (first pieces of mixed lengths put the units out of phase and every
                        //    whole tile gets slower, HBM-bound): one cut fraction for all cut tiles
  size_t slab_bytes = 0;// bytes of one parked accumulator tile x CTAs per unit (workspace sizing)
};

namespace plan_detail {

// Which tiles are cut and where.  The last (He + Hl) data tiles of the raster are cut in two:
//   early tiles (the first He of them): first piece (fraction fe) at the very start of the kernel,
//   late tiles  (the other Hl):         first piece (fraction fl) after the whole tiles,
// and all second pieces at the very end.  pieces > 2 (tests): He tiles in `pieces` equal pieces, first pieces early.
struct Cut {
  int He = 0, Hl = 0;
  double fe = 0.5, fl = 0.5;
  int pieces = 2;
};

// k-block boundaries of cut tile i
inline std::vector<int> boundaries(const PlanInput &in, const Cut &c, int i) {
  std::vector<int> b;
  b.push_back(0);
  if (c.pieces > 2) {
    for (int s = 1; s < c.pieces; ++s) b.push_back(static_cast<int>(static_cast<long long>(in.num_kb) * s / c.pieces));
  } else {
    int kb = static_cast<int>(in.num_kb * (i < c.He ? c.fe : c.fl) + 0.5);
    kb = std::max(4, std::min(in.num_kb - 4, kb));
    b.push_back(kb);
  }
  b.push_back(in.num_kb);
  return b;
}

// list scheduling in global item order; returns the (penalised) makespan, optionally records the assignment
inline double schedule(const PlanInput &in, const Cut &c, Plan *out) {
  typedef std::pair<double, int> LU;  // (load, unit): least load first, ties to the lowest unit id
  std::priority_queue<LU, std::vector<LU>, std::greater<LU>> pq;
  for (int u = 0; u < in.units; ++u) pq.push(LU(0.0, u));
  std::vector<std::vector<PlanItem>> lists;
  if (out) lists.resize(in.units);
  std::vector<double> first_whole(in.units, -1.0);
  double makespan = 0.0;
  auto give = [&](const PlanItem &it, double cost, double release, bool is_whole) -> double {
    LU lu = pq.top();
    pq.pop();
    if (lu.first < release) lu.first = release;  // the unit idles until the item's input exists
    if (is_whole && first_whole[lu.second] < 0.0) first_whole[lu.second] = lu.first;
    lu.first += cost + in.item_overhead;
    if (lu.first > makespan) makespan = lu.first;
    if (out) lists[lu.second].push_back(it);
    pq.push(lu);
    return lu.first;
  };
  const int H = c.He + c.Hl, whole = in.n_data_tiles - H;
  const int first_cut = in.n_chk_tiles + whole;
  std::vector<std::vector<int>> bnd(H);
  std::vector<double> ready(H, 0.0);  // when the next piece of cut tile i may start
  int max_pieces = 1;
  for (int i = 0; i < H; ++i) {
    bnd[i] = boundaries(in, c, i);
    max_pieces = std::max(max_pieces, static_cast<int>(bnd[i].size()) - 1);
  }
  auto piece = [&](int i, int p) {
    const int np = static_cast<int>(bnd[i].size()) - 1;
    const int kind = p == 0 ? 1 : (p == np - 1 ? 2 : 3);
    const double len = static_cast<double>(bnd[i][p + 1] - bnd[i][p]) / in.num_kb;
    const double end = give(PlanItem{first_cut + i, bnd[i][p], bnd[i][p + 1], kind, p, i},
                            len + (p > 0 ? in.seed_overhead : 0.0), ready[i], false);
    ready[i] = end + in.park_latency;
  };
  for (int i = 0; i < c.He; ++i) piece(i, 0);
  {
    const int S = in.chk_slices > 1 ? in.chk_slices : 1, per_slice = in.n_chk_tiles / S;
    for (int t = 0; t < in.n_chk_tiles; ++t) {
      const int sl = t / per_slice, r = t - sl * per_slice;
      const int kb0 = static_cast<int>(static_cast<long long>(in.num_kb) * sl / S);
      const int kb1 = static_cast<int>(static_cast<long long>(in.num_kb) * (sl + 1) / S);
      give(PlanItem{t, kb0, kb1, 0, sl, -1}, in.chk_col_cost[static_cast<size_t>(r / in.tiles_m)] / S, in.chk_release, false);
    }
  }
  for (int d = 0; d < whole; ++d)
    give(PlanItem{in.n_chk_tiles + d, 0, in.num_kb, 0, 0, -1}, 1.0, 0.0, true);
  for (int i = c.He; i < H; ++i) piece(i, 0);
  for (int p = 1; p < max_pieces; ++p) {
    std::vector<int> order;
    for (int i = 0; i < H; ++i)
      if (p < static_cast<int>(bnd[i].size()) - 1) order.push_back(i);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {  // longest first levels best
      return bnd[a][p + 1] - bnd[a][p] > bnd[b][p + 1] - bnd[b][p];
    });
    for (int i : order) piece(i, p);
  }
  // Operands that do not fit in L2: units that share A / B panels must stream the same k range at the same time.
  // (Units out of phase -- behind checksum items or first pieces of mixed lengths -- make every whole tile slower.)
  if (in.lockstep) {
    double lo = 1e30, hi = -1.0;
    for (int u = 0; u < in.units; ++u)
      if (first_whole[u] >= 0.0) {
        lo = std::min(lo, first_whole[u]);
        hi = std::max(hi, first_whole[u]);
      }
    if (hi - lo > 0.15) makespan *= 1.025;
  }
  if (out) {
    out->units = in.units;
    out->sk_tiles = H;
    out->sk_slices = H > 0 ? max_pieces : 1;
    out->makespan = makespan;
    out->offsets.assign(1, 0);
    out->items.clear();
    for (int u = 0; u < in.units; ++u) {
      out->items.insert(out->items.end(), lists[u].begin(), lists[u].end());
      out->offsets.push_back(static_cast<int>(out->items.size()));
    }
  }
  return makespan;
}


inline void add_unique(std::vector<int> *v, int x, int lo, int hi) {
  if (x >= lo && x <= hi && std::find(v->begin(), v->end(), x) == v->end()) v->push_back(x);
}

}  // namespace plan_detail

inline Plan build_plan(const PlanInput &in) {
  using namespace plan_detail;
  const Cut no_cut;
  const double base = schedule(in, no_cut, nullptr);
  Cut best_cut;
  double best = -1.0;  // best makespan among the cut candidates
  const int P = in.units, T = in.n_data_tiles;
  const bool forced = in.force_slices > 1;
  // more than ~40 waves: the quantisation loss is below the 1.5 % a cut has to buy
  if (in.max_slices > 1 && T > 0 && in.num_kb >= 8 && (forced || T < 40 * P)) {
    const int pieces = forced ? in.force_slices : 2;
    const size_t slab_cap = std::min<size_t>((static_cast<size_t>(256) << 20) / std::max<size_t>(1, in.slab_bytes * (pieces - 1)),
                                             65536 / (8 * sizeof(int) * (pieces - 1)));
    const int hcap = static_cast<int>(std::min<size_t>(slab_cap, static_cast<size_t>(T)));
    auto consider = [&](const Cut &c) {
      if (c.He + c.Hl <= 0 || c.He + c.Hl > hcap) return;
      const double t = schedule(in, c, nullptr);
      if (best < 0.0 || t < best) {
        best = t;
        best_cut = c;
      }
    };
    if (in.num_kb / pieces >= 4) {  // keep pieces at least 4 k-blocks long
      if (forced) {
        std::vector<int> hs;
        const int extra[] = {T % P, P / 2, P, T, 2 * P};
        for (int e : extra) add_unique(&hs, e, 1, T);
        for (int H : hs) {
          Cut c;
          c.He = H;
          c.pieces = pieces;
          consider(c);
        }
      } else {
        // early cuts: first pieces as long as a checksum item keep every unit in step (He = units without one)
        const double chk0 = in.n_chk_tiles > 0 ? in.chk_col_cost[0] : 0.5;
        const int n_chk_units = std::min(in.n_chk_tiles, P);
        std::vector<int> he, hl;
        const bool reduced = !in.full_search && T >= 8 * P;  // planning time: 0.3-0.5 s -> 20 ms for 4000+ tiles
        he.push_back(0);
        hl.push_back(0);
        if (reduced) {
          const int e_extra[] = {P - n_chk_units, P};
          for (int e : e_extra) add_unique(&he, e, 1, T);
          const int l_extra[] = {T % P, (T % P) / 2, P / 2, P};
          for (int e : l_extra) add_unique(&hl, e, 1, T);
        } else {
          const int e_extra[] = {P - n_chk_units, T % P, P / 2, P, P / 4, (3 * P) / 4, 2 * P - n_chk_units};
          for (int e : e_extra) add_unique(&he, e, 1, T);
          const int l_extra[] = {P / 8, P / 4, (3 * P) / 8, P / 2, (5 * P) / 8, (3 * P) / 4, P, T % P, (T % P) / 2};
          for (int e : l_extra) add_unique(&hl, e, 1, T);
        }
        const double fes[] = {chk0, 0.5, 0.25, 1.0 / 3, 2.0 / 3, 0.75};
        const double fls[] = {0.5, 1.0 / 3, 2.0 / 3};
        const int n_fe = reduced ? 2 : 6;
        for (int He : he)
          for (int Hl : hl) {
            if (He + Hl <= 0 || He + Hl > T) continue;
            for (int a = 0; a < (He > 0 ? n_fe : 1); ++a)
              for (int b = 0; b < (Hl > 0 ? 3 : 1); ++b) {
                Cut c;
                c.He = He;
                c.Hl = Hl;
                c.fe = fes[a];
                c.fl = fls[b];
                consider(c);
              }
          }
      }
    }
  }
  // a cut must buy at least 1.5 % (unless a test forces it)
  if (best < 0.0 || (!forced && best > base * 0.985)) best_cut = no_cut;
  Plan p;
  schedule(in, best_cut, &p);
  return p;
}

}  // namespace ftsgemm
