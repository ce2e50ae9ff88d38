#include "ik_chol_sched.h"

#include "ik_chol_sched.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <set>
#include <tuple>

namespace mb2 {

namespace {

struct BitRows {
  int n, words;
  std::vector<uint64_t> b;
  BitRows(int n_) : n(n_), words((n_ + 63) / 64), b(size_t(n_) * ((n_ + 63) / 64), 0) {}
  uint64_t* row(int i) { return b.data() + size_t(i) * words; }
  const uint64_t* row(int i) const { return b.data() + size_t(i) * words; }
  void set(int i, int j) { row(i)[j >> 6] |= 1ull << (j & 63); }
  void clear(int i, int j) { row(i)[j >> 6] &= ~(1ull << (j & 63)); }
  bool test(int i, int j) const { return (row(i)[j >> 6] >> (j & 63)) & 1ull; }
  int count(int i) const {
    int c = 0;
    for (int w = 0; w < words; ++w) c += __builtin_popcountll(row(i)[w]);
    return c;
  }
};

// Minimum-degree ordering on the symmetric pattern; ties go to a neighbour of the vertex eliminated
// last (keeps the parameters of one kinematic chain contiguous), then to the lowest index.
std::vector<int> minimumDegreeOrder(BitRows& adj, const std::vector<int>* priority) {
  const int n = adj.n;
  std::vector<int> order;
  order.reserve(n);
  std::vector<uint8_t> done(n, 0);
  std::vector<int> degree(n);
  for (int i = 0; i < n; ++i) degree[i] = adj.count(i);
  int last = -1;
  for (int step = 0; step < n; ++step) {
    int best = -1;
    for (int i = 0; i < n; ++i) {
      if (done[i]) continue;
      if (best < 0 || degree[i] < degree[best]) { best = i; continue; }
      if (degree[i] != degree[best]) continue;
      const int pi = priority ? (*priority)[i] : 0, pb = priority ? (*priority)[best] : 0;
      if (pi > pb) best = i;
      else if (pi == pb && last >= 0 && adj.test(last, i) && !adj.test(last, best)) best = i;
    }
    // eliminate `best`: its remaining neighbours become a clique
    std::vector<int> nb;
    for (int j = 0; j < n; ++j)
      if (!done[j] && j != best && adj.test(best, j)) nb.push_back(j);
    for (int u : nb) {
      uint64_t* ru = adj.row(u);
      const uint64_t* rv = adj.row(best);
      for (int w = 0; w < adj.words; ++w) ru[w] |= rv[w];
      adj.clear(u, u);
      adj.clear(u, best);
    }
    for (int u : nb) {
      int c = 0;
      for (int j : nb) c += (j != u) ? 1 : 0; // lower bound; exact count below
      (void)c;
      // exact remaining degree: neighbours that are not eliminated
      int d = 0;
      const uint64_t* ru = adj.row(u);
      for (int j = 0; j < n; ++j)
        if (!done[j] && j != best && ((ru[j >> 6] >> (j & 63)) & 1ull)) ++d;
      degree[u] = d;
    }
    done[best] = 1;
    order.push_back(best);
    last = best;
  }
  return order;
}

} // namespace

std::string buildCholSchedule(int n, const std::vector<std::vector<int>>& cliques, bool forceDense, CholSchedule& out, const std::vector<int>* priority) {
  out = CholSchedule();
  if (n <= 0) return "empty system";
  out.n = n;
  out.nParams = n;

  // 1. ordering
  std::vector<int> order(n);
  BitRows pattern(n);
  for (int i = 0; i < n; ++i) pattern.set(i, i);
  if (forceDense) {
    for (int i = 0; i < n; ++i) order[i] = i;
  } else {
    for (const auto& c : cliques)
      for (int a : c) {
        if (a < 0 || a >= n) continue;
        for (int b : c)
          if (b >= 0 && b < n) pattern.set(a, b);
      }
    BitRows work = pattern;
    for (int i = 0; i < n; ++i) work.clear(i, i);
    if (priority != nullptr && int(priority->size()) != n) return "priority must have one entry per column";
    order = minimumDegreeOrder(work, priority);
  }
  // 1b. supernodes of the element-level factor (columns with nested structure) decide where tiles may
  //     break: a supernode that fits in one tile is never split across two (padding instead), because a
  //     split chain would make consecutive tile columns depend on each other and serialise the levels.
  std::vector<int> slot(n); // padded position of the i-th eliminated parameter
  {
    std::vector<int> rank(n);
    for (int i = 0; i < n; ++i) rank[order[i]] = i;
    BitRows F(n); // filled lower pattern in elimination order: F[i][j], i > j
    for (int a = 0; a < n; ++a)
      for (int b = 0; b < n; ++b)
        if (a != b && (forceDense || pattern.test(a, b))) { const int i = rank[a], j = rank[b]; if (i > j) F.set(i, j); }
    std::vector<int> parent(n, -1), cnt(n, 0);
    // column structures via row-merge: struct(j) = {i > j : F[i][j]}; fill: struct(parent(j)) |= struct(j) \ {parent(j)}
    std::vector<std::vector<int>> col(n);
    for (int j = 0; j < n; ++j) {
      for (int i = j + 1; i < n; ++i) if (F.test(i, j)) col[j].push_back(i);
      cnt[j] = int(col[j].size());
      if (!col[j].empty()) {
        const int pj = col[j][0];
        parent[j] = pj;
        for (size_t k = 1; k < col[j].size(); ++k) F.set(col[j][k], pj);
      }
    }
    int fill = 0, start = 0; // greedy packing of supernodes into tiles
    int padded = 0;
    auto closeTile = [&]() { if (fill != 0) { padded += kCholTile - fill; fill = 0; } };
    auto flushSupernode = [&](int first, int lastExcl) {
      const int sz = lastExcl - first;
      if (sz <= kCholTile) {
        if (fill + sz > kCholTile) closeTile(); // do not split: pad to the tile boundary
      } else {
        // A chain longer than one tile is a sequence of dependent tile columns whatever we do: keep that sequence as short as
        // possible by giving it whole tiles of its own, the partial one FIRST (its leading entries are the deepest joints, which
        // depend on nothing outside the chain, so that tile still sits in an early level).
        closeTile();
        const int head = sz % kCholTile;
        for (int j = first; j < first + head; ++j) { slot[j] = padded++; fill = (fill + 1) % kCholTile; }
        closeTile();
        first += head;
      }
      for (int j = first; j < lastExcl; ++j) { slot[j] = padded++; fill = (fill + 1) % kCholTile; }
    };
    for (int j = 1; j <= n; ++j) {
      const bool joins = j < n && parent[j - 1] == j && cnt[j - 1] == cnt[j] + 1;
      if (!joins) { flushSupernode(start, j); start = j; }
    }
    (void)fill;
    const int T0 = (padded + kCholTile - 1) / kCholTile;
    out.numTileCols = T0;
    out.nPad = T0 * kCholTile;
  }
  const int T = out.numTileCols;
  if (T > 512) return "system too large for the tile schedule";
  out.perm.assign(out.nPad, int16_t(-1));
  std::vector<int> pos(n);
  for (int i = 0; i < n; ++i) { out.perm[slot[i]] = int16_t(order[i]); pos[order[i]] = slot[i]; }

  // 2. tile-level pattern (lower) + symbolic factorisation
  std::vector<std::vector<uint8_t>> S(T, std::vector<uint8_t>(T, 0));
  for (int I = 0; I < T; ++I) S[I][I] = 1;
  if (forceDense) {
    for (int I = 0; I < T; ++I) for (int J = 0; J <= I; ++J) S[I][J] = 1;
  } else {
    for (int a = 0; a < n; ++a)
      for (int b = 0; b < n; ++b)
        if (pattern.test(a, b)) {
          const int I = pos[a] / kCholTile, J = pos[b] / kCholTile;
          if (I >= J) S[I][J] = 1;
        }
    for (int K = 0; K < T; ++K) {
      std::vector<int> st;
      for (int I = K + 1; I < T; ++I) if (S[I][K]) st.push_back(I);
      for (size_t a = 0; a < st.size(); ++a)
        for (size_t b = 0; b <= a; ++b) S[st[a]][st[b]] = 1;
    }
  }
  // 3. tiles, elimination tree, levels
  std::vector<std::vector<int>> tileId(T, std::vector<int>(T, -1));
  out.diagTile.assign(T, -1);
  for (int J = 0; J < T; ++J)
    for (int I = J; I < T; ++I)
      if (S[I][J]) {
        tileId[I][J] = int(out.tileRow.size());
        out.tileRow.push_back(int16_t(I));
        out.tileCol.push_back(int16_t(J));
        if (I == J) out.diagTile[J] = tileId[I][J];
      }
  out.numTiles = int(out.tileRow.size());
  out.tileIdTable.assign(size_t(T) * T, int16_t(-1));
  for (int I = 0; I < T; ++I) for (int J = 0; J <= I; ++J) out.tileIdTable[size_t(I) * T + J] = int16_t(tileId[I][J]);
  out.pos.resize(n);
  for (int i = 0; i < n; ++i) out.pos[i] = int16_t(pos[i]);
  std::vector<int> level(T, 0);
  std::vector<std::vector<int>> st(T);
  for (int K = 0; K < T; ++K) {
    for (int I = K + 1; I < T; ++I) if (S[I][K]) st[K].push_back(I);
    if (!st[K].empty()) level[st[K][0]] = std::max(level[st[K][0]], level[K] + 1);
  }
  int numLevels = 0;
  for (int K = 0; K < T; ++K) numLevels = std::max(numLevels, level[K] + 1);
  out.numLevels = numLevels;

  // 4. per-level work lists
  out.levelColStart.assign(1, 0);
  out.levelPanelStart.assign(1, 0);
  out.levelTaskStart.assign(1, 0);
  out.levelVTaskStart.assign(1, 0);
  out.taskPairStart.assign(1, 0);
  out.vtaskSrcStart.assign(1, 0);
  for (int L = 0; L < numLevels; ++L) {
    std::map<int, std::vector<std::pair<int, int>>> tasks; // dst tile -> (A,B) pairs
    std::map<int, std::vector<std::pair<int, int>>> vtasks; // block row -> (tile, K)
    for (int K = 0; K < T; ++K) {
      if (level[K] != L) continue;
      out.levelCols.push_back(K);
      for (int I : st[K]) {
        out.panelTile.push_back(tileId[I][K]);
        out.panelDiag.push_back(out.diagTile[K]);
        out.panelRow.push_back(I);
        vtasks[I].push_back({tileId[I][K], K});
      }
      for (size_t a = 0; a < st[K].size(); ++a)
        for (size_t b = 0; b <= a; ++b) {
          const int I = st[K][a], J = st[K][b];
          tasks[tileId[I][J]].push_back({tileId[I][K], tileId[J][K]}); // D(I,J)(r, c) -= sum_k L(I,K)(r, k) L(J,K)(c, k)
          out.tileOps++;
        }
    }
    for (auto& kv : tasks) {
      out.taskDst.push_back(kv.first);
      for (auto& pr : kv.second) { out.pairA.push_back(pr.first); out.pairB.push_back(pr.second); }
      out.taskPairStart.push_back(int(out.pairA.size()));
    }
    for (auto& kv : vtasks) {
      out.vtaskRow.push_back(kv.first);
      for (auto& pr : kv.second) { out.vsrcTile.push_back(pr.first); out.vsrcCol.push_back(pr.second); }
      out.vtaskSrcStart.push_back(int(out.vsrcTile.size()));
    }
    out.levelColStart.push_back(int(out.levelCols.size()));
    out.levelPanelStart.push_back(int(out.panelTile.size()));
    out.levelTaskStart.push_back(int(out.taskDst.size()));
    out.levelVTaskStart.push_back(int(out.vtaskRow.size()));
  }
  for (int W : {8, 16}) {
    std::vector<int32_t>& start = W == 8 ? out.levelOrderStart8 : out.levelOrderStart16;
    std::vector<int32_t>& order = W == 8 ? out.taskOrder8 : out.taskOrder16;
    start.assign(1, 0);
    for (int L = 0; L < numLevels; ++L) {
      std::vector<int> ids;
      for (int t = out.levelTaskStart[L]; t < out.levelTaskStart[L + 1]; ++t) ids.push_back(t);
      std::stable_sort(ids.begin(), ids.end(), [&](int a, int b) { return out.taskPairStart[a + 1] - out.taskPairStart[a] > out.taskPairStart[b + 1] - out.taskPairStart[b]; });
      std::vector<std::vector<int>> ofWarp(W);
      std::vector<int64_t> load(W, 0);
      for (int t : ids) {
        int w = 0;
        for (int k = 1; k < W; ++k) if (load[k] < load[w]) w = k;
        ofWarp[w].push_back(t);
        load[w] += 2 * (out.taskPairStart[t + 1] - out.taskPairStart[t]) + 1; // k-steps + the read-modify-write of the destination
      }
      size_t rounds = 0;
      for (const auto& v : ofWarp) rounds = std::max(rounds, v.size());
      const size_t base = order.size();
      order.resize(base + rounds * W, -1);
      for (int w = 0; w < W; ++w)
        for (size_t r = 0; r < ofWarp[w].size(); ++r) order[base + r * W + w] = ofWarp[w][r];
      start.push_back(int32_t(order.size()));
    }
  }
  out.colPanelStart.assign(1, 0);
  for (int K = 0; K < T; ++K) {
    for (int I : st[K]) { out.colPanelTile.push_back(tileId[I][K]); out.colPanelRow.push_back(I); }
    out.colPanelStart.push_back(int(out.colPanelTile.size()));
  }
  for (int K = 0; K < T; ++K) { const int64_t r = T - 1 - K; out.denseTileOps += r * (r + 1) / 2; }
  out.order = order;
  if (getenv("MB2_SCHED_DUMP") != nullptr) { // planner diagnostics (host only): the shape of every level
    fprintf(stderr, "chol schedule: n %d nPad %d tile columns %d tiles %d levels %d tile ops %lld (dense %lld)\n", n, out.nPad, T, out.numTiles, numLevels, (long long)out.tileOps, (long long)out.denseTileOps);
    for (int L = 0; L < numLevels; ++L) {
      int maxPairs = 0, pairs = 0;
      for (int t = out.levelTaskStart[L]; t < out.levelTaskStart[L + 1]; ++t) { const int p = out.taskPairStart[t + 1] - out.taskPairStart[t]; pairs += p; maxPairs = std::max(maxPairs, p); }
      fprintf(stderr, "  level %d: %d diagonal tiles, %d panel tiles, %d update tasks (%d pairs, longest %d), %d vector tasks; columns:", L, out.levelColStart[L + 1] - out.levelColStart[L],
              out.levelPanelStart[L + 1] - out.levelPanelStart[L], out.levelTaskStart[L + 1] - out.levelTaskStart[L], pairs, maxPairs, out.levelVTaskStart[L + 1] - out.levelVTaskStart[L]);
      for (int ci = out.levelColStart[L]; ci < out.levelColStart[L + 1]; ++ci) fprintf(stderr, " %d(%d)", out.levelCols[ci], int(st[out.levelCols[ci]].size()));
      fprintf(stderr, "\n");
    }
  }
  return "";
}

std::string buildGramPlan(const CholSchedule& s, const std::vector<int32_t>& cellRow0, const std::vector<int32_t>& cellRows, const std::vector<int32_t>& cellCol,
                          int numRows, GramPlan& out) {
  out = GramPlan();
  out.numTiles = s.numTiles;
  out.numTileCols = s.numTileCols;
  const int T = s.numTileCols;
  std::map<std::pair<int, int>, int> stripId; // (quad, tile column) -> strip, in (quad, K) order
  for (size_t i = 0; i < cellCol.size(); ++i) {
    const int d = cellCol[i];
    if (d < 0 || d >= s.n || s.pos[d] < 0) return "Jacobian cell in a column outside the schedule";
    const int K = s.pos[d] >> 4;
    for (int q = cellRow0[i] >> 2; q <= (cellRow0[i] + cellRows[i] - 1) >> 2; ++q) stripId[{q, K}] = 0;
  }
  int next = 0;
  for (auto& kv : stripId) kv.second = next++;
  out.numStrips = next;
  out.stripCoord.resize(size_t(next) * 2);
  std::vector<std::vector<int>> ofCol(T);
  for (const auto& kv : stripId) {
    const int q = kv.first.first, K = kv.first.second;
    out.stripCoord[2 * kv.second] = 4 * q;
    out.stripCoord[2 * kv.second + 1] = s.perm[16 * K]; // first slot of a tile column is always a real device column
    ofCol[K].push_back(kv.second);
  }
  // Pairs: tile (I,J) needs strip(q,I)^T strip(q,J) only when ONE row of quad q touches both tile columns. Rows of a unit share
  // their columns, so the pairs of a quad are the union over the units with rows in it (one-row units packed into the same quad
  // do not couple each other's columns: those products are exactly zero and their tiles need not exist).
  std::map<int, std::set<int>> colsOfUnit; // keyed by the unit's first row
  std::map<int, int> rowsOfUnit;
  for (size_t i = 0; i < cellCol.size(); ++i) { colsOfUnit[cellRow0[i]].insert(s.pos[cellCol[i]] >> 4); rowsOfUnit[cellRow0[i]] = cellRows[i]; }
  std::set<std::tuple<int, int, int>> quadPairs; // (quad, I, J), I >= J
  for (const auto& kv : colsOfUnit) {
    const int r0 = kv.first, r1 = r0 + rowsOfUnit[r0] - 1;
    for (int q = r0 >> 2; q <= r1 >> 2; ++q)
      for (int I : kv.second)
        for (int J : kv.second)
          if (I >= J) quadPairs.insert(std::make_tuple(q, I, J));
  }
  std::vector<std::vector<std::pair<int, int>>> pairs(s.numTiles);
  for (const auto& qp : quadPairs) {
    const int q = std::get<0>(qp), I = std::get<1>(qp), J = std::get<2>(qp);
    const int t = s.tileIdTable[size_t(I) * T + J];
    if (t < 0) return "Gram plan: a Jacobian row couples two tile columns whose tile is not in the schedule";
    pairs[t].push_back({stripId[{q, I}], stripId[{q, J}]});
  }
  out.residOff = out.numStrips * 64;
  out.stride = (out.residOff + ((numRows + 3) & ~3) + 63) / 64 * 64; // whole strips, so that "strip stride / 64" is the all-zero strip the kernel appends
  const int zeroStrip = out.stride / 64;
  out.tilePairStart.assign(s.numTiles + 1, 0);
  for (int t = 0; t < s.numTiles; ++t) {
    out.macs += int64_t(pairs[t].size()) * 16 * 16 * 4;
    if (pairs[t].size() % 2) pairs[t].push_back({zeroStrip, zeroStrip}); // the kernel consumes two pairs per step
    out.tilePairStart[t + 1] = out.tilePairStart[t] + int(pairs[t].size());
    for (const auto& pr : pairs[t]) { out.pairA.push_back(pr.first); out.pairB.push_back(pr.second); }
  }
  out.tileQuadStart.assign(s.numTiles + 1, 0);
  for (int t = 0; t < s.numTiles; ++t) {
    out.tileQuadStart[t + 1] = out.tileQuadStart[t] + (out.tilePairStart[t + 1] - out.tilePairStart[t]) / 2;
    for (int p = out.tilePairStart[t]; p < out.tilePairStart[t + 1]; p += 2) {
      out.quad.push_back(out.pairA[p] * 64); out.quad.push_back(out.pairB[p] * 64);
      out.quad.push_back(out.pairA[p + 1] * 64); out.quad.push_back(out.pairB[p + 1] * 64);
    }
  }
  // Tiles are dealt to the kGramWarps warps of a CTA / instance group: longest first, each to the least loaded warp (the root tile of
  // a humanoid collects 42 pairs, the median tile 2). tileOrder is the resulting [rounds][kGramWarps] table, -1 = nothing this round:
  // warp w walks entries w, w + kGramWarps, ...
  {
    std::vector<int> byLoad(s.numTiles);
    for (int t = 0; t < s.numTiles; ++t) byLoad[t] = t;
    std::stable_sort(byLoad.begin(), byLoad.end(), [&](int a, int b) { return pairs[a].size() > pairs[b].size(); });
    std::vector<std::vector<int>> ofWarp(kGramWarps);
    std::vector<int64_t> load(kGramWarps, 0);
    for (int t : byLoad) {
      int w = 0;
      for (int k = 1; k < kGramWarps; ++k) if (load[k] < load[w]) w = k;
      ofWarp[w].push_back(t);
      load[w] += int64_t(pairs[t].size()) / 2 + 2; // mma steps + the tile's fixed cost (epilogue)
    }
    size_t rounds = 0;
    for (const auto& v : ofWarp) rounds = std::max(rounds, v.size());
    out.tileOrder.assign(rounds * kGramWarps, -1);
    for (int w = 0; w < kGramWarps; ++w)
      for (size_t r = 0; r < ofWarp[w].size(); ++r) out.tileOrder[r * kGramWarps + w] = ofWarp[w][r];
  }
  // where each cell writes: strips of one quad are consecutive (ascending tile column); a multi-row unit owns its quads, so its
  // quads all have the same tile columns and the same cell is a constant number of strips further in the next quad
  std::map<int, int> stripsOfQuad;
  for (const auto& kv : stripId) ++stripsOfQuad[kv.first.first];
  out.cellStripOff.resize(cellCol.size());
  out.cellQuadStride.resize(cellCol.size());
  for (size_t i = 0; i < cellCol.size(); ++i) {
    const int d = cellCol[i], K = s.pos[d] >> 4, q0 = cellRow0[i] >> 2;
    out.cellStripOff[i] = uint32_t(stripId[{q0, K}]) * 64u + uint32_t(d - s.perm[16 * K]) * 4u;
    out.cellQuadStride[i] = uint16_t(stripsOfQuad[q0]);
    for (int q = q0 + 1; q <= (cellRow0[i] + cellRows[i] - 1) >> 2; ++q)
      if (stripsOfQuad[q] != stripsOfQuad[q0] || stripId[{q, K}] != stripId[{q0, K}] + (q - q0) * stripsOfQuad[q0]) return "Gram plan: row quads of one unit are not laid out uniformly";
  }
  out.colStripStart.assign(T + 1, 0);
  for (int K = 0; K < T; ++K) {
    out.colStripStart[K + 1] = out.colStripStart[K] + int(ofCol[K].size());
    out.colStrip.insert(out.colStrip.end(), ofCol[K].begin(), ofCol[K].end());
  }
  return "";
}

void makeGramBlob(const GramPlan& g, const CholSchedule& s, std::vector<int32_t>& blob, int32_t offsets[8]) {
  blob.clear();
  int k = 0;
  auto add = [&](const std::vector<int32_t>& v) { offsets[k++] = int32_t(blob.size()); blob.insert(blob.end(), v.begin(), v.end()); while (blob.size() % 4) blob.push_back(0); };
  add(g.tileOrder); add(g.tileQuadStart); add(g.quad); add(std::vector<int32_t>()); add(g.colStripStart); add(g.colStrip);
  std::vector<int32_t> stripRow(g.numStrips), info(s.numTiles);
  for (int i = 0; i < g.numStrips; ++i) stripRow[i] = g.stripCoord[2 * i];
  auto validOf = [&](int K) { int v = 0; while (v < kCholTile && s.perm[16 * K + v] >= 0) ++v; return v; };
  for (int t = 0; t < s.numTiles; ++t) info[t] = validOf(s.tileRow[t]) | (validOf(s.tileCol[t]) << 8) | ((s.tileRow[t] == s.tileCol[t] ? 1 : 0) << 16);
  add(stripRow); add(info);
  if (blob.empty()) blob.push_back(0);
}

std::string makeGramCholTables(const GramPlan& g, const CholSchedule& s, GramCholTables& out) {
  out = GramCholTables();
  std::vector<uint16_t>& t = out.tab;
  bool fits = true;
  auto put = [&](int64_t v) { fits = fits && v >= 0 && v <= 0xFFFF; t.push_back(uint16_t(v)); };
  auto section = [&]() { while (t.size() % 4) t.push_back(0); return int32_t(t.size()); };
  auto validOf = [&](int K) { int v = 0; while (v < kCholTile && s.perm[16 * K + v] >= 0) ++v; return v; };
  out.L.gram = section();
  for (int32_t tile : g.tileOrder) {
    if (tile < 0) { put(0xFFFF); put(0); put(0); put(0); continue; }
    fits = fits && tile < 0xFFFF;
    put(tile);
    put(validOf(s.tileRow[tile]) | (validOf(s.tileCol[tile]) << 8) | ((s.tileRow[tile] == s.tileCol[tile] ? 1 : 0) << 15));
    put(g.tileQuadStart[tile]); put(g.tileQuadStart[tile + 1]);
  }
  out.L.quad = section();
  for (int32_t v : g.quad) put(v);
  out.L.col = section();
  for (int32_t v : g.colStripStart) put(v);
  out.L.colEnt = section();
  for (int32_t sidx : g.colStrip) { put(int64_t(sidx) * 64); put(g.stripCoord[2 * sidx]); }
  out.L.level = section();
  for (int L = 0; L <= s.numLevels; ++L) { put(s.levelColStart[L]); put(s.levelPanelStart[L]); put(s.levelOrderStart8[L]); put(s.levelVTaskStart[L]); }
  out.L.diag = section();
  for (int32_t K : s.levelCols) { put(K); put(s.diagTile[K]); put(s.colPanelStart[K]); put(s.colPanelStart[K + 1]); }
  out.L.panel = section();
  for (size_t pi = 0; pi < s.panelTile.size(); ++pi) { put(s.panelTile[pi]); put(s.panelDiag[pi]); }
  out.L.order = section();
  for (int32_t ti : s.taskOrder8) {
    if (ti < 0) { put(0xFFFF); put(0); put(0); put(0); continue; }
    fits = fits && s.taskDst[ti] < 0xFFFF;
    put(s.taskDst[ti]); put(s.taskPairStart[ti]); put(s.taskPairStart[ti + 1]); put(0);
  }
  out.L.pair = section();
  for (size_t p = 0; p < s.pairA.size(); ++p) { put(s.pairA[p]); put(s.pairB[p]); }
  out.L.vtask = section();
  for (size_t vi = 0; vi < s.vtaskRow.size(); ++vi) { put(s.vtaskRow[vi]); put(s.vtaskSrcStart[vi]); put(s.vtaskSrcStart[vi + 1]); put(0); }
  out.L.vsrc = section();
  for (size_t p = 0; p < s.vsrcTile.size(); ++p) { put(s.vsrcTile[p]); put(s.vsrcCol[p]); }
  out.L.colPanel = section();
  for (size_t p = 0; p < s.colPanelTile.size(); ++p) { put(s.colPanelTile[p]); put(s.colPanelRow[p]); }
  section();
  const int64_t onStrips = (int64_t(g.stride) + 64 + 255) / 256;
  out.parkTiles = int32_t(std::min<int64_t>(s.numTiles, onStrips));
  return fits ? "" : "Gram + Cholesky tables: an entry does not fit in 16 bits";
}

void layoutDeviceColumns(CholSchedule& s, std::vector<int32_t>& deviceColumnOrder) {
  deviceColumnOrder.clear();
  s.nParams = s.n;
  for (int K = 0; K < s.numTileCols; ++K) {
    while (deviceColumnOrder.size() % 4 != 0) deviceColumnOrder.push_back(-1);
    for (int j = 0; j < kCholTile; ++j) {
      int16_t& p = s.perm[16 * K + j];
      if (p < 0) continue;
      const int dev = int(deviceColumnOrder.size());
      deviceColumnOrder.push_back(p);
      p = int16_t(dev);
    }
  }
  s.n = int32_t(deviceColumnOrder.size());
  s.pos.assign(s.n, int16_t(-1));
  for (int slot = 0; slot < s.nPad; ++slot) if (s.perm[slot] >= 0) s.pos[s.perm[slot]] = int16_t(slot);
  s.order.assign(deviceColumnOrder.begin(), deviceColumnOrder.end());
}

} // namespace mb2

namespace mb2 {

void makeScheduleBlob(const CholSchedule& s, std::vector<int32_t>& blob, CholSchedDev& dev) {
  blob.clear();
  std::vector<size_t> offs;
  auto add16 = [&](const std::vector<int16_t>& v) { offs.push_back(blob.size()); for (int16_t x : v) blob.push_back(int32_t(x)); while (blob.size() % 4) blob.push_back(0); };
  auto add32 = [&](const std::vector<int32_t>& v) { offs.push_back(blob.size()); blob.insert(blob.end(), v.begin(), v.end()); while (blob.size() % 4) blob.push_back(0); };
  add16(s.perm); add16(s.pos); add16(s.tileIdTable); add16(s.tileRow); add16(s.tileCol);
  add32(s.diagTile); add32(s.levelColStart); add32(s.levelCols); add32(s.levelPanelStart); add32(s.panelTile); add32(s.panelDiag);
  add32(s.levelTaskStart); add32(s.taskDst); add32(s.taskPairStart); add32(s.pairA); add32(s.pairB); add32(s.levelVTaskStart); add32(s.vtaskRow);
  add32(s.vtaskSrcStart); add32(s.vsrcTile); add32(s.vsrcCol); add32(s.colPanelStart); add32(s.colPanelTile); add32(s.colPanelRow);
  add32(s.levelOrderStart8); add32(s.taskOrder8); add32(s.levelOrderStart16); add32(s.taskOrder16);
  {
    std::vector<int32_t> info(size_t(s.numTiles) * 3, 0);
    auto validOf = [&](int K) { int v = 0; while (v < kCholTile && s.perm[16 * K + v] >= 0) ++v; return v; };
    for (int t = 0; t < s.numTiles; ++t) {
      const int I = s.tileRow[t], J = s.tileCol[t];
      const int vI = validOf(I), vJ = validOf(J);
      info[3 * t] = vI > 0 ? s.perm[16 * I] : 0;
      info[3 * t + 1] = vJ > 0 ? s.perm[16 * J] : 0;
      info[3 * t + 2] = vI | (vJ << 8) | ((I == J ? 1 : 0) << 16);
    }
    add32(info);
  }
  if (blob.empty()) blob.push_back(0);
  dev = CholSchedDev();
  dev.n = s.n; dev.nPad = s.nPad; dev.numTileCols = s.numTileCols; dev.numTiles = s.numTiles; dev.numLevels = s.numLevels;
  const int32_t* b = blob.data();
  dev.blob = b;
  dev.blobInts = int32_t(blob.size());
  int k = 0;
  dev.perm = b + offs[k++]; dev.pos = b + offs[k++]; dev.tileIdTable = b + offs[k++]; dev.tileRow = b + offs[k++]; dev.tileCol = b + offs[k++];
  dev.diagTile = b + offs[k++]; dev.levelColStart = b + offs[k++]; dev.levelCols = b + offs[k++]; dev.levelPanelStart = b + offs[k++];
  dev.panelTile = b + offs[k++]; dev.panelDiag = b + offs[k++]; dev.levelTaskStart = b + offs[k++]; dev.taskDst = b + offs[k++];
  dev.taskPairStart = b + offs[k++]; dev.pairA = b + offs[k++]; dev.pairB = b + offs[k++]; dev.levelVTaskStart = b + offs[k++]; dev.vtaskRow = b + offs[k++];
  dev.vtaskSrcStart = b + offs[k++]; dev.vsrcTile = b + offs[k++]; dev.vsrcCol = b + offs[k++]; dev.colPanelStart = b + offs[k++];
  dev.colPanelTile = b + offs[k++]; dev.colPanelRow = b + offs[k++];
  dev.levelOrderStart8 = b + offs[k++]; dev.taskOrder8 = b + offs[k++]; dev.levelOrderStart16 = b + offs[k++]; dev.taskOrder16 = b + offs[k++];
  dev.tileInfo = b + offs[k++];
}

} // namespace mb2
