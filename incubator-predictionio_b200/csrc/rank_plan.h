// rank_plan.h -- how a pio_als_rank_lists call is cut up and which path each query takes.  Pure host C++17: no CUDA
// header and no handle, so the rules can be checked without a GPU (tests/test_rank_plan.py compiles this header alone
// and compares it with the model in tests/productranking_ref.py).  pio_als.cu asks for the plan and runs it.
//
//   parts   consecutive queries; a part closes before the query whose entries would take it over the budget, and holds
//           at least one query, so a single query over the budget forms a part of its own
//   radix   a query whose list is longer than RL_TILE entries: scored into (order key, entry) pairs, then two stable
//           radix sorts (by order key, then by the query)
//   tiles   the other non-empty queries of a part, packed in order into tiles of at most RL_TILE entries: a tile
//           closes before a query that would overflow it.  One CTA per tile scores and sorts it in shared memory.
//   empty   a query with an empty list takes no path: it is not ranked, and it has no entry to write.
#pragma once
#include <stdint.h>

#include <vector>

namespace pio {

constexpr int RL_TILE = 2048;   // entries of one tile: one CTA of RL_TILE / 2 threads, two entries each

struct RankPart {
  int q0 = 0, q1 = 0;               // queries [q0, q1)
  long long e0 = 0, e1 = 0;         // their entries [e0, e1) = [list_ptr[q0], list_ptr[q1])
  std::vector<int> radix;           // queries on the radix path, in query order
  std::vector<int> tile_q;          // queries on the tile path, in query order
  std::vector<int> tile_ptr{0};     // tile t holds tile_q[tile_ptr[t] .. tile_ptr[t + 1])
  std::vector<int> tile_off;        // entry offset of tile_q[j] inside its tile
  std::vector<int> tile_n;          // entries of each tile
  int n_tiles() const { return (int)tile_n.size(); }
};

// The parts of a call of n queries with offsets list_ptr[0 .. n] (already checked: list_ptr[0] == 0, non-decreasing,
// every list shorter than 2^31) under an entries budget >= 1.
inline std::vector<RankPart> plan_rank_lists(const int64_t* list_ptr, int n, long long budget) {
  std::vector<RankPart> parts;
  long long acc = 0;
  for (int q = 0; q < n; ++q) {
    const long long len = list_ptr[q + 1] - list_ptr[q];
    if (parts.empty() || acc + len > budget) {
      parts.emplace_back();
      parts.back().q0 = q;
      parts.back().e0 = list_ptr[q];
      acc = 0;
    }
    acc += len;
    RankPart& p = parts.back();
    p.q1 = q + 1;
    p.e1 = list_ptr[q + 1];
    if (len > RL_TILE) {
      p.radix.push_back(q);
    } else if (len > 0) {
      if (p.tile_n.empty() || p.tile_n.back() + len > RL_TILE) {
        if (!p.tile_n.empty()) p.tile_ptr.push_back((int)p.tile_q.size());
        p.tile_n.push_back(0);
      }
      p.tile_q.push_back(q);
      p.tile_off.push_back(p.tile_n.back());
      p.tile_n.back() += (int)len;
    }
  }
  for (RankPart& p : parts)
    if (!p.tile_n.empty()) p.tile_ptr.push_back((int)p.tile_q.size());
  return parts;
}

}  // namespace pio
