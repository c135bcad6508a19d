// Host-side work lists of the persistent Schur SYRK kernels (csrc/ba_schur.cu FP64 DMMA, csrc/syrk_i8.cu Ozaki INT8):
// the upper 128 x 128 tiles of Zt^T Zt, each cut into k ranges of 64-row blocks.
#pragma once
#include <algorithm>
#include <utility>
#include <vector>

namespace vgg {

struct SyrkTileJob {
  int bi, bj;                  // row block bi <= column block bj
  int kb0 = 0, kb1 = -1;       // k-block range in which BOTH row blocks can be non-zero (kb1 < 0: all of K)
};

// Upper tiles of an nb x nb block grid.  ranges (the band hint, [lo, hi) k blocks per row block, empty = dense): tiles
// whose two ranges do not meet are left out, the others are clipped to the intersection.
inline std::vector<SyrkTileJob> syrk_tile_jobs(int nb, const std::vector<int>& ranges) {
  const bool banded = (int)ranges.size() == 2 * nb;
  std::vector<SyrkTileJob> jobs;
  for (int bi = 0; bi < nb; ++bi)
    for (int bj = 0; bj <= bi; ++bj) {
      SyrkTileJob jb{bj, bi};
      if (banded) {
        jb.kb0 = std::max(ranges[2 * bi], ranges[2 * bj]);
        jb.kb1 = std::min(ranges[2 * bi + 1], ranges[2 * bj + 1]);
        if (jb.kb1 <= jb.kb0) continue;
      }
      jobs.push_back(jb);
    }
  return jobs;
}

// Work items are handed out statically (item w goes to CTA w mod nworkers, longest first), so the finishing time is the
// heaviest residue class.  Every job is done once per entry of group_cost, at group_cost[g] units per k block (the
// Ozaki kernel's order groups cost their pair count; a plain FP64 product has one group of cost 1).  The k-split
// granularity is chosen by simulating that assignment for a few candidate targets and keeping the best makespan, with
// epilogue_cost units charged per item.  No item spans more than max_item_kb k blocks.
template <class Work, class Make>
void build_work_list(const std::vector<int>& group_cost, const std::vector<SyrkTileJob>& jobs, int KB, int nworkers,
                     int max_item_kb, long long epilogue_cost, Make make, std::vector<Work>* out) {
  long long total = 0, cost_all = 0;
  for (int c : group_cost) cost_all += c;
  for (const SyrkTileJob& jb : jobs) total += cost_all * (long long)((jb.kb1 < 0 ? KB : jb.kb1) - jb.kb0);
  long long best = -1;
  for (int div = 2; div <= 10; ++div) {
    const long long target = std::max<long long>(1, total / ((long long)nworkers * div));
    std::vector<std::pair<long long, Work>> items;
    for (const SyrkTileJob& jb : jobs) {
      const int jk0 = jb.kb0, jk1 = jb.kb1 < 0 ? KB : jb.kb1, len = jk1 - jk0;
      if (len <= 0) continue;
      for (int g = 0; g < (int)group_cost.size(); ++g) {
        const long long cost = (long long)group_cost[g] * len;
        int parts = (int)std::min<long long>(16, std::max<long long>(1, (cost + target / 2) / target));
        parts = std::max(parts, (len + max_item_kb - 1) / max_item_kb);
        parts = std::min(parts, len);
        for (int p = 0; p < parts; ++p) {
          const int k0 = jk0 + (int)((long long)len * p / parts), k1 = jk0 + (int)((long long)len * (p + 1) / parts);
          items.push_back({(long long)group_cost[g] * (k1 - k0), make(jb, g, k0, k1)});
        }
      }
    }
    std::stable_sort(items.begin(), items.end(), [](const auto& a, const auto& b) { return a.first > b.first; });
    std::vector<long long> load(nworkers, 0);
    for (size_t i = 0; i < items.size(); ++i) load[i % nworkers] += items[i].first + epilogue_cost;
    const long long makespan = *std::max_element(load.begin(), load.end());
    if (best < 0 || makespan < best) {
      best = makespan;
      out->clear();
      for (auto& it : items) out->push_back(it.second);
    }
  }
}

}  // namespace vgg
