// tc_schedule.h -- how the work items of a tensor-core conv launch are dealt to the persistent CTAs (plain C++,
// host only; tc_conv.cu and tc_wgrad.cu fill it, the kernels walk it, tests compile it on its own).
//
// Both kernels run one CTA per SM over a list of work items whose K loops have known lengths (in K blocks).  Dealt
// round robin, CTA g runs items g, g + grid, ...; a launch lasts as long as its most loaded CTA, and the last wave
// leaves SMs idle.  The stream-K schedule keeps round robin for all but the last one or two waves (data-parallel,
// DP) and spreads the K blocks of the rest over the grid (stream-K, SK):
//   * items [0, dp_items), dp_items = W * grid, W = items / grid (one less when the division leaves a remainder):
//     CTA g runs items g, g + grid, ... with their whole K loops, as round robin does;
//   * items [dp_items, items) -- between grid and 2 * grid - 1 of them, or all when items < grid -- are laid end to
//     end, item-major, and cut into grid consecutive ranges, one per CTA, sized so that every CTA ends at the same
//     time: a CTA whose DP items are short (the classes of a transposed layer have unequal tap counts) gets a
//     longer range.  Cuts fall only on multiples of `chunk` K blocks from an item's start, so every wgmma
//     accumulation chunk stays whole (tc_conv.cu, "Accuracy").  Consecutive CTAs get consecutive ranges: the items
//     that run side by side are still neighbours in the item order and share their input boxes in L2.
// A range starts at (sk_item[g], sk_k[g]) -- SK item (counted from dp_items) and K block within it -- and ends
// where range g + 1 starts; range grid ends at (items - dp_items, 0).  Each (item, K range) piece of a range is
// one SEGMENT.  An item cut by one or more range boundaries is SPLIT: several CTAs run one segment of it each.
//
// A split item costs more than its K blocks: its segments refill the pipeline, and tc_conv adds the partial sums
// of its segments in a fixup.  make_sk_schedule charges kSkSplitCost chunks for every segment of a split item and
// keeps plain round robin (dp_items = items, no ranges, grid = min(items, grid)) unless the stream-K schedule ends
// the launch at least one chunk sooner.  Launches whose items are shorter than a chunk, whose last wave is nearly
// full, or whose DP waves are long beside the tail therefore stay round robin, and compute exactly what they
// computed without this schedule.
#pragma once

namespace unflow {
namespace tc {

constexpr int kSkMaxGrid = 132;       // CTAs of a launch (one per SM of an H100 SXM)
constexpr int kSkSplitCost = 1;       // model cost of one segment of a split item, in chunks

struct SkSchedule {
  int grid;                           // CTAs to launch
  int dp_items;                       // items run whole, round robin (= all items when stream-K does not pay)
  int sk_item[kSkMaxGrid + 1];        // start of CTA g's SK range: SK item ...
  int sk_k[kSkMaxGrid + 1];           // ... and K block within it
};

// `len(i)`: K blocks of item i (>= 0).  `grid` <= kSkMaxGrid, `chunk` >= 1.  Returns the modelled length of the
// launch (K blocks of its most loaded CTA, split costs included).
template <class Len>
inline long long make_sk_schedule(SkSchedule &s, int items, int grid, int chunk, Len len) {
  // plain round robin: the fallback, and the length to beat
  long long rr[kSkMaxGrid] = {}, rr_span = 0;
  for (int i = 0; i < items; ++i) rr[i % grid] += len(i);
  for (int g = 0; g < grid; ++g) rr_span = rr[g] > rr_span ? rr[g] : rr_span;
  auto round_robin = [&]() {
    s.grid = items < grid ? items : grid;
    s.dp_items = items;
    for (int g = 0; g <= kSkMaxGrid; ++g) s.sk_item[g] = s.sk_k[g] = 0;
    return rr_span;
  };
  const int waves = items / grid;
  const int dp_items = (items % grid ? (waves > 0 ? waves - 1 : 0) : waves) * grid;
  const int n_sk = items - dp_items;
  if (n_sk == 0) return round_robin();
  long long dp[kSkMaxGrid] = {}, total = 0, dp_max = 0;
  for (int i = 0; i < dp_items; ++i) dp[i % grid] += len(i);
  for (int j = 0; j < n_sk; ++j) total += len(dp_items + j);
  for (int g = 0; g < grid; ++g) dp_max = dp[g] > dp_max ? dp[g] : dp_max;
  if (total == 0) return round_robin();
  // the level every CTA should end at: the least one whose room above the DP loads holds the SK K blocks
  long long lo = 0, hi = dp_max + total;
  while (lo < hi) {
    const long long mid = (lo + hi) / 2;
    long long room = 0;
    for (int g = 0; g < grid; ++g) room += mid > dp[g] ? mid - dp[g] : 0;
    if (room >= total) hi = mid; else lo = mid + 1;
  }
  // range g starts at the first allowed cut at or after its share of the SK K blocks: the room of CTAs 0 .. g - 1
  // scaled to the total (the room at that level exceeds the total by less than a K block per CTA; scaling spreads
  // the excess).  The walk over the items only moves forward because the targets grow with g.
  long long room_all = 0;
  for (int g = 0; g < grid; ++g) room_all += lo > dp[g] ? lo - dp[g] : 0;
  s.grid = grid;
  s.dp_items = dp_items;
  int j = 0;
  long long off = 0, room = 0;        // off: K blocks of the SK items before item j
  for (int g = 0; g <= grid; ++g) {
    if (g > 0) room += lo > dp[g - 1] ? lo - dp[g - 1] : 0;
    const long long target = g == grid ? total : total * room / room_all;
    while (j < n_sk && off + len(dp_items + j) <= target) { off += len(dp_items + j); ++j; }
    if (j == n_sk) { s.sk_item[g] = n_sk; s.sk_k[g] = 0; continue; }
    const long long k = (target - off + chunk - 1) / chunk * chunk;
    if (k < len(dp_items + j)) {
      s.sk_item[g] = j; s.sk_k[g] = (int)k;
    } else {                          // past the last chunk start of item j: the next item's start
      s.sk_item[g] = j + 1; s.sk_k[g] = 0;
    }
  }
  for (int g = grid + 1; g <= kSkMaxGrid; ++g) { s.sk_item[g] = n_sk; s.sk_k[g] = 0; }
  // the modelled length: DP load + range + the split cost of every segment of a split item
  long long span = 0;
  for (int g = 0; g < grid; ++g) {
    long long load = dp[g];
    for (int jj = s.sk_item[g]; jj <= s.sk_item[g + 1] && jj < n_sk; ++jj) {
      const int L = len(dp_items + jj);
      const long long k0 = jj == s.sk_item[g] ? s.sk_k[g] : 0, k1 = jj == s.sk_item[g + 1] ? s.sk_k[g + 1] : L;
      if (k1 <= k0) continue;
      load += k1 - k0;
      if (k0 > 0 || k1 < L) load += (long long)kSkSplitCost * chunk;
    }
    span = load > span ? load : span;
  }
  if (span + chunk > rr_span) return round_robin();
  return span;
}

}  // namespace tc
}  // namespace unflow
