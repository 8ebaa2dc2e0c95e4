// The ordinary sliced decode's rules (coverm_b200/csrc/cmb_slices.hpp) compiled as plain C++.
//
// Pair cut: random tid / eligibility streams, sorted and unsorted, walked in slices of random record counts the way
// decode_sliced walks them -- every slice but the last submits the records before its cut and the next slice starts at the
// cut; the order fold runs over each slice's eligible tids with the earlier slices' largest tid as its carry.  Checked against
// a brute-force walk of the whole stream:
//   - the records are submitted exactly once, in file order;
//   - every tid's eligible records fall in one slice;
//   - a slice whose records after the first eligible one are one run is reported (cut 0), never looped on, and only then;
//   - the fold flags a stream exactly when some eligible tid is below an earlier one, also when the drop lies across a slice
//     edge.
// Budget: decode_slice_budget leaves room for the event list's projected peak and the slice's other buffers.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include "cmb_slices.hpp"

namespace {
int failures = 0;
#define CHECK(cond, ...)                  \
  do {                                    \
    if (!(cond)) {                        \
      if (failures++ < 20) {              \
        fprintf(stderr, "FAIL: " __VA_ARGS__); \
        fprintf(stderr, "\n");            \
      }                                   \
    }                                     \
  } while (0)

struct Rec {
  bool eligible;
  uint32_t tid;
};

// The fold of one slice: whether an eligible tid drops below the largest before it (carry included), and the new largest
uint32_t fold(const std::vector<Rec>& r, uint32_t a, uint32_t b, uint32_t carry, bool* drop) {
  uint32_t largest = carry;
  for (uint32_t i = a; i < b; ++i) {
    if (!r[i].eligible) continue;
    *drop = *drop || pair_order_drop(r[i].tid, largest);
    largest = std::max(largest, r[i].tid);
  }
  return largest;
}

// The cut of slice [a, b) by the two reductions the kernels do, relative to a
uint32_t cut_of(const std::vector<Rec>& r, uint32_t a, uint32_t b, uint32_t last) {
  const uint32_t n = b - a;
  uint32_t after = 0, cut = n;
  for (uint32_t i = 0; i < n; ++i) after = std::max(after, pair_cut_after(r[a + i].eligible, r[a + i].tid, last, i));
  for (uint32_t i = 0; i < n; ++i) cut = std::min(cut, pair_cut_at(r[a + i].eligible, r[a + i].tid, last, after, i, n));
  return cut;
}

std::vector<Rec> stream(std::mt19937& rng, bool sorted) {
  const uint32_t n = 1 + rng() % 400, n_tids = 1 + rng() % 12;
  const uint32_t p_elig = rng() % 101;
  std::vector<Rec> r(n);
  for (auto& x : r) {
    x.eligible = rng() % 100 < p_elig;
    x.tid = rng() % 8 == 0 ? 0xffffffffu : rng() % n_tids;  // some unplaced (tid -1: last in unsigned order)
  }
  if (sorted) std::sort(r.begin(), r.end(), [](const Rec& a, const Rec& b) { return a.tid < b.tid; });
  return r;
}

void check_pairs(std::mt19937& rng, bool sorted, uint32_t max_slice) {
  const std::vector<Rec> r = stream(rng, sorted);
  const uint32_t n = (uint32_t)r.size();
  // brute force: a drop anywhere among the eligible records
  bool want_drop = false;
  for (uint32_t i = 0, hi = 0; i < n; ++i)
    if (r[i].eligible) {
      want_drop = want_drop || r[i].tid < hi;
      hi = std::max(hi, r[i].tid);
    }
  std::vector<uint32_t> submitted, slice_of(n, ~0u);
  uint32_t at = 0, carry = 0, slice = 0, checked_end = 0;
  bool drop = false, declined = false;
  for (uint32_t iter = 0; at < n; ++iter) {
    CHECK(iter <= n, "the walk does not progress");
    if (iter > n) return;
    const uint32_t b = std::min(n, at + 1 + (uint32_t)(rng() % max_slice));
    const uint32_t largest = fold(r, at, b, carry, &drop);
    checked_end = b;
    if (drop) break;  // mate matching gives up: the sample declines
    uint32_t cut = b - at;
    if (b < n) {
      cut = cut_of(r, at, b, largest);
      if (cut == 0) {
        // only when every eligible record of the slice has tid `largest` and the first record is one of them
        bool one_run = r[at].eligible && r[at].tid == largest;
        for (uint32_t i = at; i < b; ++i) one_run = one_run && (!r[i].eligible || r[i].tid == largest);
        CHECK(one_run, "cut 0 for a slice that is not one run (at %u)", at);
        declined = true;
        break;
      }
      // the held-back records are eligible of tid `largest` or not eligible, and the first of them is eligible
      CHECK(cut == b - at || (r[at + cut].eligible && r[at + cut].tid == largest), "held-back run starts at a wrong record");
      for (uint32_t i = at + cut; i < b; ++i) CHECK(!r[i].eligible || r[i].tid == largest, "held back a record of another tid");
    }
    for (uint32_t i = at; i < at + cut; ++i) {
      submitted.push_back(i);
      slice_of[i] = slice;
    }
    carry = largest;
    at += cut;
    ++slice;
  }
  bool want_checked_drop = false;  // a drop among the records the walk folded
  for (uint32_t i = 0, hi = 0; i < checked_end; ++i)
    if (r[i].eligible) {
      want_checked_drop = want_checked_drop || r[i].tid < hi;
      hi = std::max(hi, r[i].tid);
    }
  CHECK(drop == want_checked_drop, "fold flagged %d, brute force %d (sorted %d)", (int)drop, (int)want_checked_drop, (int)sorted);
  CHECK(!drop || want_drop, "a drop flagged in a stream without one");
  if (sorted) CHECK(!drop, "a sorted stream flagged");
  if (drop || declined) return;
  CHECK(!want_drop, "a drop was missed");
  CHECK(submitted.size() == n, "%zu of %u records submitted", submitted.size(), n);
  for (uint32_t i = 0; i < submitted.size(); ++i) CHECK(submitted[i] == i, "record %u submitted out of order", i);
  std::vector<uint32_t> tid_slice;  // every tid's eligible records in one slice
  std::vector<uint32_t> tids;
  for (uint32_t i = 0; i < n; ++i) {
    if (!r[i].eligible) continue;
    auto it = std::find(tids.begin(), tids.end(), r[i].tid);
    if (it == tids.end()) {
      tids.push_back(r[i].tid);
      tid_slice.push_back(slice_of[i]);
    } else {
      CHECK(tid_slice[it - tids.begin()] == slice_of[i], "tid %u split over slices %u and %u", r[i].tid, tid_slice[it - tids.begin()], slice_of[i]);
    }
  }
}

// An order drop exactly at a slice edge: slice 1 ends with tid 5, slice 2 starts with tid 3
void check_edge_drop() {
  std::vector<Rec> r;
  for (int i = 0; i < 10; ++i) r.push_back({true, 5});
  for (int i = 0; i < 10; ++i) r.push_back({true, 3});
  bool drop = false;
  uint32_t carry = fold(r, 0, 10, 0, &drop);
  CHECK(!drop && carry == 5, "first slice");
  fold(r, 10, 20, carry, &drop);
  CHECK(drop, "a drop across the slice edge was not flagged");
  bool alone = false;
  fold(r, 10, 20, 0, &alone);
  CHECK(!alone, "the second slice alone is in order");
}

void check_budget(std::mt19937& rng) {
  for (int t = 0; t < 20000; ++t) {
    const uint64_t room = (64ull << 20) + rng() % (80ull << 30);
    const uint64_t total = 1 + rng() % (200ull << 30), done = rng() % (total + 1);
    const uint64_t iv_done = done / (100 + rng() % 3000);
    const uint64_t held = iv_done * SLICE_EVENT_BYTES * (rng() % 3);
    const double side = (rng() % 100) / 100.0;
    const bool events = rng() & 1;
    const uint64_t b = decode_slice_budget(room, events, held, done, total, iv_done, side);
    if (done == 0) {
      CHECK(b == room / 2, "the first slice takes half the room");
      continue;
    }
    double peak = 0;  // the event list's projected final size, twice (old and new during grow_keep), less what is held
    if (events && done < total) peak = std::max(0.0, 2.0 * SLICE_EVENT_BYTES * (double)iv_done * (double)total / (double)done - (double)held);
    if (done < total && b) CHECK((double)b * (1 + side) + peak <= (double)room * (1 + 1e-9) + 2, "budget %llu over the room", (unsigned long long)b);
    if (!b) CHECK(peak >= (double)room * (1 - 1e-9) - 2, "no budget although the event list leaves room");
    // more room never gives a smaller slice
    CHECK(decode_slice_budget(room + (1ull << 30), events, held, done, total, iv_done, side) >= b, "budget not monotonic in the room");
  }
}
}  // namespace

int main() {
  std::mt19937 rng(20261017);
  for (int t = 0; t < 20000; ++t) check_pairs(rng, t % 2 == 0, 1 + rng() % 120);
  check_edge_drop();
  check_budget(rng);
  if (failures) {
    fprintf(stderr, "%d failures\n", failures);
    return 1;
  }
  printf("ok decode slices\n");
  return 0;
}
