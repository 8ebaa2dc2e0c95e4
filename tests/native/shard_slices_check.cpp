// The sliced decode's slice planner (coverm_b200/csrc/cmb_slices.hpp) on random block tables: the slices cover the
// record blocks exactly once and in order, each fits the budget unless it is one block that alone exceeds it, each is as long as
// the budget allows, and a budget below one block is reported slice by slice instead of looping.  Prints "ok <cases>".
#include <cstdio>
#include <random>

#include "cmb_slices.hpp"

static int fails = 0;
#define CHECK(cond, ...)                        \
  do {                                          \
    if (!(cond)) {                              \
      if (fails++ < 10) {                       \
        fprintf(stderr, "FAIL %s: ", #cond);    \
        fprintf(stderr, __VA_ARGS__);           \
        fprintf(stderr, "\n");                  \
      }                                         \
    }                                           \
  } while (0)

int main() {
  std::mt19937_64 rng(7);
  int cases = 0;
  for (int t = 0; t < 3000; ++t) {
    const uint32_t nb = 1 + rng() % 300;
    std::vector<uint64_t> coff(nb), ustart(nb + 1, 0);
    std::vector<uint32_t> clen(nb);
    uint64_t o = 100 + rng() % 5000;  // the file's header block(s) lie in front
    for (uint32_t b = 0; b < nb; ++b) {
      const bool eof = b + 1 == nb && rng() % 2;  // the empty BGZF end-of-file block
      const uint32_t isize = eof ? 0 : (uint32_t)(rng() % 4 == 0 ? 1 + rng() % 200 : 1 + rng() % 65280);
      clen[b] = eof ? 2 : 1 + (uint32_t)(rng() % (isize + 64));
      coff[b] = o + 18;
      o += 18 + clen[b] + 8;
      ustart[b + 1] = ustart[b] + isize;
    }
    const SliceBlocks f{nb, o, coff.data(), clen.data(), ustart.data()};
    const uint32_t first = (uint32_t)(rng() % nb);
    const uint64_t tail = rng() % 3 == 0 ? 0 : 1 + rng() % 200000;
    const uint64_t whole = slice_bytes(f, first, nb, tail);
    const uint64_t budget = rng() % 8 == 0 ? rng() % 100 : rng() % (whole + whole / 4 + 1);
    uint32_t n_over = 0;
    const auto plan = plan_slices(f, first, budget, tail, &n_over);
    uint32_t at = first, over = 0;
    for (const auto& s : plan) {
      CHECK(s.first == at && s.second > s.first && s.second <= nb, "case %d: slice [%u, %u) after %u of %u", t, s.first, s.second, at, nb);
      const uint64_t bytes = slice_bytes(f, s.first, s.second, tail);
      if (bytes > budget) {
        ++over;
        CHECK(s.second == s.first + 1, "case %d: slice [%u, %u) of %llu bytes over a budget of %llu", t, s.first, s.second,
              (unsigned long long)bytes, (unsigned long long)budget);
      } else if (s.second < nb) {
        CHECK(slice_bytes(f, s.first, s.second + 1, tail) > budget, "case %d: slice [%u, %u) could take one more block", t, s.first, s.second);
      }
      at = s.second;
    }
    CHECK(at == nb, "case %d: the slices end at %u of %u", t, at, nb);
    CHECK(over == n_over, "case %d: %u slices over the budget, %u reported", t, over, n_over);
    if (budget >= whole) CHECK(plan.size() == 1, "case %d: a shard that fits is %zu slices", t, plan.size());
    ++cases;
  }
  if (fails) {
    fprintf(stderr, "%d failures\n", fails);
    return 1;
  }
  printf("ok %d\n", cases);
  return 0;
}
