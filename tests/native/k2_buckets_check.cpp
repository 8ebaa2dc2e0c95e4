// Contig mode's K2 rounds built from word buckets (coverm_b200/csrc/cmb_k2_slots.cuh: k2_round_words, k2_bucket_row,
// k2_round_events) compiled as plain C++.  Random events go into a dense delta arena and, as K1 + K1b + K1e would put them,
// into per-word buckets of (element % 1024) | sign << 10 codes, shuffled inside each bucket.  Every round of every chunk is
// then built in K2's order -- 32 lanes striding its bucket range, the first `cap` entries from a copy of the 16-B units the
// fetch stage stages, the rest straight from the buckets -- and compared with the same 32 rows cut from the arena.  Each event
// must land in exactly one round.  Chunks sparse and dense (thresholds 0, 160, 257), rounds that share a word with their
// neighbours, many events on one position, events on word and chunk edges, and stages of 1024, 64 and 8 entries.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include "cmb_k2_slots.cuh"

namespace {
constexpr uint32_t SPAN = 32, CHUNK_SPANS = 256, CHUNK = SPAN * CHUNK_SPANS, WORD = 1024;

struct Case {
  uint32_t n_chunks = 0;
  std::vector<int32_t> delta;
  std::vector<uint32_t> bits, count, wo;
  std::vector<uint16_t> buckets;
  uint64_t n_events = 0;
};

// kind: 0 uniform, 1 a few spans with many events, 2 word and chunk edges, 3 every span of a chunk, 4 thousands of events on
// a few positions
Case make_case(std::mt19937& rng, uint32_t kind) {
  Case c;
  c.n_chunks = 1 + rng() % 4;
  const uint64_t elems = (uint64_t)c.n_chunks * CHUNK;
  c.delta.assign(elems, 0);
  c.bits.assign(c.n_chunks * 8, 0);
  c.count.assign(c.n_chunks * 8, 0);
  std::vector<std::pair<uint32_t, uint16_t>> ev;  // (word, code)
  auto event = [&](uint64_t e) {
    const bool minus = rng() % 2;
    c.delta[e] += minus ? -1 : 1;
    c.bits[e / WORD] |= 1u << ((e / SPAN) % 32);
    c.count[e / WORD] += 1;
    ev.emplace_back((uint32_t)(e / WORD), (uint16_t)((e % WORD) | (uint32_t)minus << 10));
  };
  const uint32_t n = rng() % 3 == 0 ? rng() % 40 : rng() % 3000;
  std::vector<uint64_t> hot;
  for (uint32_t i = 0; i < 1 + rng() % 6; ++i) hot.push_back(rng() % elems);
  for (uint32_t i = 0; i < n; ++i) {
    switch (kind) {
      case 0: event(rng() % elems); break;
      case 1: event(hot[rng() % hot.size()] / SPAN * SPAN + rng() % SPAN); break;
      case 2: {
        const uint64_t w = rng() % (elems / WORD);
        const uint32_t at[] = {0, 31, 32, 33, 991, 992, 1023};
        const uint64_t e = rng() % 4 == 0 ? (rng() % c.n_chunks) * (uint64_t)CHUNK + (rng() % 2 ? CHUNK - 1 : 0) : w * WORD + at[rng() % 7];
        event(e);
        break;
      }
      case 3: {
        const uint64_t k = rng() % c.n_chunks;
        for (uint32_t s = 0; s < CHUNK_SPANS; s += 1 + rng() % 2) event(k * CHUNK + s * SPAN + rng() % SPAN);
        i += CHUNK_SPANS;
        break;
      }
      default: event(hot[rng() % 2 % hot.size()]); break;
    }
  }
  c.n_events = ev.size();
  c.wo.assign(c.count.size() + 1, 0);
  for (size_t w = 0; w < c.count.size(); ++w) c.wo[w + 1] = c.wo[w] + c.count[w];
  c.buckets.assign(c.n_events + 8, 0xffff);  // K2 may stage up to 8 entries past the last event
  std::vector<uint32_t> fill(c.count.size(), 0);
  for (const auto& x : ev) c.buckets[c.wo[x.first] + fill[x.first]++] = x.second;
  for (size_t w = 0; w < c.count.size(); ++w) std::shuffle(c.buckets.begin() + c.wo[w], c.buckets.begin() + c.wo[w + 1], rng);
  return c;
}

// Builds every round of every chunk as K2 does and compares it with the arena; returns false on the first difference.
bool check(const Case& c, uint32_t dense_spans, uint32_t cap, uint32_t* shared_words) {
  uint64_t added = 0;
  for (uint32_t k = 0; k < c.n_chunks; ++k) {
    uint32_t w[8];
    uint32_t pop = 0;
    for (uint32_t q = 0; q < 8; ++q) pop += k2_popc(w[q] = c.bits[k * 8 + q]);
    const bool dense = pop >= dense_spans;
    const uint32_t nslots = dense ? CHUNK_SPANS : pop, nr = dense ? CHUNK_SPANS / 32 : (pop + 31) / 32;
    const uint32_t* wo = c.wo.data() + k * 8;
    uint32_t prev_wl = 99;
    for (uint32_t r = 0; r < nr; ++r) {
      uint32_t wf, wl;
      k2_round_words(w, nslots, dense, r, wf, wl);
      if (wf == prev_wl) ++*shared_words;
      prev_wl = wl;
      // the fetch stage: 16-B units from the one holding the first entry, at most cap entries
      const uint32_t b0 = wo[wf], b1 = wo[wl + 1], base = b0 & ~7u, units = std::min((b1 - base + 7) / 8, cap / 8);
      std::vector<uint16_t> stage(c.buckets.begin() + base, c.buckets.begin() + base + units * 8);
      int32_t rows[32][32] = {};
      for (uint32_t lane = 0; lane < 32; ++lane)
        k2_round_events(
            w, wo, dense, r, wf, wl, lane, 32,
            [&](uint32_t p) { return p - base < cap ? (uint32_t)stage.at(p - base) : (uint32_t)c.buckets.at(p); },
            [&](uint32_t row, uint32_t e, int d) {
              rows[row][e] += d;
              ++added;
            });
      for (uint32_t i = 0; i < 32; ++i) {
        const uint32_t j = r * 32 + i;
        const uint32_t sp = j < nslots ? k2_slot_span(w, j, dense) : CHUNK_SPANS;
        for (uint32_t e = 0; e < 32; ++e) {
          const int32_t want = sp < CHUNK_SPANS ? c.delta[(uint64_t)k * CHUNK + sp * SPAN + e] : 0;
          if (rows[i][e] != want) {
            printf("chunk %u round %u row %u pos %u: %d, arena %d (dense %d, cap %u)\n", k, r, i, e, rows[i][e], want, (int)dense, cap);
            return false;
          }
        }
      }
    }
  }
  if (added != c.n_events) {
    printf("%llu events added, %llu in the buckets\n", (unsigned long long)added, (unsigned long long)c.n_events);
    return false;
  }
  return true;
}
}  // namespace

int main() {
  std::mt19937 rng(20261016);
  uint32_t tests = 0, fails = 0, shared_words = 0, overflows = 0;
  const uint32_t thresholds[] = {0, 160, 257}, caps[] = {1024, 64, 8};
  for (uint32_t it = 0; it < 200; ++it) {
    const Case c = make_case(rng, it % 5);
    for (uint32_t t : thresholds)
      for (uint32_t cap : caps) {
        ++tests;
        if (!check(c, t, cap, &shared_words)) ++fails;
      }
    for (size_t w = 0; w + 1 < c.wo.size(); ++w) overflows += c.wo[w + 1] - c.wo[w] > 1024;
  }
  printf("%u tests, %u fails (%u rounds sharing a word with the previous one, %u words over 1024 events)\n", tests, fails,
         shared_words, overflows);
  return fails ? 1 : 0;
}
