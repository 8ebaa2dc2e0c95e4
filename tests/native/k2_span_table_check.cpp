// K2's per-chunk slot -> span table (coverm_b200/csrc/cmb_k2_slots.cuh: k2_span_table_lane) compiled as plain C++: for random
// bitmaps -- empty, single-bit, full and sparse words, whole chunks -- the 32 lanes build the table as the kernel's warp does,
// and every entry must equal k2_slot_span.  pre[] is checked against the popcounts of the words before, the table-based
// k2_round_words against the bitmap-based one, and the pre[]-taking k2_round_events against the one that counts bits.
#include <cstdint>
#include <cstdio>
#include <random>

#include "cmb_k2_slots.cuh"

namespace {
uint32_t random_word(std::mt19937& rng) {
  switch (rng() % 6) {
    case 0: return 0u;
    case 1: return 1u << (rng() % 32);
    case 2: return ~0u;
    case 3: return rng() & rng() & rng();
    default: return rng();
  }
}

// The kernel's spread(): lanes 0..7 scan the (dense: all-ones) words, lane l builds byte l % 4 of word l / 4.
void build(const uint32_t (&w)[8], bool dense, uint8_t* span, uint8_t* pre) {
  uint32_t mw[8], before[8], acc = 0;
  for (uint32_t q = 0; q < 8; ++q) {
    mw[q] = dense ? ~0u : w[q];
    before[q] = acc;
    acc += k2_popc(mw[q]);
    pre[q] = (uint8_t)before[q];
  }
  for (uint32_t lane = 0; lane < 32; ++lane) k2_span_table_lane(mw[lane / 4], before[lane / 4], lane, span);
}
}  // namespace

int main() {
  std::mt19937 rng(20261017);
  uint32_t tests = 0, fails = 0;
  for (uint32_t it = 0; it < 20000 && fails < 10; ++it) {
    uint32_t w[8], pop = 0;
    for (uint32_t q = 0; q < 8; ++q) pop += k2_popc(w[q] = random_word(rng));
    for (bool dense : {false, true}) {
      ++tests;
      uint8_t span[K2_CHUNK_SPANS + 1], pre[8];
      for (uint8_t& s : span) s = 0xaa;
      build(w, dense, span, pre);
      const uint32_t nslots = dense ? K2_CHUNK_SPANS : pop;
      bool ok = span[K2_CHUNK_SPANS] == 0xaa;  // nothing past the table
      for (uint32_t j = 0; j < nslots; ++j) ok &= span[j] == k2_slot_span(w, j, dense);
      for (uint32_t j = nslots; j < K2_CHUNK_SPANS; ++j) ok &= span[j] == 0xaa;  // nothing past the chunk's slots
      for (uint32_t q = 0, before = 0; q < 8; before += dense ? 32 : k2_popc(w[q]), ++q) ok &= pre[q] == before;
      for (uint32_t r = 0; r * 32 < nslots; ++r) {
        uint32_t wf0, wl0, wf1, wl1;
        k2_round_words(w, nslots, dense, r, wf0, wl0);
        k2_round_words(span, nslots, r, wf1, wl1);
        ok &= wf0 == wf1 && wl0 == wl1;
        // one random entry per word (code: position in the word, sign at bit 10), through both k2_round_events
        uint32_t wo[9], codes[8];
        for (uint32_t q = 0; q < 8; ++q) {
          wo[q] = q;
          codes[q] = rng() % 2048;
        }
        wo[8] = 8;
        uint32_t got0 = 0, got1 = 0;
        for (uint32_t lane = 0; lane < 32; ++lane) {
          k2_round_events(w, wo, dense, r, wf0, wl0, lane, 32, [&](uint32_t p) { return codes[p]; },
                          [&](uint32_t row, uint32_t e, int d) { got0 = got0 * 31 + row * 64 + e * 2 + (d > 0); });
          k2_round_events(w, pre, wo, dense, r, wf1, wl1, lane, 32, [&](uint32_t p) { return codes[p]; },
                          [&](uint32_t row, uint32_t e, int d) { got1 = got1 * 31 + row * 64 + e * 2 + (d > 0); });
        }
        ok &= got0 == got1;
      }
      if (!ok) {
        printf("bitmap %08x %08x %08x %08x %08x %08x %08x %08x dense %d: table differs\n", w[0], w[1], w[2], w[3], w[4], w[5], w[6],
               w[7], (int)dense);
        ++fails;
      }
    }
  }
  printf("%u tests, %u fails\n", tests, fails);
  return fails != 0;
}
