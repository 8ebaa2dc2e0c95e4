// K2's slot arithmetic (coverm_b200/csrc/cmb_k2_slots.cuh) compiled as plain C++, walked over random arenas in the kernel's
// order -- chunks, rounds of 32 slots, the depth carried between rounds, the chunk's head stretch -- and compared against a
// per-position prefix sum: covered_full, covered_window, sum_depth_window, every histogram bin and the highest bin.
// Dense thresholds 0 (every chunk whole), 160 and 257 (never whole).
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include "cmb_k2_slots.cuh"

namespace {
constexpr uint32_t SPAN = 32, CHUNK_SPANS = 256, CHUNK = SPAN * CHUNK_SPANS;
const uint32_t EDGE_LENS[] = {1, 31, 32, 33, 1023, 1024, 1025, 8191, 8192, 8193, 3 * 8192 + 5};

struct Stats {
  uint64_t cov_full = 0, cov_win = 0, sum_win = 0;
  uint32_t hi = 0;
  std::vector<uint64_t> bins;  // depth 1.. (index = depth)
  bool operator==(const Stats& o) const {
    return cov_full == o.cov_full && cov_win == o.cov_win && sum_win == o.sum_win && hi == o.hi && bins == o.bins;
  }
};

struct Arena {
  std::vector<uint32_t> len, off_span, chunk_first;
  std::vector<int32_t> delta, carry_in;
  std::vector<uint32_t> bits;  // 8 words per chunk
  uint32_t n_chunks = 0, E = 0;
};

Arena make_arena(std::mt19937& rng, bool edge) {
  Arena a;
  const uint32_t n = 1 + rng() % 12;
  uint32_t spans = 0;
  for (uint32_t i = 0; i < n; ++i) {
    uint32_t L;
    if (edge || rng() % 2) L = EDGE_LENS[rng() % 11];
    else L = 1 + rng() % 40000;
    a.len.push_back(L);
    a.off_span.push_back(spans);
    spans += std::max<uint32_t>(1, (L + SPAN - 1) / SPAN);
  }
  a.off_span.push_back(spans);
  a.n_chunks = std::max<uint32_t>(1, (spans + CHUNK_SPANS - 1) / CHUNK_SPANS);
  a.delta.assign((size_t)a.n_chunks * CHUNK, 0);
  a.bits.assign((size_t)a.n_chunks * 8, 0);
  auto event = [&](uint32_t c, uint32_t pos, int d) {  // as K1 adds one: its span's bit is set even if deltas cancel
    const uint64_t e = (uint64_t)a.off_span[c] * SPAN + pos;
    a.delta[e] += d;
    a.bits[e / 1024] |= 1u << ((e / SPAN) % 32);
  };
  for (uint32_t c = 0; c < n; ++c) {
    const uint32_t L = a.len[c];
    const uint32_t reads = rng() % 4 == 0 ? 0 : rng() % (2 + L / (50 + rng() % 2000));
    const uint32_t maxlen = 1 + (rng() % 3 == 0 ? 20000 : 300);
    for (uint32_t r = 0; r < reads; ++r) {
      const uint32_t s = rng() % L, e = s + 1 + rng() % maxlen;
      event(c, s, +1);
      if (e < L) event(c, e, -1);
    }
  }
  a.E = rng() % 3 == 0 ? 0 : (rng() % 2 ? rng() % 100 : rng() % 9000);
  // chunk_first and carry_in as cmb_set_reference and K1b make them
  a.chunk_first.resize(a.n_chunks + 1);
  a.carry_in.assign(a.n_chunks, 0);
  uint32_t ci = 0;
  for (uint32_t k = 0; k < a.n_chunks; ++k) {
    while (ci + 1 < n && a.off_span[ci + 1] <= k * CHUNK_SPANS) ++ci;
    a.chunk_first[k] = ci;
    if (a.off_span[ci] < k * CHUNK_SPANS) {
      int d = 0;
      for (uint64_t e = (uint64_t)a.off_span[ci] * SPAN; e < (uint64_t)k * CHUNK; ++e) d += a.delta[e];
      a.carry_in[k] = d;
    }
  }
  a.chunk_first[a.n_chunks] = n - 1;
  return a;
}

std::vector<Stats> reference(const Arena& a) {
  std::vector<Stats> out(a.len.size());
  for (size_t c = 0; c < a.len.size(); ++c) {
    const uint32_t L = a.len[c];
    const K2Win w = k2_window(L, a.E);
    Stats& s = out[c];
    int d = 0;
    for (uint32_t p = 0; p < L; ++p) {
      d += a.delta[(uint64_t)a.off_span[c] * SPAN + p];
      if (d > 0) ++s.cov_full;
      if (p >= w.w0 && p < w.w1) {
        s.sum_win += (uint64_t)(int64_t)d;
        if (d > 0) {
          ++s.cov_win;
          if (s.bins.size() <= (size_t)d) s.bins.resize(d + 1, 0);
          ++s.bins[d];
          s.hi = std::max<uint32_t>(s.hi, d);
        }
      }
    }
  }
  return out;
}

// The kernel's walk: what every lane of every round computes, with the warp scans written out.
std::vector<Stats> model(const Arena& a, uint32_t dense_spans) {
  std::vector<Stats> out(a.len.size());
  auto hist = [&](uint32_t c, int d, uint32_t n) {
    Stats& s = out[c];
    if (s.bins.size() <= (size_t)d) s.bins.resize(d + 1, 0);
    s.bins[d] += n;
    s.hi = std::max<uint32_t>(s.hi, d);
  };
  auto add = [&](uint32_t c, const K2Acc& acc) {
    out[c].cov_full += acc.cov_full;
    out[c].cov_win += acc.cov_win;
    out[c].sum_win += acc.sum_win;
  };
  for (uint32_t k = 0; k < a.n_chunks; ++k) {
    uint32_t w[8];
    uint32_t pop = 0;
    for (uint32_t q = 0; q < 8; ++q) pop += k2_popc(w[q] = a.bits[k * 8 + q]);
    const bool dense = pop >= dense_spans;
    const uint32_t nslots = dense ? CHUNK_SPANS : pop, nr = dense ? 8 : (pop + 31) / 32;
    const uint32_t cf = a.chunk_first[k], cl = a.chunk_first[k + 1], span0 = k * CHUNK_SPANS;
    const int cin = a.carry_in[k];
    uint32_t pc = cf, c_first = UINT32_MAX;
    int pd = cin;
    for (uint32_t r = 0; r < nr; ++r) {
      uint32_t c[32], s[32], sn[32];
      int total[32];
      uint32_t ev[32];
      for (uint32_t l = 0; l < 32; ++l) {
        const uint32_t j = r * 32 + l;
        s[l] = k2_slot_span(w, j, dense);
        sn[l] = k2_slot_span(w, j + 1, dense);
        c[l] = UINT32_MAX;
        total[l] = 0;
        ev[l] = 0;
        if (j >= nslots) continue;
        if (s[l] >= CHUNK_SPANS || sn[l] <= s[l] || sn[l] > CHUNK_SPANS) {
          printf("bad slot span %u -> %u\n", s[l], sn[l]);
          exit(1);
        }
        uint32_t lo = cf, hi = cl;
        while (lo < hi) {
          const uint32_t mid = (lo + hi + 1) >> 1;
          if (a.off_span[mid] <= span0 + s[l]) lo = mid;
          else hi = mid - 1;
        }
        c[l] = lo;
        for (uint32_t e = 0; e < 32; ++e) {
          const int d = a.delta[(uint64_t)(span0 + s[l]) * SPAN + e];
          total[l] += d;
          if (d) ev[l] |= 1u << e;
        }
      }
      int out_depth[32];
      for (uint32_t l = 0; l < 32; ++l) {
        int incl = total[l];  // the segmented inclusive scan: lanes before l in the same contig
        for (uint32_t m = l; m-- > 0 && c[m] == c[l];) incl += total[m];
        const int depth = incl - total[l] + (c[l] == pc ? pd : 0);
        out_depth[l] = 0;
        if (r * 32 + l >= nslots) continue;
        const uint32_t cstart = a.off_span[c[l]];
        const uint32_t rel = (span0 + s[l] - cstart) * SPAN;
        const uint32_t from = r == 0 && l == 0 && c[l] == cf ? (span0 - cstart) * SPAN : rel;
        const uint32_t to = rel + (sn[l] - s[l]) * SPAN;
        const K2Win win = k2_window(a.len[c[l]], a.E);
        K2Acc acc{0, 0, 0};
        const uint32_t cc = c[l];
        const uint64_t base = (uint64_t)(span0 + s[l]) * SPAN;
        out_depth[l] = k2_slot_runs(
            acc, win, depth, ev[l], rel, from, to, [&](uint32_t e) { return a.delta[base + e]; },
            [&](int d, uint32_t n) {
              if (d < 0) {
                printf("negative depth\n");
                exit(1);
              }
              hist(cc, d, n);
            });
        add(cc, acc);
      }
      pc = c[31];
      pd = out_depth[31];
      if (r == 0) c_first = c[0];
    }
    if (cin != 0 && c_first != cf) {
      const uint32_t cstart = a.off_span[cf];
      const K2Win win = k2_window(a.len[cf], a.E);
      const uint32_t s0 = k2_slot_span(w, 0, dense);
      K2Acc acc{0, 0, 0};
      const uint32_t nw = k2_close_run(acc, win, cin, (span0 - cstart) * SPAN, (span0 + s0 - cstart) * SPAN);
      if (nw) hist(cf, cin, nw);
      add(cf, acc);
    }
  }
  for (Stats& s : out)  // the reference only sizes bins up to the highest depth seen
    if (!s.bins.empty()) s.bins.resize(s.hi + 1);
  return out;
}

bool nth_bit_ok(std::mt19937& rng) {
  for (int t = 0; t < 20000; ++t) {
    uint32_t x = rng();
    if (t % 3 == 0) x &= rng();
    if (t % 7 == 0) x = 1u << (t % 32);
    if (!x) continue;
    uint32_t n = 0;
    for (uint32_t b = 0; b < 32; ++b)
      if ((x >> b) & 1u) {
        if (k2_nth_bit(x, n) != b) return false;
        ++n;
      }
  }
  return true;
}
}  // namespace

int main() {
  std::mt19937 rng(1234);
  int tests = 0, fails = 0;
  if (!nth_bit_ok(rng)) {
    printf("k2_nth_bit wrong\n");
    ++fails;
  }
  for (int it = 0; it < 600; ++it) {
    const Arena a = make_arena(rng, it % 4 == 0);
    const std::vector<Stats> want = reference(a);
    for (uint32_t dense : {0u, 160u, 257u}) {
      ++tests;
      const std::vector<Stats> got = model(a, dense);
      for (size_t c = 0; c < want.size(); ++c)
        if (!(got[c] == want[c])) {
          printf("arena %d dense %u contig %zu (L=%u E=%u): cov_full %llu/%llu cov_win %llu/%llu sum %llu/%llu hi %u/%u\n", it, dense,
                 c, a.len[c], a.E, (unsigned long long)got[c].cov_full, (unsigned long long)want[c].cov_full,
                 (unsigned long long)got[c].cov_win, (unsigned long long)want[c].cov_win, (unsigned long long)got[c].sum_win,
                 (unsigned long long)want[c].sum_win, got[c].hi, want[c].hi);
          ++fails;
          break;
        }
    }
  }
  printf("%d tests, %d fails\n", tests, fails);
  return fails != 0;
}
