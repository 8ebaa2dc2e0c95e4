// K2's per-slot arithmetic as plain integer code, shared by k2_scan_reduce and tests/native/k2_slots_check.cpp (which
// compiles it with g++ and walks random arenas in the kernel's order against a per-position prefix sum), and the building of
// a round's rows from word buckets, shared with tests/native/k2_buckets_check.cpp (against rows cut from a dense arena).
//
// A chunk's slots are all 256 of its spans when it is dense, else only its occupied spans, in order.  Slot j covers the
// positions from its span's start up to the next slot's span (the chunk's end for the last slot): past the span's last
// event the depth stays constant, so the event-free spans after a slot are counted with the slot's last run.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define K2_HD __host__ __device__ __forceinline__
#else
#define K2_HD inline
#endif

constexpr uint32_t K2_CHUNK_SPANS = 256;  // spans per chunk = 8 bitmap words of 32

K2_HD uint32_t k2_popc(uint32_t x) {
#ifdef __CUDA_ARCH__
  return __popc(x);
#else
  return (uint32_t)__builtin_popcount(x);
#endif
}

K2_HD uint32_t k2_low_bit(uint32_t x) {  // x != 0
#ifdef __CUDA_ARCH__
  return (uint32_t)__ffs((int)x) - 1u;
#else
  return (uint32_t)__builtin_ctz(x);
#endif
}

// Position of the n-th (from 0) set bit of x; n < popcount(x).  Five halving steps, the same code on host and device.
K2_HD uint32_t k2_nth_bit(uint32_t x, uint32_t n) {
  uint32_t pos = 0;
#pragma unroll
  for (uint32_t w = 16; w; w >>= 1) {
    const uint32_t lo = k2_popc(x & ((1u << w) - 1u));
    if (n >= lo) {
      n -= lo;
      x >>= w;
      pos += w;
    }
  }
  return pos;
}

// Span (0..255) of slot j of a chunk with bitmap words w[0..7]; K2_CHUNK_SPANS when there is no slot j.
K2_HD uint32_t k2_slot_span(const uint32_t (&w)[8], uint32_t j, bool dense) {
  if (dense) return j < K2_CHUNK_SPANS ? j : K2_CHUNK_SPANS;
  uint32_t base = 0, word = 0, rem = j;
  bool found = false;
#pragma unroll
  for (uint32_t q = 0; q < 8; ++q) {
    const uint32_t p = k2_popc(w[q]);
    if (!found) {
      if (rem < p) {
        found = true;
        base = 32 * q;
        word = w[q];
      } else {
        rem -= p;
      }
    }
  }
  return found ? base + k2_nth_bit(word, rem) : K2_CHUNK_SPANS;
}

// ---- A chunk's slot -> span table, built once when K2 enters the chunk so that its rounds read spans instead of counting
// bits: span[j] = k2_slot_span(w, j, dense) for j < nslots, and pre[q] = the slots of the words before word q (32 q when
// dense).  Lane `lane` (0..31) writes the slots of byte lane % 4 of word q = lane / 4: `word` is w[q] (all ones when the
// chunk is dense) and `before` is pre[q].
K2_HD void k2_span_table_lane(uint32_t word, uint32_t before, uint32_t lane, uint8_t* span) {
  const uint32_t q = lane / 4, sh = (lane % 4) * 8;
  uint32_t m = (word >> sh) & 255u, j = before + k2_popc(word & ((1u << sh) - 1u));
  while (m) {
    span[j++] = (uint8_t)(32 * q + sh + k2_low_bit(m));
    m &= m - 1;
  }
}

// ---- A round's rows from word buckets (contig mode).  K1e puts each event of bitmap word q of a chunk into the word's bucket
// as the u16 code (element % 1024) | sign << 10 (sign 1: the -1 at a block's end); the bucket of word q is the entries
// [wo[q], wo[q + 1]).  Row i of round r is slot 32 r + i: span 32 r + i of a dense chunk, else the (32 r + i)-th occupied span.

// The first and last bitmap word (0..7) that round r's slots lie in, of a chunk with nslots slots (nslots > 32 r)
K2_HD void k2_round_words(const uint32_t (&w)[8], uint32_t nslots, bool dense, uint32_t r, uint32_t& wf, uint32_t& wl) {
  const uint32_t j1 = r * 32 + 31 < nslots ? r * 32 + 31 : nslots - 1;
  wf = k2_slot_span(w, r * 32, dense) / 32;
  wl = k2_slot_span(w, j1, dense) / 32;
}
// The same from the chunk's slot -> span table
K2_HD void k2_round_words(const uint8_t* span, uint32_t nslots, uint32_t r, uint32_t& wf, uint32_t& wl) {
  const uint32_t j1 = r * 32 + 31 < nslots ? r * 32 + 31 : nslots - 1;
  wf = span[r * 32] / 32u;
  wl = span[j1] / 32u;
}

// Row of round r for an event of word q with code `code`, `before` the slots of the words before q: its span's slot minus
// 32 r, 32 or more when the slot is another round's (a word the round shares with its neighbours)
K2_HD uint32_t k2_bucket_row(const uint32_t (&w)[8], bool dense, uint32_t r, uint32_t q, uint32_t before, uint32_t code) {
  const uint32_t b = (code & 1023u) / 32u;  // span within word q
  if (dense) return q * 32 + b - r * 32;
  return before + k2_popc(w[q] & ((1u << b) - 1u)) - r * 32;  // wraps past 32 for an earlier round's slot
}

// The events of round r, whose slots lie in words wf..wl: bucket entries p = wo[wf] + p0, + step, ... below wo[wl + 1]
// (K2: p0 = lane, step = 32).  code(p) reads entry p; add(row, e, delta) is called for each event of the round's slots, e
// its position in the span.  pre[q] is the slots of the words before word q (the chunk's table, k2_span_table_lane).
template <class Code, class Add>
K2_HD void k2_round_events(const uint32_t (&w)[8], const uint8_t* pre, const uint32_t* wo, bool dense, uint32_t r, uint32_t wf,
                           uint32_t wl, uint32_t p0, uint32_t step, Code code, Add add) {
  uint32_t q = wf, before = pre[wf];  // the word of entry p and the slots of the words before it
  const uint32_t p1 = wo[wl + 1];
  for (uint32_t p = wo[wf] + p0; p < p1; p += step) {
    while (q < wl && wo[q + 1] <= p) before = pre[++q];
    const uint32_t c = code(p);
    const uint32_t row = k2_bucket_row(w, dense, r, q, before, c);
    if (row < 32) add(row, c & 31u, (c >> 10) & 1u ? -1 : 1);
  }
}
// The same with pre[] counted from the bitmap words
template <class Code, class Add>
K2_HD void k2_round_events(const uint32_t (&w)[8], const uint32_t* wo, bool dense, uint32_t r, uint32_t wf, uint32_t wl,
                           uint32_t p0, uint32_t step, Code code, Add add) {
  uint8_t pre[8];
  for (uint32_t q = 0, before = 0; q < 8; before += k2_popc(w[q++])) pre[q] = (uint8_t)before;
  k2_round_events(w, pre, wo, dense, r, wf, wl, p0, step, code, add);
}

// A contig's length and its end-trimmed window [w0, w1) (empty when 2E >= L), in contig coordinates.
struct K2Win {
  uint32_t L, w0, w1;
};
K2_HD K2Win k2_window(uint32_t L, uint32_t E) {
  K2Win w{L, 0u, 0u};
  if (2ull * E < L) {
    w.w0 = E;
    w.w1 = L - E;
  }
  return w;
}

// What a contig gains from its runs (EST:393-404, 447-465, 494-501).
struct K2Acc {
  uint32_t cov_full, cov_win;
  uint64_t sum_win;
};

// The run [from, to) at `depth`, clipped to [0, L) and to the window; returns its window positions (its histogram count).
K2_HD uint32_t k2_close_run(K2Acc& a, const K2Win& w, int depth, uint32_t from, uint32_t to) {
  const uint32_t nc = (to < w.L ? to : w.L) - (from < w.L ? from : w.L);
  const uint32_t t1 = to < w.w0 ? w.w0 : (to > w.w1 ? w.w1 : to), f1 = from < w.w0 ? w.w0 : (from > w.w1 ? w.w1 : from);
  const uint32_t nw = t1 - f1;
  if (depth > 0) {
    a.cov_full += nc;
    a.cov_win += nw;
  }
  a.sum_win += (uint64_t)(int64_t)depth * nw;
  return nw;
}

// The runs of one slot: `from` .. `to` in contig coordinates, `rel` the position of its span's first element, `ev` the
// positions of that span with a delta (delta(j) reads it), `depth` the depth entering the slot.  hist(depth, n) is called
// for every run at a depth other than 0 with n > 0 window positions.  Returns the depth leaving the slot.
template <class Delta, class Hist>
K2_HD int k2_slot_runs(K2Acc& a, const K2Win& w, int depth, uint32_t ev, uint32_t rel, uint32_t from, uint32_t to, Delta delta,
                       Hist hist) {
  while (ev) {
    const uint32_t j = k2_low_bit(ev);
    ev &= ev - 1;
    const uint32_t nw = k2_close_run(a, w, depth, from, rel + j);
    if (nw && depth != 0) hist(depth, nw);
    depth += delta(j);
    from = rel + j;
  }
  const uint32_t nw = k2_close_run(a, w, depth, from, to);
  if (nw && depth != 0) hist(depth, nw);
  return depth;
}
