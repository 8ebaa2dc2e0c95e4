// The block slices a sliced device decode walks: a shard of sharded input (cmb_shard_add), or an ordinary stream whose whole
// decode does not fit (cmb_submit_bgzf).  Host-only, so that tests can check the plan natively.
//
// A slice decodes the records that START in blocks [b0, b1).  Its device footprint is what a ranged decode uploads and inflates:
// the compressed bytes of blocks [b0, data_end) and their inflated bytes, where data_end extends b1 by the following blocks that
// hold at least `tail` inflated bytes (the bytes of a record straddling out of the slice).  BgzfCall::prepare computes the same.
#pragma once
#include <cstdint>
#include <utility>
#include <vector>

struct ShardBlocks {
  uint32_t nb;                // blocks in the file
  uint64_t size;              // file bytes
  const uint64_t* coffset;    // per block: offset of its deflate payload
  const uint32_t* clen;       // payload length (the 8-byte footer follows it)
  const uint64_t* ustart;     // [nb + 1]: offset of every block in the inflated stream
};

// First block past the tail of a slice ending at b1
inline uint32_t slice_data_end(const ShardBlocks& f, uint32_t b1, uint64_t tail) {
  uint32_t e = b1;
  while (e < f.nb && f.ustart[e] - f.ustart[b1] < tail) ++e;
  return e;
}

// Device bytes of the slice [b0, b1): compressed plus inflated, tail included
inline uint64_t slice_bytes(const ShardBlocks& f, uint32_t b0, uint32_t b1, uint64_t tail) {
  const uint32_t e = slice_data_end(f, b1, tail);
  const uint64_t byte_hi = e == f.nb ? f.size : f.coffset[e - 1] + f.clen[e - 1] + 8;
  return (byte_hi - f.coffset[b0]) + (f.ustart[e] - f.ustart[b0]);
}

// The end of the longest slice from b0 whose bytes fit `budget`; b0 + 1 with *over set when even one block does not fit.
inline uint32_t slice_end(const ShardBlocks& f, uint32_t b0, uint64_t budget, uint64_t tail, bool* over) {
  *over = slice_bytes(f, b0, b0 + 1, tail) > budget;
  if (*over) return b0 + 1;
  uint32_t lo = b0 + 1, hi = f.nb;  // slice_bytes grows with b1: the last b1 that fits, by bisection
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo + 1) / 2;
    if (slice_bytes(f, b0, mid, tail) <= budget) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// The slices of blocks [first, nb) under a fixed budget, in order; *n_over counts the slices of one block that exceed it.  For
// tests only: the device loop (decode_in_slices) calls slice_end itself, with a budget recomputed before every slice, each slice
// starting at the block that holds the previous slice's exit offset (past the planned end when a record spans whole blocks),
// its end lowered when its buffers fail to allocate and its tail doubled for a long record.
inline std::vector<std::pair<uint32_t, uint32_t>> plan_slices(const ShardBlocks& f, uint32_t first, uint64_t budget, uint64_t tail,
                                                              uint32_t* n_over) {
  std::vector<std::pair<uint32_t, uint32_t>> out;
  *n_over = 0;
  for (uint32_t b0 = first; b0 < f.nb;) {
    bool over = false;
    const uint32_t b1 = slice_end(f, b0, budget, tail, &over);
    *n_over += over;
    out.emplace_back(b0, b1);
    b0 = b1;
  }
  return out;
}
