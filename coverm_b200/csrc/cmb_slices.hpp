// The block slices of a sliced device decode: a shard of sharded input (cmb_shard_add), or an ordinary stream whose whole
// decode does not fit (cmb_submit_bgzf).  The slice plan, and for the ordinary stream the budget of the next slice and the
// pair-mode cut.  Plain C++ outside nvcc, so that tests can check them natively.
//
// A slice decodes the records that START in blocks [b0, b1).  Its device footprint is what a ranged decode uploads and inflates:
// the compressed bytes of blocks [b0, data_end) and their inflated bytes, where data_end extends b1 by the following blocks that
// hold at least `tail` inflated bytes (the bytes of a record straddling out of the slice).  BgzfCall::prepare computes the same.
#pragma once
#include <cstdint>
#include <utility>
#include <vector>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

// The block table of a sliced decode
struct SliceBlocks {
  uint32_t nb;                // blocks in the file
  uint64_t size;              // file bytes
  const uint64_t* coffset;    // per block: offset of its deflate payload
  const uint32_t* clen;       // payload length (the 8-byte footer follows it)
  const uint64_t* ustart;     // [nb + 1]: offset of every block in the inflated stream
};

// First block past the tail of a slice ending at b1
inline uint32_t slice_data_end(const SliceBlocks& f, uint32_t b1, uint64_t tail) {
  uint32_t e = b1;
  while (e < f.nb && f.ustart[e] - f.ustart[b1] < tail) ++e;
  return e;
}

// Device bytes of the slice [b0, b1): compressed plus inflated, tail included
inline uint64_t slice_bytes(const SliceBlocks& f, uint32_t b0, uint32_t b1, uint64_t tail) {
  const uint32_t e = slice_data_end(f, b1, tail);
  const uint64_t byte_hi = e == f.nb ? f.size : f.coffset[e - 1] + f.clen[e - 1] + 8;
  return (byte_hi - f.coffset[b0]) + (f.ustart[e] - f.ustart[b0]);
}

// The end of the longest slice from b0 whose bytes fit `budget`; b0 + 1 with *over set when even one block does not fit.
inline uint32_t slice_end(const SliceBlocks& f, uint32_t b0, uint64_t budget, uint64_t tail, bool* over) {
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
inline std::vector<std::pair<uint32_t, uint32_t>> plan_slices(const SliceBlocks& f, uint32_t first, uint64_t budget, uint64_t tail,
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

// ---- the ordinary stream (decode_sliced)

// Device bytes of the sample's event list per interval (aligned block): two u64 events, allocated with 1/8 slack
constexpr uint64_t SLICE_EVENT_BYTES = 18;

// Compressed plus inflated bytes (slice_bytes) the next slice may take.
//   room         bytes for the decode buffers and the sample's event list: free device memory plus the decode buffers held
//   events       whether K1 appends to the event list (contig mode)
//   events_held  bytes the event list holds now (not part of `room`)
//   done, total  inflated bytes of the stream walked by the slices so far / to walk in all
//   iv_done      intervals those slices submitted
//   side         bytes a slice needed beside its compressed and inflated bytes (tuples, record offsets, mate matching), per
//                byte of them, as the last slice measured
// The reserve is the event list's growth: at its last growth Buf::grow_keep holds the old and the new list together, so the
// sample still needs up to twice the final list, less what it holds.  The first slice has no estimate and takes half the room.
inline uint64_t decode_slice_budget(uint64_t room, bool events, uint64_t events_held, uint64_t done, uint64_t total, uint64_t iv_done,
                                    double side) {
  if (done == 0 || done >= total) return room / 2;
  uint64_t reserve = 0;
  if (events) {
    const double final_list = (double)SLICE_EVENT_BYTES * (double)iv_done * ((double)total / (double)done);
    reserve = 2 * final_list > (double)events_held ? (uint64_t)(2 * final_list) - events_held : 0;
  }
  if (room <= reserve) return 0;
  return (uint64_t)((double)(room - reserve) / (1.0 + (side > 0 ? side : 0)));
}

// Pair mode: a slice that does not reach the end of the stream submits only the records before the trailing run of its last
// eligible tid `last` (mate matching's eligibility and unsigned tid order, cmb_pairs.cuh), so that every tid's eligible
// records are matched within one slice.  The run starts at the first eligible record of tid `last` after every eligible
// record of another tid.  Over the slice's records i:
//   after = max of pair_cut_after(...)      one past the last eligible record of another tid (0: none)
//   cut   = min of pair_cut_at(..., after)  the run's first record (n: no eligible record of `last`, so nothing to hold back)
// The next slice starts at record `cut`.  cut == 0 means the run is the whole slice: it cannot be split, and the sample declines.
__host__ __device__ inline uint32_t pair_cut_after(bool eligible, uint32_t tid, uint32_t last, uint32_t i) {
  return eligible && tid != last ? i + 1 : 0;
}
__host__ __device__ inline uint32_t pair_cut_at(bool eligible, uint32_t tid, uint32_t last, uint32_t after, uint32_t i, uint32_t n) {
  return eligible && tid == last && i >= after ? i : n;
}

// The eligible tids of a slice are in order (kd_pair_order / kd_pair_order_fold) when none is below the largest eligible tid
// before it, the earlier slices' largest (`carry`, 0 for none) included.
__host__ __device__ inline bool pair_order_drop(uint32_t tid, uint32_t largest_before) { return tid < largest_before; }
