// The ordinary (non-sharded) device decode in block slices (cmb_submit_bgzf when the whole-stream buffers do not fit): the
// budget of the next slice, and the pair-mode cut.  Plain C++ outside nvcc, so that tests can check both natively.
#pragma once
#include <cstdint>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

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
