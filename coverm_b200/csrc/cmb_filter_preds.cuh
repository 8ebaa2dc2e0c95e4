// The read-filter predicates of ReferenceSortedBamFilter over a record's decoded columns, shared by K1 (cmb_k1.cuh) and
// `coverm filter` (cmb_filter.cuh), and compiled as plain C++ by tests/native/pairs_check.cpp (which shims the rounding
// intrinsics as IEEE float operations).
#pragma once

struct RecView {
  uint32_t flag, mapq, nm_state, nm, l_seq, aligned, del;
};

// filter.rs:243-279.  Sets *nm_err when the reference would reach nm() on a record without a usable NM tag.
__device__ __forceinline__ bool single_read_passes(const RecView& r, const cmb_params& p, bool* nm_err) {
  if (p.min_mapq != 255 && (r.mapq < p.min_mapq || r.mapq == 255)) return false;
  if (r.nm_state != 1) *nm_err = true;
  const float aligned_f = __uint2float_rn(r.aligned);
  return r.aligned >= p.min_aligned_length_single &&
         __fdiv_rn(aligned_f, __uint2float_rn(r.l_seq)) >= p.min_aligned_percent_single &&
         __fsub_rn(1.0f, __fdiv_rn(__uint2float_rn(r.nm), aligned_f)) >= p.min_percent_identity_single;
}
// filter.rs:281-336 (D is not part of the pair aligned length).
__device__ __forceinline__ bool read_pair_passes(const RecView& a, const RecView& b, const cmb_params& p, bool* nm_err) {
  if (p.min_mapq != 255 && (a.mapq < p.min_mapq || b.mapq < p.min_mapq || a.mapq == 255 || b.mapq == 255)) return false;
  if (a.nm_state != 1 || b.nm_state != 1) *nm_err = true;
  const uint32_t aligned = (a.aligned - a.del) + (b.aligned - b.del);
  const float aligned_f = __uint2float_rn(aligned);
  const float seq_f = __ull2float_rn((unsigned long long)a.l_seq + (unsigned long long)b.l_seq);
  const float edit_f = __ull2float_rn((unsigned long long)a.nm + (unsigned long long)b.nm);
  return aligned >= p.min_aligned_length_pair && __fdiv_rn(aligned_f, seq_f) >= p.min_aligned_percent_pair &&
         __fsub_rn(1.0f, __fdiv_rn(edit_f, aligned_f)) >= p.min_percent_identity_pair;
}
