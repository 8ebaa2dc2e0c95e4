// `coverm filter` on the device (src/bin/coverm.rs:408-472): which records ReferenceSortedBamFilter::read (filter.rs:86-234)
// returns, and in which order, for a sample that cmb_decode_bgzf left in HBM (inflated stream, record offsets, tuple columns,
// mate table).  filter_out = !--inverse.
//   singles path (filter_single_reads && !filter_pairs, filter.rs:88-116): records in file order;
//   pair path (filter.rs:117-233): unmapped records (inverse only) and improper pairs (inverse only) at their own position, a
//   passing pair as (stored first mate, second mate) at the SECOND mate's position.
// Every emitted record is given an anchor (the file position at which the reference returns it) and a rank inside the anchor;
// an exclusive scan of the bytes per anchor gives each record its place in the output, which kf_gather then fills.
#pragma once
#include "cmb_filter_preds.cuh"

struct FilterArgs {
  const uint8_t* data;
  const uint64_t* rec_off;
  uint32_t n;
  const uint16_t* flag;
  const uint8_t* mapq;
  const uint8_t* nm_state;
  const uint32_t* nm;
  const uint32_t* l_seq;
  const uint32_t* aligned;
  const uint32_t* del;
  const int32_t* mate;  // pair path: partner index or -1
  cmb_params p;
  uint8_t filter_single, pair_path, filter_out;
  unsigned long long* anchor_bytes;  // [n + 1]: bytes returned at anchor i; after kf_scan: exclusive offsets, [n] = total
  uint8_t* role;                     // [n]: 0 not returned, 1 at its own anchor, 2 as the stored first mate of mate[i]
  uint32_t* error_flags;
  unsigned long long* n_emit;
  uint8_t* out;                      // kf_gather: the returned records back to back
};

__device__ __forceinline__ RecView filter_view(const FilterArgs& a, uint32_t i) {
  RecView r;
  r.flag = a.flag[i];
  r.mapq = a.mapq[i];
  r.nm_state = a.nm_state[i];
  r.nm = a.nm[i];
  r.l_seq = a.l_seq[i];
  r.aligned = a.aligned[i];
  r.del = a.del[i];
  return r;
}

__global__ void __launch_bounds__(256) kf_decide(const FilterArgs a) {
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= a.n) return;
  const RecView r = filter_view(a, i);
  const bool unmapped = r.flag & 0x4, secondary = r.flag & 0x100, supplementary = r.flag & 0x800, proper = r.flag & 0x2;
  const unsigned long long size_i = 4ull + ldu32(a.data + a.rec_off[i]);
  uint32_t role = 0;
  unsigned long long bytes = 0;
  bool nm_err = false;
  if (!a.pair_path) {
    if (unmapped && !a.filter_out) role = 1;
    else {
      const bool passes_filter1 = !unmapped && (a.p.include_supplementary || !supplementary) && (a.p.include_secondary || !secondary);
      if (passes_filter1 && single_read_passes(r, a.p, &nm_err) == (bool)a.filter_out) role = 1;
    }
    if (role) bytes = size_i;
  } else {
    if (unmapped && !a.filter_out) {
      role = 1;
      bytes = size_i;
    } else if (secondary || supplementary) {
    } else if (!proper) {
      if (!a.filter_out) {
        role = 1;
        bytes = size_i;
      }
    } else {
      const int32_t m = a.mate[i];
      if (m >= 0) {
        const RecView o = filter_view(a, (uint32_t)m);
        const bool i_is_second = (uint32_t)m < i;
        const RecView& first = i_is_second ? o : r;
        const RecView& second = i_is_second ? r : o;
        bool ok = true;
        if (a.filter_single) ok = single_read_passes(first, a.p, &nm_err) && single_read_passes(second, a.p, &nm_err);
        if (ok) ok = read_pair_passes(second, first, a.p, &nm_err);
        if (ok == (bool)a.filter_out) {
          if (i_is_second) {
            role = 1;
            bytes = size_i + 4ull + ldu32(a.data + a.rec_off[m]);
          } else {
            role = 2;
          }
        }
      }
    }
  }
  a.role[i] = (uint8_t)role;
  a.anchor_bytes[i] = bytes;
  if (role) atomicAdd(a.n_emit, 1ull);
  if (nm_err) atomicOr(a.error_flags, ERR_NM);
}

// Exclusive scan of v[0..n) in place, v[n] = total (single CTA; n is tens of millions at most).
__global__ void __launch_bounds__(1024) kf_scan(unsigned long long* v, uint32_t n) {
  __shared__ unsigned long long s[1024];
  const uint32_t t = threadIdx.x;
  const uint32_t per = (n + 1023) / 1024;
  const uint32_t i0 = min(n, t * per), i1 = min(n, i0 + per);
  unsigned long long sum = 0;
  for (uint32_t i = i0; i < i1; ++i) sum += v[i];
  s[t] = sum;
  __syncthreads();
  for (uint32_t d = 1; d < 1024; d <<= 1) {
    const unsigned long long x = t >= d ? s[t - d] : 0;
    __syncthreads();
    s[t] += x;
    __syncthreads();
  }
  unsigned long long run = s[t] - sum;
  for (uint32_t i = i0; i < i1; ++i) {
    const unsigned long long x = v[i];
    v[i] = run;
    run += x;
  }
  if (t == 1023) v[n] = s[1023];
}

// One warp per returned record: copy it to its place.
__global__ void __launch_bounds__(256) kf_gather(const FilterArgs a) {
  const uint32_t i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= a.n) return;
  const uint32_t role = a.role[i];
  if (!role) return;
  const uint8_t* src = a.data + a.rec_off[i];
  const uint32_t size = 4u + ldu32(src);
  unsigned long long dst;
  if (role == 2) dst = a.anchor_bytes[a.mate[i]];                                          // first of its pair, at the second's anchor
  else if (a.pair_path && a.mate[i] >= 0 && a.role[a.mate[i]] == 2) dst = a.anchor_bytes[i] + 4ull + ldu32(a.data + a.rec_off[a.mate[i]]);  // after its first mate
  else dst = a.anchor_bytes[i];
  uint8_t* out = a.out + dst;
  for (uint32_t k = lane; k < size; k += 32) out[k] = src[k];
}
