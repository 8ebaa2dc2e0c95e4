// Device-side mate matching for the pair path of ReferenceSortedBamFilter::read (filter.rs:117-233), so that
// `--proper-pairs-only` / the *-pair thresholds stay on the device decoder (the read names are in HBM after the inflate).
//
// The reference walks the records in file order with a BTreeMap `first_set` of qname -> stored first mate that is
// cleared whenever the reference id of an eligible record changes:
//     eligible  = !secondary && !supplementary && proper_pair, and mapped when filter_out is false (filter.rs:133-147:
//                 `coverm filter --inverse` returns an unmapped record at once, before it can reach first_set)
//     not found : stored[qname] = record, but only if record.mtid == current tid      (filter.rs:166-176)
//     found     : the pair (stored, record) is tested and, if it passes, both are emitted (filter.rs:185-219)
// When the tids of the eligible records are non-decreasing in file order, every tid's eligible records form one run, the set
// is cleared exactly between runs, and the walk is a two-state machine per (tid, qname) over that key's eligible records in
// file order: different keys never interact.  A stream whose eligible tids go down somewhere is declined
// (DEC_ERR_PAIR_ORDER) and the host's HostMates walks it in file order instead; a reference-sorted file never is (the
// unsigned comparison puts unplaced records, tid -1, last).  Otherwise the matching parallelises over keys:
//   kd_pair_keys       one thread per record: eligibility, a 64-bit hash of (tid, qname), mate[i] = -1
//   kd_pair_order      one thread per PAIR_ORDER_CHUNK records: the chunk's first and last eligible tid, and whether they
//                      go down inside it; kd_pair_order_fold then compares every chunk with the largest tid before it
//   kd_pair_insert     eligible records enter an open-addressing table keyed by the hash (atomicCAS on the tag); the
//                      records of a key form a linked list (atomicExch on the head)
//   kd_pair_resolve    one thread per table slot: collect the list, sort it by record index (= file order), split it by
//                      EXACT (tid, qname) (hash collisions cost time, never correctness), run the state machine and write
//                      mate[first] = second, mate[second] = first
// K1 then evaluates the pair predicates with the partner's columns (mate[i] instead of the host path's i ^ 1 layout);
// records stay in file order.  The emitted order of the reference (stored mate first, at the second mate's position) is
// irrelevant downstream: both mates carry the same tid, and no eligible record of another tid can lie between them (the
// eligible tids are non-decreasing), so the sortedness check (contig.rs:129-132) over the kept records in file order fails
// exactly when it fails over the emitted stream.
#pragma once
#include "cmb_slices.hpp"

struct PairArgs {
  const uint8_t* data;       // inflated stream
  const uint64_t* rec_off;   // per record: offset of its block_size field
  uint32_t n_records;
  uint64_t* key;             // per record: hash of (tid, qname); 0 = not eligible
  int32_t* mate;             // per record: partner index or -1
  uint32_t* next;            // per record: next record of the same table slot
  unsigned long long* slot_tag;  // table: 0 = empty
  uint32_t* slot_head;           // table: list head (0xffffffff = nil)
  uint32_t table_mask;           // table size - 1 (power of two)
  uint32_t* flags;               // [0] error bits (DEC_ERR_*)
  uint2* order;                  // per PAIR_ORDER_CHUNK records: {first, last} eligible tid (unsigned; {~0u, 0} = none)
  uint8_t filter_out;            // ReferenceSortedBamFilter's filter_out: 0 for `coverm filter --inverse`
};
constexpr uint32_t PAIR_NIL = 0xffffffffu;
constexpr uint32_t PAIR_MAX_GROUP = 24;       // eligible records sharing one table slot; more -> the stream is declined
constexpr uint32_t PAIR_ORDER_CHUNK = 64;     // records per kd_pair_order thread
constexpr uint32_t DEC_ERR_PAIRS = 8u;        // a table slot holds more than PAIR_MAX_GROUP eligible records
constexpr uint32_t DEC_ERR_PAIR_ORDER = 16u;  // the tids of the eligible records go down somewhere in file order

__device__ __forceinline__ uint64_t pair_mix(uint64_t h) {  // splitmix64 finaliser
  h ^= h >> 30;
  h *= 0xbf58476d1ce4e5b9ull;
  h ^= h >> 27;
  h *= 0x94d049bb133111ebull;
  h ^= h >> 31;
  return h;
}

__global__ void __launch_bounds__(256) kd_pair_keys(const PairArgs a) {
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= a.n_records) return;
  const uint8_t* rec = a.data + a.rec_off[i];
  const uint8_t* o = rec + 4;
  const uint32_t tid = ldu32(o), w2 = ldu32(o + 8), flag = ldu32(o + 12) >> 16;
  const uint32_t l_read_name = w2 & 0xff;
  a.mate[i] = -1;
  a.next[i] = PAIR_NIL;
  const bool eligible = !(flag & 0x900) && (flag & 0x2) && (a.filter_out || !(flag & 0x4));
  uint64_t h = 0;
  if (eligible) {
    h = 0xcbf29ce484222325ull ^ ((uint64_t)tid * 0x9e3779b97f4a7c15ull);
    const uint8_t* q = o + 32;
    const uint32_t n = l_read_name ? l_read_name - 1 : 0;  // without the NUL
    for (uint32_t k = 0; k < n; ++k) h = (h ^ q[k]) * 0x100000001b3ull;  // FNV-1a over the name
    h = pair_mix(h);
    if (h == 0) h = 1;
  }
  a.key[i] = h;
}

// Eligible tids in file order, compared as unsigned: a chunk's first and last, and a flag when they go down inside it.
__global__ void __launch_bounds__(256) kd_pair_order(const PairArgs a) {
  const uint32_t c = blockIdx.x * 256 + threadIdx.x;
  const uint32_t i0 = c * PAIR_ORDER_CHUNK;
  if (i0 >= a.n_records) return;
  const uint32_t i1 = min(a.n_records, i0 + PAIR_ORDER_CHUNK);
  uint32_t first = 0xffffffffu, last = 0;
  bool any = false, down = false;
  for (uint32_t i = i0; i < i1; ++i) {
    if (!a.key[i]) continue;
    const uint32_t tid = ldu32(a.data + a.rec_off[i] + 4);
    if (!any) first = tid;
    down = down || (any && tid < last);
    any = true;
    last = tid;
  }
  a.order[c] = make_uint2(first, last);
  if (down) atomicOr(a.flags, DEC_ERR_PAIR_ORDER);
}

// Across chunks (one CTA): chunk c's first eligible tid must be >= the last eligible tid of every chunk before it and >= `carry`,
// the largest eligible tid of the earlier slices of a sliced decode (0: none).  `largest` (when given) receives the largest
// eligible tid so far, carry included: the next slice's carry.
__global__ void __launch_bounds__(1024) kd_pair_order_fold(const uint2* order, uint32_t n_chunks, uint32_t* flags, uint32_t carry,
                                                           uint32_t* largest) {
  __shared__ uint32_t s_max[1024];
  const uint32_t t = threadIdx.x;
  const uint32_t per = (n_chunks + 1023) / 1024;
  const uint32_t c0 = min(n_chunks, t * per), c1 = min(n_chunks, c0 + per);
  uint32_t lmax = carry;
  bool bad = false;
  for (uint32_t c = c0; c < c1; ++c) {
    const uint2 r = order[c];
    bad = bad || pair_order_drop(r.x, lmax);
    lmax = max(lmax, r.y);
  }
  s_max[t] = lmax;
  __syncthreads();
  uint32_t before = carry;
  for (uint32_t k = 0; k < t; ++k) before = max(before, s_max[k]);
  for (uint32_t c = c0; c < c1 && !bad; ++c) bad = pair_order_drop(order[c].x, before);
  if (bad) atomicOr(flags, DEC_ERR_PAIR_ORDER);
  if (largest && t == 1023) *largest = max(before, lmax);
}

__global__ void __launch_bounds__(256) kd_pair_insert(const PairArgs a) {
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= a.n_records) return;
  const uint64_t h = a.key[i];
  if (!h) return;
  uint32_t s = (uint32_t)(h >> 20) & a.table_mask;
  for (;;) {
    unsigned long long cur = a.slot_tag[s];
    if (cur == 0) cur = atomicCAS(a.slot_tag + s, 0ull, (unsigned long long)h);
    if (cur == 0 || cur == h) break;
    s = (s + 1) & a.table_mask;
  }
  a.next[i] = atomicExch(a.slot_head + s, i);
}

// exact identity of two eligible records: same tid and the same name bytes
__device__ __forceinline__ bool pair_same_name(const uint8_t* data, uint64_t off_a, uint64_t off_b) {
  const uint8_t* ra = data + off_a + 4;
  const uint8_t* rb = data + off_b + 4;
  if (ldu32(ra) != ldu32(rb)) return false;
  const uint32_t la = ra[8], lb = rb[8];
  if (la != lb) return false;
  for (uint32_t k = 0; k < la; ++k)
    if (ra[32 + k] != rb[32 + k]) return false;
  return true;
}

__global__ void __launch_bounds__(256) kd_pair_resolve(const PairArgs a) {
  const uint32_t s = blockIdx.x * 256 + threadIdx.x;
  if (s > a.table_mask) return;
  uint32_t head = a.slot_head[s];
  if (head == PAIR_NIL) return;
  uint32_t idx[PAIR_MAX_GROUP];
  uint32_t n = 0;
  for (uint32_t r = head; r != PAIR_NIL; r = a.next[r]) {
    if (n == PAIR_MAX_GROUP) {
      atomicOr(a.flags, DEC_ERR_PAIRS);
      return;
    }
    idx[n++] = r;
  }
  for (uint32_t x = 1; x < n; ++x) {  // file order
    const uint32_t v = idx[x];
    uint32_t y = x;
    while (y > 0 && idx[y - 1] > v) {
      idx[y] = idx[y - 1];
      --y;
    }
    idx[y] = v;
  }
  // one pass per distinct exact name (normally a single one): `done` marks the records already handled
  uint32_t done = 0;
  for (uint32_t g = 0; g < n; ++g) {
    if (done & (1u << g)) continue;
    const uint64_t off_g = a.rec_off[idx[g]];
    int32_t stored = -1;  // first_set entry of this qname (filter.rs:166-176)
    for (uint32_t x = g; x < n; ++x) {
      if (done & (1u << x)) continue;
      if (x != g && !pair_same_name(a.data, off_g, a.rec_off[idx[x]])) continue;
      done |= 1u << x;
      const uint32_t i = idx[x];
      if (stored < 0) {
        const uint8_t* o = a.data + a.rec_off[i] + 4;
        if ((int32_t)ldu32(o + 20) == (int32_t)ldu32(o)) stored = (int32_t)i;  // record.mtid() == current_reference
      } else {
        a.mate[stored] = (int32_t)i;
        a.mate[i] = stored;
        stored = -1;
      }
    }
  }
}

#ifdef __CUDACC__
// The pair-mode cut of a slice (cmb_slices.hpp) over its n records, `last` = its largest eligible tid
// (kd_pair_order_fold): *after = max of pair_cut_after, then *cut_back = n - min of pair_cut_at (0: no record is held back).
__global__ void __launch_bounds__(256) kd_pair_cut_after(const uint64_t* key, const int32_t* tid, uint32_t n, const uint32_t* last,
                                                         uint32_t* after) {
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = pair_cut_after(key[i] != 0, (uint32_t)tid[i], *last, i);
  if (v) atomicMax(after, v);
}
__global__ void __launch_bounds__(256) kd_pair_cut_at(const uint64_t* key, const int32_t* tid, uint32_t n, const uint32_t* last,
                                                      const uint32_t* after, uint32_t* cut_back) {
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = pair_cut_at(key[i] != 0, (uint32_t)tid[i], *last, *after, i, n);
  if (v < n) atomicMax(cut_back, n - v);
}
#endif
