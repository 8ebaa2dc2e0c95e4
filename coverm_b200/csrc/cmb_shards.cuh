// Sharded input (ReadSortedShardedBamReader, src/shard_bam_reader.rs): the per-record scan of one shard's decoded stream, the
// per-pair choice of the best shard, and the counting sort of the winners by tid.  Included from cmb_shard_input.cu; the plain
// structs the context stores (ShardStore, PairState) are in cmb_context.cuh.
//
// Errors are not traps: each kernel folds what it finds into one 64-bit key with atomicMin, ordered like the reference's serial
// loop meets them -- the primary-set index first (the reference reads set s of every shard, then decides pair s/2 after its second
// set), then the phase inside that step (reading shard k, then scoring shard k, the pair's choice, cloning the winner), then the
// kind.  The host turns the smallest key into the reference's message.

constexpr uint32_t SH_NONE = 0xffffffffu;
// error kinds (4 bits of the key)
constexpr uint32_t SHE_UNPAIRED = 1, SHE_NAME = 2, SHE_AS_MISSING = 5, SHE_AS_TYPE = 6, SHE_EXCLUDED = 7, SHE_NM_TYPE = 8,
                   SHE_NM_MISSING = 9, SHE_NO_SEPARATOR = 10;
// phases: reading shard k = k, scoring shard k = SHP_SCORE + k, the pair's choice, cloning the winner's records
constexpr uint32_t SHP_SCORE = 0x100, SHP_CHOOSE = 0x200, SHP_CLONE = 0x300;
// key: set index (40 bits) | phase (12 bits) | kind (4 bits) | detail (8 bits: the AS tag's type)
__device__ __forceinline__ unsigned long long sh_key(uint64_t set, uint32_t phase, uint32_t kind, uint32_t detail) {
  return (set << 24) | ((unsigned long long)(phase & 0xfff) << 12) | ((kind & 0xf) << 8) | (detail & 0xff);
}

// info byte of a stored primary: bits 0-1 NM tag (0 absent, 1 type C, 2 another type), bit 2 n_cigar > 0
constexpr uint8_t SHI_NM_MASK = 3, SHI_HAS_CIGAR = 4;
// AS state of a stored primary (aux_as, lib.rs:160-178): 0 absent, 1 type C or S, else the tag's type character

// One block slice of a shard (cmb_shard_add): its records are scanned and their primaries appended to the shard's store at
// prim_base / iv_base, so that every index below (the store's, hash0's, the error keys') counts from the shard's first record.
struct ShardScanArgs {
  const uint8_t* data;          // biased base of the inflated stream
  const uint64_t* rec_off;
  cmb_read_batch tb;            // the decoder's tuples of this slice
  uint64_t n_records;
  unsigned long long* scan;     // [n_records + 1]: packed (primaries << 32 | interval slots), exclusive after kf_scan
  ShardStore st;                // this shard's store (ks_compact)
  uint64_t prim_base;           // primaries of the shard's earlier slices
  uint32_t iv_base;             // their interval slots
  int32_t* as_val;              // [primaries] this shard's AS values (ks_pairs reads them)
  uint8_t* as_state;
  unsigned long long* hash0;    // shard 0's name hashes; written by shard 0, compared by the others
  unsigned long long* names;    // group runs, shards k > 0: this shard's name hashes, compared later by ks_names
  uint64_t n0;                  // primaries of shard 0 (complete before shard 1's first slice)
  uint32_t shard;
  int32_t tid_offset;
  unsigned long long* err;
};

__global__ void __launch_bounds__(256) ks_mark(const ShardScanArgs a) {
  const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= a.n_records) return;
  const bool prim = !(a.tb.flag[i] & 0x900);
  a.scan[i] = prim ? ((1ull << 32) | (a.tb.iv_begin[i + 1] - a.tb.iv_begin[i])) : 0ull;
}

__device__ __forceinline__ unsigned long long sh_mix(unsigned long long x) {  // splitmix64 finaliser
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

// One thread per record: the unpaired check for every record, and for a primary its tuple, intervals, AS, NM type and name hash
// into the store.
__global__ void __launch_bounds__(256) ks_compact(const ShardScanArgs a) {
  const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= a.n_records) return;
  const unsigned long long s = a.scan[i];
  const uint64_t j = a.prim_base + (s >> 32);
  const uint32_t ivo = a.iv_base + (uint32_t)s;
  const uint32_t flag = a.tb.flag[i];
  // "This code can only handle paired-end input" (shard_bam_reader.rs:79-87): met while reading set j of this shard
  if (!(flag & 0x1)) atomicMin(a.err, sh_key(j, a.shard, SHE_UNPAIRED, 0));
  if (flag & 0x900) return;
  const cmb_read_batch& o = a.st.b;
  const int32_t tid = a.tb.tid[i];
  o.tid[j] = tid + a.tid_offset;  // set_tid(tid + tid_offsets[winner]) (shard_bam_reader.rs:194, 285)
  o.pos[j] = a.tb.pos[i];
  o.flag[j] = (uint16_t)flag;
  o.mapq[j] = a.tb.mapq[i];
  o.nm_state[j] = a.tb.nm_state[i];
  o.nm[j] = a.tb.nm[i];
  o.l_seq[j] = a.tb.l_seq[i];
  o.aligned[j] = a.tb.aligned[i];
  o.del[j] = a.tb.del[i];
  o.ins[j] = a.tb.ins[i];
  o.iv_begin[j] = ivo;
  const uint32_t i0 = a.tb.iv_begin[i], n_iv = a.tb.iv_begin[i + 1] - i0;
  for (uint32_t k = 0; k < n_iv; ++k) {
    o.iv_start[ivo + k] = a.tb.iv_start[i0 + k];
    o.iv_len[ivo + k] = a.tb.iv_len[i0 + k];
  }
  // the record again, for what the decoder's tuple does not carry (the decoder has validated its layout)
  const uint8_t* rec = a.data + a.rec_off[i];
  const uint8_t* p = rec + 4;
  const uint8_t* end = p + ldu32(rec);
  const uint32_t l_read_name = p[8], n_cigar = ldu16(p + 12), l_seq = ldu32(p + 16);
  unsigned long long h = 0xcbf29ce484222325ull;  // FNV-1a of the name (without its NUL)
  const uint8_t* name = p + 32;
  for (uint32_t k = 0; k + 1 < l_read_name; ++k) h = (h ^ name[k]) * 0x100000001b3ull;
  h = sh_mix(h ^ l_read_name);
  uint32_t as_state = 0, nm_type = 0;
  int32_t as_val = 0;
  const uint8_t* q = name + l_read_name + 4ull * n_cigar + (l_seq + 1) / 2 + l_seq;
  while (q + 3 <= end) {  // first AS / first NM win, as htslib's bam_aux_get
    const uint32_t t0 = q[0], t1 = q[1], ty = q[2];
    q += 3;
    uint64_t sz;
    if (ty == 'A' || ty == 'c' || ty == 'C') sz = 1;
    else if (ty == 's' || ty == 'S') sz = 2;
    else if (ty == 'i' || ty == 'I' || ty == 'f') sz = 4;
    else if (ty == 'Z' || ty == 'H') {
      const uint8_t* e = q;
      while (e < end && *e) ++e;
      sz = (uint64_t)(e - q) + 1;
    } else if (ty == 'B') {
      if (q + 5 > end) break;
      const uint32_t sub = q[0];
      sz = 5 + ((sub == 'c' || sub == 'C') ? 1ull : (sub == 's' || sub == 'S') ? 2ull : 4ull) * ldu32(q + 1);
    } else {
      break;
    }
    if (t0 == 'A' && t1 == 'S' && as_state == 0) {
      if (ty == 'C') { as_state = 1; as_val = q[0]; }
      else if (ty == 'S') { as_state = 1; as_val = (int32_t)ldu16(q); }
      else as_state = ty;
    }
    if (t0 == 'N' && t1 == 'M' && nm_type == 0) nm_type = ty == 'C' ? 1 : 2;
    q += sz;
  }
  a.st.info[j] = (uint8_t)(nm_type | (n_cigar ? SHI_HAS_CIGAR : 0));
  a.as_val[j] = as_val;
  a.as_state[j] = (uint8_t)as_state;
  // the name check of read_a_record_set (shard_bam_reader.rs:88-108): set j of every shard carries one read name
  if (a.shard == 0) a.hash0[j] = h;
  else if (a.names) a.names[j] = h;
  else if (j < a.n0 && a.hash0[j] != h) atomicMin(a.err, sh_key(j, a.shard, SHE_NAME, 0));
}

struct ShardPairArgs {
  ShardStore st;
  const int32_t* as_val;
  const uint8_t* as_state;
  const uint8_t* excluded;  // per global tid
  PairState* state;
  uint64_t n_pairs;         // pairs this shard and shard 0 both hold
  uint32_t shard;
  int32_t tid_offset;
  unsigned long long* err;
  int32_t* score;           // ks_score: this shard's column of the score table
  uint64_t n_score;         // its length: the pairs every shard holds
};

// the t-th tied candidate (t >= 2) replaces the winner with probability 1/t
__device__ __forceinline__ bool sh_take_tie(uint64_t pair, uint32_t shard, uint32_t t) {
  const unsigned long long r = sh_mix(sh_mix(pair) ^ ((unsigned long long)shard << 32 | t));
  return (uint32_t)(((r >> 32) * (unsigned long long)t) >> 32) == 0;
}

// Pair j's summed AS in this shard; false when the shard is no candidate for it or its records are in error (the error folded)
__device__ __forceinline__ bool sh_pair_score(const ShardPairArgs& a, uint64_t j, long long& score) {
  const uint64_t m1 = 2 * j, m2 = m1 + 1;
  const int32_t tid = a.st.b.tid[m1];
  const int32_t local = tid - a.tid_offset;
  // a shard is a candidate unless its first mate is placed on an excluded contig; the second mate is not looked at
  if (local >= 0 && a.excluded && a.excluded[tid] == 2) {  // the contig's name has no genome separator: the reference panics
    atomicMin(a.err, sh_key(m2, SHP_SCORE + a.shard, SHE_NO_SEPARATOR, 0));
    return false;
  }
  if (local >= 0 && a.excluded && a.excluded[tid]) return false;
  score = 0;
  const uint64_t at = m2;  // the choice follows the pair's second set
  if (!(a.st.b.flag[m1] & 0x4)) {
    if (a.as_state[m1] != 1) {
      atomicMin(a.err, sh_key(at, SHP_SCORE + a.shard, a.as_state[m1] ? SHE_AS_TYPE : SHE_AS_MISSING, a.as_state[m1]));
      return false;
    }
    score += a.as_val[m1];
  }
  if (!(a.st.b.flag[m2] & 0x4)) {
    if (a.as_state[m2] != 1) {
      atomicMin(a.err, sh_key(at, SHP_SCORE + a.shard, a.as_state[m2] ? SHE_AS_TYPE : SHE_AS_MISSING, a.as_state[m2]));
      return false;
    }
    score += a.as_val[m2];
  }
  return true;
}

// The running winner after shard k: first candidate or higher score takes the pair, the t-th tie takes it when sh_take_tie says so
__device__ __forceinline__ bool sh_update(PairState& s, uint64_t j, uint32_t shard, long long score) {
  if (s.winner == SH_NONE || score > s.best) {
    s.best = score;
    s.winner = shard;
    s.ties = 1;
  } else if (score == s.best) {
    s.ties += 1;
    if (sh_take_tie(j, shard, s.ties)) s.winner = shard;
  } else {
    return false;
  }
  return true;
}

__global__ void __launch_bounds__(256) ks_pairs(const ShardPairArgs a) {
  const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (j >= a.n_pairs) return;
  long long score;
  if (!sh_pair_score(a, j, score)) return;
  PairState s = a.state[j];
  if (sh_update(s, j, a.shard, score)) a.state[j] = s;
}

// ---- group runs (several GPUs, each decoding a run of whole shards): the choice goes through a table of scores instead of the
// running state, so that the ranks can exchange it.  A column holds one int32 per pair: AS values are of type C or S, so a
// pair's sum is below 2^17, and the sentinels are negative.
constexpr int32_t SH_SCORE_NONE = -1;  // the shard is no candidate for the pair
constexpr int32_t SH_SCORE_ERR = -2;   // the pair's records in this shard are in error (folded into the rank's error key)

// One thread per pair the shard holds with shard 0: its errors folded as ks_pairs folds them, its score into the column
__global__ void __launch_bounds__(256) ks_score(const ShardPairArgs a) {
  const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (j >= a.n_pairs) return;
  long long score = 0;
  const uint64_t m1 = 2 * j;
  const int32_t tid = a.st.b.tid[m1];
  const bool candidate = sh_pair_score(a, j, score);
  const bool excluded = tid - a.tid_offset >= 0 && a.excluded && a.excluded[tid] == 1;
  if (j < a.n_score) a.score[j] = candidate ? (int32_t)score : excluded ? SH_SCORE_NONE : SH_SCORE_ERR;
}

// The name check of read_a_record_set for a shard decoded away from shard 0: its primary j against shard 0's, once hash0 arrived
__global__ void __launch_bounds__(256) ks_names(const unsigned long long* names, const unsigned long long* hash0, uint64_t n, uint32_t shard,
                                                unsigned long long* err) {
  const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (j < n && names[j] != hash0[j]) atomicMin(err, sh_key(j, shard, SHE_NAME, 0));
}

// One thread per pair: the columns walked in shard order with ks_pairs' rule, so every rank reaches the winner one GPU reaches
__global__ void __launch_bounds__(256) ks_choose(const int32_t* score, uint64_t n_pairs, uint32_t n_shards, PairState* state) {
  const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (j >= n_pairs) return;
  PairState s{0, SH_NONE, 0};
  for (uint32_t k = 0; k < n_shards; ++k) {
    const int32_t v = score[(uint64_t)k * n_pairs + j];
    if (v >= 0) sh_update(s, j, k, v);
  }
  state[j] = s;
}

struct ShardSortArgs {
  const ShardStore* stores;   // [n_shards], device copy
  const int32_t* tid_offsets; // [n_shards]
  const PairState* state;
  uint64_t n_pairs;
  uint32_t n_contigs;
  unsigned long long* tid_count;  // [n_contigs + 1]: winners per tid, then (kf_scan) their first slot, then (scatter) cursors
  unsigned long long* src;        // [emitted]: (shard << 40 | primary index) of each sorted slot
  unsigned long long* slot_iv;    // [emitted + 1]: interval slots of each sorted record, then (kf_scan) their offsets
  cmb_read_batch out;
  uint64_t n_out;
  unsigned long long* err;
  uint32_t own_begin, own_end;    // the shards whose winners this context sorts (a group rank's run; else all)
};

// A winner's record goes to the coverage loop when it is mapped (contig.rs:124 skips the others; they still count as reads)
__device__ __forceinline__ bool sh_emitted(const ShardStore& s, uint64_t m) { return !(s.b.flag[m] & 0x4) && s.b.tid[m] >= 0; }

// One thread per pair: no candidate is an error; the winners' NM tags are checked as clone_record_into does
// (shard_bam_reader.rs:151-175), and their mapped records counted by tid.
__global__ void __launch_bounds__(256) ks_count(const ShardSortArgs a) {
  const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (j >= a.n_pairs) return;
  const uint32_t w = a.state[j].winner;
  if (w == SH_NONE) {
    atomicMin(a.err, sh_key(2 * j + 1, SHP_CHOOSE, SHE_EXCLUDED, 0));
    return;
  }
  if (w < a.own_begin || w >= a.own_end) return;
  const ShardStore s = a.stores[w];
  for (uint64_t m = 2 * j; m < 2 * j + 2; ++m) {
    const uint32_t info = s.info[m];
    const uint32_t nm = info & SHI_NM_MASK;
    if (nm == 2) atomicMin(a.err, sh_key(2 * j + 1, SHP_CLONE + (uint32_t)(m & 1), SHE_NM_TYPE, 0));
    else if (nm == 0 && s.b.tid[m] - a.tid_offsets[w] >= 0 && (info & SHI_HAS_CIGAR))
      atomicMin(a.err, sh_key(2 * j + 1, SHP_CLONE + (uint32_t)(m & 1), SHE_NM_MISSING, 0));
    if (sh_emitted(s, m) && (uint32_t)s.b.tid[m] < a.n_contigs) atomicAdd(a.tid_count + s.b.tid[m], 1ull);
  }
}

// One thread per pair: each emitted record takes the next slot of its tid.  The order inside a tid is free: K1 checks tids only and
// every per-contig statistic is an integer sum (sum_identity is a floating-point sum).
__global__ void __launch_bounds__(256) ks_scatter(const ShardSortArgs a) {
  const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (j >= a.n_pairs) return;
  const uint32_t w = a.state[j].winner;
  if (w == SH_NONE || w < a.own_begin || w >= a.own_end) return;
  const ShardStore s = a.stores[w];
  for (uint64_t m = 2 * j; m < 2 * j + 2; ++m) {
    if (!sh_emitted(s, m) || (uint32_t)s.b.tid[m] >= a.n_contigs) continue;
    const unsigned long long slot = atomicAdd(a.tid_count + s.b.tid[m], 1ull);
    a.src[slot] = ((unsigned long long)w << 40) | m;
    a.slot_iv[slot] = s.b.iv_begin[m + 1] - s.b.iv_begin[m];
  }
}

// One thread per sorted slot: the record's tuple and intervals into the output batch.
__global__ void __launch_bounds__(256) ks_gather(const ShardSortArgs a) {
  const uint64_t o = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (o >= a.n_out) return;
  const unsigned long long src = a.src[o];
  const ShardStore s = a.stores[src >> 40];
  const uint64_t m = src & ((1ull << 40) - 1);
  const cmb_read_batch& d = a.out;
  d.tid[o] = s.b.tid[m];
  d.pos[o] = s.b.pos[m];
  d.flag[o] = s.b.flag[m];
  d.mapq[o] = s.b.mapq[m];
  d.nm_state[o] = s.b.nm_state[m];
  d.nm[o] = s.b.nm[m];
  d.l_seq[o] = s.b.l_seq[m];
  d.aligned[o] = s.b.aligned[m];
  d.del[o] = s.b.del[m];
  d.ins[o] = s.b.ins[m];
  const uint32_t ivo = (uint32_t)a.slot_iv[o];
  d.iv_begin[o] = ivo;
  if (o + 1 == a.n_out) d.iv_begin[a.n_out] = (uint32_t)a.slot_iv[a.n_out];
  const uint32_t i0 = s.b.iv_begin[m], n_iv = s.b.iv_begin[m + 1] - i0;
  for (uint32_t k = 0; k < n_iv; ++k) {
    d.iv_start[ivo + k] = s.b.iv_start[i0 + k];
    d.iv_len[ivo + k] = s.b.iv_len[i0 + k];
  }
}
