// Multi-GPU contig sharding of ONE sample (SURVEY.md 8e): which contigs a rank owns and which BGZF blocks hold them.
//
// The reference processes a BAM front to back and flushes per tid (contig.rs:40-104, 140-155); contigs never interact,
// and a reference-sorted file keeps a tid range in one contiguous run of the record stream.  So rank r of N
//   * owns the tid range [cut[r], cut[r+1]) -- cuts balance the summed contig length, i.e. the O(L) work of the scan;
//   * uploads and inflates only the BGZF blocks that can hold records of that range, found by a binary search over
//     "tid of the first record that starts at or after block b" (a few host-side block inflations);
//   * its walk starts one block early (the block before the first one whose first record already belongs to the
//     range), so neighbouring ranks overlap by a block; every record is still COUNTED by exactly one rank (by tid).
// Both cuts and block boundaries are pure functions of the file, so every rank derives the same partition without
// talking to the others.
#pragma once
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

#include "bam_source.hpp"

namespace cmbh {

// cut[r] = first tid of rank r; cut[n_ranks] = n_ref.  Greedy on the cumulative length: rank r starts at the first contig
// whose preceding length reaches r/N of the total.
inline std::vector<uint32_t> tid_cuts_by_length(const std::vector<uint64_t>& lens, int n_ranks) {
  std::vector<uint32_t> cut((size_t)n_ranks + 1, (uint32_t)lens.size());
  cut[0] = 0;
  unsigned __int128 total = 0;
  for (uint64_t l : lens) total += std::max<uint64_t>(1, l);
  unsigned __int128 acc = 0;
  int r = 1;
  for (uint32_t t = 0; t < lens.size() && r < n_ranks; ++t) {
    while (r < n_ranks && acc * (unsigned)n_ranks >= total * (unsigned)r) cut[r++] = t;
    acc += std::max<uint64_t>(1, lens[t]);
  }
  return cut;
}

// 32-base spans the contigs [b, e) take in one device context's layout (at least one per contig, cmb_set_reference); a
// context holds at most CMB_MAX_SPANS of them.
// Sharded input over a group: rank r decodes the whole shards [cuts[r], cuts[r + 1]).  The runs are contiguous and the cut
// minimises the largest run's summed size (compressed bytes); the smallest such bound is packed greedily from the first rank,
// so ranks beyond the shards (n_ranks > shards) own empty runs at the end.
inline std::vector<uint32_t> shard_run_cuts(const std::vector<uint64_t>& sizes, int n_ranks) {
  const uint32_t K = (uint32_t)sizes.size();
  auto pack = [&](uint64_t cap, std::vector<uint32_t>* cuts) {  // ranks used when each takes shards while they fit `cap`
    int used = 0;
    for (uint32_t k = 0; k < K; ++used) {
      if (cuts) cuts->push_back(k);
      uint64_t sum = 0;
      do sum += sizes[k++];
      while (k < K && sum + sizes[k] <= cap);
    }
    return used;
  };
  uint64_t lo = 0, hi = 0;
  for (uint64_t x : sizes) {
    lo = std::max(lo, x);
    hi += x;
  }
  while (lo < hi) {  // the smallest cap that n_ranks runs can hold
    const uint64_t mid = lo + (hi - lo) / 2;
    if (pack(mid, nullptr) <= n_ranks) hi = mid;
    else lo = mid + 1;
  }
  std::vector<uint32_t> cuts;
  pack(lo, &cuts);
  while ((int)cuts.size() <= n_ranks) cuts.push_back(K);
  return cuts;
}

inline uint64_t layout_spans(const std::vector<uint64_t>& lens, uint32_t b, uint32_t e) {
  uint64_t s = 0;
  for (uint32_t t = b; t < e; ++t) s += std::max<uint64_t>(1, (lens[t] + 31) / 32);
  return s;
}

// The smallest number of GPUs whose contig cuts (tid_cuts_by_length) keep every rank's contigs within CMB_MAX_SPANS, or 0 when
// no number up to one GPU per contig does.
inline int gpus_for_layout(const std::vector<uint64_t>& lens) {
  const uint64_t total = layout_spans(lens, 0, (uint32_t)lens.size());
  for (uint64_t n = std::max<uint64_t>(1, (total + CMB_MAX_SPANS - 1) / CMB_MAX_SPANS); n <= std::max<size_t>(1, lens.size()); ++n) {
    const std::vector<uint32_t> cut = tid_cuts_by_length(lens, (int)n);
    bool fits = true;
    for (uint64_t r = 0; r < n && fits; ++r) fits = layout_spans(lens, cut[r], cut[r + 1]) <= CMB_MAX_SPANS;
    if (fits) return (int)n;
  }
  return 0;
}

// Per-gene coverage (--gff): a contig's share of the work is its genes' arena, every gene padded to whole 32-base spans (the
// device lays a rank's arena out over the genes of its contigs, cmb_set_genes_range).  seg_tid / seg_len: contig and length of
// each gene.  Cutting these weights with tid_cuts_by_length keeps the cuts on contig boundaries: a contig's genes never split
// across ranks, and the block-range search by tid is the one of contig mode.
inline std::vector<uint64_t> padded_gene_bases(size_t n_ref, const std::vector<uint32_t>& seg_tid, const std::vector<uint64_t>& seg_len) {
  constexpr uint64_t SPAN = 32;
  std::vector<uint64_t> w(n_ref, 0);
  for (size_t g = 0; g < seg_tid.size(); ++g) w[seg_tid[g]] += std::max<uint64_t>(1, (seg_len[g] + SPAN - 1) / SPAN) * SPAN;
  return w;
}

// The row cuts of gene mode: rank r's rows are the genes of its contigs, [first_of_tid[cut[r]], first_of_tid[cut[r+1]]), and
// the rank whose range ends with the last contig also holds the placeholder row of an empty gene set (n_rows = max(1, genes)).
// The same rule as cmb_set_genes_range's, so these are the cuts cmb_allgather_stats checks against each rank's context.
inline std::vector<uint32_t> gene_row_cuts(const std::vector<uint32_t>& tid_cuts, const std::vector<uint32_t>& first_of_tid, uint32_t n_rows) {
  const uint32_t n_ref = (uint32_t)first_of_tid.size() - 1;
  std::vector<uint32_t> rc(tid_cuts.size());
  for (size_t r = 0; r < tid_cuts.size(); ++r) {
    const uint32_t t = tid_cuts[r];
    rc[r] = t == 0 && r == 0 ? 0 : t == n_ref ? n_rows : first_of_tid[t];
  }
  return rc;
}

struct BlockRange {
  uint32_t walk_begin = 0, walk_end = 0;  // records starting in blocks [walk_begin, walk_end) are this rank's to decode
  uint64_t records_at = 0;                // uncompressed offset of the first record that starts in walk_begin
  uint32_t excl_end = 0;                  // == the next rank's walk_begin (walk_end for the last rank)
  uint32_t probes = 0;                    // blocks inflated on the host to find the range
};

class BlockRangeFinder {
 public:
  // hint_min_blocks: files with fewer blocks are bisected even when a hint is given (fewer probes than galloping)
  BlockRangeFinder(const BlockIndex& bx, uint32_t n_ref, uint64_t records_at, uint32_t hint_min_blocks = 1024)
      : bx_(bx), n_ref_(n_ref), hint_min_blocks_(hint_min_blocks), records_at_(records_at) {
    nb_ = (uint32_t)bx.blocks.size();
    first_ = (uint32_t)(std::upper_bound(bx.ustart.begin(), bx.ustart.end(), records_at) - bx.ustart.begin()) - 1;
    if (first_ > nb_) first_ = nb_;
  }
  uint32_t probes() const { return probes_; }

  // Range of rank `rank`: tids [t_lo, t_hi); `last` = this rank also takes the unplaced tail (tid < 0) and runs to the end.
  // Throws Panic on a stream whose record boundaries cannot be established (the caller then decodes the whole file).
  // frac_lo / frac_hi (optional, in [0, 1]): where the records of t_lo / t_hi are expected to start as a fraction of the record
  // stream -- the caller's cumulative contig length is a good guess when reads cover the reference evenly.  A hint only
  // changes WHERE the search starts (galloping from the guess before bisecting), never its result.
  BlockRange find(uint32_t t_lo, uint32_t t_hi, bool first_rank, bool last, double frac_lo = -1.0, double frac_hi = -1.0) {
    hint_lo_ = frac_lo;
    hint_hi_ = frac_hi;
    t_lo_ = t_lo;
    t_hi_ = t_hi;
    BlockRange r;
    if (first_rank || t_lo == 0) {
      r.walk_begin = first_;
      r.records_at = records_at_;
    } else {
      range_begin(t_lo, &r.walk_begin, &r.records_at);
    }
    if (last) {
      r.walk_end = nb_;
      r.excl_end = nb_;
    } else {
      r.walk_end = lower_bound_block(t_hi);
      uint64_t unused;
      range_begin(t_hi, &r.excl_end, &unused);
    }
    if (r.walk_end < r.walk_begin) r.walk_end = r.walk_begin;
    r.excl_end = std::min(std::max(r.excl_end, r.walk_begin), r.walk_end);
    r.probes = probes_;
    return r;
  }

 private:
  // Sort key of a record's tid: unplaced records (tid < 0) come after every reference.
  static int64_t key_of(int32_t tid) { return tid < 0 ? (int64_t)INT32_MAX + 1 : (int64_t)tid; }

  // The first record that STARTS in block b: false when none does (the block lies inside one long record, or is empty).
  bool first_record_in(uint32_t b, int32_t* tid, uint64_t* uoff) {
    if (b >= nb_ || b < first_) return false;
    if (b < cache_.size() && cache_[b].state) {
      *tid = cache_[b].tid;
      *uoff = cache_[b].uoff;
      return cache_[b].state == 1;
    }
    if (cache_.size() < nb_) cache_.resize(nb_);
    // inflate b and a little of what follows, enough to test six consecutive headers of ordinary records (a chain that runs
    // off the inflated data counts as confirmed, like in the host decoder)
    uint32_t e = b + 1;
    uint64_t have = bx_.blocks[b].isize;
    while (e < nb_ && e < b + 3 && have < bx_.blocks[b].isize + (64u << 10)) have += bx_.blocks[e++].isize;
    buf_.resize((size_t)have + 8);
    bx_.inflate(b, e, buf_.data(), inf_);
    probes_ += e - b;
    const size_t usize = (size_t)have;
    const size_t own = bx_.blocks[b].isize;
    size_t start = (size_t)-1;
    if (b == first_) {
      start = (size_t)(records_at_ - bx_.ustart[b]);  // known exactly
      if (start >= own) start = (size_t)-1;
    } else {
      // A run of six consistent headers confirms a guess; so does a shorter run that reaches the end of the inflated data.  A
      // candidate whose FIRST record already points past the data (a very long read -- or four stray bytes that happen to look like
      // a multi-megabyte block_size in front of the real header, e.g. the tail `NM:C:0` of the previous record) proves nothing
      // by itself: it is only taken when no other offset of the block yields a checked run.
      size_t unchecked = (size_t)-1, landed = (size_t)-1;
      const bool to_eof = e == nb_;
      for (size_t s = 0; s < own && start == (size_t)-1; ++s) {
        if (!record_plausible(buf_.data(), s, usize, n_ref_)) continue;
        size_t q = s;
        int ok = 0;
        bool ran_off = false;
        while (ok < 6) {
          if (q + 36 > usize) {
            ran_off = true;
            break;
          }
          if (!record_plausible(buf_.data(), q, usize, n_ref_)) break;
          q += 4 + (size_t)rd_u32(buf_.data() + q);
          ++ok;
        }
        if (ok >= 6 || (ran_off && ok >= 2)) start = s;
        else if (ran_off && q == usize && to_eof) start = s;  // its record ends exactly where the file's records end
        else if (ran_off && q <= usize && landed == (size_t)-1) landed = s;  // the next header would start inside the data
        else if (ran_off && unchecked == (size_t)-1) unchecked = s;
      }
      if (start == (size_t)-1) start = landed != (size_t)-1 ? landed : unchecked;
    }
    Probe& c = cache_[b];
    if (start == (size_t)-1 || start + 8 > usize) {
      c.state = 2;
      return false;
    }
    c.state = 1;
    c.tid = (int32_t)rd_u32(buf_.data() + start + 4);
    c.uoff = bx_.ustart[b] + start;
    *tid = c.tid;
    *uoff = c.uoff;
    return true;
  }

  // key(b): sort key of the first record that starts at or after block b (past the end: +inf).
  int64_t key_at_or_after(uint32_t b) {
    for (; b < nb_; ++b) {
      int32_t tid;
      uint64_t uoff;
      if (first_record_in(b, &tid, &uoff)) return key_of(tid);
    }
    return INT64_MAX;
  }

  // Smallest block b in [first_, nb_] with key(b) >= t  (every record with a smaller tid starts before block b's first record).
  uint32_t lower_bound_block(uint32_t t) {
    if (bound_cached_[0].first == (int64_t)t) return bound_cached_[0].second;
    if (bound_cached_[1].first == (int64_t)t) return bound_cached_[1].second;
    uint32_t lo = first_, hi = nb_;
    // invariant: the answer lies in [lo, hi]; key(hi) >= t or hi == nb_; key(b) < t for every b < lo
    const double frac = t == t_lo_ ? hint_lo_ : t == t_hi_ ? hint_hi_ : -1.0;
    if (frac >= 0.0 && frac <= 1.0 && nb_ - first_ > hint_min_blocks_) {
      uint32_t g = first_ + (uint32_t)(frac * (double)(nb_ - first_));
      if (g >= nb_) g = nb_ - 1;
      uint32_t step = 8;
      if (key_at_or_after(g) >= (int64_t)t) {  // the answer is at or before g: gallop backwards
        hi = g;
        while (hi > lo) {
          const uint32_t p = hi - lo > step ? hi - step : lo;
          if (key_at_or_after(p) >= (int64_t)t) {
            hi = p;
            step *= 4;
          } else {
            lo = p + 1;
            break;
          }
        }
      } else {  // after g: gallop forwards
        lo = g + 1;
        while (lo < hi) {
          const uint32_t p = hi - lo > step ? lo + step : hi;
          if (p >= hi) break;
          if (key_at_or_after(p) >= (int64_t)t) {
            hi = p;
            break;
          }
          lo = p + 1;
          step *= 4;
        }
      }
    }
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (key_at_or_after(mid) >= (int64_t)t) hi = mid;
      else lo = mid + 1;
    }
    bound_cached_[bound_cached_[0].first < 0 ? 0 : 1] = {(int64_t)t, lo};
    return lo;
  }

  // Where the walk of the rank whose first tid is t starts: the last block before lower_bound_block(t) in which a record
  // starts (records of tid t may begin there, after its first record), with that record's offset.  The offset is a
  // speculative alignment; it is confirmed against the block before it: the record chain started from THAT block's own guess
  // must land exactly on it.
  void range_begin(uint32_t t, uint32_t* block, uint64_t* uoff) {
    const uint32_t beta = lower_bound_block(t);
    uint32_t b = beta > first_ ? beta - 1 : first_;
    int32_t tid;
    for (;;) {
      if (first_record_in(b, &tid, uoff)) break;
      if (b == first_) {  // no record starts anywhere before beta: start at beta itself (or at the very first record)
        if (beta < nb_ && first_record_in(beta, &tid, uoff)) {
          *block = beta;
          return;
        }
        *block = first_;
        *uoff = records_at_;
        return;
      }
      --b;
    }
    *block = b;
    if (b > first_) confirm_alignment(b, *uoff);
  }

  void confirm_alignment(uint32_t b, uint64_t want) {
    uint32_t p = b - 1;
    int32_t tid;
    uint64_t g;
    while (!first_record_in(p, &tid, &g)) {
      if (p == first_) return;  // nothing to compare against
      --p;
    }
    // walk the chain from g to `want`
    uint32_t e = p;
    uint64_t have = 0;
    while (e < nb_ && bx_.ustart[e] < want + 36) have += bx_.blocks[e++].isize;
    buf_.resize((size_t)have + 8);
    bx_.inflate(p, e, buf_.data(), inf_);
    probes_ += e - p;
    uint64_t pos = g;
    const uint64_t base = bx_.ustart[p];
    while (pos < want) {
      if (pos + 4 - base > have) break;
      pos += 4 + (uint64_t)rd_u32(buf_.data() + (pos - base));
    }
    if (pos != want) throw Panic("Error reading BAM record: record alignment of a block range could not be confirmed");
  }

  struct Probe {
    uint8_t state = 0;  // 0 unknown, 1 a record starts here, 2 none does
    int32_t tid = 0;
    uint64_t uoff = 0;
  };
  const BlockIndex& bx_;
  uint32_t n_ref_, hint_min_blocks_, nb_ = 0, first_ = 0, probes_ = 0;
  uint32_t t_lo_ = 0, t_hi_ = 0;
  double hint_lo_ = -1.0, hint_hi_ = -1.0;
  std::pair<int64_t, uint32_t> bound_cached_[2] = {{-1, 0}, {-1, 0}};  // lower_bound_block results of this find()
  uint64_t records_at_;
  BgzfInflater inf_;
  std::vector<uint8_t> buf_;
  std::vector<Probe> cache_;
};

}  // namespace cmbh
