// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_bam.hpp header).
//
// Literal single-threaded CPU restatement of CoverM v0.8.0's coverage path.
// Every function cites the reference file:line it follows (paths relative to
// the CoverM source tree).  f32/f64 usage and operation order are kept exactly as in
// the reference; compile with -ffp-contract=off.
#pragma once
#include <charconv>
#include <cmath>
#include <functional>
#include <memory>
#include <optional>
#include <set>
#include <sstream>

#include "oracle_bam.hpp"

namespace oracle {

// ---------------------------------------------------------------- formatting
// Rust `{}` on f32/f64: shortest round-trip digits, never exponent notation.
template <class F>
inline std::string fmt_float(F v) {
  if (std::isnan(v)) return "NaN";
  if (std::isinf(v)) return v < 0 ? "-inf" : "inf";
  char buf[512];
  auto res = std::to_chars(buf, buf + sizeof buf, v, std::chars_format::fixed);
  return std::string(buf, res.ptr);
}

// ---------------------------------------------------------------- lib.rs
struct ReadsMapped {  // lib.rs:53-57
  uint64_t num_mapped_reads = 0;
  uint64_t num_reads = 0;
};

struct FlagFilter {  // lib.rs:59-79
  bool include_improper_pairs = true;
  bool include_supplementary = true;
  bool include_secondary = false;
  bool passes(const Record& r) const {
    if (!include_secondary && r.is_secondary()) return false;
    if (!include_supplementary && r.is_supplementary()) return false;
    if (!include_improper_pairs && !r.is_proper_pair()) return false;
    return true;
  }
};

// ---------------------------------------------------------------- filter.rs
static const uint8_t MAPQ_UNAVAILABLE = 255;  // filter.rs:13

// filter.rs:243-279
inline bool single_read_passes_filter(const Record& record, uint32_t min_aligned_length_single,
                                      float min_percent_identity_single, float min_aligned_percent_single,
                                      uint8_t min_mapq_single) {
  if (min_mapq_single != MAPQ_UNAVAILABLE && (record.mapq < min_mapq_single || record.mapq == MAPQ_UNAVAILABLE))
    return false;
  uint64_t edit_distance1 = nm(record);
  uint32_t aligned = 0;
  for (auto& c : record.cigar)
    if (c.op == 0 || c.op == 1 || c.op == 2 || c.op == 8 || c.op == 7) aligned += c.len;
  return aligned >= min_aligned_length_single &&
         (float)aligned / (float)record.l_seq >= min_aligned_percent_single &&
         1.0f - (float)edit_distance1 / (float)aligned >= min_percent_identity_single;
}

// filter.rs:281-336
inline bool read_pair_passes_filter(const Record& record1, const Record& record2, uint32_t min_aligned_length_pair,
                                    float min_percent_identity_pair, float min_aligned_percent_pair,
                                    uint8_t min_mapq_single) {
  if (min_mapq_single != MAPQ_UNAVAILABLE &&
      (record1.mapq < min_mapq_single || record2.mapq < min_mapq_single || record1.mapq == MAPQ_UNAVAILABLE ||
       record2.mapq == MAPQ_UNAVAILABLE))
    return false;
  uint64_t edit_distance1 = nm(record1);
  uint64_t edit_distance2 = nm(record2);
  uint32_t aligned_length1 = 0, aligned_length2 = 0;
  for (auto& c : record1.cigar)
    if (c.op == 0 || c.op == 1 || c.op == 8 || c.op == 7) aligned_length1 += c.len;
  for (auto& c : record2.cigar)
    if (c.op == 0 || c.op == 1 || c.op == 8 || c.op == 7) aligned_length2 += c.len;
  uint32_t aligned = aligned_length1 + aligned_length2;
  return aligned >= min_aligned_length_pair &&
         (float)aligned / (float)((size_t)record1.l_seq + (size_t)record2.l_seq) >= min_aligned_percent_pair &&
         1.0f - ((float)(edit_distance1 + edit_distance2) / (float)aligned) >= min_percent_identity_pair;
}

// trait NamedBamReader, bam_generator.rs:21-38
struct NamedBamReader {
  virtual ~NamedBamReader() {}
  virtual const std::string& name() const = 0;
  virtual bool read(Record& r) = 0;
  virtual const Header& header() const = 0;
  virtual uint64_t num_detected_primary_alignments() const = 0;
};

inline std::string file_stem(const std::string& path) {  // Path::file_stem, bam_generator.rs:360-365
  size_t s = path.find_last_of('/');
  std::string base = s == std::string::npos ? path : path.substr(s + 1);
  size_t d = base.find_last_of('.');
  if (d == std::string::npos || d == 0) return base;
  return base.substr(0, d);
}

// BamFileNamedReader, bam_generator.rs:103-144
struct BamFileNamedReader : NamedBamReader {
  std::string stoit_name;
  AlignmentFile bam;
  uint64_t primaries = 0;
  BamFileNamedReader(const std::string& path, int threads) : stoit_name(file_stem(path)), bam(path, threads) {}
  const std::string& name() const override { return stoit_name; }
  bool read(Record& r) override {
    bool ok = bam.read(r);
    if (ok && !r.is_secondary() && !r.is_supplementary()) primaries += 1;
    return ok;
  }
  const Header& header() const override { return bam.header; }
  uint64_t num_detected_primary_alignments() const override { return primaries; }
};

// ReferenceSortedBamFilter (filter.rs:15-234) behind FilteredBamReader
// (bam_generator.rs:524-560).
struct FilteredBamReader : NamedBamReader {
  std::string stoit_name;
  AlignmentFile reader;
  std::map<std::string, Record> first_set;
  int32_t current_reference = -1;
  std::optional<Record> known_next_read;
  bool filter_single_reads, filter_pairs;
  uint32_t min_aligned_length_single;
  float min_percent_identity_single, min_aligned_percent_single;
  uint8_t min_mapq_single;
  uint32_t min_aligned_length_pair;
  float min_percent_identity_pair, min_aligned_percent_pair;
  uint64_t primaries = 0;
  FlagFilter flag_filters;
  bool filter_out;

  FilteredBamReader(const std::string& path, int threads, FlagFilter ff, uint32_t mals, float mpis, float maps,
                    uint8_t mapq, uint32_t malp, float mpip, float mapp, bool filter_out_)
      : stoit_name(file_stem(path)), reader(path, threads), min_aligned_length_single(mals),
        min_percent_identity_single(mpis), min_aligned_percent_single(maps), min_mapq_single(mapq),
        min_aligned_length_pair(malp), min_percent_identity_pair(mpip), min_aligned_percent_pair(mapp),
        flag_filters(ff), filter_out(filter_out_) {
    // filter.rs:48-61
    bool filtering_single_initial = mals > 0 || mpis > 0.0f || maps > 0.0f;
    bool filtering_pairs_initial = malp > 0 || mpip > 0.0f || mapp > 0.0f;
    filter_single_reads = filtering_single_initial || (!filtering_pairs_initial && mapq != MAPQ_UNAVAILABLE);
    filter_pairs = filtering_pairs_initial ||
                   ((!filter_single_reads || !ff.include_improper_pairs) && mapq != MAPQ_UNAVAILABLE);
  }
  const std::string& name() const override { return stoit_name; }
  const Header& header() const override { return reader.header; }
  uint64_t num_detected_primary_alignments() const override { return primaries; }

  bool read(Record& record) override {  // filter.rs:86-234
    if (filter_single_reads && !filter_pairs) {
      for (;;) {
        if (!reader.read(record)) return false;
        if (!record.is_supplementary() && !record.is_secondary()) primaries += 1;
        if (record.is_unmapped() && !filter_out) return true;
        bool passes_filter1 = !record.is_unmapped() &&
                              (flag_filters.include_supplementary || !record.is_supplementary()) &&
                              (flag_filters.include_secondary || !record.is_secondary());
        if (passes_filter1) {
          bool passes_filter2 = single_read_passes_filter(record, min_aligned_length_single,
                                                          min_percent_identity_single, min_aligned_percent_single,
                                                          min_mapq_single);
          if (passes_filter2 == filter_out) return true;
        }
      }
    } else if (!known_next_read.has_value()) {
      while (reader.read(record)) {
        if (!record.is_supplementary() && !record.is_secondary()) primaries += 1;
        if (record.is_unmapped() && !filter_out) return true;
        if (record.is_secondary() || record.is_supplementary()) continue;
        if (!record.is_proper_pair()) {
          if (filter_out) continue;
          return true;
        }
        if (record.tid != current_reference) {
          current_reference = record.tid;
          first_set.clear();
        }
        const std::string qname = record.qname;
        auto it = first_set.find(qname);
        if (it == first_set.end()) {
          if (record.mtid == current_reference) first_set.emplace(qname, record);
          // else: warned and dropped (filter.rs:179-183)
        } else {
          Record record1 = std::move(it->second);
          first_set.erase(it);
          bool passes_filter =
              (!filter_single_reads ||
               (single_read_passes_filter(record1, min_aligned_length_single, min_percent_identity_single,
                                          min_aligned_percent_single, min_mapq_single) &&
                single_read_passes_filter(record, min_aligned_length_single, min_percent_identity_single,
                                          min_aligned_percent_single, min_mapq_single))) &&
              read_pair_passes_filter(record, record1, min_aligned_length_pair, min_percent_identity_pair,
                                      min_aligned_percent_pair, min_mapq_single);
          if (passes_filter == filter_out) {
            known_next_read = record;
            record = record1;
            return true;
          }
        }
      }
      return false;
    } else {
      record = *known_next_read;
      known_next_read.reset();
      return true;
    }
  }
};

// ---------------------------------------------------------------- takers
struct CoverageEntry {  // coverage_takers.rs:40-44
  size_t entry_index;
  float coverage;
};
struct EntryAndCoverages {  // coverage_takers.rs:222-227
  size_t entry_index, stoit_index;
  std::vector<float> coverages;
};

// enum CoverageTakerType + trait CoverageTaker, coverage_takers.rs:8-219
struct CoverageTaker {
  enum Kind { Streaming, Pileup, Cached } kind;
  std::ostream* print_stream = nullptr;
  std::optional<std::string> current_stoit, current_entry;
  // cached
  std::vector<std::string> stoit_names;
  std::vector<std::optional<std::string>> entry_names;
  std::vector<std::vector<CoverageEntry>> coverages;
  size_t current_stoit_index = 0, current_entry_index = 0;
  size_t num_coverages = 0;

  static CoverageTaker streaming(std::ostream* s) { CoverageTaker t; t.kind = Streaming; t.print_stream = s; return t; }
  static CoverageTaker pileup(std::ostream* s) { CoverageTaker t; t.kind = Pileup; t.print_stream = s; return t; }
  static CoverageTaker cached(size_t n) { CoverageTaker t; t.kind = Cached; t.num_coverages = n; return t; }

  void start_stoit(const std::string& stoit_name) {  // :75-98
    if (kind == Cached) {
      stoit_names.push_back(stoit_name);
      coverages.emplace_back();
      current_stoit_index = stoit_names.size() - 1;
    } else {
      current_stoit = stoit_name;
    }
  }
  void start_entry(size_t entry_order_id, const std::string& entry_name) {  // :100-151
    switch (kind) {
      case Streaming: *print_stream << *current_stoit << "\t" << entry_name; break;
      case Pileup: current_entry = entry_name; break;
      case Cached:
        if (entry_order_id >= entry_names.size()) entry_names.resize(entry_order_id + 1);
        if (!entry_names[entry_order_id].has_value()) entry_names[entry_order_id] = entry_name;
        if (*entry_names[entry_order_id] != entry_name)
          throw ExitError(1, "Found a difference amongst the reference sets used for mapping. For this "
                             "(non-streaming) usage of CoverM, all BAM files must have the same set of reference "
                             "sequences. Previous entry was " + *entry_names[entry_order_id] + ", new is " + entry_name);
        current_entry_index = entry_order_id;
        break;
    }
  }
  void add_single_coverage(float coverage) {  // :153-181
    switch (kind) {
      case Streaming:
        if (coverage == 0.0f) *print_stream << "\t0";
        else *print_stream << "\t" << fmt_float(coverage);
        break;
      case Pileup: throw Panic("unreachable");
      case Cached: coverages[current_stoit_index].push_back({current_entry_index, coverage}); break;
    }
  }
  void add_coverage_entry(size_t num_reads, uint64_t num_bases) {  // :186-207
    if (kind != Pileup) throw Panic("unreachable");
    *print_stream << *current_stoit << "\t" << *current_entry << "\t" << num_reads << "\t" << num_bases << "\n";
  }
  void finish_entry() {  // :209-218
    if (kind == Streaming) *print_stream << "\n";
  }

  // CoverageTakerTypeIterator, coverage_takers.rs:229-377: for each stoit in
  // turn, yields every entry index present in ANY stoit (ascending), with
  // zeros where the current stoit lacks it.
  std::vector<EntryAndCoverages> iterate() const {
    std::vector<EntryAndCoverages> out;
    std::vector<size_t> next(stoit_names.size(), 0);
    size_t cur = 0;
    std::optional<size_t> last;
    while (cur <= stoit_names.size()) {
      std::optional<size_t> lowest;
      for (size_t s = 0; s < next.size(); ++s) {
        if (next[s] < coverages[s].size()) {
          const CoverageEntry& e = coverages[s][next[s]];
          if (!last.has_value() || e.entry_index > *last) {
            if (!lowest.has_value() || e.entry_index < *lowest) lowest = e.entry_index;
          }
        }
      }
      if (lowest.has_value()) {
        size_t chosen = next[cur];
        const auto& lst = coverages[cur];
        EntryAndCoverages ec;
        ec.entry_index = *lowest;
        ec.stoit_index = cur;
        if (chosen >= lst.size() || lst[chosen].entry_index != *lowest) {
          ec.coverages.assign(num_coverages, 0.0f);
        } else {
          for (size_t k = 0; k < num_coverages; ++k) ec.coverages.push_back(lst[chosen++].coverage);
        }
        for (size_t s = 0; s < stoit_names.size(); ++s)
          if (coverages[s].size() > next[s] && coverages[s][next[s]].entry_index == *lowest) next[s] += num_coverages;
        last = *lowest;
        out.push_back(std::move(ec));
      } else {
        cur += 1;
        if (cur >= stoit_names.size()) return out;
        next.assign(stoit_names.size(), 0);
        last.reset();
      }
    }
    return out;
  }
};

// ---------------------------------------------------------------- estimators
// enum CoverageEstimator, mosdepth_genome_coverage_estimators.rs:3-81 (EST)
struct CoverageEstimator {
  enum Kind { Mean, TrimmedMean, PileupCounts, CoveredFraction, CoveredBases, RPKM, TPM, Variance, Length, ReadCount,
              ReadsPerBase, ANIr } kind;
  uint64_t total_count = 0, total_bases = 0, num_covered_bases = 0, num_mapped_reads = 0, total_mismatches = 0;
  uint64_t observed_contig_length = 0;
  std::vector<uint64_t> counts;
  double sum_identity = 0.0;
  // configuration
  float min_fraction_covered_bases = 0.0f;
  uint64_t contig_end_exclusion = 0;
  bool exclude_mismatches = false;
  float min = 0.0f, max = 0.0f;

  static CoverageEstimator make(Kind k, float minfrac = 0.0f, uint64_t excl = 0) {
    CoverageEstimator e;
    e.kind = k;
    e.min_fraction_covered_bases = minfrac;
    e.contig_end_exclusion = excl;
    return e;
  }

  std::vector<std::string> column_headers() const {  // EST:84-104
    switch (kind) {
      case Mean: return {"Mean"};
      case TrimmedMean: return {"Trimmed Mean"};
      case PileupCounts: return {"Coverage", "Bases"};
      case CoveredFraction: return {"Covered Fraction"};
      case CoveredBases: return {"Covered Bases"};
      case RPKM: return {"RPKM"};
      case TPM: return {"TPM"};
      case Variance: return {"Variance"};
      case Length: return {"Length"};
      case ReadCount: return {"Read Count"};
      case ReadsPerBase: return {"Reads per base"};
      case ANIr: return {"ANIr"};
    }
    return {};
  }

  static uint64_t calculate_unobserved_bases(const std::vector<uint64_t>& unobserved, uint64_t excl) {  // EST:226-242
    uint64_t s = 0;
    uint64_t e = 2 * excl;
    for (uint64_t l : unobserved) s += (l < e) ? l : l - e;
    return s;
  }

  void setup() {  // EST:268-364
    total_count = total_bases = num_covered_bases = num_mapped_reads = total_mismatches = 0;
    observed_contig_length = 0;
    counts.clear();
    sum_identity = 0.0;
  }

  void add_contig(const std::vector<int32_t>& ups_and_downs, uint64_t num_mapped_reads_in_contig,
                  uint64_t total_mismatches_in_contig, double sum_identity_in_contig) {  // EST:366-528
    switch (kind) {
      case Mean: {
        num_mapped_reads += num_mapped_reads_in_contig;
        total_mismatches += total_mismatches_in_contig;
        size_t len = ups_and_downs.size();
        if (contig_end_exclusion * 2 < (uint64_t)len) total_bases += (uint64_t)len - 2 * contig_end_exclusion;
        else return;
        int32_t cumulative_sum = 0;
        size_t start_from = (size_t)contig_end_exclusion;
        size_t end_at = len - (size_t)contig_end_exclusion - 1;
        for (size_t i = 0; i < len; ++i) {
          cumulative_sum += ups_and_downs[i];
          if (i >= start_from && i <= end_at) {
            if (cumulative_sum > 0) num_covered_bases += 1;
            total_count += (uint64_t)(int64_t)cumulative_sum;  // `as u64`
          }
        }
        break;
      }
      case TrimmedMean:
      case PileupCounts:
      case Variance: {
        num_mapped_reads = num_mapped_reads_in_contig;  // assignment (EST:434)
        size_t len1 = ups_and_downs.size();
        if (contig_end_exclusion * 2 < (uint64_t)len1) observed_contig_length += (uint64_t)len1 - 2 * contig_end_exclusion;
        else return;
        int32_t cumulative_sum = 0;
        size_t start_from = (size_t)contig_end_exclusion;
        size_t end_at = len1 - (size_t)contig_end_exclusion - 1;
        for (size_t i = 0; i < len1; ++i) {
          cumulative_sum += ups_and_downs[i];
          if (i >= start_from && i <= end_at) {
            if (cumulative_sum > 0) num_covered_bases += 1;
            size_t idx = (size_t)(int64_t)cumulative_sum;
            if (counts.size() <= idx) counts.resize(idx + 1, 0);
            counts[idx] += 1;
          }
        }
        break;
      }
      case CoveredFraction:
      case CoveredBases:
      case RPKM:
      case TPM: {
        num_mapped_reads += num_mapped_reads_in_contig;
        total_bases += (uint64_t)ups_and_downs.size();
        int32_t cumulative_sum = 0;
        for (int32_t current : ups_and_downs) {
          cumulative_sum += current;
          if (cumulative_sum > 0) num_covered_bases += 1;
        }
        break;
      }
      case Length:
      case ReadsPerBase:
        observed_contig_length += (uint64_t)ups_and_downs.size();
        num_mapped_reads += num_mapped_reads_in_contig;
        break;
      case ReadCount: num_mapped_reads += num_mapped_reads_in_contig; break;
      case ANIr:
        num_mapped_reads += num_mapped_reads_in_contig;  // `num_reads`
        sum_identity += sum_identity_in_contig;
        break;
    }
  }

  float calculate_coverage(const std::vector<uint64_t>& unobserved_contig_lengths) {  // EST:530-839
    auto sum_unobs = [&]() { uint64_t s = 0; for (auto l : unobserved_contig_lengths) s += l; return s; };
    switch (kind) {
      case Mean: {
        uint64_t final_total_bases = total_bases + calculate_unobserved_bases(unobserved_contig_lengths, contig_end_exclusion);
        if (final_total_bases == 0 || ((float)num_covered_bases / (float)final_total_bases) < min_fraction_covered_bases)
          return 0.0f;
        float num = exclude_mismatches ? (float)(total_count - total_mismatches) : (float)total_count;
        return num / (float)final_total_bases;
      }
      case TrimmedMean: {
        uint64_t unobserved_contig_length = calculate_unobserved_bases(unobserved_contig_lengths, contig_end_exclusion);
        uint64_t total_bases_ = observed_contig_length + unobserved_contig_length;
        if (total_bases_ == 0) return 0.0f;
        if (((float)num_covered_bases / (float)total_bases_) < min_fraction_covered_bases) return 0.0f;
        size_t min_index = (size_t)std::floor(min * (float)total_bases_);
        size_t max_index = (size_t)std::ceil(max * (float)total_bases_);
        if (num_covered_bases == 0) return 0.0f;
        counts[0] += unobserved_contig_length;
        size_t num_accounted_for = 0, total = 0;
        bool started = false;
        for (size_t i = 0; i < counts.size(); ++i) {
          size_t num_covered = (size_t)counts[i];
          num_accounted_for += num_covered;
          if (num_accounted_for >= min_index) {
            if (started) {
              if (num_accounted_for > max_index) {
                size_t num_excess = num_accounted_for - num_covered;
                size_t num_wanted = (max_index >= num_excess) ? max_index - num_excess + 1 : 0;
                total += num_wanted * i;
                break;
              } else {
                total += num_covered * i;
              }
            } else if (num_accounted_for > max_index) {
              total = (max_index - min_index + 1) * i;
              started = true;
            } else if (num_accounted_for < min_index) {
            } else {
              size_t num_wanted = num_accounted_for - min_index + 1;
              total = num_wanted * i;
              started = true;
            }
          }
        }
        return (float)total / (float)(max_index - min_index);
      }
      case PileupCounts: {
        if (observed_contig_length == 0) return 0.0f;
        uint64_t total_bases_ = observed_contig_length + calculate_unobserved_bases(unobserved_contig_lengths, contig_end_exclusion);
        if (((float)num_covered_bases / (float)total_bases_) < min_fraction_covered_bases) return 0.0f;
        return (float)(total_bases_ - num_covered_bases + 1);
      }
      case CoveredFraction: {
        uint64_t f = total_bases + sum_unobs();
        if (f == 0 || ((float)num_covered_bases / (float)f) < min_fraction_covered_bases) return 0.0f;
        return (float)num_covered_bases / (float)f;
      }
      case CoveredBases: {
        uint64_t f = total_bases + sum_unobs();
        if (f == 0 || ((float)num_covered_bases / (float)f) < min_fraction_covered_bases) return 0.0f;
        return (float)num_covered_bases;
      }
      case RPKM: {
        uint64_t f = total_bases + sum_unobs();
        if (f == 0 || ((float)num_covered_bases / (float)f) < min_fraction_covered_bases) return 0.0f;
        return (float)(num_mapped_reads * 1000000000ULL) / (float)f;
      }
      case TPM: {
        uint64_t f = total_bases + sum_unobs();
        if (f == 0 || ((float)num_covered_bases / (float)f) < min_fraction_covered_bases) return 0.0f;
        return (float)std::exp(std::log((double)num_mapped_reads) - std::log((double)f));
      }
      case Variance: {
        uint64_t unobserved_contig_length = calculate_unobserved_bases(unobserved_contig_lengths, contig_end_exclusion);
        uint64_t total_bases_ = observed_contig_length + unobserved_contig_length;
        if (total_bases_ == 0) return 0.0f;
        if (((float)num_covered_bases / (float)total_bases_) < min_fraction_covered_bases || total_bases_ < 3 || counts.empty())
          return 0.0f;
        counts[0] += unobserved_contig_length;
        size_t k = 0;
        while (counts[k] == 0) k += 1;
        size_t ex = 0, ex2 = 0;  // usize, wrapping in release builds
        for (size_t x = 0; x < counts.size(); ++x) {
          if (counts[x] == 0) continue;
          size_t nc = (size_t)counts[x];
          ex += (x - k) * nc;
          ex2 += (x - k) * (x - k) * nc;
        }
        return ((float)ex2 - (float)(ex * ex) / (float)total_bases_) / (float)(total_bases_ - 1);
      }
      case Length: return (float)(observed_contig_length + sum_unobs());
      case ReadCount: return (float)num_mapped_reads;
      case ReadsPerBase: return (float)num_mapped_reads / (float)(observed_contig_length + sum_unobs());
      case ANIr:
        if (num_mapped_reads == 0) return 0.0f;
        return (float)(sum_identity / (double)num_mapped_reads);
    }
    return 0.0f;
  }

  void print_coverage(float coverage, CoverageTaker& t) const {  // EST:936-969
    if (kind != PileupCounts) {
      t.add_single_coverage(coverage);
      return;
    }
    for (size_t i = 0; i < counts.size(); ++i) {
      uint64_t cov;
      if (i == 0) {
        uint64_t c = (uint64_t)std::floor(coverage);
        cov = c == 0 ? 0 : c - 1;
      } else {
        cov = counts[i];
      }
      t.add_coverage_entry(i, cov);
    }
  }
  void print_zero_coverage(CoverageTaker& t, uint64_t entry_length) const {  // EST:971-991
    if (kind == PileupCounts) return;
    if (kind == Length) t.add_single_coverage((float)entry_length);
    else t.add_single_coverage(0.0f);
  }
};

// ---------------------------------------------------------------- printers
// enum CoveragePrinter, coverage_printer.rs:9-17
struct CoveragePrinter {
  enum Kind { Streamed, SparseCached, DenseCached, MetabatAdjusted } kind = Streamed;
  std::string entry_type;
  std::vector<std::string> estimator_headers;

  void print_headers(const std::string& entry_type_str, const std::vector<std::string>& headers, std::ostream& os) {  // :123-152
    switch (kind) {
      case Streamed:
      case SparseCached:
        os << "Sample\t" << entry_type_str;
        for (auto& h : headers) os << "\t" << h;
        os << "\n";
        break;
      case DenseCached:
        entry_type = entry_type_str;
        estimator_headers = headers;
        break;
      case MetabatAdjusted: break;
    }
  }

  static bool contains(const std::vector<size_t>& v, size_t i) {
    for (auto x : v) if (x == i) return true;
    return false;
  }
  static std::string trim_cr(const std::string& s) {
    size_t e = s.size();
    while (e > 0 && s[e - 1] == '\r') --e;
    return s.substr(0, e);
  }
  static size_t count_tabs(const std::string& s) {
    size_t n = 0;
    for (char c : s) if (c == '\t') ++n;
    return n;
  }

  void finalise_printing(const CoverageTaker& taker, std::ostream& os, const std::vector<ReadsMapped>* rm,
                         const std::vector<size_t>& columns_to_normalise, std::optional<size_t> rpkm_column,
                         std::optional<size_t> tpm_column) {  // :20-121
    switch (kind) {
      case Streamed: break;
      case SparseCached: print_sparse(taker, os, rm, columns_to_normalise, rpkm_column, tpm_column); break;
      case DenseCached: print_dense(taker, os, rm, columns_to_normalise, rpkm_column, tpm_column); break;
      case MetabatAdjusted: print_metabat(taker, os); break;
    }
  }

  void print_metabat(const CoverageTaker& taker, std::ostream& os) {  // :57-119
    os << "contigName\tcontigLen\ttotalAvgDepth";
    for (auto& stoit : taker.stoit_names) os << "\t" << stoit << ".bam\t" << stoit << ".bam-var";
    os << "\n";
    std::vector<std::vector<EntryAndCoverages>> sbe;
    for (auto& ecs : taker.iterate()) {
      if (sbe.size() <= ecs.stoit_index) sbe.emplace_back();
      sbe[ecs.stoit_index].push_back(ecs);
    }
    if (sbe.empty()) throw Panic("index out of bounds: the len is 0 but the index is 0");
    for (size_t entry_i = 0; entry_i < sbe[0].size(); ++entry_i) {
      float total_depth = 0.0f;
      for (auto& stoit : sbe) total_depth += stoit[entry_i].coverages[1];
      os << *taker.entry_names[entry_i] << "\t" << fmt_float(sbe[0][entry_i].coverages[0]) << "\t"
         << fmt_float(std::round((double)total_depth * 10000.0 / (double)taker.coverages.size()) / 10000.0);
      for (auto& stoit : sbe) {
        auto& c = stoit[entry_i].coverages;
        os << "\t" << fmt_float(std::round((double)c[1] * 10000.0) / 10000.0) << "\t"
           << fmt_float(std::round((double)c[2] * 10000.0) / 10000.0);
      }
      os << "\n";
    }
  }

  void print_sparse(const CoverageTaker& taker, std::ostream& os, const std::vector<ReadsMapped>* rm,
                    const std::vector<size_t>& columns_to_normalise, std::optional<size_t> rpkm_column,
                    std::optional<size_t> tpm_column) {  // :155-356
    size_t num_coverages = taker.num_coverages;
    size_t num_extra_entry_columns = 0;
    for (auto& n : taker.entry_names)
      if (n.has_value()) { num_extra_entry_columns = count_tabs(*n); break; }
    std::vector<std::vector<float>> cur_cov;
    std::vector<size_t> cur_idx;
    size_t cur_stoit = 0;
    auto print_previous_stoit = [&](const std::vector<std::vector<float>>& covs, const std::vector<size_t>& idxs,
                                    size_t stoit_index) {
      std::vector<std::optional<float>> mult(num_coverages), totals(num_coverages);
      for (size_t i : columns_to_normalise) {
        float total_coverage = 0.0f;
        for (auto& cs : covs) total_coverage += cs[i];
        totals[i] = total_coverage;
        if (rm) {
          const ReadsMapped& r = (*rm)[stoit_index];
          mult[i] = (float)r.num_mapped_reads / (float)r.num_reads;
        }
      }
      if (tpm_column.has_value()) {
        float total_coverage = 0.0f;
        for (auto& cs : covs) total_coverage += cs[*tpm_column];
        totals[*tpm_column] = total_coverage;
      }
      if (stoit_index >= taker.stoit_names.size()) throw Panic("index out of bounds");
      const std::string& stoit = taker.stoit_names[stoit_index];
      if (!columns_to_normalise.empty()) {
        os << stoit << "\tunmapped";
        for (size_t k = 0; k < num_extra_entry_columns; ++k) os << "\t";
        for (size_t i = 0; i < columns_to_normalise.size(); ++i) {
          size_t column = columns_to_normalise[i];
          if (i == 0) { for (size_t k = 0; k < column; ++k) os << "\tNA"; }
          else { for (size_t k = columns_to_normalise[i - 1] + 1; k < column; ++k) os << "\tNA"; }
          os << "\t" << fmt_float(100.0f * (1.0f - *mult[column]));
        }
        for (size_t k = columns_to_normalise.back() + 1; k < num_coverages; ++k) os << "\tNA";
        os << "\n";
      }
      for (size_t e = 0; e < idxs.size(); ++e) {
        const auto& coverages = covs[e];
        if (!taker.entry_names[idxs[e]].has_value()) throw ExitError(1, "Didn't find entry name string as expected");
        os << stoit << "\t" << trim_cr(*taker.entry_names[idxs[e]]);
        for (size_t i = 0; i < num_coverages; ++i) {
          if (contains(columns_to_normalise, i)) {
            os << "\t" << fmt_float(coverages[i] * 100.0f * *mult[i] / *totals[i]);
          } else if (rpkm_column == i) {
            uint64_t n = (*rm)[stoit_index].num_mapped_reads;
            os << "\t" << fmt_float(n == 0 ? 0.0f : coverages[i] / (float)n);
          } else if (tpm_column == i) {
            uint64_t n = (*rm)[stoit_index].num_mapped_reads;
            double v = n == 0 ? 0.0 : (double)std::exp(std::log(coverages[i]) - std::log(*totals[i])) * (double)1000000ULL;
            os << "\t" << fmt_float(v);
          } else {
            os << "\t" << fmt_float(coverages[i]);
          }
        }
        os << "\n";
      }
    };
    for (auto& ec : taker.iterate()) {
      if (cur_stoit != ec.stoit_index) {
        print_previous_stoit(cur_cov, cur_idx, cur_stoit);
        cur_cov.clear();
        cur_idx.clear();
        cur_stoit = ec.stoit_index;
      }
      cur_cov.push_back(ec.coverages);
      cur_idx.push_back(ec.entry_index);
    }
    print_previous_stoit(cur_cov, cur_idx, cur_stoit);
  }

  void print_dense(const CoverageTaker& taker, std::ostream& os, const std::vector<ReadsMapped>* rm,
                   const std::vector<size_t>& columns_to_normalise, std::optional<size_t> rpkm_column,
                   std::optional<size_t> tpm_column) {  // :359-553
    size_t num_coverages = taker.num_coverages;
    os << entry_type;
    for (auto& stoit_name : taker.stoit_names)
      for (auto& h : estimator_headers) os << "\t" << stoit_name << " " << h;
    os << "\n";
    std::vector<float> mult;
    if (rm) for (auto& r : *rm) mult.push_back((float)r.num_mapped_reads / (float)r.num_reads);
    std::vector<std::vector<EntryAndCoverages>> sbe;
    if (!columns_to_normalise.empty()) {
      os << "unmapped";
      for (size_t k = 0; k < count_tabs(entry_type); ++k) os << "\t";
      for (size_t stoit_i = 0; stoit_i < taker.stoit_names.size(); ++stoit_i) {
        for (size_t i = 0; i < columns_to_normalise.size(); ++i) {
          size_t column = columns_to_normalise[i];
          if (i == 0) { for (size_t k = 0; k < column; ++k) os << "\tNA"; }
          else { for (size_t k = columns_to_normalise[i - 1] + 1; k < column; ++k) os << "\tNA"; }
          os << "\t" << fmt_float(100.0f * (1.0f - mult[stoit_i]));
        }
        for (size_t k = columns_to_normalise.back() + 1; k < num_coverages; ++k) os << "\tNA";
      }
      os << "\n";
    }
    std::vector<std::vector<std::optional<float>>> totals(taker.stoit_names.size(),
                                                          std::vector<std::optional<float>>(num_coverages));
    for (auto& ecs : taker.iterate()) {
      for (size_t i : columns_to_normalise) {
        auto& t = totals[ecs.stoit_index][i];
        t = t.has_value() ? *t + ecs.coverages[i] : ecs.coverages[i];
      }
      if (tpm_column.has_value()) {
        auto& t = totals[ecs.stoit_index][*tpm_column];
        t = t.has_value() ? *t + ecs.coverages[*tpm_column] : ecs.coverages[*tpm_column];
      }
      if (sbe.size() <= ecs.stoit_index) sbe.emplace_back();
      sbe[ecs.stoit_index].push_back(ecs);
    }
    if (sbe.empty()) throw Panic("index out of bounds: the len is 0 but the index is 0");
    for (size_t my_entry_i = 0; my_entry_i < sbe[0].size(); ++my_entry_i) {
      os << trim_cr(*taker.entry_names[sbe[0][my_entry_i].entry_index]);
      for (size_t stoit_i = 0; stoit_i < sbe.size(); ++stoit_i) {
        const EntryAndCoverages& ecs = sbe[stoit_i][my_entry_i];
        const auto& coverages = ecs.coverages;
        for (size_t i = 0; i < coverages.size(); ++i) {
          if (contains(columns_to_normalise, i)) {
            os << "\t" << fmt_float(coverages[i] / *totals[ecs.stoit_index][i] * 100.0f * mult[stoit_i]);
          } else if (rpkm_column == i) {
            uint64_t n = (*rm)[stoit_i].num_mapped_reads;
            os << "\t" << fmt_float(n == 0 ? 0.0f : coverages[i] / (float)n);
          } else if (tpm_column == i) {
            uint64_t n = (*rm)[stoit_i].num_mapped_reads;
            float v = n == 0 ? 0.0f
                             : std::exp(std::log(coverages[i]) - std::log(*totals[ecs.stoit_index][i])) * (float)1000000ULL;
            os << "\t" << fmt_float(v);
          } else {
            os << "\t" << fmt_float(coverages[i]);
          }
        }
      }
      os << "\n";
    }
  }
};

// ---------------------------------------------------------------- contig.rs
using ReaderFactory = std::function<std::unique_ptr<NamedBamReader>()>;

static const char* UNSORTED_MSG =
    "BAM file appears to be unsorted. Input BAM files must be sorted by reference (i.e. by samtools sort)";

// CIGAR walk shared by contig.rs:166-202 / genome.rs:179-214, 683-718.
inline void accumulate_cigar(const Record& record, std::vector<int32_t>& ups_and_downs, uint64_t& total_indels,
                             uint64_t& aligned_len) {
  size_t cursor = (size_t)(int64_t)record.pos;
  for (auto& cig : record.cigar) {
    switch (cig.op) {
      case 0: case 8: case 7: {
        if (cursor >= ups_and_downs.size()) throw Panic("index out of bounds (read starts beyond contig end)");
        ups_and_downs[cursor] += 1;
        size_t final_pos = cursor + cig.len;
        if (final_pos < ups_and_downs.size()) ups_and_downs[final_pos] -= 1;
        cursor += cig.len;
        aligned_len += cig.len;
        break;
      }
      case 2: cursor += cig.len; total_indels += cig.len; aligned_len += cig.len; break;
      case 3: cursor += cig.len; break;
      case 1: total_indels += cig.len; aligned_len += cig.len; break;
      default: break;
    }
  }
}

// contig.rs:255-277
inline void print_previous_zero_coverage_contigs(int32_t last_tid, int32_t current_tid,
                                                 const std::vector<CoverageEstimator>& ests, const Header& header,
                                                 CoverageTaker& taker) {
  int32_t my_tid = last_tid + 1;
  while (my_tid < current_tid) {
    taker.start_entry((size_t)my_tid, header.names[my_tid]);
    for (auto& e : ests) e.print_zero_coverage(taker, header.lens[my_tid]);
    taker.finish_entry();
    my_tid += 1;
  }
}

// contig.rs:13-253
inline std::vector<ReadsMapped> contig_coverage(std::vector<ReaderFactory>& bam_readers, CoverageTaker& coverage_taker,
                                                std::vector<CoverageEstimator>& coverage_estimators,
                                                bool print_zero_coverage_contigs, const FlagFilter& flag_filters) {
  std::vector<ReadsMapped> reads_mapped_vector;
  for (auto& gen : bam_readers) {
    std::unique_ptr<NamedBamReader> bam_generated = gen();
    std::string stoit_name = bam_generated->name();
    coverage_taker.start_stoit(stoit_name);
    Record record;
    int32_t last_tid = -2;
    std::vector<int32_t> ups_and_downs;
    const Header& header = bam_generated->header();
    uint64_t num_mapped_reads_total = 0, num_mapped_reads_in_current_contig = 0, total_indels_in_current_contig = 0,
             total_edit_distance_in_current_contig = 0;
    double sum_identity_in_current_contig = 0.0;

    auto process_previous_contigs = [&](int32_t last_tid_, int32_t tid) {  // :40-104
      if (last_tid_ != -2) {
        for (auto& e : coverage_estimators)
          e.add_contig(ups_and_downs, num_mapped_reads_in_current_contig,
                       total_edit_distance_in_current_contig - total_indels_in_current_contig,
                       sum_identity_in_current_contig);
        std::vector<float> coverages;
        for (auto& e : coverage_estimators) coverages.push_back(e.calculate_coverage({0}));
        bool has_nonzero = false;
        for (float c : coverages) if (c > 0.0f) has_nonzero = true;
        if (has_nonzero) num_mapped_reads_total += num_mapped_reads_in_current_contig;
        if (print_zero_coverage_contigs || has_nonzero) {
          coverage_taker.start_entry((size_t)last_tid_, header.names[last_tid_]);
          for (size_t i = 0; i < coverages.size(); ++i) coverage_estimators[i].print_coverage(coverages[i], coverage_taker);
          coverage_taker.finish_entry();
        }
        for (auto& e : coverage_estimators) e.setup();
        sum_identity_in_current_contig = 0.0;
      }
      if (print_zero_coverage_contigs)
        print_previous_zero_coverage_contigs(last_tid_ == -2 ? -1 : last_tid_, tid, coverage_estimators, header,
                                             coverage_taker);
    };

    while (bam_generated->read(record)) {
      if (!flag_filters.passes(record)) continue;
      int32_t tid = record.tid;
      if (!record.is_unmapped()) {
        if (tid != last_tid) {
          if (tid < last_tid) throw Panic(UNSORTED_MSG);
          process_previous_contigs(last_tid, tid);
          if (tid < 0 || (size_t)tid >= header.lens.size()) throw Panic("Corrupt BAM file?");
          ups_and_downs.assign((size_t)header.lens[tid], 0);
          last_tid = tid;
          num_mapped_reads_in_current_contig = 0;
          total_edit_distance_in_current_contig = 0;
          total_indels_in_current_contig = 0;
          sum_identity_in_current_contig = 0.0;
        }
        if (!record.is_supplementary() && !record.is_secondary()) num_mapped_reads_in_current_contig += 1;
        uint64_t aligned_len = 0;
        accumulate_cigar(record, ups_and_downs, total_indels_in_current_contig, aligned_len);
        uint64_t edit = nm(record);
        total_edit_distance_in_current_contig += edit;
        if (!record.is_supplementary() && !record.is_secondary() && aligned_len > 0)
          sum_identity_in_current_contig += ((double)aligned_len - (double)edit) / (double)aligned_len;
      }
    }
    process_previous_contigs(last_tid, (int32_t)header.names.size());
    ReadsMapped rm;
    rm.num_mapped_reads = num_mapped_reads_total;
    rm.num_reads = bam_generated->num_detected_primary_alignments();
    reads_mapped_vector.push_back(rm);
  }
  return reads_mapped_vector;
}

// ---------------------------------------------------------------- genes.rs
struct Gene {  // genes.rs:16-25
  std::string id, contig;
  uint64_t start = 0, end = 0;  // 0-based, half-open
};
struct GeneDefinitions {
  std::vector<Gene> genes;
};

inline std::string rust_trim(const std::string& x) {  // str::trim: Unicode White_Space; the ASCII members suffice here
  size_t a = 0, b = x.size();
  auto ws = [](unsigned char c) { return c == ' ' || (c >= 9 && c <= 13); };
  while (a < b && ws((unsigned char)x[a])) ++a;
  while (b > a && ws((unsigned char)x[b - 1])) --b;
  return x.substr(a, b - a);
}

// genes.rs:146-164: `key=value` (GFF3) or `key "value"` (GTF) among the `;`-separated attributes
inline std::optional<std::string> parse_gff_attribute(const std::string& attributes, const std::string& key) {
  size_t a = 0;
  for (;;) {
    size_t b = attributes.find(';', a);
    std::string entry = rust_trim(attributes.substr(a, b == std::string::npos ? std::string::npos : b - a));
    if (!entry.empty()) {
      if (entry.compare(0, key.size() + 1, key + "=") == 0) return rust_trim(entry.substr(key.size() + 1));
      if (entry.compare(0, key.size() + 1, key + " ") == 0) {
        std::string v = rust_trim(entry.substr(key.size() + 1));
        size_t x = 0, y = v.size();
        while (x < y && v[x] == '"') ++x;
        while (y > x && v[y - 1] == '"') --y;
        return v.substr(x, y - x);
      }
    }
    if (b == std::string::npos) break;
    a = b + 1;
  }
  return std::nullopt;
}
inline std::optional<std::string> parse_gff_id(const std::string& attributes) {  // genes.rs:131-142
  for (const char* key : {"ID", "locus_tag", "gene_id", "Name", "gene", "Parent"}) {
    auto v = parse_gff_attribute(attributes, key);
    if (v && !v->empty()) return v;
  }
  return std::nullopt;
}

// GeneDefinitions::read_gff, genes.rs:44-126
inline GeneDefinitions read_gff(const std::string& path, const std::optional<std::string>& feature_type) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) throw Panic("Failed to open GFF file " + path);
  std::string text;
  char chunk[1 << 16];
  size_t got;
  while ((got = fread(chunk, 1, sizeof chunk, f)) > 0) text.append(chunk, got);
  fclose(f);
  GeneDefinitions defs;
  uint64_t auto_id = 0;
  size_t a = 0;
  while (a < text.size()) {
    size_t b = text.find('\n', a);
    if (b == std::string::npos) b = text.size();
    std::string line = text.substr(a, b - a);
    a = b + 1;
    if (!line.empty() && line.back() == '\r') line.pop_back();  // BufRead::lines strips "\r\n"
    {  // trim_end
      size_t e = line.size();
      while (e > 0 && (line[e - 1] == ' ' || ((unsigned char)line[e - 1] >= 9 && (unsigned char)line[e - 1] <= 13))) --e;
      line.resize(e);
    }
    if (line.empty() || line[0] == '#') continue;
    std::vector<std::string> fields;
    {
      size_t x = 0;
      for (;;) {
        size_t y = line.find('\t', x);
        if (y == std::string::npos) { fields.push_back(line.substr(x)); break; }
        fields.push_back(line.substr(x, y - x));
        x = y + 1;
      }
    }
    if (fields.size() < 8) continue;  // warn!: malformed line
    if (feature_type && fields[2] != *feature_type) continue;
    auto parse_u64 = [](const std::string& t, uint64_t& v) {  // str::parse::<u64>: optional '+', digits only, no overflow
      size_t i = 0;
      if (!t.empty() && t[0] == '+') i = 1;
      if (i >= t.size()) return false;
      unsigned __int128 acc = 0;
      for (; i < t.size(); ++i) {
        if (t[i] < '0' || t[i] > '9') return false;
        acc = acc * 10 + (unsigned)(t[i] - '0');
        if (acc > (unsigned __int128)UINT64_MAX) return false;
      }
      v = (uint64_t)acc;
      return true;
    };
    uint64_t start_1based, end_1based;
    if (!parse_u64(fields[3], start_1based)) continue;
    if (!parse_u64(fields[4], end_1based)) continue;
    if (start_1based == 0 || end_1based < start_1based) continue;
    const std::string attributes = fields.size() > 8 ? fields[8] : std::string();
    Gene g;
    g.contig = fields[0];
    auto id = parse_gff_id(attributes);
    if (id) g.id = *id;
    else {
      auto_id += 1;
      g.id = g.contig + "_gene_" + std::to_string(auto_id);
    }
    g.start = start_1based - 1;
    g.end = end_1based;
    defs.genes.push_back(g);
  }
  return defs;
}

struct ResolvedGene {  // genes.rs:168-173
  size_t entry_id = 0;
  std::string name;
  size_t start = 0, end = 0;
};
using GenomeNamer = std::function<std::optional<std::string>(const std::string&)>;

// genes.rs:351-432
inline std::vector<std::vector<ResolvedGene>> resolve_genes_against_header(const GeneDefinitions& defs, const Header& header,
                                                                          const GenomeNamer* genome_namer) {
  std::unordered_map<std::string, size_t> name_to_tid;
  for (size_t tid = 0; tid < header.names.size(); ++tid) name_to_tid[header.names[tid]] = tid;  // later duplicates win, like HashMap::insert
  std::vector<std::vector<ResolvedGene>> genes_by_tid(header.names.size());
  for (auto& gene : defs.genes) {
    auto it = name_to_tid.find(gene.contig);
    if (it == name_to_tid.end()) continue;
    const size_t tid = it->second;
    const uint64_t contig_len = header.lens[tid];
    const uint64_t start = std::min(gene.start, contig_len), end = std::min(gene.end, contig_len);
    if (start >= end) continue;
    ResolvedGene r;
    if (genome_namer) {
      auto genome = (*genome_namer)(gene.contig);
      if (!genome) continue;
      r.name = gene.id + "\t" + gene.contig + "\t" + *genome;
    } else {
      r.name = gene.id + "\t" + gene.contig;
    }
    r.start = (size_t)start;
    r.end = (size_t)end;
    genes_by_tid[tid].push_back(r);
  }
  size_t next_entry_id = 0;
  for (auto& genes : genes_by_tid) {
    std::stable_sort(genes.begin(), genes.end(), [](const ResolvedGene& x, const ResolvedGene& y) { return x.start < y.start; });  // sort_by_key is stable
    for (auto& g : genes) g.entry_id = next_entry_id++;
  }
  return genes_by_tid;
}

// genes.rs:467-552
inline void emit_genes_for_contig(const std::vector<ResolvedGene>& genes, const std::vector<int32_t>& ups_and_downs,
                                  const std::vector<uint64_t>& read_starts, const std::vector<uint64_t>& read_is_primary,
                                  const std::vector<uint64_t>& read_mismatches, const std::vector<double>& read_identities,
                                  std::vector<CoverageEstimator>& ests, CoverageTaker& taker, bool print_zero_coverage_genes) {
  if (genes.empty()) return;
  const size_t contig_len = ups_and_downs.size();
  std::vector<int32_t> coverage_at_base(contig_len, 0);
  int32_t running = 0;
  for (size_t i = 0; i < contig_len; ++i) {
    running += ups_and_downs[i];
    coverage_at_base[i] = running;
  }
  const size_t n = read_starts.size();
  std::vector<uint64_t> prefix_primary(n + 1, 0), prefix_mismatches(n + 1, 0);
  std::vector<double> prefix_identity(n + 1, 0.0);
  for (size_t i = 0; i < n; ++i) {
    prefix_primary[i + 1] = prefix_primary[i] + read_is_primary[i];
    prefix_mismatches[i + 1] = prefix_mismatches[i] + read_mismatches[i];
    prefix_identity[i + 1] = prefix_identity[i] + read_identities[i];
  }
  for (auto& gene : genes) {
    const size_t start = gene.start, end = std::min(gene.end, contig_len);
    if (start >= end) continue;
    const size_t len = end - start;
    std::vector<int32_t> gene_ups_and_downs(len, 0);
    gene_ups_and_downs[0] = coverage_at_base[start];
    for (size_t i = 1; i < len; ++i) gene_ups_and_downs[i] = ups_and_downs[start + i];
    // partition_point: first index whose start is not < bound (read_starts ascends within a sorted contig)
    auto pp = [&](size_t bound) {
      size_t lo = 0, hi = n;
      while (lo < hi) {
        size_t mid = lo + (hi - lo) / 2;
        if ((size_t)read_starts[mid] < bound) lo = mid + 1;
        else hi = mid;
      }
      return lo;
    };
    const size_t lo = pp(start), hi = pp(end);
    const uint64_t num_mapped_reads = prefix_primary[hi] - prefix_primary[lo];
    const uint64_t mismatches = prefix_mismatches[hi] - prefix_mismatches[lo];
    const double sum_identity = prefix_identity[hi] - prefix_identity[lo];
    for (auto& e : ests) e.add_contig(gene_ups_and_downs, num_mapped_reads, mismatches, sum_identity);
    std::vector<float> coverages;
    for (auto& e : ests) coverages.push_back(e.calculate_coverage({0}));
    bool has_nonzero = false;
    for (float c : coverages) if (c > 0.0f) has_nonzero = true;
    if (print_zero_coverage_genes || has_nonzero) {
      taker.start_entry(gene.entry_id, gene.name);
      for (size_t i = 0; i < coverages.size(); ++i) ests[i].print_coverage(coverages[i], taker);
      taker.finish_entry();
    }
    for (auto& e : ests) e.setup();
  }
}

// genes.rs:182-344
inline std::vector<ReadsMapped> gene_coverage(std::vector<ReaderFactory>& bam_readers, CoverageTaker& coverage_taker,
                                              std::vector<CoverageEstimator>& coverage_estimators, const GeneDefinitions& gene_definitions,
                                              const GenomeNamer* genome_namer, bool print_zero_coverage_genes,
                                              const FlagFilter& flag_filters) {
  std::vector<ReadsMapped> reads_mapped_vector;
  for (auto& gen : bam_readers) {
    std::unique_ptr<NamedBamReader> bam_generated = gen();
    coverage_taker.start_stoit(bam_generated->name());
    const Header& header = bam_generated->header();
    const auto genes_by_tid = resolve_genes_against_header(gene_definitions, header, genome_namer);
    Record record;
    int32_t last_tid = -2;
    std::vector<int32_t> ups_and_downs;
    std::vector<uint64_t> read_starts, read_is_primary, read_mismatches;
    std::vector<double> read_identities;
    uint64_t num_mapped_reads_total = 0;
    auto process_previous_genes = [&](int32_t last_tid_, int32_t current_tid) {  // :434-465
      if (last_tid_ != -2)
        emit_genes_for_contig(genes_by_tid[(size_t)last_tid_], ups_and_downs, read_starts, read_is_primary, read_mismatches, read_identities,
                              coverage_estimators, coverage_taker, print_zero_coverage_genes);
      if (print_zero_coverage_genes) {
        for (int32_t my_tid = last_tid_ == -2 ? 0 : last_tid_ + 1; my_tid < current_tid; ++my_tid) {
          for (auto& gene : genes_by_tid[(size_t)my_tid]) {  // emit_zero_coverage_genes :554-568
            coverage_taker.start_entry(gene.entry_id, gene.name);
            for (auto& e : coverage_estimators) e.print_zero_coverage(coverage_taker, (uint64_t)(gene.end - gene.start));
            coverage_taker.finish_entry();
          }
        }
      }
    };
    while (bam_generated->read(record)) {
      if (!flag_filters.passes(record)) continue;
      if (record.is_unmapped()) continue;
      const int32_t tid = record.tid;
      if (tid != last_tid) {
        if (tid < last_tid) throw Panic("BAM file appears to be unsorted.");
        process_previous_genes(last_tid, tid);
        if (tid < 0 || (size_t)tid >= header.lens.size()) throw Panic("Corrupt BAM file?");
        ups_and_downs.assign((size_t)header.lens[tid], 0);
        last_tid = tid;
        read_starts.clear();
        read_is_primary.clear();
        read_mismatches.clear();
        read_identities.clear();
      }
      const bool is_primary = !record.is_supplementary() && !record.is_secondary();
      if (is_primary) num_mapped_reads_total += 1;
      uint64_t aligned_len = 0, indels = 0;
      accumulate_cigar(record, ups_and_downs, indels, aligned_len);
      const uint64_t edit = nm(record);
      read_starts.push_back((uint64_t)(int64_t)record.pos);
      read_is_primary.push_back(is_primary ? 1 : 0);
      read_mismatches.push_back(edit >= indels ? edit - indels : 0);  // saturating_sub
      read_identities.push_back(is_primary && aligned_len > 0 ? ((double)aligned_len - (double)edit) / (double)aligned_len : 0.0);
    }
    process_previous_genes(last_tid, (int32_t)genes_by_tid.size());
    ReadsMapped rm;
    rm.num_mapped_reads = num_mapped_reads_total;
    rm.num_reads = bam_generated->num_detected_primary_alignments();
    reads_mapped_vector.push_back(rm);
  }
  return reads_mapped_vector;
}

// ---------------------------------------------------------------- genome.rs
struct GenomesAndContigs {  // genomes_and_contigs.rs:7-58
  std::vector<std::string> genomes;
  std::map<std::string, size_t> contig_to_genome;
  std::optional<size_t> genome_index_of_contig(const std::string& c) const {
    auto it = contig_to_genome.find(c);
    if (it == contig_to_genome.end()) return std::nullopt;
    return it->second;
  }
};

// genome_parsing.rs:75-142
inline GenomesAndContigs read_genome_definition_file(const std::string& path) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) throw Panic("Unable to find/read genome definition file " + path);
  std::string text;
  char buf[65536];
  size_t n;
  while ((n = fread(buf, 1, sizeof buf, f)) > 0) text.append(buf, n);
  fclose(f);
  std::map<std::string, std::string> contig_to_genome;
  std::map<std::string, std::vector<std::string>> genome_to_contig;
  std::vector<std::string> genome_order;
  size_t a = 0;
  while (a < text.size()) {
    size_t b = text.find('\n', a);
    std::string line = text.substr(a, b == std::string::npos ? std::string::npos : b - a);
    a = b == std::string::npos ? text.size() : b + 1;
    if (!line.empty() && line.back() == '\r') line.pop_back();  // BufRead::lines strips \r\n
    std::vector<std::string> v;
    size_t s = 0;
    for (;;) {
      size_t t = line.find('\t', s);
      if (t == std::string::npos) { v.push_back(line.substr(s)); break; }
      v.push_back(line.substr(s, t - s));
      s = t + 1;
    }
    if (v.size() == 2) {
      auto is_ws = [](char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\x0c' || c == '\x0b'; };
      std::string genome = v[0];
      size_t g0 = 0, g1 = genome.size();
      while (g0 < g1 && is_ws(genome[g0])) ++g0;
      while (g1 > g0 && is_ws(genome[g1 - 1])) --g1;
      genome = genome.substr(g0, g1 - g0);
      size_t c0 = 0;
      while (c0 < v[1].size() && is_ws(v[1][c0])) ++c0;
      size_t c1 = c0;
      while (c1 < v[1].size() && !is_ws(v[1][c1])) ++c1;
      if (c1 == c0) throw Panic("Failed to split contig name by whitespace in genome definition file");
      std::string contig = v[1].substr(c0, c1 - c0);
      auto it = contig_to_genome.find(contig);
      if (it != contig_to_genome.end()) {
        if (it->second != genome) throw ExitError(1, "The contig name '" + contig + "' was assigned to multiple genomes");
      } else {
        contig_to_genome[contig] = genome;
      }
      if (genome_to_contig.count(genome)) genome_to_contig[genome].push_back(contig);
      else { genome_to_contig[genome] = {contig}; genome_order.push_back(genome); }
    } else {
      throw ExitError(1, "The line \"" + line + "\" in the genome definition file is not a genome name and contig name separated by a tab");
    }
  }
  GenomesAndContigs gc;
  for (auto& genome : genome_order) {
    size_t idx = gc.genomes.size();
    gc.genomes.push_back(genome);
    for (auto& contig : genome_to_contig[genome]) {
      if (gc.contig_to_genome.count(contig))
        throw ExitError(1, "The contig '" + contig + "' has been assigned to multiple genomes");
      gc.contig_to_genome[contig] = idx;
    }
  }
  return gc;
}

// genome.rs:17-322
inline std::vector<ReadsMapped> mosdepth_genome_coverage_with_contig_names(
    std::vector<ReaderFactory>& bam_readers, const GenomesAndContigs& contigs_and_genomes, CoverageTaker& coverage_taker,
    bool print_zero_coverage_genomes, const FlagFilter& flag_filters, std::vector<CoverageEstimator>& coverage_estimators) {
  std::vector<ReadsMapped> reads_mapped_vector;
  for (auto& gen : bam_readers) {
    std::unique_ptr<NamedBamReader> bam_generated = gen();
    std::string stoit_name = bam_generated->name();
    coverage_taker.start_stoit(stoit_name);
    const Header& header = bam_generated->header();
    std::vector<std::optional<size_t>> reference_number_to_genome_index;
    uint32_t num_refs_in_genomes = 0;
    std::vector<std::vector<uint32_t>> genome_index_to_references(contigs_and_genomes.genomes.size());
    std::vector<uint64_t> reads_mapped_in_each_genome(contigs_and_genomes.genomes.size(), 0);
    for (size_t tid = 0; tid < header.names.size(); ++tid) {
      auto gi = contigs_and_genomes.genome_index_of_contig(header.names[tid]);
      reference_number_to_genome_index.push_back(gi);
      if (gi.has_value()) { num_refs_in_genomes += 1; genome_index_to_references[*gi].push_back((uint32_t)tid); }
    }
    if (num_refs_in_genomes == 0)
      throw ExitError(1, "Error: There are no found reference sequences that are a part of a genome");
    std::vector<std::vector<CoverageEstimator>> per_genome(contigs_and_genomes.genomes.size(), coverage_estimators);

    uint32_t last_tid = 0;
    bool doing_first = true;
    std::vector<int32_t> ups_and_downs;
    Record record;
    std::set<uint32_t> seen_ref_ids;
    uint64_t num_mapped_reads_in_current_contig = 0, total_edit_distance_in_current_contig = 0,
             total_indels_in_current_contig = 0;
    double sum_identity_in_current_contig = 0.0;
    while (bam_generated->read(record)) {
      if (!flag_filters.passes(record)) continue;
      int32_t original_tid = record.tid;
      if (!record.is_unmapped()) {
        uint32_t tid = (uint32_t)original_tid;
        if (tid != last_tid || doing_first) {
          if (doing_first) {
            doing_first = false;
          } else {
            if (tid < last_tid) throw Panic(UNSORTED_MSG);
            if (reference_number_to_genome_index[last_tid].has_value()) {
              size_t genome_index = *reference_number_to_genome_index[last_tid];
              for (auto& e : per_genome[genome_index])
                e.add_contig(ups_and_downs, num_mapped_reads_in_current_contig,
                             total_edit_distance_in_current_contig - total_indels_in_current_contig,
                             sum_identity_in_current_contig);
            }
          }
          if (tid >= header.lens.size()) throw Panic("Corrupt BAM file?");
          ups_and_downs.assign((size_t)header.lens[tid], 0);
          num_mapped_reads_in_current_contig = 0;
          total_edit_distance_in_current_contig = 0;
          total_indels_in_current_contig = 0;
          sum_identity_in_current_contig = 0.0;
          last_tid = tid;
          seen_ref_ids.insert(tid);
        }
        if (reference_number_to_genome_index[tid].has_value()) {
          size_t genome_index = *reference_number_to_genome_index[tid];
          reads_mapped_in_each_genome[genome_index] += 1;
          num_mapped_reads_in_current_contig += 1;
          uint64_t aligned_len = 0;
          accumulate_cigar(record, ups_and_downs, total_indels_in_current_contig, aligned_len);
          uint64_t edit = nm(record);
          total_edit_distance_in_current_contig += edit;
          if (!record.is_supplementary() && aligned_len > 0)
            sum_identity_in_current_contig += ((double)aligned_len - (double)edit) / (double)aligned_len;
        }
      }
    }
    uint64_t num_mapped_reads_total = 0;
    if (doing_first && bam_generated->num_detected_primary_alignments() == 0) {
      // warn only (genome.rs:230-234)
    } else {
      if (last_tid >= reference_number_to_genome_index.size()) throw Panic("index out of bounds");
      if (reference_number_to_genome_index[last_tid].has_value()) {
        size_t genome_index = *reference_number_to_genome_index[last_tid];
        for (auto& e : per_genome[genome_index])
          e.add_contig(ups_and_downs, num_mapped_reads_in_current_contig,
                       total_edit_distance_in_current_contig - total_indels_in_current_contig,
                       sum_identity_in_current_contig);
      }
      std::vector<std::vector<uint64_t>> unobserved_lengths(contigs_and_genomes.genomes.size());
      for (size_t ref_id = 0; ref_id < reference_number_to_genome_index.size(); ++ref_id) {
        if (reference_number_to_genome_index[ref_id].has_value() && !seen_ref_ids.count((uint32_t)ref_id))
          unobserved_lengths[*reference_number_to_genome_index[ref_id]].push_back(header.lens[ref_id]);
      }
      for (size_t i = 0; i < contigs_and_genomes.genomes.size(); ++i) {
        std::vector<float> coverages;
        for (auto& e : per_genome[i]) coverages.push_back(e.calculate_coverage(unobserved_lengths[i]));
        bool any_nonzero = false;
        for (float c : coverages) if (c > 0.0f) any_nonzero = true;
        if (any_nonzero) num_mapped_reads_total += reads_mapped_in_each_genome[i];
        if (print_zero_coverage_genomes || any_nonzero) {
          coverage_taker.start_entry(i, contigs_and_genomes.genomes[i]);
          for (size_t j = 0; j < per_genome[i].size(); ++j) {
            float coverage = coverages[j];
            if (coverage > 0.0f) {
              per_genome[i][j].print_coverage(coverage, coverage_taker);
            } else {
              uint64_t total_len = 0;
              for (uint32_t tid : genome_index_to_references[i]) total_len += header.lens[tid];
              per_genome[i][j].print_zero_coverage(coverage_taker, total_len);
            }
          }
          coverage_taker.finish_entry();
        }
      }
    }
    ReadsMapped rm;
    rm.num_mapped_reads = num_mapped_reads_total;
    rm.num_reads = bam_generated->num_detected_primary_alignments();
    reads_mapped_vector.push_back(rm);
  }
  return reads_mapped_vector;
}

struct UnobservedLengthAndFirstTid {  // genome.rs:324-328
  std::vector<uint64_t> unobserved_contig_lengths;
  size_t first_tid = 0;
};

// genome.rs:799-805
inline std::string extract_genome(uint32_t tid, const Header& header, uint8_t split_char) {
  const std::string& target_name = header.names.at(tid);
  size_t offset = target_name.find((char)split_char);
  if (offset == std::string::npos)
    throw Panic("Contig name " + target_name + " does not contain split symbol, so cannot determine which genome it belongs to");
  return target_name.substr(0, offset);
}

// genome.rs:807-853
inline UnobservedLengthAndFirstTid fill_genome_length_backwards(uint32_t current_tid, const std::string& target_genome,
                                                                bool single_genome, const Header& header,
                                                                uint8_t split_char) {
  UnobservedLengthAndFirstTid r;
  if (current_tid == 0) { r.first_tid = 0; return r; }
  uint32_t my_tid = current_tid - 1;
  while (single_genome || extract_genome(my_tid, header, split_char) == target_genome) {
    r.unobserved_contig_lengths.push_back(header.lens[my_tid]);
    if (my_tid == 0) { r.first_tid = 0; return r; }
    my_tid -= 1;
  }
  r.first_tid = (size_t)(my_tid + 1);
  return r;
}

// genome.rs:859-929
inline void print_previous_zero_coverage_genomes2(const std::optional<std::string>& last_genome,
                                                  const std::string& current_genome, uint32_t current_tid,
                                                  const std::vector<CoverageEstimator>& ests, const Header& header,
                                                  uint8_t split_char, CoverageTaker& taker) {
  std::string my_current_genome = current_genome;
  uint32_t tid = current_tid;
  std::vector<std::string> genomes_to_print;
  std::vector<size_t> genome_first_tids;
  std::vector<uint64_t> genomes_unobserved_length;
  uint64_t unobserved_length = 0;
  std::optional<uint32_t> last_first_id;
  for (;;) {
    std::string genome = extract_genome(tid, header, split_char);
    if (last_genome.has_value() && genome == *last_genome) {
      break;
    } else if (genome != my_current_genome) {
      if (last_first_id.has_value()) {
        if (!last_genome.has_value() || genome != *last_genome) {
          genome_first_tids.push_back(*last_first_id);
          genomes_to_print.push_back(my_current_genome);
          genomes_unobserved_length.push_back(unobserved_length);
        }
      }
      my_current_genome = genome;
      last_first_id = tid;
      unobserved_length = header.lens[tid];
    } else if (genome != current_genome) {
      last_first_id = tid;
      unobserved_length += header.lens[tid];
    }
    if (tid == 0) break;
    tid -= 1;
  }
  if (last_first_id.has_value()) {
    genome_first_tids.push_back(*last_first_id);
    genomes_to_print.push_back(my_current_genome);
    genomes_unobserved_length.push_back(unobserved_length);
  }
  for (size_t k = genomes_to_print.size(); k-- > 0;) {
    taker.start_entry(genome_first_tids[k], genomes_to_print[k]);
    for (auto& e : ests) e.print_zero_coverage(taker, genomes_unobserved_length[k]);
    taker.finish_entry();
  }
}

// genome.rs:331-416
inline bool print_last_genomes(uint64_t num_mapped_reads_in_current_contig, const std::optional<std::string>& last_genome,
                               UnobservedLengthAndFirstTid& unobs, const std::vector<int32_t>& ups_and_downs,
                               uint64_t total_edit_distance, uint64_t total_indels, double sum_identity,
                               const std::string& current_genome, std::vector<CoverageEstimator>& ests,
                               CoverageTaker& taker, bool print_zero_coverage_genomes, bool single_genome,
                               const Header& header, uint8_t split_char, uint32_t tid_to_print_zeros_to) {
  for (auto& e : ests) e.add_contig(ups_and_downs, num_mapped_reads_in_current_contig, total_edit_distance - total_indels, sum_identity);
  std::vector<float> coverages;
  for (auto& e : ests) coverages.push_back(e.calculate_coverage(unobs.unobserved_contig_lengths));
  bool positive_coverage = false;
  for (float c : coverages) if (c > 0.0f) positive_coverage = true;
  if (print_zero_coverage_genomes || positive_coverage) {
    if (last_genome.has_value()) {
      taker.start_entry(unobs.first_tid, *last_genome);
      for (size_t i = 0; i < ests.size(); ++i) {
        if (coverages[i] > 0.0f) ests[i].print_coverage(coverages[i], taker);
        else ests[i].print_zero_coverage(taker, 9);
      }
      taker.finish_entry();
    }
  }
  for (auto& e : ests) e.setup();
  if (print_zero_coverage_genomes && !single_genome)
    print_previous_zero_coverage_genomes2(last_genome, current_genome, tid_to_print_zeros_to, ests, header, split_char, taker);
  return positive_coverage;
}

// genome.rs:419-797
inline std::vector<ReadsMapped> mosdepth_genome_coverage(std::vector<ReaderFactory>& bam_readers, uint8_t split_char,
                                                         CoverageTaker& coverage_taker, bool print_zero_coverage_genomes,
                                                         std::vector<CoverageEstimator>& coverage_estimators,
                                                         const FlagFilter& flag_filters, bool single_genome) {
  std::vector<ReadsMapped> reads_mapped_vector;
  for (auto& gen : bam_readers) {
    std::unique_ptr<NamedBamReader> bam_generated = gen();
    std::string stoit_name = bam_generated->name();
    coverage_taker.start_stoit(stoit_name);
    const Header& header = bam_generated->header();

    auto fill_genome_length_forwards = [&](uint32_t current_tid, const std::optional<std::string>& target_genome) {  // :448-475
      std::vector<uint64_t> extras;
      if (!target_genome.has_value()) return extras;
      uint32_t total_refs = header.target_count();
      uint32_t my_tid = current_tid + 1;
      while (my_tid < total_refs) {
        if (single_genome || extract_genome(my_tid, header, split_char) == *target_genome) {
          extras.push_back(header.lens[my_tid]);
          my_tid += 1;
        } else break;
      }
      return extras;
    };
    auto fill_genome_length_backwards_to_last = [&](uint32_t current_tid, uint32_t last_tid, const std::string& target_genome) {  // :477-499
      std::vector<uint64_t> extras;
      if (current_tid == 0) return extras;
      uint32_t my_tid = last_tid + 1;
      while (my_tid < current_tid) {
        if (single_genome || extract_genome(my_tid, header, split_char) == target_genome) {
          extras.push_back(header.lens[my_tid]);
          my_tid += 1;
        } else break;
      }
      return extras;
    };

    uint32_t last_tid = 0;
    bool doing_first = true;
    std::optional<std::string> last_genome;
    UnobservedLengthAndFirstTid unobs;
    std::vector<int32_t> ups_and_downs;
    Record record;
    uint64_t num_mapped_reads_total = 0, num_mapped_reads_in_current_contig = 0, num_mapped_reads_in_current_genome = 0,
             total_edit_distance_in_current_contig = 0, total_indels_in_current_contig = 0;
    double sum_identity_in_current_contig = 0.0;
    while (bam_generated->read(record)) {
      if (!flag_filters.passes(record)) continue;
      int32_t original_tid = record.tid;
      if (!record.is_unmapped()) {
        uint32_t tid = (uint32_t)original_tid;
        std::string current_genome = single_genome ? std::string("") : extract_genome(tid, header, split_char);
        if (tid != last_tid || doing_first) {
          if (!doing_first && tid < last_tid) throw Panic(UNSORTED_MSG);
          if (doing_first) {
            for (auto& e : coverage_estimators) e.setup();
            unobs = fill_genome_length_backwards(tid, current_genome, single_genome, header, split_char);
            last_genome = current_genome;
            doing_first = false;
            if (print_zero_coverage_genomes && !single_genome)
              print_previous_zero_coverage_genomes2(std::nullopt, current_genome, tid, coverage_estimators, header, split_char, coverage_taker);
          } else if (current_genome == *last_genome) {
            for (auto& e : coverage_estimators)
              e.add_contig(ups_and_downs, num_mapped_reads_in_current_contig,
                           total_edit_distance_in_current_contig - total_indels_in_current_contig,
                           sum_identity_in_current_contig);
            auto extra = fill_genome_length_backwards_to_last(tid, last_tid, current_genome);
            unobs.unobserved_contig_lengths.insert(unobs.unobserved_contig_lengths.end(), extra.begin(), extra.end());
          } else {
            auto extra = fill_genome_length_backwards_to_last(tid, last_tid, *last_genome);
            unobs.unobserved_contig_lengths.insert(unobs.unobserved_contig_lengths.end(), extra.begin(), extra.end());
            bool positive_coverage = print_last_genomes(
                num_mapped_reads_in_current_contig, last_genome, unobs, ups_and_downs, total_edit_distance_in_current_contig,
                total_indels_in_current_contig, sum_identity_in_current_contig, current_genome, coverage_estimators,
                coverage_taker, print_zero_coverage_genomes, single_genome, header, split_char, tid);
            if (positive_coverage) num_mapped_reads_total += num_mapped_reads_in_current_genome;
            num_mapped_reads_in_current_genome = 0;
            last_genome = current_genome;
            unobs = fill_genome_length_backwards(tid, current_genome, single_genome, header, split_char);
          }
          if (tid >= header.lens.size()) throw Panic("Corrupt BAM file?");
          ups_and_downs.assign((size_t)header.lens[tid], 0);
          num_mapped_reads_in_current_contig = 0;
          total_edit_distance_in_current_contig = 0;
          total_indels_in_current_contig = 0;
          sum_identity_in_current_contig = 0.0;
          last_tid = tid;
        }
        if (!record.is_supplementary()) {
          num_mapped_reads_in_current_contig += 1;
          num_mapped_reads_in_current_genome += 1;
        }
        uint64_t aligned_len = 0;
        accumulate_cigar(record, ups_and_downs, total_indels_in_current_contig, aligned_len);
        uint64_t edit = nm(record);
        total_edit_distance_in_current_contig += edit;
        if (!record.is_supplementary() && !record.is_secondary() && aligned_len > 0)
          sum_identity_in_current_contig += ((double)aligned_len - (double)edit) / (double)aligned_len;
      }
    }
    if (doing_first && bam_generated->num_detected_primary_alignments() == 0) {
      // warn only (genome.rs:731-735)
    } else {
      if (single_genome) last_genome = std::string("genome1");
      auto extra = fill_genome_length_forwards(last_tid, last_genome);
      unobs.unobserved_contig_lengths.insert(unobs.unobserved_contig_lengths.end(), extra.begin(), extra.end());
      bool positive_coverage = print_last_genomes(
          num_mapped_reads_in_current_contig, last_genome, unobs, ups_and_downs, total_edit_distance_in_current_contig,
          total_indels_in_current_contig, sum_identity_in_current_contig, std::string(""), coverage_estimators,
          coverage_taker, print_zero_coverage_genomes, single_genome, header, split_char, header.target_count() - 1);
      if (positive_coverage) num_mapped_reads_total += num_mapped_reads_in_current_genome;
    }
    ReadsMapped rm;
    rm.num_mapped_reads = num_mapped_reads_total;
    rm.num_reads = bam_generated->num_detected_primary_alignments();
    reads_mapped_vector.push_back(rm);
  }
  return reads_mapped_vector;
}

}  // namespace oracle
