// `coverm contig` / `coverm genome` in --bam-files mode on top of libcoverm_b200.
//
// Mirrors the reference's CLI surface for this path: flag names and defaults from src/cli.rs:1670-2582
// (genome :1670-2263, contig :2265-2582), FilterParameters (coverm.rs:1648-1704), EstimatorsAndTaker
// (coverm.rs:1315-1520), parse_percentage (coverm.rs:1296-1312), run_contig / run_genome (coverm.rs:2088-2131,
// 1539-1628), per-gene coverage with --gff (coverm.rs:488-509, 1554-1590), sharded BAMs (--sharded, coverm.rs:96-239, 565-578).
// Read mapping, dereplication and FASTA genome definitions are out of scope.
//
// Library-level switches (they expose the constructor arguments the reference's unit tests use directly;
// contig.rs:290-322, genome.rs:940-1086):  --lib-estimators SPEC;SPEC  --lib-streaming  --lib-flags I,S,SEC
//   --print-reads-mapped   --timing
#pragma once
#include <algorithm>
#include <fstream>
#include <memory>
#include <iostream>
#include <sstream>
#include <thread>
#include <unordered_set>

#include "drivers.hpp"
#include "filter_command.hpp"

namespace cmbh {

struct CliOptions {
  std::string sub;
  std::vector<std::string> bam_files, methods, output_bam_files;
  bool inverse = false;
  bool device_deflate = false;  // `filter --device-deflate`: the output BAM compressed on the GPU (cmb_deflate_*)
  std::optional<uint32_t> min_read_aligned_length, min_read_aligned_length_pair;
  std::optional<float> min_read_percent_identity, min_read_aligned_percent, min_read_percent_identity_pair,
      min_read_aligned_percent_pair;
  std::optional<uint8_t> min_mapq;
  bool proper_pairs_only = false, exclude_supplementary = false, include_secondary = false, no_zeros = false;
  float min_covered_fraction = 0.0f, trim_min = 5.0f, trim_max = 95.0f;
  uint64_t contig_end_exclusion = 75;
  std::string output_format = "dense";
  std::optional<std::string> output_file, separator, genome_definition, lib_estimators, lib_flags, gff, gff_feature_type;
  bool single_genome = false, lib_streaming = false, print_reads_mapped = false, timing = false, quiet = false;
  bool sharded = false;
  std::optional<std::string> exclude_genomes_from_deshard;
  int threads = 1;
  int device = 0;
  int gpus = 1;  // > 1: every sample is range-partitioned by contig over GPUs device .. device+gpus-1 (one NCCL gather per sample)
};

struct CliResult {
  int status = 0;
  std::vector<ReadsMapped> reads_mapped;
  std::vector<SampleTiming> timings;
  std::vector<uint64_t> record_counts;
};

[[noreturn]] inline void usage(const std::string& m) { throw ExitError(2, "error: " + m); }

inline float to_f32(const std::string& s) {
  char* e = nullptr;
  const float v = strtof(s.c_str(), &e);
  if (s.empty() || *e) usage("invalid value '" + s + "': invalid float literal");
  return v;
}

inline CliOptions parse_cli(const std::vector<std::string>& args) {
  CliOptions o;
  if (args.empty()) usage("a subcommand (contig | genome) is required");
  o.sub = args[0];
  const bool filter_sub = o.sub == "filter" || o.sub == "filter-names";
  if (o.sub != "contig" && o.sub != "genome" && !filter_sub) usage("unrecognized subcommand '" + o.sub + "'");
  if (o.sub == "genome") {
    o.min_covered_fraction = 10.0f;  // cli.rs:2065
    o.methods = {"relative_abundance"};
  } else {
    o.methods = {"mean"};  // cli.rs:2521
  }
  bool methods_given = false;
  std::vector<std::string>* list = nullptr;
  for (size_t i = 1; i < args.size(); ++i) {
    const std::string& a = args[i];
    const bool flagish = a.size() >= 2 && a[0] == '-' && !((a[1] >= '0' && a[1] <= '9') || a[1] == '.');
    if (!flagish) {
      if (!list) usage("unexpected argument '" + a + "' found");
      list->push_back(a);
      continue;
    }
    list = nullptr;
    auto value = [&]() -> const std::string& {
      if (i + 1 >= args.size()) usage("a value is required for '" + a + "' but none was supplied");
      return args[++i];
    };
    if (a == "-b" || a == "--bam-files") list = &o.bam_files;
    else if (filter_sub && (a == "-o" || a == "--output-bam-files")) list = &o.output_bam_files;
    else if (filter_sub && a == "--inverse") o.inverse = true;
    else if (o.sub == "filter" && a == "--device-deflate") o.device_deflate = true;
    else if (a == "-m" || a == "--methods" || a == "--method") {
      if (!methods_given) o.methods.clear();
      methods_given = true;
      list = &o.methods;
    }
    else if (a == "--min-read-aligned-length") o.min_read_aligned_length = (uint32_t)std::stoul(value());
    else if (a == "--min-read-percent-identity") o.min_read_percent_identity = to_f32(value());
    else if (a == "--min-read-aligned-percent") o.min_read_aligned_percent = to_f32(value());
    else if (a == "--min-read-aligned-length-pair") o.min_read_aligned_length_pair = (uint32_t)std::stoul(value());
    else if (a == "--min-read-percent-identity-pair") o.min_read_percent_identity_pair = to_f32(value());
    else if (a == "--min-read-aligned-percent-pair") o.min_read_aligned_percent_pair = to_f32(value());
    else if (a == "--min-mapq") o.min_mapq = (uint8_t)std::stoul(value());
    else if (a == "--proper-pairs-only") o.proper_pairs_only = true;
    else if (a == "--exclude-supplementary") o.exclude_supplementary = true;
    else if (a == "--include-secondary") o.include_secondary = true;
    else if (a == "--no-zeros") o.no_zeros = true;
    else if (a == "--min-covered-fraction") o.min_covered_fraction = to_f32(value());
    else if (a == "--contig-end-exclusion") o.contig_end_exclusion = std::stoull(value());
    else if (a == "--trim-min") o.trim_min = to_f32(value());
    else if (a == "--trim-max") o.trim_max = to_f32(value());
    else if (a == "--output-format") o.output_format = value();
    else if (a == "-o" || a == "--output-file") o.output_file = value();
    else if ((a == "-s" || a == "--separator") && o.sub == "genome") o.separator = value();
    else if (a == "--single-genome" && o.sub == "genome") o.single_genome = true;
    else if (a == "--genome-definition" && o.sub == "genome") o.genome_definition = value();
    else if (a == "--sharded" && !filter_sub) o.sharded = true;
    else if (a == "--exclude-genomes-from-deshard" && o.sub == "genome") o.exclude_genomes_from_deshard = value();
    else if (a == "--gff") o.gff = value();
    else if (a == "--gff-feature-type") o.gff_feature_type = value();
    else if (a == "-t" || a == "--threads") o.threads = std::stoi(value());
    else if (a == "--device") o.device = std::stoi(value());
    else if (a == "--gpus") o.gpus = std::max(1, std::stoi(value()));
    else if (a == "--lib-estimators") o.lib_estimators = value();
    else if (a == "--lib-flags") o.lib_flags = value();
    else if (a == "--lib-streaming") o.lib_streaming = true;
    else if (a == "--print-reads-mapped") o.print_reads_mapped = true;
    else if (a == "--timing") o.timing = true;
    else if (a == "-q" || a == "--quiet") o.quiet = true;
    else if (a == "-v" || a == "--verbose") {}
    else usage("unexpected argument '" + a + "' found");
  }
  if (!o.lib_flags && !o.proper_pairs_only &&
      (o.min_read_aligned_length_pair || o.min_read_percent_identity_pair || o.min_read_aligned_percent_pair))
    usage("the following required arguments were not provided: --proper-pairs-only");  // cli.rs `requires`
  if (o.exclude_genomes_from_deshard && !o.sharded) usage("the following required arguments were not provided: --sharded");  // cli.rs:1698-1701
  if (o.output_format != "sparse" && o.output_format != "dense") usage("invalid value '" + o.output_format + "' for '--output-format'");
  if (o.bam_files.empty()) usage("--bam-files is required: this build implements the BAM-input coverage path only");
  return o;
}

inline float parse_percentage(std::optional<float> given) {  // coverm.rs:1296-1312
  if (!given) return 0.0f;
  float p = *given;
  if (p >= 1.0f && p <= 100.0f) p /= 100.0f;
  else if (!(p >= 0.0f && p <= 100.0f)) throw ExitError(1, "Invalid alignment percentage: '" + rust_display(p) + "'");
  return p;
}

struct Plan {  // EstimatorsAndTaker (coverm.rs:1315-1504) + FilterParameters (coverm.rs:1648-1704)
  std::vector<CoverageEstimator> estimators;
  std::vector<size_t> columns_to_normalise;
  std::optional<size_t> rpkm_column, tpm_column;
  enum class TakerKind { Streaming, Pileup, Cached } taker = TakerKind::Cached;
  CoveragePrinter printer;
  cmb_params params{};
};

inline bool wants_metabat(const CliOptions& o) {  // coverm.rs:1630-1646
  const bool has = std::find(o.methods.begin(), o.methods.end(), "metabat") != o.methods.end();
  if (has && o.methods.size() > 1) throw ExitError(1, "Cannot specify the metabat method with any other coverage methods");
  return has;
}

inline Plan make_plan(const CliOptions& o) {
  using K = CoverageEstimator::Kind;
  Plan p;
  // ---- filters
  cmb_params& f = p.params;
  f.include_improper_pairs = !o.proper_pairs_only;
  f.include_secondary = o.include_secondary;
  f.include_supplementary = !o.exclude_supplementary;
  f.min_aligned_length_single = o.min_read_aligned_length.value_or(0);
  f.min_percent_identity_single = parse_percentage(o.min_read_percent_identity);
  f.min_aligned_percent_single = parse_percentage(o.min_read_aligned_percent);
  f.min_mapq = o.min_mapq.value_or(255);
  f.min_aligned_length_pair = o.min_read_aligned_length_pair.value_or(0);
  f.min_percent_identity_pair = parse_percentage(o.min_read_percent_identity_pair);
  f.min_aligned_percent_pair = parse_percentage(o.min_read_aligned_percent_pair);
  const bool metabat = wants_metabat(o);
  if (metabat && o.sub != "contig") usage("invalid value 'metabat' for '--methods <methods>...'");
  if (metabat) {  // add_metabat_filtering_if_required (coverm.rs:1680-1693)
    f.min_percent_identity_single = 0.97001f;
    f.include_improper_pairs = f.include_supplementary = f.include_secondary = 1;
  }
  if (o.lib_flags) {
    int i, s, sec;
    if (sscanf(o.lib_flags->c_str(), "%d,%d,%d", &i, &s, &sec) != 3) usage("--lib-flags expects I,S,SEC");
    f.include_improper_pairs = i != 0;
    f.include_supplementary = s != 0;
    f.include_secondary = sec != 0;
  }
  f.filtering = f.min_percent_identity_single > 0.0f || f.min_percent_identity_pair > 0.0f || f.min_aligned_percent_single > 0.0f ||
                f.min_mapq < 255 || f.min_aligned_percent_pair > 0.0f || f.min_aligned_length_single > 0 ||
                f.min_aligned_length_pair > 0;  // doing_filtering (coverm.rs:1695-1703)

  // ---- estimators
  auto split = [](const std::string& s, char d) {
    std::vector<std::string> v;
    std::stringstream ss(s);
    std::string item;
    while (std::getline(ss, item, d)) v.push_back(item);
    return v;
  };
  const float min_fraction_covered = parse_percentage(o.min_covered_fraction);
  const uint64_t E = o.contig_end_exclusion;
  if (o.lib_estimators) {
    for (auto& spec : split(*o.lib_estimators, ';')) {
      const auto q = split(spec, ':');
      auto fl = [&](size_t i) { return to_f32(q.at(i)); };
      auto un = [&](size_t i) { return (uint64_t)std::stoull(q.at(i)); };
      CoverageEstimator e;
      if (q[0] == "mean") { e = CoverageEstimator::make(K::Mean, fl(1), un(2)); e.exclude_mismatches = q.size() > 3 && q[3] == "1"; }
      else if (q[0] == "trimmed_mean") { e = CoverageEstimator::make(K::TrimmedMean, fl(3), un(4)); e.min = fl(1); e.max = fl(2); }
      else if (q[0] == "coverage_histogram") e = CoverageEstimator::make(K::PileupCounts, fl(1), un(2));
      else if (q[0] == "variance") e = CoverageEstimator::make(K::Variance, fl(1), un(2));
      else if (q[0] == "covered_fraction") e = CoverageEstimator::make(K::CoveredFraction, fl(1));
      else if (q[0] == "covered_bases") e = CoverageEstimator::make(K::CoveredBases, fl(1));
      else if (q[0] == "rpkm") e = CoverageEstimator::make(K::RPKM, fl(1));
      else if (q[0] == "tpm") e = CoverageEstimator::make(K::TPM, fl(1));
      else if (q[0] == "length") e = CoverageEstimator::make(K::Length);
      else if (q[0] == "count") e = CoverageEstimator::make(K::ReadCount);
      else if (q[0] == "reads_per_base") e = CoverageEstimator::make(K::ReadsPerBase);
      else if (q[0] == "anir") e = CoverageEstimator::make(K::ANIr);
      else usage("bad --lib-estimators spec '" + spec + "'");
      p.estimators.push_back(e);
    }
    p.taker = (p.estimators.size() == 1 && p.estimators[0].kind == K::PileupCounts) ? Plan::TakerKind::Pileup : Plan::TakerKind::Streaming;
    p.printer.kind = CoveragePrinter::Kind::Streamed;
  } else if (metabat) {
    p.estimators = {CoverageEstimator::make(K::Length), CoverageEstimator::make(K::Mean, min_fraction_covered, E),
                    CoverageEstimator::make(K::Variance, min_fraction_covered, E)};
    p.taker = Plan::TakerKind::Cached;
    p.printer.kind = CoveragePrinter::Kind::MetabatAdjusted;
  } else {
    bool histogram = false;
    for (size_t i = 0; i < o.methods.size(); ++i) {
      const std::string& m = o.methods[i];
      if (m == "mean") p.estimators.push_back(CoverageEstimator::make(K::Mean, min_fraction_covered, E));
      else if (m == "coverage_histogram") { p.estimators.push_back(CoverageEstimator::make(K::PileupCounts, min_fraction_covered, E)); histogram = true; }
      else if (m == "trimmed_mean") {
        CoverageEstimator e = CoverageEstimator::make(K::TrimmedMean, min_fraction_covered, E);
        e.min = parse_percentage(o.trim_min);
        e.max = parse_percentage(o.trim_max);
        p.estimators.push_back(e);
      }
      else if (m == "covered_fraction") p.estimators.push_back(CoverageEstimator::make(K::CoveredFraction, min_fraction_covered));
      else if (m == "covered_bases") p.estimators.push_back(CoverageEstimator::make(K::CoveredBases, min_fraction_covered));
      else if (m == "rpkm") {
        if (p.rpkm_column) throw ExitError(1, "The RPKM column cannot be specified more than once");
        p.rpkm_column = i;
        p.estimators.push_back(CoverageEstimator::make(K::RPKM, min_fraction_covered));
      }
      else if (m == "tpm") {
        if (p.tpm_column) throw ExitError(1, "The TPM column cannot be specified more than once");
        p.tpm_column = i;
        p.estimators.push_back(CoverageEstimator::make(K::TPM, min_fraction_covered));
      }
      else if (m == "variance") p.estimators.push_back(CoverageEstimator::make(K::Variance, min_fraction_covered, E));
      else if (m == "length") p.estimators.push_back(CoverageEstimator::make(K::Length));
      else if (m == "relative_abundance" && o.sub == "genome") {
        p.columns_to_normalise.push_back(i);
        p.estimators.push_back(CoverageEstimator::make(K::Mean, min_fraction_covered, E));
      }
      else if (m == "count") p.estimators.push_back(CoverageEstimator::make(K::ReadCount));
      else if (m == "reads_per_base") p.estimators.push_back(CoverageEstimator::make(K::ReadsPerBase));
      else if (m == "anir") p.estimators.push_back(CoverageEstimator::make(K::ANIr));
      else usage("invalid value '" + m + "' for '--methods <methods>...'");
    }
    if (histogram) {
      if (o.methods.size() > 1) throw ExitError(1, "Cannot specify the coverage_histogram method with any other coverage methods");
      p.taker = Plan::TakerKind::Pileup;
      p.printer.kind = CoveragePrinter::Kind::Streamed;
    } else if (p.columns_to_normalise.empty() && !p.rpkm_column && !p.tpm_column && o.output_format == "sparse") {
      p.taker = Plan::TakerKind::Streaming;
      p.printer.kind = CoveragePrinter::Kind::Streamed;
    } else {
      p.taker = Plan::TakerKind::Cached;
      p.printer.kind = o.output_format == "sparse" ? CoveragePrinter::Kind::SparseCached : CoveragePrinter::Kind::DenseCached;
    }
  }
  if (!o.lib_estimators && min_fraction_covered != 0.0f) {  // coverm.rs:1473-1494
    for (auto& e : p.estimators) {
      const char* name = e.kind == K::ReadCount ? "counts" : e.kind == K::Length ? "length" : e.kind == K::ReadsPerBase ? "reads_per_base"
                         : e.kind == K::ANIr ? "anir" : nullptr;
      if (name)
        throw ExitError(1, std::string("The '") + name + "' coverage estimator cannot be used when --min-covered-fraction is > 0 as it does not calculate the covered fraction. You may wish to set the --min-covered-fraction to 0 and/or run this estimator separately.");
    }
  }
  // ---- what the GPU has to produce
  f.contig_end_exclusion = 0;
  f.trim_min = f.trim_max = 0.0f;
  bool need_hist = false, need_csr = false, have_window = false;
  for (auto& e : p.estimators) {
    if (e.kind == K::Mean || e.needs_histogram()) {
      if (have_window && f.contig_end_exclusion != e.contig_end_exclusion)
        throw ExitError(1, "estimators with different contig-end-exclusion values cannot share one GPU pass");
      f.contig_end_exclusion = e.contig_end_exclusion;
      have_window = true;
    }
    if (e.needs_histogram()) need_hist = true;
    if (e.kind == K::PileupCounts) need_csr = true;
    if (e.kind == K::TrimmedMean) {
      f.trim_min = e.min;
      f.trim_max = e.max;
    }
  }
  if (need_hist && o.sub == "genome") need_csr = true;  // per-genome histograms are merged from per-contig pairs
  f.want = (need_hist ? CMB_WANT_HIST : 0u) | (need_csr ? CMB_WANT_HIST_CSR : 0u);
  return p;
}

// The sample's name: the file stem, or the shards' stems joined with '|' (shard_bam_reader.rs:536-551)
inline std::string sample_name(const InputSpec& in) {
  if (in.shards.empty()) return file_stem(in.path);
  std::string name;
  for (const InputSpec& s : in.shards) name += (name.empty() ? "" : "|") + file_stem(s.path);
  return name;
}

// --exclude-genomes-from-deshard (coverm.rs:96-155, genome_exclusion.rs): genome names, one per line (empty lines skipped); a
// contig is excluded when its genome -- the name up to the separator (-s), or its genome in the definition file -- is listed.
// --single-genome excludes nothing.
inline void sharded_exclusion(const CliOptions& o, InputSpec& all) {
  if (!o.exclude_genomes_from_deshard) return;
  std::ifstream f(*o.exclude_genomes_from_deshard, std::ios::binary);
  if (!f) throw Panic("Failed to open file '" + *o.exclude_genomes_from_deshard + "' containing list of excluded genomes");
  auto names = std::make_shared<std::unordered_set<std::string>>();
  std::string line;
  while (std::getline(f, line))
    if (!line.empty()) names->insert(line);
  if (names->empty() || o.single_genome) return;
  if (o.separator) {
    if (o.separator->size() != 1) usage("invalid value '" + *o.separator + "' for '--separator <separator>': too many characters in string");
    const char sep = (*o.separator)[0];
    all.excluded = [names, sep](const std::string& contig) -> uint8_t {
      const size_t at = contig.find(sep);
      if (at == std::string::npos) return 2;
      return names->count(contig.substr(0, at)) ? 1 : 0;
    };
    all.unknown_genome_panic = "Contig name " + std::to_string((unsigned)(uint8_t)sep) +
                               " does not contain split symbol, so cannot determine which genome it belongs to";
  } else if (o.genome_definition) {
    auto gc = std::make_shared<GenomesAndContigs>(read_genome_definition_file(*o.genome_definition));
    all.excluded = [names, gc](const std::string& contig) -> uint8_t {
      const auto it = gc->contig_to_genome.find(contig);
      return it != gc->contig_to_genome.end() && names->count(gc->genomes[it->second]) ? 1 : 0;
    };
  }
}

// Runs one CLI invocation on one session (one rank).  `memory_inputs` optionally supplies BAM bytes for paths given with -b
// (matched by path).
inline CliResult run_cli_rank(const std::vector<std::string>& args, const std::vector<InputSpec>& memory_inputs, std::ostream& out,
                         std::ostream& err, DeviceSession* shared_session = nullptr) {
  CliResult res;
  try {
    const CliOptions o = parse_cli(args);
    if (o.sub == "filter" || o.sub == "filter-names") {  // coverm.rs:408-472
      if (o.sub == "filter" && o.bam_files.size() != o.output_bam_files.size())
        throw ExitError(1, "The number of input BAM files must be the same as the number output");
      cmb_params fp{};  // FilterParameters::generate_from_clap (coverm.rs:1648-1678)
      fp.include_improper_pairs = !o.proper_pairs_only;
      fp.include_secondary = o.include_secondary;
      fp.include_supplementary = !o.exclude_supplementary;
      if (o.lib_flags) {
        int i, s2, sec;
        if (sscanf(o.lib_flags->c_str(), "%d,%d,%d", &i, &s2, &sec) != 3) usage("--lib-flags expects I,S,SEC");
        fp.include_improper_pairs = i != 0;
        fp.include_supplementary = s2 != 0;
        fp.include_secondary = sec != 0;
      }
      fp.min_aligned_length_single = o.min_read_aligned_length.value_or(0);
      fp.min_percent_identity_single = parse_percentage(o.min_read_percent_identity);
      fp.min_aligned_percent_single = parse_percentage(o.min_read_aligned_percent);
      fp.min_mapq = o.min_mapq.value_or(255);
      fp.min_aligned_length_pair = o.min_read_aligned_length_pair.value_or(0);
      fp.min_percent_identity_pair = parse_percentage(o.min_read_percent_identity_pair);
      fp.min_aligned_percent_pair = parse_percentage(o.min_read_aligned_percent_pair);
      fp.filtering = 1;  // the filter always runs; which of its two paths is decided by the thresholds (filter.rs:48-61)
      std::unique_ptr<DeviceSession> own;
      DeviceSession* session = shared_session;
      if (!session) {
        own = std::make_unique<DeviceSession>(o.device, o.threads);
        session = own.get();
      }
      for (size_t k = 0; k < o.bam_files.size(); ++k) {
        InputSpec in;
        in.path = o.bam_files[k];
        for (auto& m : memory_inputs)
          if (m.path == in.path) in = m;
        if (o.sub == "filter-names") {  // printed once the input is done: an input that ends in an error prints nothing of it
          RecordsSink names;
          const FilterRun run = filter_one_input(*session, in, fp, o.inverse, names);
          if (o.timing) err << "#filter\tsample=" << k << "\trecords_out=" << run.n_records << "\tdevice=" << (run.on_device ? 1 : 0) << '\n';
          for (size_t off = 0; off + 4 <= names.bytes.size(); off += 4 + (size_t)rd_u32(names.bytes.data() + off)) out << bam_qname(names.bytes.data() + off) << '\n';
        } else if (o.device_deflate) {
          DeviceDeflateBamSink bam(o.output_bam_files[k], session->ctx());
          const FilterRun run = filter_one_input(*session, in, fp, o.inverse, bam);
          if (o.timing) {
            const cmb_deflate_stats& z = bam.stats();
            err << "#filter\tsample=" << k << "\trecords_out=" << run.n_records << "\tdevice=" << (run.on_device ? 1 : 0) << '\n';
            err << "#deflate\tsample=" << k << "\traw_bytes=" << z.raw_bytes << "\tbgzf_bytes=" << z.bgzf_bytes << "\tblocks=" << z.blocks
                << "\tstored_blocks=" << z.stored_blocks << "\tsink_calls=" << z.sink_calls << "\tdeflate_ms=" << z.ms_deflate
                << "\td2h_ms=" << z.ms_d2h << '\n';
          }
        } else {
          BamFileSink bam(o.output_bam_files[k], session->pool());
          const FilterRun run = filter_one_input(*session, in, fp, o.inverse, bam);
          if (o.timing) err << "#filter\tsample=" << k << "\trecords_out=" << run.n_records << "\tdevice=" << (run.on_device ? 1 : 0) << '\n';
        }
      }
      out.flush();
      res.status = 0;
      return res;
    }
    Plan plan = make_plan(o);
    std::ofstream file;
    std::ostream* os = &out;
    if (o.output_file && *o.output_file != "-") {
      file.open(*o.output_file);
      if (!file) throw Panic("Failed to create output file: " + *o.output_file);
      os = &file;
    }
    std::vector<InputSpec> inputs;
    for (auto& path : o.bam_files) {
      InputSpec in;
      in.path = path;
      for (auto& m : memory_inputs)
        if (m.path == path) in = m;
      inputs.push_back(in);
    }
    // --sharded makes the BAMs one sample, unless a read filter is given: then the reference ignores it (coverm.rs:168-187, 546-563)
    if (o.sharded && !plan.params.filtering) {
      InputSpec all;
      all.path = o.bam_files[0];
      all.shards = inputs;
      if (o.sub == "genome") sharded_exclusion(o, all);
      inputs = {all};
    }
    const bool output_rank = !shared_session || shared_session->is_output_rank();  // multi-GPU: only rank 0 prints
    CoverageTaker taker = plan.taker == Plan::TakerKind::Streaming ? CoverageTaker::streaming(os)
                          : plan.taker == Plan::TakerKind::Pileup  ? CoverageTaker::pileup(os)
                                                                   : CoverageTaker::cached(plan.estimators.size());
    if (!o.lib_streaming && output_rank) {  // EstimatorsAndTaker::print_headers (coverm.rs:1506-1519)
      std::vector<std::string> headers;
      for (auto& e : plan.estimators)
        for (auto& h : e.column_headers()) headers.push_back(h);
      for (size_t i : plan.columns_to_normalise) headers[i] = "Relative Abundance (%)";
      // entry type: coverm.rs:67-74 (genome), 513-520 (contig)
      plan.printer.print_headers(o.sub == "contig" ? (o.gff ? "Gene\tContig" : "Contig") : (o.gff ? "Gene\tContig\tGenome" : "Genome"), headers, *os);
    }
    std::optional<GeneDefinitions> gene_definitions;
    if (o.gff) {
      if (o.sub == "contig" && wants_metabat(o)) throw ExitError(1, "The metabat method cannot be used with --gff");
      gene_definitions = read_gff(*o.gff, o.gff_feature_type);
    }
    std::unique_ptr<DeviceSession> own;
    DeviceSession* session = shared_session;
    if (!session) {
      own = std::make_unique<DeviceSession>(o.device, o.threads);
      session = own.get();
    }
    plan.printer.pool = &session->pool();
    HostRange nvtx_drivers("host: coverage drivers (samples, estimator replay)");
    const double t_driver0 = now_s();
    DriverIO io{session, plan.params, &res.timings, &res.record_counts, (o.quiet || !output_rank) ? nullptr : &err};
    if (o.sub == "contig") {
      if (gene_definitions) res.reads_mapped = gene_coverage(inputs, taker, plan.estimators, *gene_definitions, nullptr, !o.no_zeros, io);
      else res.reads_mapped = contig_coverage(inputs, taker, plan.estimators, !o.no_zeros, io);
    } else {
      std::optional<uint8_t> separator;  // parse_separator (coverm.rs:1522-1537)
      if (o.single_genome) separator = (uint8_t)'0';
      else if (o.separator) {
        if (o.separator->size() != 1) usage("invalid value '" + *o.separator + "' for '--separator <separator>': too many characters in string");
        separator = (uint8_t)(*o.separator)[0];
      }
      if (gene_definitions) {  // coverm.rs:1554-1590: single-genome and separator modes win over a genome definition file
        GenomesAndContigs gc;
        GenomeNamer namer;
        if (o.single_genome) namer = [](const std::string&) { return std::optional<std::string>("genome1"); };
        else if (separator) {
          const char sep = (char)*separator;
          namer = [sep](const std::string& contig) -> std::optional<std::string> {
            const size_t at = contig.find(sep);
            if (at == std::string::npos) return std::nullopt;
            return contig.substr(0, at);
          };
        } else {
          if (!o.genome_definition) usage("a genome definition (--separator, --single-genome or --genome-definition) is required when using --gff in genome mode");
          gc = read_genome_definition_file(*o.genome_definition);
          namer = [&gc](const std::string& contig) -> std::optional<std::string> {
            auto it = gc.contig_to_genome.find(contig);
            if (it == gc.contig_to_genome.end()) return std::nullopt;
            return gc.genomes[it->second];
          };
        }
        res.reads_mapped = gene_coverage(inputs, taker, plan.estimators, *gene_definitions, &namer, !o.no_zeros, io);
      } else if (separator || o.single_genome) {
        res.reads_mapped = mosdepth_genome_coverage(inputs, *separator, taker, !o.no_zeros, plan.estimators, o.single_genome, io);
      } else {
        if (!o.genome_definition)
          usage("one of --separator, --single-genome or --genome-definition is required (FASTA genome definitions are out of scope)");
        const GenomesAndContigs gc = read_genome_definition_file(*o.genome_definition);
        res.reads_mapped = mosdepth_genome_coverage_with_contig_names(inputs, gc, taker, !o.no_zeros, plan.estimators, io);
      }
    }
    nvtx_drivers.end();
    HostRange nvtx_print("host: print");
    const double t_print0 = now_s();
    if (output_rank) plan.printer.finalise_printing(taker, *os, res.reads_mapped, plan.columns_to_normalise, plan.rpkm_column, plan.tpm_column);
    os->flush();
    if (o.timing) err << "#timing_run\tdrivers_s=" << (t_print0 - t_driver0) << "\tprint_s=" << (now_s() - t_print0) << '\n';
    if (o.print_reads_mapped)
      for (size_t i = 0; i < res.reads_mapped.size(); ++i)
        err << "#reads_mapped\t" << sample_name(inputs[i]) << '\t' << res.reads_mapped[i].num_mapped_reads << '\t'
            << res.reads_mapped[i].num_reads << '\n';
    if (o.timing)
      for (size_t i = 0; i < res.timings.size(); ++i) {
        const SampleTiming& t = res.timings[i];
        err << "#timing\tsample=" << i << "\trecords=" << res.record_counts[i] << "\ttotal_s=" << t.total_s << "\tdecode_s=" << t.decode_s
            << "\tsubmit_wait_s=" << t.submit_wait_s << "\tend_sample_s=" << t.end_sample_s << "\theader_s=" << t.header_s << "\tindex_s=" << t.index_s
            << "\tdevice_call_s=" << t.device_call_s << "\tgather_s=" << t.gather_s << "\tk0_ms=" << t.device.ms_zero
            << "\tk1_ms=" << t.device.ms_accumulate << "\tk2_ms=" << t.device.ms_scan << "\tk3_ms=" << t.device.ms_finalize << '\n';
      }
    res.status = 0;
  } catch (const Panic& p) {
    out.flush();
    err << "thread 'main' panicked: " << p.what() << '\n';
    res.status = 101;
  } catch (const ExitError& e) {
    out.flush();
    err << "[ERROR] " << e.what() << '\n';
    res.status = e.code;
  } catch (const std::exception& e) {
    out.flush();
    err << "thread 'main' panicked: " << e.what() << '\n';
    res.status = 101;
  }
  return res;
}

// Runs one CLI invocation.  With `--gpus N` (and no session handed in) the process drives N GPUs itself: one session and one
// host thread per GPU, an NCCL communicator over them (cmb_comm_init_local), every sample range-partitioned by contig
// (DeviceSession::process in group mode); each rank then runs the ordinary driver on the gathered table and rank 0's
// output is the result.
inline CliResult run_cli(const std::vector<std::string>& args, const std::vector<InputSpec>& memory_inputs, std::ostream& out,
                         std::ostream& err, DeviceSession* shared_session = nullptr) {
  int gpus = 1, device = 0, threads = 1;
  for (size_t i = 1; i + 1 < args.size(); ++i) {
    try {
      if (args[i] == "--gpus") gpus = std::max(1, std::stoi(args[i + 1]));
      else if (args[i] == "--device") device = std::stoi(args[i + 1]);
      else if (args[i] == "-t" || args[i] == "--threads") threads = std::stoi(args[i + 1]);
    } catch (...) {  // malformed numbers are reported by parse_cli below
    }
  }
  if (shared_session || gpus <= 1) return run_cli_rank(args, memory_inputs, out, err, shared_session);
  std::vector<std::unique_ptr<DeviceSession>> sessions;
  try {
    std::vector<cmb_ctx*> ctxs;
    for (int r = 0; r < gpus; ++r) {
      sessions.push_back(std::make_unique<DeviceSession>(device + r, std::max(1, threads / gpus)));
      ctxs.push_back(sessions.back()->ctx());
    }
    const int rc = cmb_comm_init_local(ctxs.data(), gpus);
    if (rc) throw ExitError(1, std::string("cannot create the NCCL communicator over the GPUs: ") + cmb_last_error(ctxs[0]));
    for (int r = 0; r < gpus; ++r) sessions[(size_t)r]->adopt_local_group(r, gpus);
  } catch (const std::exception& e) {
    err << "[ERROR] " << e.what() << '\n';
    CliResult res;
    res.status = 1;
    return res;
  }
  std::vector<std::thread> others;
  for (int r = 1; r < gpus; ++r)
    others.emplace_back([&, r]() {
      std::ostringstream o, e;  // the other ranks compute the same table; only rank 0's text is kept
      std::vector<std::string> a = args;
      for (size_t i = 1; i + 1 < a.size(); ++i)
        if (a[i] == "-o" || a[i] == "--output-file") a[i + 1] = "-";
      run_cli_rank(a, memory_inputs, o, e, sessions[(size_t)r].get());
    });
  CliResult res = run_cli_rank(args, memory_inputs, out, err, sessions[0].get());
  for (auto& t : others) t.join();
  return res;
}

}  // namespace cmbh
