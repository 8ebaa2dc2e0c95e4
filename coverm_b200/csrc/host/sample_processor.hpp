// One BAM file ("stoit") through the device library: decode -> pinned SoA batches -> cmb_submit_batch -> per-contig
// integer statistics.  This is the record loop of contig.rs:107-215 / genome.rs:109-227, 516-729 with the CIGAR walk
// and the filters moved onto the GPU; the host keeps only what needs read names (mate matching, filter.rs:149-224).
#pragma once
#include <chrono>
#include <cstdio>

#include "bam_source.hpp"
#include "decode_runner.hpp"
#include "genes.hpp"
#include "shard_range.hpp"

// Referenced weakly: the host code also links against stand-ins of the device library that predate per-gene sharding (the CPU
// emulator of the ABI).  With such a library a group run with --gff stops with an error; libcoverm_b200 always defines it.
extern "C" int cmb_set_genes_range(cmb_ctx* ctx, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes,
                                   uint32_t tid_begin, uint32_t tid_end) __attribute__((weak));

// Referenced weakly for the same reason: the emulator without the sharded-input entry points stops a --sharded run with an error.
extern "C" int cmb_shard_begin(cmb_ctx* ctx, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded) __attribute__((weak));
extern "C" int cmb_shard_add(cmb_ctx* ctx, const cmb_bgzf_input* in, cmb_bgzf_result* out) __attribute__((weak));
extern "C" int cmb_shard_finish(cmb_ctx* ctx, cmb_shard_result* out) __attribute__((weak));
// ... and so are the entry points of sharded input over a group of ranks: without them a group --sharded run stops on every rank.
extern "C" int cmb_shard_begin_range(cmb_ctx* ctx, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded, uint32_t shard_begin,
                                     uint32_t shard_end) __attribute__((weak));
extern "C" int cmb_shard_score(cmb_ctx* ctx, const uint64_t* n_primary) __attribute__((weak));
extern "C" int cmb_shard_exchange(cmb_ctx* ctx, const uint32_t* shard_cuts) __attribute__((weak));
extern "C" int cmb_shard_export(cmb_ctx* ctx, uint32_t shard, int32_t* scores, uint64_t* names) __attribute__((weak));
extern "C" int cmb_shard_import(cmb_ctx* ctx, uint32_t shard, const int32_t* scores, const uint64_t* names) __attribute__((weak));
extern "C" int cmb_shard_choose(cmb_ctx* ctx, uint64_t* err_key) __attribute__((weak));
extern "C" int cmb_shard_finish_group(cmb_ctx* ctx, uint64_t err_key, cmb_shard_result* out) __attribute__((weak));

namespace cmbh {

// NVTX range of a host-side stage (cmb_nvtx_push / cmb_nvtx_pop of the device library; no-ops without a profiler)
struct HostRange {
  bool open = true;
  explicit HostRange(const char* name) { cmb_nvtx_push(name); }
  void end() {
    if (open) {
      cmb_nvtx_pop();
      open = false;
    }
  }
  ~HostRange() { end(); }
  HostRange(const HostRange&) = delete;
  HostRange& operator=(const HostRange&) = delete;
};

inline double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

inline std::string file_stem(const std::string& path) {  // Path::file_stem (bam_generator.rs:360-365)
  size_t s = path.find_last_of('/');
  std::string base = s == std::string::npos ? path : path.substr(s + 1);
  size_t d = base.find_last_of('.');
  if (d == std::string::npos || d == 0) return base;
  return base.substr(0, d);
}

struct SampleTiming {
  double total_s = 0, decode_s = 0, submit_wait_s = 0, end_sample_s = 0;
  double header_s = 0, index_s = 0, device_call_s = 0;  // inside decode_s: header parse, BGZF block index (+ range probes), cmb_submit_bgzf
  cmb_sample_timing device{};
  uint64_t h2d_bytes = 0;
  bool device_decode = false;
  cmb_bgzf_result bgzf{};
  uint32_t decode_launches = 0;
  // multi-GPU contig sharding
  uint32_t group_ranks = 1, shard_blocks = 0, total_blocks = 0, range_probes = 0, tid_begin = 0, tid_end = 0;
  double gather_s = 0;
};

struct SampleResult {
  std::string stoit_name;
  std::shared_ptr<Header> hdr = std::make_shared<Header>();  // shared with the session's header cache
  const Header& header() const { return *hdr; }
  const cmb_contig_stats* rows = nullptr;  // n_ref rows in the session's page-locked buffer; valid until the next process()
  std::vector<cmb_hist_pair> pairs;
  uint64_t num_detected_primary_alignments = 0;  // bam_generator.rs:113-119 / filter.rs:94-96,129-131
  uint64_t n_records = 0;                        // every record read from the file
  SampleTiming timing;
  // gene mode (--gff): rows are per gene (genes->entries order)
  std::shared_ptr<const ResolvedGenes> genes;
  std::vector<uint8_t> contig_seen;  // per tid: a record that passed the filters mapped here
  uint64_t kept_primary = 0;         // primaries among those records (genes.rs:249-252)
};

[[noreturn]] inline void throw_device_error(cmb_ctx* ctx, int rc) {
  const std::string msg = cmb_last_error(ctx);
  if (rc == CMB_E_UNSORTED || rc == CMB_E_NM || rc == CMB_E_BOUNDS || rc == CMB_E_SHARD_PANIC) throw Panic(msg);
  if (rc == CMB_E_SHARD_EXIT) throw ExitError(1, msg);
  throw ExitError(1, "device error " + std::to_string(rc) + ": " + msg);
}

class DeviceSession {
 public:
  DeviceSession(int device, int threads, uint32_t batch_records = 1u << 20) : pool_(threads) {
    if (const char* e = getenv("CMB_BATCH_RECORDS")) batch_records = std::max(40000u, (uint32_t)strtoul(e, nullptr, 10));
    cmb_device_cfg cfg{};
    cfg.device = device;
    cfg.batch_records = batch_records;
    cfg.batch_intervals = batch_records + batch_records / 2;
    cfg.n_staging = 4;
    int rc = cmb_create(&cfg, &ctx_);
    if (rc != CMB_OK) throw ExitError(1, std::string("cannot create the CUDA coverage context: ") + cmb_last_error(nullptr));
    batch_records_ = cfg.batch_records;
    batch_intervals_ = cfg.batch_intervals;
    n_staging_ = cfg.n_staging;
  }
  ~DeviceSession() {
    cmb_host_free(rows_buf_);
    cmb_destroy(ctx_);
  }
  DeviceSession(const DeviceSession&) = delete;
  ThreadPool& pool() { return pool_; }
  cmb_ctx* ctx() { return ctx_; }

  // Restrict this session to the contig shard [begin, end) (multi-GPU); (0, UINT32_MAX) = everything.
  void set_shard(uint32_t begin, uint32_t end) { shard_begin_ = begin; shard_end_ = end; ref_lens_.clear(); }

  // Per-gene coverage: the following samples report one row per gene of `defs` (resolved against each sample's header)
  // instead of one per contig; nullptr returns to contig rows.
  void set_gene_definitions(const GeneDefinitions* defs, const GenomeNamer* namer) {
    gene_defs_ = defs;
    gene_namer_ = namer;
    ref_lens_.clear();
    gene_cache_.reset();
  }

  // Makes this session rank `rank` of `n_ranks` that process every sample TOGETHER (contigs range-partitioned by summed
  // length, each rank decoding only its BGZF block range, one gather of the per-contig table; SURVEY.md 8e).  The ranks
  // exchange either over NCCL inside the device library (`nccl_id` from cmb_comm_unique_id, shared by the caller) or, for
  // hosts without NCCL between them (MPI, gloo, tests), through the caller's own all-gather of host buffers.
  typedef int (*AllGatherFn)(void* user, const void* send, size_t bytes_per_rank, void* recv);
  void set_group(int rank, int n_ranks, const uint8_t* nccl_id, AllGatherFn fn, void* user) {
    if (n_ranks < 1 || rank < 0 || rank >= n_ranks) throw ExitError(1, "set_group: bad rank / group size");
    if (n_ranks > 1 && !nccl_id && !fn) throw ExitError(1, "set_group: a group needs an NCCL id or an all-gather callback");
    if (group_nccl_) cmb_comm_destroy(ctx_);
    group_rank_ = rank;
    group_n_ = n_ranks;
    group_nccl_ = false;
    group_fn_ = fn;
    group_user_ = user;
    if (n_ranks > 1 && nccl_id) {
      const int rc = cmb_comm_init(ctx_, nccl_id, rank, n_ranks);
      if (rc) throw ExitError(1, std::string("cannot create the NCCL communicator: ") + cmb_last_error(ctx_));
      group_nccl_ = true;
    }
    ref_lens_.clear();
  }
  // cmb_comm_init_local was called on this session's context by the owner of all the ranks (one process, several GPUs)
  void adopt_local_group(int rank, int n_ranks) {
    group_rank_ = rank;
    group_n_ = n_ranks;
    group_nccl_ = n_ranks > 1;
    group_fn_ = nullptr;
    ref_lens_.clear();
  }
  int group_rank() const { return group_rank_; }
  int group_size() const { return group_n_; }
  // After the gather every rank holds the complete table, but only one needs to turn it into text: rank 0 replays the
  // estimators and prints, the others return an empty table -- unless every_rank_prints (tests: proves the gather is complete
  // everywhere).
  void set_every_rank_prints(bool v) { every_rank_prints_ = v; }
  bool is_output_rank() const { return group_n_ <= 1 || group_rank_ == 0 || every_rank_prints_; }

  // One sample.  In a group every rank must call this for the same input (it is collective).
  SampleResult process(const InputSpec& in, const cmb_params& params) {
    if (group_n_ <= 1) return in.shards.empty() ? process_local(in, params, nullptr) : process_sharded(in, params);
    // ---- local phase: this rank's contigs, from this rank's block range (sharded input: from this rank's shards).  Nothing
    //      may escape before the ranks have compared notes: a rank that failed still takes part in the exchange, and then
    //      every rank fails the same way.
    ShardState sh;
    SampleResult res;
    RankSummary mine = attempt([&](RankSummary& mine) {
      res = in.shards.empty() ? process_local(in, params, &sh) : process_sharded_group(in, params, sh);
      mine.n_records = res.n_records;
      mine.n_primary = res.num_detected_primary_alignments;
      mine.counts_global = sh.counts_global ? 1 : 0;
      mine.n_pairs = sh.n_pairs;
      mine.kept_primary = res.kept_primary;
      int32_t lo = INT32_MAX, hi = INT32_MIN;
      if (!sh.counts_global) cmb_kept_tid_range(ctx_, &lo, &hi);
      mine.min_tid = lo;
      mine.max_tid = hi;
    });
    HostRange nvtx_gather("host: rank summaries + table gather");
    const double t_g0 = now_s();
    std::vector<RankSummary> all((size_t)group_n_);
    group_allgather(&mine, all.data(), sizeof(RankSummary));
    for (const RankSummary& s : all) {  // the lowest failing rank's error, on every rank
      if (s.kind == 1) throw Panic(s.message);
      if (s.kind == 2) throw ExitError(s.code, s.message);
    }
    check_rank_order(all);
    // ---- the gather of the path: every rank ends up with the complete per-contig (gene mode: per-gene) table + histogram pairs
    const uint32_t n_ref = (uint32_t)res.hdr->names.size();
    std::vector<uint64_t> pair_base((size_t)group_n_ + 1, 0);
    for (int r = 0; r < group_n_; ++r) pair_base[(size_t)r + 1] = pair_base[(size_t)r] + all[(size_t)r].n_pairs;
    const bool csr = params.want & CMB_WANT_HIST_CSR;
    res.pairs.clear();
    if (csr) res.pairs.resize(pair_base[(size_t)group_n_]);
    ensure_rows(res.genes ? std::max<uint32_t>(1, (uint32_t)res.genes->entries.size()) : n_ref);
    if (res.genes && res.genes->entries.empty()) {
      // no gene rows to report (every printed row is a gene's): nothing to gather
    } else if (group_nccl_) {
      const int rc = cmb_allgather_stats(ctx_, sh.row_cuts.data(), csr ? pair_base.data() : nullptr, rows_buf_, csr ? res.pairs.data() : nullptr);
      if (rc) throw_device_error(ctx_, rc);
    } else {
      gather_rows_through_host(sh, res, all, pair_base, csr);
    }
    if (res.genes) gather_contig_seen(sh, res);
    res.rows = rows_buf_;
    fold_counters(all, res);
    res.timing.gather_s = now_s() - t_g0;
    res.timing.total_s += res.timing.gather_s;
    res.timing.group_ranks = (uint32_t)group_n_;
    return res;
  }

 private:
  struct ShardState {
    std::vector<uint32_t> cuts;      // contig (tid) cuts: rank r owns the records of contigs [cuts[r], cuts[r+1])
    std::vector<uint32_t> row_cuts;  // the ranks' row ranges: == cuts, or in gene mode the genes of those contigs
    bool counts_global = false;  // this rank read the whole file (host decode): its counters cover every record
    uint64_t n_pairs = 0;
  };
  struct RankSummary {  // what the ranks tell each other before the table gather (fixed size: it travels by all-gather)
    int32_t kind;       // 0 fine, 1 Panic, 2 ExitError
    int32_t code;
    uint64_t n_records, n_primary, n_pairs;
    uint64_t kept_primary;  // gene mode: primaries among the kept records of the rank's own contigs
    int32_t min_tid, max_tid;
    uint32_t counts_global, reserved;
    char message[208];
  };

  // `f` run with its failure, if any, recorded as what this rank tells the others (the fields f filled are kept)
  template <class F>
  static RankSummary attempt(F&& f) {
    RankSummary mine{};
    try {
      f(mine);
    } catch (const Panic& e) {
      mine.kind = 1;
      mine.code = 101;
      snprintf(mine.message, sizeof mine.message, "%s", e.what());
    } catch (const ExitError& e) {
      mine.kind = 2;
      mine.code = e.code;
      snprintf(mine.message, sizeof mine.message, "%s", e.what());
    } catch (const std::exception& e) {
      mine.kind = 1;
      mine.code = 101;
      snprintf(mine.message, sizeof mine.message, "%s", e.what());
    }
    return mine;
  }

  // Every rank's summary and `bytes` of payload behind it (all ranks send the same size); the lowest failing rank's error is
  // thrown on every rank.  Returns the ranks' payloads, rank after rank.
  std::vector<uint8_t> agree(const RankSummary& mine, const void* payload, size_t bytes) {
    const size_t each = sizeof(RankSummary) + bytes;
    std::vector<uint8_t> send(each), recv(each * (size_t)group_n_), out(bytes * (size_t)group_n_);
    memcpy(send.data(), &mine, sizeof mine);
    if (bytes) memcpy(send.data() + sizeof mine, payload, bytes);
    group_allgather(send.data(), recv.data(), each);
    for (int r = 0; r < group_n_; ++r) {
      RankSummary s;
      memcpy(&s, recv.data() + (size_t)r * each, sizeof s);
      if (s.kind == 1) throw Panic(s.message);
      if (s.kind == 2) throw ExitError(s.code, s.message);
      if (bytes) memcpy(out.data() + (size_t)r * bytes, recv.data() + (size_t)r * each + sizeof s, bytes);
    }
    return out;
  }

  // The cross-rank half of the sortedness check (contig.rs:129-132): each rank has verified its own (overlapping) stretch of
  // the stream; the kept tids of the ranks' exclusive shares must not decrease from rank to rank either.
  static void check_rank_order(const std::vector<RankSummary>& all) {
    int64_t seen_max = INT64_MIN;
    for (const RankSummary& s : all) {
      if (s.counts_global || s.min_tid > s.max_tid) continue;
      if ((int64_t)s.min_tid < seen_max)
        throw Panic("BAM file appears to be unsorted. Input BAM files must be sorted by reference (i.e. by samtools sort)");
      seen_max = std::max<int64_t>(seen_max, s.max_tid);
    }
  }
  // The whole-file counters: taken from the first rank that had to read the whole file, else summed over the ranks' owned records.
  // kept_primary is always summed: whichever part of the file a rank read, K1 counted only its own contigs' records.
  static void fold_counters(const std::vector<RankSummary>& all, SampleResult& res) {
    res.kept_primary = 0;
    for (const RankSummary& s : all) res.kept_primary += s.kept_primary;
    res.n_records = res.num_detected_primary_alignments = 0;
    for (const RankSummary& s : all) {
      if (s.counts_global) {
        res.n_records = s.n_records;
        res.num_detected_primary_alignments = s.n_primary;
        return;
      }
      res.n_records += s.n_records;
      res.num_detected_primary_alignments += s.n_primary;
    }
  }

  void group_allgather(const void* send, void* recv, size_t bytes) {
    if (group_nccl_) {
      const int rc = cmb_comm_allgather(ctx_, send, recv, bytes);
      if (rc) throw ExitError(1, std::string("all-gather over NCCL failed: ") + cmb_last_error(ctx_));
    } else if (group_fn_(group_user_, send, bytes, recv) != 0) {
      throw ExitError(1, "the caller's all-gather failed");
    }
  }

  void ensure_rows(uint32_t n_ref) {
    if (rows_cap_ < (size_t)n_ref + 1) {
      cmb_host_free(rows_buf_);
      rows_cap_ = 0;
      rows_buf_ = (cmb_contig_stats*)cmb_host_alloc(sizeof(cmb_contig_stats) * ((size_t)n_ref + 1));
      if (!rows_buf_) throw ExitError(1, "cannot allocate the page-locked result buffer");
      rows_cap_ = (size_t)n_ref + 1;
    }
  }

  // Table gather without NCCL: own row range (and own pairs, offsets made global) through the caller's all-gather, padded
  // to the largest share.
  void gather_rows_through_host(const ShardState& sh, SampleResult& res, const std::vector<RankSummary>& all,
                                const std::vector<uint64_t>& pair_base, bool csr) {
    const int N = group_n_, me = group_rank_;
    size_t max_rows = 0, max_pairs = 0;
    for (int r = 0; r < N; ++r) {
      max_rows = std::max<size_t>(max_rows, sh.row_cuts[(size_t)r + 1] - sh.row_cuts[(size_t)r]);
      max_pairs = std::max<size_t>(max_pairs, all[(size_t)r].n_pairs);
    }
    const std::vector<uint32_t>& cuts = sh.row_cuts;
    const uint32_t b = cuts[(size_t)me], e = cuts[(size_t)me + 1];
    if (max_rows) {
      std::vector<cmb_contig_stats> send(max_rows), recv(max_rows * (size_t)N);
      for (uint32_t t = b; t < e; ++t) {
        send[t - b] = rows_buf_[t];
        if (csr && send[t - b].hist_count) send[t - b].hist_offset += pair_base[(size_t)me];
      }
      group_allgather(send.data(), recv.data(), max_rows * sizeof(cmb_contig_stats));
      for (int r = 0; r < N; ++r)
        for (uint32_t t = cuts[(size_t)r]; t < cuts[(size_t)r + 1]; ++t) rows_buf_[t] = recv[(size_t)r * max_rows + (t - cuts[(size_t)r])];
    }
    if (csr && max_pairs) {
      std::vector<cmb_hist_pair> send(max_pairs), recv(max_pairs * (size_t)N);
      std::copy(local_pairs_.begin(), local_pairs_.end(), send.begin());
      group_allgather(send.data(), recv.data(), max_pairs * sizeof(cmb_hist_pair));
      for (int r = 0; r < N; ++r)
        std::copy(recv.begin() + (ptrdiff_t)((size_t)r * max_pairs), recv.begin() + (ptrdiff_t)((size_t)r * max_pairs + all[(size_t)r].n_pairs),
                  res.pairs.begin() + (ptrdiff_t)pair_base[(size_t)r]);
    }
  }

  // Gene mode: each rank's contig_seen covers its own contigs only; the ranks' slices, padded to the largest, complete it.
  void gather_contig_seen(const ShardState& sh, SampleResult& res) {
    const int N = group_n_, me = group_rank_;
    size_t max_tids = 0;
    for (int r = 0; r < N; ++r) max_tids = std::max<size_t>(max_tids, sh.cuts[(size_t)r + 1] - sh.cuts[(size_t)r]);
    if (!max_tids) return;
    std::vector<uint8_t> send(max_tids, 0), recv(max_tids * (size_t)N);
    std::copy(res.contig_seen.begin() + sh.cuts[(size_t)me], res.contig_seen.begin() + sh.cuts[(size_t)me + 1], send.begin());
    group_allgather(send.data(), recv.data(), max_tids);
    for (int r = 0; r < N; ++r)
      std::copy(recv.begin() + (ptrdiff_t)((size_t)r * max_tids), recv.begin() + (ptrdiff_t)((size_t)r * max_tids + sh.cuts[(size_t)r + 1] - sh.cuts[(size_t)r]),
                res.contig_seen.begin() + sh.cuts[(size_t)r]);
  }

  // cmb_set_params; whether the parameters filter read pairs
  bool set_params(const cmb_params& params) {
    cmb_filter_mode mode{};
    const int rc = cmb_set_params(ctx_, &params, &mode);
    if (rc) throw_device_error(ctx_, rc);
    return mode.filter_pairs;
  }

  SampleResult process_local(const InputSpec& in, const cmb_params& params, ShardState* shard) {
    HostRange nvtx_sample("host: sample");
    SampleCall c(*this, in, params, shard);
    c.header();
    c.reference();
    {
      HostRange nvtx_index("host: BGZF block index (+ range probes in a group)");
      const double t_index0 = now_s();
      const BlockIndex& bx = c.index(t_index0);
      // Device-side decode first (compressed blocks cross PCIe, the GPU inflates and parses them); the host pipeline runs
      // when the input is not BGZF, when CMB_HOST_DECODE is set, or when the device declines the stream.  Pair filtering
      // included: the device matches mates itself (cmb_pairs.cuh); the host's map-based matching is the fallback.
      if (bx.bgzf && !getenv("CMB_HOST_DECODE")) c.device_decode(bx, nvtx_index, t_index0);
      if (!c.decoded_on_device && !c.pair_mode) c.host_pipeline(bx);
    }
    if (!c.decoded_on_device && c.pair_mode) c.pair_fallback();
    return c.end_sample();
  }

  // Ends the sample a sharded run began when the run stops on an error, so that the session can take the next sample
  struct SampleCloser {
    cmb_ctx* ctx;
    bool open = false;
    ~SampleCloser() {
      uint64_t n_pairs = 0;
      if (open) cmb_end_sample(ctx, nullptr, nullptr, 0, &n_pairs);
    }
  };

  // --sharded (ReadSortedShardedBamReader, shard_bam_reader.rs): the shards' headers concatenated into one reference, every
  // shard decoded on the device in turn, each pair's best shard chosen there and the winners accumulated as one sample.
  SampleResult process_sharded(const InputSpec& in, const cmb_params& params) {
    HostRange nvtx_sample("host: sharded sample");
    const double t0 = now_s();
    if (!cmb_shard_begin || !cmb_shard_add || !cmb_shard_finish) throw ExitError(1, "this device library has no cmb_shard_*: --sharded needs it");
    if (set_params(params)) throw ExitError(1, "--sharded input takes no read-pair filter");
    SampleResult res;
    const size_t K = in.shards.size();
    std::vector<uint32_t> offsets;
    sharded_header(in, res, offsets, nullptr);
    const uint32_t n_ref = (uint32_t)res.hdr->names.size();
    const uint32_t n_rows = sharded_reference(res, nullptr, 0, n_ref);
    SampleCloser closer{ctx_, true};
    const std::vector<uint8_t> excluded = sharded_excluded(in, res);
    int rc;
    if ((rc = cmb_shard_begin(ctx_, (uint32_t)K, offsets.data(), in.excluded ? excluded.data() : nullptr))) throw_device_error(ctx_, rc);
    double decode_s = 0;
    for (size_t k = 0; k < K; ++k) add_shard(in, k, res, decode_s);
    cmb_shard_result sr{};
    if ((rc = cmb_shard_finish(ctx_, &sr))) throw_shard_error(in, rc);
    res.num_detected_primary_alignments = sr.n_records;
    print_shard_stats(K, sr);
    const double t_dec = now_s();
    closer.open = false;
    sharded_end(res, params, n_ref, n_rows, nullptr);
    const double t1 = now_s();
    res.timing.total_s = t1 - t0;
    res.timing.decode_s = decode_s;
    res.timing.end_sample_s = t1 - t_dec;
    return res;
  }

  // --sharded over the ranks of a group: rank r decodes the whole shards [cuts[r], cuts[r + 1]) (shard_run_cuts over the files'
  // sizes) and owns their contigs.  A pair's winning records lie on the winning shard's contigs, so only every pair's scores
  // travel: exchange A the shards' primary counts, exchange B the score columns and shard 0's name hashes, exchange C the
  // smallest error key.  Every rank then reaches the winners and the error the one-GPU run reaches, sorts and submits the
  // winners of its own shards, and leaves its rows to the group's gather (process()).
  SampleResult process_sharded_group(const InputSpec& in, const cmb_params& params, ShardState& sh) {
    HostRange nvtx_sample("host: sharded sample (group)");
    const double t0 = now_s();
    const int N = group_n_, me = group_rank_;
    const size_t K = in.shards.size();
    SampleResult res;
    std::vector<uint32_t> offsets, scut;
    std::vector<uint64_t> n_prim(K, 0);
    double decode_s = 0;
    uint32_t n_ref = 0, n_rows = 0;
    int rc;
    SampleCloser closer{ctx_};
    // ---- this rank's shards, decoded and compacted
    RankSummary mine = attempt([&](RankSummary&) {
      if (!cmb_shard_begin_range || !cmb_shard_add || !cmb_shard_score || !cmb_shard_choose || !cmb_shard_finish_group ||
          (group_nccl_ ? !cmb_shard_exchange : (!cmb_shard_export || !cmb_shard_import)))
        throw ExitError(1, "this device library has no cmb_shard_begin_range / cmb_shard_score / cmb_shard_choose / cmb_shard_finish_group "
                           "(and cmb_shard_exchange, or cmb_shard_export / cmb_shard_import): --sharded over several ranks needs them");
      if (set_params(params)) throw ExitError(1, "--sharded input takes no read-pair filter");
      std::vector<uint64_t> sizes;
      sharded_header(in, res, offsets, &sizes);
      n_ref = (uint32_t)res.hdr->names.size();
      scut = shard_run_cuts(sizes, N);
      sh.cuts.assign((size_t)N + 1, n_ref);
      for (int r = 0; r <= N; ++r)
        if (scut[(size_t)r] < K) sh.cuts[(size_t)r] = offsets[scut[(size_t)r]];
      n_rows = sharded_reference(res, &sh, sh.cuts[(size_t)me], sh.cuts[(size_t)me + 1]);
      closer.open = true;
      const std::vector<uint8_t> excluded = sharded_excluded(in, res);
      if ((rc = cmb_shard_begin_range(ctx_, (uint32_t)K, offsets.data(), in.excluded ? excluded.data() : nullptr, scut[(size_t)me], scut[(size_t)me + 1])))
        throw_device_error(ctx_, rc);
      for (uint32_t k = scut[(size_t)me]; k < scut[(size_t)me + 1]; ++k) n_prim[k] = add_shard(in, k, res, decode_s);
    });
    // ---- exchange A: every shard's primaries (each from its owner; the others send 0)
    double xs = 0;
    double a = now_s();
    const std::vector<uint8_t> counts = agree(mine, n_prim.data(), 8 * K);
    for (size_t k = 0; k < K; ++k) {
      n_prim[k] = 0;
      for (int r = 0; r < N; ++r) {
        uint64_t v;
        memcpy(&v, counts.data() + ((size_t)r * K + k) * 8, 8);
        n_prim[k] += v;
      }
    }
    xs += now_s() - a;
    const uint64_t n0 = n_prim[0], n_pairs = *std::min_element(n_prim.begin(), n_prim.end()) / 2;
    agree(attempt([&](RankSummary&) {
            if ((rc = cmb_shard_score(ctx_, n_prim.data()))) throw_device_error(ctx_, rc);
          }),
          nullptr, 0);
    // ---- exchange B: the score table and shard 0's names on every rank
    a = now_s();
    if (group_nccl_) {
      if ((rc = cmb_shard_exchange(ctx_, scut.data()))) throw ExitError(1, std::string("score exchange over NCCL failed: ") + cmb_last_error(ctx_));
    } else {
      exchange_scores_through_host(scut, n_pairs, n0);
    }
    xs += now_s() - a;
    // ---- exchange C: the choice on every rank, and the smallest error key of the group
    a = now_s();
    uint64_t key = ~0ull;
    const std::vector<uint8_t> keys = agree(attempt([&](RankSummary&) {
                                              if ((rc = cmb_shard_choose(ctx_, &key))) throw_device_error(ctx_, rc);
                                            }),
                                            &key, 8);
    for (int r = 0; r < N; ++r) {
      uint64_t v;
      memcpy(&v, keys.data() + (size_t)r * 8, 8);
      key = std::min(key, v);
    }
    xs += now_s() - a;
    cmb_shard_result sr{};
    if ((rc = cmb_shard_finish_group(ctx_, key, &sr))) throw_shard_error(in, rc);
    // the sample's primaries are a global count: rank 0 alone reports them, the group's sum of the ranks' counters is then right
    res.num_detected_primary_alignments = me == 0 ? sr.n_records : 0;
    print_shard_stats(K, sr);
    if (getenv("CMB_PIPELINE_STATS"))
      fprintf(stderr, "#shard_exchange\tbytes=%llu\tms=%.3f\trank=%d\tshards=%u..%u\tdecode_ms=%.3f\tchoose_ms=%.3f\tsort_ms=%.3f\n",
              (unsigned long long)(4 * K * n_pairs + 8 * n0), xs * 1e3, me, scut[(size_t)me], scut[(size_t)me + 1], sr.ms_decode, sr.ms_choose, sr.ms_sort);
    const double t_dec = now_s();
    closer.open = false;
    sharded_end(res, params, n_ref, n_rows, &sh);
    const double t1 = now_s();
    res.timing.total_s = t1 - t0;
    res.timing.decode_s = decode_s;
    res.timing.end_sample_s = t1 - t_dec;
    return res;
  }

  // Exchange B without NCCL: each rank's columns (shard 0's owner: its names first) through the caller's all-gather, padded to
  // the largest share
  void exchange_scores_through_host(const std::vector<uint32_t>& scut, uint64_t n_pairs, uint64_t n0) {
    const int N = group_n_, me = group_rank_;
    auto owns0 = [&](int r) { return scut[(size_t)r] == 0 && scut[(size_t)r + 1] > 0; };
    auto share = [&](int r) { return (size_t)(scut[(size_t)r + 1] - scut[(size_t)r]) * n_pairs * 4 + (owns0(r) ? 8 * n0 : 0); };
    size_t max_b = 0;
    for (int r = 0; r < N; ++r) max_b = std::max(max_b, share(r));
    if (!max_b) return;
    std::vector<uint8_t> send(max_b), recv(max_b * (size_t)N);
    // names (8-byte aligned) at the front, then the columns in shard order
    auto columns = [&](int r, uint8_t* base, bool out) {
      uint64_t* names = owns0(r) ? (uint64_t*)base : nullptr;
      int32_t* col = (int32_t*)(base + (names ? 8 * n0 : 0));
      for (uint32_t k = scut[(size_t)r]; k < scut[(size_t)r + 1]; ++k, col += n_pairs) {
        const int rc = out ? cmb_shard_export(ctx_, k, col, k == 0 ? names : nullptr) : cmb_shard_import(ctx_, k, col, k == 0 ? names : nullptr);
        if (rc) throw_device_error(ctx_, rc);
      }
    };
    columns(me, send.data(), true);
    group_allgather(send.data(), recv.data(), max_b);
    for (int r = 0; r < N; ++r)
      if (r != me) columns(r, recv.data() + (size_t)r * max_b, false);
  }

  // The shards' headers concatenated (shard_bam_reader.rs:315-336) into res.hdr: offsets[k] = the targets of shards 0 .. k-1;
  // `sizes` (when given): the shard files' bytes
  void sharded_header(const InputSpec& in, SampleResult& res, std::vector<uint32_t>& offsets, std::vector<uint64_t>* sizes) {
    const size_t K = in.shards.size();
    offsets.assign(K, 0);
    auto hdr = std::make_shared<Header>();
    for (size_t k = 0; k < K; ++k) {
      res.stoit_name += (k ? "|" : "") + file_stem(in.shards[k].path);
      const BamInput input(in.shards[k]);
      if (sizes) sizes->push_back(input.size());
      InflateStream stream(input.data(), input.size(), pool_, 1u << 20);
      std::vector<uint8_t> buf;
      const BamHeader h = read_bam_header(stream, buf, in.shards[k].path);
      offsets[k] = (uint32_t)hdr->names.size();
      hdr->names.insert(hdr->names.end(), h.header->names.begin(), h.header->names.end());
      hdr->lens.insert(hdr->lens.end(), h.header->lens.begin(), h.header->lens.end());
    }
    res.hdr = hdr;
  }

  // The device's reference (or genes) over the contigs [tb, te) -- in a group (`sh`) this rank's, with every rank's ranges in
  // sh.cuts -- and the sample begun.  Returns the rows of the table.
  uint32_t sharded_reference(SampleResult& res, ShardState* sh, uint32_t tb, uint32_t te) {
    const Header& hdr = *res.hdr;
    const uint32_t n_ref = (uint32_t)hdr.names.size();
    uint32_t n_rows = n_ref;
    int rc;
    if (gene_defs_) {
      gene_cache_ = std::make_shared<ResolvedGenes>(resolve_genes_against_header(*gene_defs_, hdr, gene_namer_));
      std::vector<cmb_gene> genes(gene_cache_->entries.size());
      for (size_t g = 0; g < genes.size(); ++g) genes[g] = cmb_gene{gene_cache_->entries[g].tid, gene_cache_->entries[g].start, gene_cache_->entries[g].end};
      n_rows = std::max<uint32_t>(1, (uint32_t)genes.size());
      if (sh) {
        if (!cmb_set_genes_range) throw ExitError(1, "this device library has no cmb_set_genes_range: --gff needs it over several ranks");
        sh->row_cuts = gene_row_cuts(sh->cuts, gene_cache_->first_of_tid, n_rows);
        rc = cmb_set_genes_range(ctx_, n_ref, hdr.lens.data(), (uint32_t)genes.size(), genes.data(), tb, te);
      } else {
        rc = cmb_set_genes(ctx_, n_ref, hdr.lens.data(), (uint32_t)genes.size(), genes.data());
      }
      res.genes = gene_cache_;
    } else {
      SampleCall::check_layout_fits(hdr.lens, sh ? sh->cuts : std::vector<uint32_t>{0, n_ref});
      if (sh) sh->row_cuts = sh->cuts;
      rc = cmb_set_reference(ctx_, n_ref, hdr.lens.data(), tb, te);
    }
    if (rc) throw_device_error(ctx_, rc);
    ref_lens_.clear();  // the next ordinary sample sets its own reference
    gene_cache_names_.clear();
    if (sh) {
      res.timing.tid_begin = tb;
      res.timing.tid_end = te;
    }
    if ((rc = cmb_begin_sample(ctx_))) throw_device_error(ctx_, rc);
    return n_rows;
  }

  static std::vector<uint8_t> sharded_excluded(const InputSpec& in, const SampleResult& res) {
    std::vector<uint8_t> excluded;
    if (in.excluded) {
      const uint32_t n_ref = (uint32_t)res.hdr->names.size();
      excluded.resize(n_ref);
      for (uint32_t t = 0; t < n_ref; ++t) excluded[t] = in.excluded(res.hdr->names[t]);
    }
    return excluded;
  }

  // Shard k through cmb_shard_add; returns its primaries
  uint64_t add_shard(const InputSpec& in, size_t k, SampleResult& res, double& decode_s) {
    const double a = now_s();
    const BamInput input(in.shards[k]);
    InflateStream stream(input.data(), input.size(), pool_, 1u << 20);
    std::vector<uint8_t> buf;
    const BamHeader h = read_bam_header(stream, buf, in.shards[k].path);
    const BlockIndex& bx = stream.index();
    if (!bx.bgzf) throw ExitError(1, "shard " + in.shards[k].path + " is not a BGZF-compressed BAM file: sharded input is decoded on the GPU only");
    BgzfInput bi(bx, (uint32_t)h.header->names.size(), h.records_at, pool_.size());
    cmb_bgzf_result br{};
    const int rc = cmb_shard_add(ctx_, &bi.in, &br);
    if (rc == CMB_E_DECLINED) throw ExitError(1, "cannot read shard " + in.shards[k].path + ": " + cmb_last_error(ctx_));
    if (rc) throw_device_error(ctx_, rc);
    res.n_records += br.n_records;
    decode_s += now_s() - a;
    return br.n_primary;
  }

  [[noreturn]] void throw_shard_error(const InputSpec& in, int rc) {
    const std::string msg = cmb_last_error(ctx_);
    if (msg.rfind("Contig name does not contain", 0) == 0 && !in.unknown_genome_panic.empty()) throw Panic(in.unknown_genome_panic);
    throw_device_error(ctx_, rc);
  }

  static void print_shard_stats(size_t K, const cmb_shard_result& sr) {
    if (getenv("CMB_PIPELINE_STATS"))
      fprintf(stderr, "#reference_bytes\tshards=%zu\tshard_store=%llu\n#sharded\tpairs=%llu\temitted=%llu\tdecode_ms=%.3f\tchoose_ms=%.3f\tsort_ms=%.3f\n", K,
              (unsigned long long)sr.store_bytes, (unsigned long long)sr.n_pairs, (unsigned long long)sr.n_emitted, sr.ms_decode, sr.ms_choose, sr.ms_sort);
  }

  // The sample ended: its rows (in a group over NCCL they stay on the device for cmb_allgather_stats), histogram pairs and
  // gene extras
  void sharded_end(SampleResult& res, const cmb_params& params, uint32_t n_ref, uint32_t n_rows, ShardState* sh) {
    ensure_rows(n_rows);
    res.rows = rows_buf_;
    uint64_t n_pairs = 0;
    int rc;
    const bool on_device = sh && group_nccl_;
    if ((rc = cmb_end_sample(ctx_, on_device ? nullptr : rows_buf_, nullptr, 0, &n_pairs))) throw_device_error(ctx_, rc);
    if (!on_device && (params.want & CMB_WANT_HIST_CSR) && n_pairs) {
      res.pairs.resize(n_pairs);
      if ((rc = cmb_fetch_pairs(ctx_, res.pairs.data(), n_pairs))) throw_device_error(ctx_, rc);
    }
    if (sh) {
      sh->n_pairs = n_pairs;
      if (!on_device) local_pairs_ = res.pairs;
    }
    if (gene_defs_) {
      res.contig_seen.assign((size_t)n_ref + 1, 0);
      if ((rc = cmb_fetch_gene_extras(ctx_, res.contig_seen.data(), &res.kept_primary))) throw_device_error(ctx_, rc);
    }
    cmb_get_timing(ctx_, &res.timing.device);
    res.timing.device_decode = true;
  }

  // One process_local call, handed from stage to stage.
  struct SampleCall {
    DeviceSession& s;
    const InputSpec& in;
    const cmb_params& params;
    ShardState* shard;
    HostRange nvtx_header{"host: open + BAM header"};
    const double t0 = now_s();
    SampleResult res;
    BamInput input;
    const bool pair_mode;
    InflateStream stream;  // only the header is read through it, unless the host's mate matching needs the records too
    std::vector<uint8_t> buf;
    size_t begin = 0;      // first unconsumed byte of buf
    bool hdr_fast = false, decoded_on_device = false;
    uint64_t records_at = 0;
    uint32_t n_ref = 0, n_rows = 0, sb = 0, se = 0;
    double wait_s = 0;     // in cmb_acquire_batch / cmb_submit_batch

    SampleCall(DeviceSession& session, const InputSpec& input_spec, const cmb_params& p, ShardState* sh)
        : s(session), in(input_spec), params(p), shard(sh), input(in), pair_mode(s.set_params(params)),
          stream(input.data(), input.size(), s.pool_, 1u << 20) {
      res.stoit_name = file_stem(in.path);
    }

    void acquire(cmb_read_batch* b) {
      const double a = now_s();
      const int rc = cmb_acquire_batch(s.ctx_, b);
      wait_s += now_s() - a;
      if (rc) throw_device_error(s.ctx_, rc);
    }
    void submit(uint32_t n_records, uint32_t n_intervals) {
      const double a = now_s();
      const int rc = cmb_submit_batch(s.ctx_, n_records, n_intervals);
      wait_s += now_s() - a;
      if (rc) throw_device_error(s.ctx_, rc);
    }

    // Header (SAMv1 §4.2).  Samples mapped to the same reference carry byte-identical headers up to the first record: the
    // parsed copy of the previous sample is reused then (500 000 names are not rebuilt per sample).
    void header() {
      // Fastest case: the file starts with the very same COMPRESSED bytes as the previous sample's header did (the same
      // file again, or samples written by one pipeline): nothing is inflated on the host at all.
      if (s.hdr_cache_ && stream.is_bgzf() && !s.hdr_comp_.empty() && input.size() >= s.hdr_comp_.size() &&
          memcmp(input.data(), s.hdr_comp_.data(), s.hdr_comp_.size()) == 0) {
        hdr_fast = true;
        res.hdr = s.hdr_cache_;
        records_at = s.hdr_records_at_;
      } else {  // otherwise the raw reference list may still be the previous sample's, behind a different @-text
        const BamHeader h = read_bam_header(stream, buf, in.path, s.hdr_raw_);
        if (h.header) {
          res.hdr = s.hdr_cache_ = h.header;
          s.hdr_raw_.assign(buf.data() + h.refs_at, buf.data() + h.records_at);
        } else {
          res.hdr = s.hdr_cache_;
        }
        records_at = h.records_at;
        begin = (size_t)records_at;
        s.hdr_comp_.clear();  // refreshed by index(), once the block table is known
      }
      n_ref = (uint32_t)res.hdr->names.size();
      res.timing.header_s = now_s() - t0;
      nvtx_header.end();
    }

    // Contig mode: every rank's contigs [cuts[r], cuts[r + 1]) fit one device context.  All ranks of a group check every
    // rank's range, so they stop together.
    static void check_layout_fits(const std::vector<uint64_t>& lens, const std::vector<uint32_t>& cuts) {
      for (size_t r = 0; r + 1 < cuts.size(); ++r) {
        const uint64_t spans = layout_spans(lens, cuts[r], cuts[r + 1]);
        if (spans <= CMB_MAX_SPANS) continue;
        const int n = gpus_for_layout(lens);
        throw ExitError(1, "the reference contigs [" + std::to_string(cuts[r]) + ", " + std::to_string(cuts[r + 1]) + ") take " +
                               std::to_string(spans) + " 32-base spans, more than one GPU holds (" + std::to_string(CMB_MAX_SPANS) +
                               ", about 2^37 bases); " +
                               (n ? "run with --gpus " + std::to_string(n) + " or more to split them over GPUs by contig"
                                  : std::string("no split by contig brings every GPU's share under that")));
      }
    }

    // The device's reference (or genes) and the sample begun.
    void reference() {
      sb = std::min<uint32_t>(s.shard_begin_, n_ref);
      se = std::min<uint32_t>(s.shard_end_, n_ref);
      if (shard && !s.gene_defs_) {
        shard->cuts = tid_cuts_by_length(res.hdr->lens, s.group_n_);
        shard->row_cuts = shard->cuts;
        sb = shard->cuts[(size_t)s.group_rank_];
        se = shard->cuts[(size_t)s.group_rank_ + 1];
      }
      n_rows = n_ref;
      int rc;
      if (s.gene_defs_) {
        const bool resolve = !s.gene_cache_ || res.hdr->lens != s.ref_lens_ || res.hdr->names != s.gene_cache_names_;
        if (resolve) {
          s.gene_cache_ = std::make_shared<ResolvedGenes>(resolve_genes_against_header(*s.gene_defs_, *res.hdr, s.gene_namer_));
          s.gene_cache_names_ = res.hdr->names;
        }
        const auto& entries = s.gene_cache_->entries;
        n_rows = std::max<uint32_t>(1, (uint32_t)entries.size());
        if (shard) {  // contigs cut by their genes' padded bases; each rank owns the genes of its contigs
          std::vector<uint32_t> seg_tid(entries.size());
          std::vector<uint64_t> seg_len(entries.size());
          for (size_t g = 0; g < entries.size(); ++g) {
            seg_tid[g] = entries[g].tid;
            seg_len[g] = entries[g].end - entries[g].start;
          }
          shard->cuts = tid_cuts_by_length(padded_gene_bases(n_ref, seg_tid, seg_len), s.group_n_);
          shard->row_cuts = gene_row_cuts(shard->cuts, s.gene_cache_->first_of_tid, n_rows);
          sb = shard->cuts[(size_t)s.group_rank_];
          se = shard->cuts[(size_t)s.group_rank_ + 1];
        }
        // the device's genes depend on the header and, in a group, on this rank's contig range
        if (resolve || (shard != nullptr) != s.gene_ranged_ || (shard && (sb != s.gene_sb_ || se != s.gene_se_))) {
          if (shard && !cmb_set_genes_range) throw ExitError(1, "this device library has no cmb_set_genes_range: --gff needs it over several ranks");
          std::vector<cmb_gene> genes(entries.size());
          for (size_t g = 0; g < genes.size(); ++g) genes[g] = cmb_gene{entries[g].tid, entries[g].start, entries[g].end};
          rc = shard ? cmb_set_genes_range(s.ctx_, n_ref, res.hdr->lens.data(), (uint32_t)genes.size(), genes.data(), sb, se)
                     : cmb_set_genes(s.ctx_, n_ref, res.hdr->lens.data(), (uint32_t)genes.size(), genes.data());
          if (rc) throw_device_error(s.ctx_, rc);
          s.ref_lens_ = res.hdr->lens;
          s.gene_ranged_ = shard != nullptr;
          s.gene_sb_ = sb;
          s.gene_se_ = se;
        }
        res.genes = s.gene_cache_;
      } else if (res.hdr->lens != s.ref_lens_ || sb != s.ref_sb_ || se != s.ref_se_) {
        check_layout_fits(res.hdr->lens, shard ? shard->cuts : std::vector<uint32_t>{sb, se});
        s.ref_sb_ = sb;
        s.ref_se_ = se;
        rc = cmb_set_reference(s.ctx_, n_ref, res.hdr->lens.data(), sb, se);
        if (rc) throw_device_error(s.ctx_, rc);
        s.ref_lens_ = res.hdr->lens;
      }
      res.timing.tid_begin = sb;
      res.timing.tid_end = se;
      rc = cmb_begin_sample(s.ctx_);
      if (rc) throw_device_error(s.ctx_, rc);
    }

    // The whole block table.  htslib flushes the BGZF block after the header (bam_hdr_write), so the records usually start
    // a block: then the compressed bytes in front of that block ARE the header, and the next sample that begins with the
    // same bytes needs no header inflate at all.
    const BlockIndex& index(double t_index0) {
      const BlockIndex& bx = stream.index();
      res.timing.index_s = now_s() - t_index0;
      if (!hdr_fast && bx.bgzf) {
        const size_t b = (size_t)(std::lower_bound(bx.ustart.begin(), bx.ustart.end(), records_at) - bx.ustart.begin());
        if (b > 0 && b < bx.blocks.size() && bx.ustart[b] == records_at && bx.blocks[b].cdata >= 18) {
          const size_t start = bx.blocks[b].cdata - 18;
          if (start <= (256u << 20) && bx.p[start] == 0x1f && bx.p[start + 1] == 0x8b) {
            s.hdr_comp_.assign(bx.p, bx.p + start);
            s.hdr_records_at_ = records_at;
          }
        }
      }
      return bx;
    }

    // cmb_submit_bgzf over the sample's blocks (in a group, over this rank's block range).
    void device_decode(const BlockIndex& bx, HostRange& nvtx_index, double t_index0) {
      BgzfInput bi(bx, n_ref, records_at, s.pool_.size());
      const bool range_ok = !shard || rank_block_range(bx, bi.in);
      cmb_bgzf_result br{};
      nvtx_index.end();
      const double a = now_s();
      res.timing.index_s = a - t_index0;  // incl. the block table and, in a group, the range probes
      const int rc = range_ok ? cmb_submit_bgzf(s.ctx_, &bi.in, &br) : CMB_E_DECLINED;
      res.timing.device_call_s = now_s() - a;
      if (rc == CMB_OK) {
        decoded_on_device = true;
        res.timing.device_decode = true;
        res.timing.bgzf = br;
        res.timing.h2d_bytes = br.h2d_bytes;
        res.timing.decode_launches = br.n_launches;
        res.n_records = br.n_records;
        res.num_detected_primary_alignments = br.n_primary;
        if (getenv("CMB_PIPELINE_STATS"))
          fprintf(stderr, "#device_decode\tblocks=%zu\thost_blocks=%u\trepairs=%u\tcopy_inflate_ms=%.2f\tchain_ms=%.2f\textract_ms=%.2f\ttotal_ms=%.2f\tcall_s=%.4f\n",
                  bx.blocks.size(), br.n_blocks_host, br.chain_repairs, br.ms_copy_inflate, br.ms_chain, br.ms_extract, br.ms_total, now_s() - a);
      } else if (rc != CMB_E_DECLINED) {
        throw_device_error(s.ctx_, rc);
      } else if (getenv("CMB_PIPELINE_STATS")) {
        fprintf(stderr, "#device_decode\tdeclined: %s\n", cmb_last_error(s.ctx_));
      }
    }

    // This rank's block range (shard_range.hpp), into `bi`; false when the stream's alignment cannot be confirmed (the
    // rank then reads the stream whole).
    bool rank_block_range(const BlockIndex& bx, cmb_bgzf_input& bi) {
      try {
        BlockRangeFinder finder(bx, n_ref, records_at);
        const bool last = s.group_rank_ == s.group_n_ - 1;
        // reads cover the reference roughly evenly, so a tid's records start near its share of the summed contig length
        double frac_lo = -1.0, frac_hi = -1.0;
        long double before_lo = 0, before_hi = 0, total = 0;
        const auto& lens = res.hdr->lens;
        for (size_t t = 0; t < lens.size(); ++t) {
          if (t == sb) before_lo = total;
          if (t == se) before_hi = total;
          total += (long double)lens[t];
        }
        if (se >= lens.size()) before_hi = total;
        if (total > 0) {
          frac_lo = (double)(before_lo / total);
          frac_hi = (double)(before_hi / total);
        }
        const BlockRange br = finder.find(sb, se, s.group_rank_ == 0, last, frac_lo, frac_hi);
        bi.ranged = 1;
        bi.walk_begin_block = br.walk_begin;
        bi.walk_end_block = br.walk_end;
        bi.records_at = br.records_at;
        bi.excl_end_block = br.excl_end;
        bi.own_tid_begin = (int32_t)sb;
        bi.own_tid_end = (int32_t)se;
        bi.own_unplaced = last ? 1u : 0u;
        res.timing.shard_blocks = br.walk_end - br.walk_begin;
        res.timing.total_blocks = (uint32_t)bx.blocks.size();
        res.timing.range_probes = br.probes;
        return true;
      } catch (const Panic&) {
        return false;
      }
    }

    // The region-parallel host decode (decode_runner.hpp): this thread only acquires / submits staging batches.
    void host_pipeline(const BlockIndex& bx) {
      if (shard) shard->counts_global = true;  // every rank's host decoder reads the whole file; K1 keeps the rank's own tids
      const PipelineCounts pc = run_decode_pipeline(
          bx, records_at, n_ref, s.pool_.size(), s.batch_records_, s.batch_intervals_, s.n_staging_, s.scratch_,
          [&](cmb_read_batch* b) { acquire(b); }, [&](uint32_t nr, uint32_t ni) { submit(nr, ni); });
      res.n_records = pc.n_records;
      res.num_detected_primary_alignments = pc.primaries;
      if (getenv("CMB_PIPELINE_STATS"))
        fprintf(stderr, "#pipeline\titems=%u\tworkers=%u\tinflate_s=%.3f\tchain_s=%.3f\textract_s=%.3f\tidle_s=%.3f (summed over workers)\n",
                pc.n_items, pc.n_workers, pc.inflate_s, pc.scan_s, pc.extract_s, pc.idle_s);
    }

    // Pair filtering when the device did not decode the stream (filter.rs:117-233): windows of records are decoded in
    // parallel, then mates are matched in stream order; only completed pairs reach the GPU, the first mate at the even index.
    void pair_fallback() {
      if (shard) shard->counts_global = true;  // mate matching reads the whole file on every rank
      if (hdr_fast) {  // the header was recognised without inflating it: skip over it now
        while (buf.size() < records_at)
          if (!stream.fill(buf)) throw Panic("Error reading BAM header: truncated");
        begin = (size_t)records_at;
      }
      stream.set_window(48u << 20);  // mate matching is sequential: decode window by window
      struct Stored {
        Tuple t;
        std::vector<int32_t> iv_start, iv_len;
      };
      HostMates<Stored> mates;
      constexpr size_t ITEM = 4096;  // records per parallel work item
      struct ItemOut {
        std::vector<int32_t> iv_start, iv_len;
      };
      std::vector<ItemOut> items;
      std::vector<size_t> rec_off;
      std::vector<Tuple> tuples;
      std::vector<uint32_t> iv_at;
      cmb_read_batch batch{};
      bool have_batch = false;
      uint32_t used_r = 0, used_i = 0;
      auto put = [&](const Tuple& t, const int32_t* ivs, const int32_t* ivl) {
        put_tuple(batch, used_r++, used_i, t, ivs, ivl);
        used_i += t.n_iv;
      };
      auto flush = [&]() {
        if (!have_batch) return;
        batch.iv_begin[used_r] = used_i;
        submit(used_r, used_i);
        have_batch = false;
      };
      for (;;) {
        // the complete records currently in buf (one window within a batch)
        rec_off.clear();
        size_t max_iv = 0;
        const size_t q = walk_records(buf.data(), begin, buf.size(), false, [&](size_t o) {
          const int64_t ops = record_cigar_ops(buf.data() + o);
          if (ops < 0) throw_bad_record_layout();
          rec_off.push_back(o);
          max_iv += (size_t)ops;
          return rec_off.size() < s.batch_records_ / 2;
        });
        if (rec_off.empty()) {
          buf.erase(buf.begin(), buf.begin() + (ptrdiff_t)begin);
          begin = 0;
          if (stream.fill(buf)) continue;
          if (!buf.empty()) throw Panic("Error reading BAM record: truncated");  // as walk_records' at_eof
          break;
        }
        const size_t nrec = rec_off.size();
        res.n_records += nrec;
        const size_t n_items = (nrec + ITEM - 1) / ITEM;
        if (items.size() < n_items) items.resize(n_items);
        if (max_iv > s.batch_intervals_) throw ExitError(1, "a window of records has more aligned blocks than a device batch holds");
        tuples.resize(nrec);
        iv_at.resize(nrec);
        const uint8_t* base = buf.data();
        s.pool_.parallel_for(n_items, [&](size_t it, int) {
          ItemOut& io = items[it];
          io.iv_start.clear();
          io.iv_len.clear();
          for (size_t r = it * ITEM; r < std::min(nrec, (it + 1) * ITEM); ++r) {
            iv_at[r] = (uint32_t)io.iv_start.size();
            decode_bam_record(base + rec_off[r], tuples[r], io.iv_start, io.iv_len);
          }
        });
        for (size_t r = 0; r < nrec; ++r) {
          const Tuple& t = tuples[r];
          if (t.flag & 0x900) continue;  // secondary / supplementary (filter.rs:138-140)
          res.num_detected_primary_alignments += 1;
          if (!(t.flag & 0x2)) continue;  // not a proper pair (filter.rs:141-147, filter_out = true)
          const ItemOut& io = items[r / ITEM];
          const int32_t* ivs = io.iv_start.data() + iv_at[r];
          const int32_t* ivl = io.iv_len.data() + iv_at[r];
          const std::optional<Stored> first = mates.match(t, bam_qname(base + rec_off[r]), [&] {
            return Stored{t, std::vector<int32_t>(ivs, ivs + t.n_iv), std::vector<int32_t>(ivl, ivl + t.n_iv)};
          });
          if (!first) continue;
          if (have_batch && (used_r + 2 > s.batch_records_ || used_i + first->t.n_iv + t.n_iv > s.batch_intervals_)) flush();
          if (!have_batch) {
            acquire(&batch);
            have_batch = true;
            used_r = used_i = 0;
          }
          put(first->t, first->iv_start.data(), first->iv_len.data());
          put(t, ivs, ivl);
        }
        begin = q;
      }
      flush();
    }

    // cmb_end_sample.  A histogram buffer of the device overflowed (very deep coverage over many small contigs): with the
    // sample's tuples still in device memory the buffers are enlarged and the kernels run again; otherwise the error stands.
    int end_device_sample(cmb_contig_stats* rows_out, uint64_t& n_pairs) {
      int rc = cmb_end_sample(s.ctx_, rows_out, nullptr, 0, &n_pairs);
      for (int attempt = 0; rc == CMB_E_CAPACITY && decoded_on_device && attempt < 8; ++attempt) {
        cmb_read_batch again{};
        uint32_t nr = 0, ni = 0;
        if (cmb_last_bgzf_batch(s.ctx_, &again, &nr, &ni) != CMB_OK) break;
        if (getenv("CMB_PIPELINE_STATS")) fprintf(stderr, "#capacity_retry\tattempt=%d\n", attempt + 1);
        if ((rc = cmb_grow_buffers(s.ctx_)) != CMB_OK) break;
        if ((rc = cmb_begin_sample(s.ctx_)) != CMB_OK) break;
        if ((rc = cmb_submit_device_batch(s.ctx_, &again, nr, ni)) != CMB_OK) break;
        rc = cmb_end_sample(s.ctx_, rows_out, nullptr, 0, &n_pairs);
      }
      return rc;
    }

    // The device's per-contig table (and histogram pairs), the gene extras, and the sample's timing.
    SampleResult end_sample() {
      const double t_dec = now_s();
      s.ensure_rows(n_rows);
      res.rows = s.rows_buf_;
      uint64_t n_pairs = 0;
      int rc;
      if (shard && s.group_nccl_) {
        // rows (and pairs) stay on the device: cmb_allgather_stats completes the table there and copies it back once
        rc = end_device_sample(nullptr, n_pairs);
        if (rc) throw_device_error(s.ctx_, rc);
        shard->n_pairs = n_pairs;
      } else {
        rc = end_device_sample(s.rows_buf_, n_pairs);
        if (rc) throw_device_error(s.ctx_, rc);
        if ((params.want & CMB_WANT_HIST_CSR) && n_pairs) {
          res.pairs.resize(n_pairs);
          rc = cmb_fetch_pairs(s.ctx_, res.pairs.data(), n_pairs);
          if (rc) throw_device_error(s.ctx_, rc);
        }
        if (shard) {
          shard->n_pairs = n_pairs;
          s.local_pairs_ = res.pairs;
        }
      }
      if (s.gene_defs_) {
        res.contig_seen.assign((size_t)n_ref + 1, 0);
        rc = cmb_fetch_gene_extras(s.ctx_, res.contig_seen.data(), &res.kept_primary);
        if (rc) throw_device_error(s.ctx_, rc);
      }
      cmb_get_timing(s.ctx_, &res.timing.device);
      if (!res.timing.device_decode) res.timing.h2d_bytes = 40ull * res.timing.device.n_records + 4 + 8ull * res.timing.device.n_intervals;
      const double t1 = now_s();
      res.timing.total_s = t1 - t0;
      res.timing.decode_s = t_dec - t0 - wait_s;
      res.timing.submit_wait_s = wait_s;
      res.timing.end_sample_s = t1 - t_dec;
      return std::move(res);
    }
  };

  std::shared_ptr<Header> hdr_cache_;  // parsed reference list of the previous sample and its raw bytes (n_ref .. first record)
  std::vector<uint8_t> hdr_raw_;
  std::vector<uint8_t> hdr_comp_;  // the compressed file prefix the last full header parse consumed, and where its records start
  uint64_t hdr_records_at_ = 0;
  cmb_contig_stats* rows_buf_ = nullptr;
  size_t rows_cap_ = 0;
  ThreadPool pool_;
  DecodeScratch scratch_;
  cmb_ctx* ctx_ = nullptr;
  uint32_t batch_records_ = 0, batch_intervals_ = 0, n_staging_ = 0;
  uint32_t shard_begin_ = 0, shard_end_ = 0xffffffffu;
  std::vector<uint64_t> ref_lens_;
  uint32_t ref_sb_ = 0, ref_se_ = 0;
  const GeneDefinitions* gene_defs_ = nullptr;
  const GenomeNamer* gene_namer_ = nullptr;
  std::shared_ptr<ResolvedGenes> gene_cache_;
  std::vector<std::string> gene_cache_names_;
  bool gene_ranged_ = false;  // the device holds the genes of the contigs [gene_sb_, gene_se_) (cmb_set_genes_range), else all
  uint32_t gene_sb_ = 0, gene_se_ = 0;
  // group (multi-GPU contig sharding)
  int group_rank_ = 0, group_n_ = 1;
  bool group_nccl_ = false, every_rank_prints_ = false;
  AllGatherFn group_fn_ = nullptr;
  void* group_user_ = nullptr;
  std::vector<cmb_hist_pair> local_pairs_;
};

}  // namespace cmbh
