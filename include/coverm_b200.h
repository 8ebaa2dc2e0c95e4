/*
 * coverm_b200.h — C ABI of libcoverm_b200.so: the H100 (sm_90a) replacement for
 * CoverM's per-contig coverage hot path.
 *
 * All citations are file:line under the reference tree (wwood/CoverM v0.8.0).
 *
 * Where it plugs in.  The reference's hot path is the body of the record loop
 * plus the per-contig flush of its three drivers:
 *     contig_coverage()                              src/contig.rs:13-253
 *     mosdepth_genome_coverage_with_contig_names()   src/genome.rs:17-322
 *     mosdepth_genome_coverage()                     src/genome.rs:419-797
 * i.e.  NamedBamReader::read (bam_generator.rs:21-38)
 *         -> [ReferenceSortedBamFilter::read  filter.rs:86-234]  -> FlagFilter::passes (lib.rs:59-79)
 *         -> CIGAR walk into `ups_and_downs: Vec<i32>` (contig.rs:166-202)
 *         -> MosdepthGenomeCoverageEstimator::add_contig(&[i32], reads, mismatches, identity)
 *            (mosdepth_genome_coverage_estimators.rs:366-528, "EST")
 *         -> calculate_coverage (EST:530-839) -> CoverageTaker (coverage_takers.rs:29-38).
 * add_contig takes a dense host array per contig, so the device boundary sits
 * one level up: the host reduces each BAM record to a fixed tuple (+ its
 * M/=/X intervals), this library does filter + delta accumulation + prefix sum
 * + every O(contig length) reduction on the GPU, and hands back per-contig
 * INTEGER sufficient statistics from which the host replays calculate_coverage
 * verbatim in f32/f64.  A Rust host binds these symbols from the same spot in
 * contig.rs / genome.rs (see INTEGRATION.md).
 *
 * Conventions: every function returns 0 on success or a negative CMB_E_* code
 * (never throws / aborts across the ABI); cmb_last_error() gives the message.
 * The caller owns every host result buffer; the library owns the pinned
 * staging buffers and all device memory.  One cmb_ctx per (GPU, host thread);
 * a ctx is not thread-safe.  There is NO CPU fallback: cmb_create fails if no
 * CUDA device is usable.
 */
#ifndef COVERM_B200_H
#define COVERM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CMB_ABI_VERSION 3

/* error codes */
#define CMB_OK 0
#define CMB_E_CUDA (-1)      /* CUDA runtime / driver failure                               */
#define CMB_E_ARG (-2)       /* bad argument / call order                                   */
#define CMB_E_NOMEM (-3)     /* device or pinned allocation failed                          */
#define CMB_E_UNSORTED (-4)  /* records not sorted by reference   (contig.rs:129-132 panic) */
#define CMB_E_NM (-5)        /* NM aux missing / wrong type where the reference calls nm()  (lib.rs:138-158 panic) */
#define CMB_E_BOUNDS (-6)    /* an aligned block starts at/after the contig end (contig.rs:178 index panic) */
#define CMB_E_CAPACITY (-7)  /* a device-side buffer (histogram records) overflowed         */
#define CMB_E_DECLINED (-8)  /* cmb_submit_bgzf: the device decoder cannot vouch for this stream; nothing was
                                accumulated -- decode on the host instead                    */

typedef struct cmb_ctx cmb_ctx;

typedef struct cmb_device_cfg {
  int32_t device;             /* CUDA device ordinal                                         */
  uint32_t batch_records;     /* capacity (records) of each pinned staging batch            */
  uint32_t batch_intervals;   /* capacity (intervals) of each pinned staging batch          */
  uint32_t n_staging;         /* number of staging batches (>= 2: decode overlaps H2D + K1) */
} cmb_device_cfg;

/* Which statistics the host needs (selects kernel variants). */
#define CMB_WANT_HIST 1u      /* depth histogram of the end-trimmed window: trimmed_mean / variance /
                                 coverage_histogram (EST:410-466)                                     */
#define CMB_WANT_HIST_CSR 2u  /* also return the merged per-contig histogram as (depth,count) pairs  */

/* Filter / estimator parameters: FlagFilter (lib.rs:59-64), ReferenceSortedBamFilter::new
 * arguments (filter.rs:36-47), FilterParameters::doing_filtering (coverm.rs:1695-1703),
 * contig_end_exclusion / trim bounds (coverm.rs:1317-1318, 1364-1372). */
typedef struct cmb_params {
  uint8_t include_improper_pairs;
  uint8_t include_supplementary;
  uint8_t include_secondary;
  uint8_t filtering;                 /* 1: a ReferenceSortedBamFilter (filter_out = true) precedes the flag filter */
  uint8_t min_mapq;                  /* 255 = no MAPQ filtering (filter.rs:13)                  */
  uint8_t reserved0[3];
  uint32_t min_aligned_length_single;
  float min_percent_identity_single;
  float min_aligned_percent_single;
  uint32_t min_aligned_length_pair;
  float min_percent_identity_pair;
  float min_aligned_percent_pair;
  uint64_t contig_end_exclusion;     /* E: the window of a contig of length L is [E, L-E) when 2E < L */
  float trim_min;                    /* trimmed-mean bounds as fractions (EST:591-592)          */
  float trim_max;
  uint32_t want;                     /* CMB_WANT_* bitmask                                      */
  uint32_t reserved1;
} cmb_params;

/* Derived filter gating (filter.rs:48-61), filled by cmb_set_params for the host:
 * when filter_pairs is set the host must perform mate matching (filter.rs:149-184)
 * and submit only completed pairs, first mate at an even index, second right after. */
typedef struct cmb_filter_mode {
  uint8_t filter_single_reads;
  uint8_t filter_pairs;
} cmb_filter_mode;

/* One staging batch, SoA.  Pointers are into pinned host memory owned by the ctx;
 * valid from cmb_acquire_batch until the matching cmb_submit_batch (several batches may
 * be acquired at once, up to n_staging; cmb_submit_batch submits the oldest one).
 * Record i covers intervals [iv_begin[i], iv_begin[i+1]) — the host writes
 * iv_begin[n_records] = n_intervals.  40 B per record + 8 B per interval.
 * An interval whose iv_start is CMB_IV_PAD is an unused pool slot and is ignored (lets
 * parallel decoders reserve interval space by an upper bound). */
#define CMB_IV_PAD INT32_MIN
typedef struct cmb_read_batch {
  uint32_t capacity_records;
  uint32_t capacity_intervals;
  int32_t* tid;       /* record.tid()                                   contig.rs:124 */
  int32_t* pos;       /* record.pos(), 0-based leftmost                  contig.rs:166 */
  uint16_t* flag;     /* BAM FLAG                                        lib.rs:67-78  */
  uint8_t* mapq;      /*                                                 filter.rs:251 */
  uint8_t* nm_state;  /* 1: NM aux present with type C/S/I; 0: absent; 2: other type (lib.rs:139-156) */
  uint32_t* nm;       /* NM value                                                       */
  uint32_t* l_seq;    /* record.seq().len()                              filter.rs:277 */
  uint32_t* aligned;  /* sum len(M,I,D,=,X)            filter.rs:261, contig.rs:171-199 */
  uint32_t* del;      /* sum len(D)  (pair filter omits D, filter.rs:304; indels contig.rs:189) */
  uint32_t* ins;      /* sum len(I)                                      contig.rs:197 */
  uint32_t* iv_begin; /* capacity_records + 1 entries                                   */
  int32_t* iv_start;  /* 0-based reference start of each M/=/X block     contig.rs:178 */
  int32_t* iv_len;    /* its length                                      contig.rs:179 */
} cmb_read_batch;

/* Per-contig integer sufficient statistics (one row per reference sequence). */
typedef struct cmb_contig_stats {
  uint64_t n_records;            /* records that survived every filter and are mapped here; "seen" iff > 0
                                    (contig.rs:125-155); names-mode read count (genome.rs:173-174)         */
  uint64_t n_primary;            /* ... and neither secondary nor supplementary   (contig.rs:157-159)      */
  uint64_t n_nonsupp;            /* ... and not supplementary                     (genome.rs:677-682)      */
  uint64_t sum_edit;             /* sum of NM                                     (contig.rs:206-207)      */
  uint64_t sum_indel;            /* sum of I+D lengths                            (contig.rs:189,197)      */
  double sum_identity_primary;   /* sum (aligned-NM)/aligned over primaries       (contig.rs:208-211)      */
  double sum_identity_nonsupp;   /* same over non-supplementary records           (genome.rs:220-223)      */
  uint64_t sum_depth_window;     /* sum of depth over the window                  (EST:402)                */
  uint64_t covered_window;       /* window bases with depth > 0                   (EST:399-401, 457-459)   */
  uint64_t covered_full;         /* all bases with depth > 0 (no end exclusion)   (EST:496-501)            */
  /* histogram-derived, valid with CMB_WANT_HIST; contig mode semantics (unobserved = [0], contig.rs:65): */
  uint64_t trimmed_total;        /* `total` of the trimmed-mean walk              (EST:598-642)            */
  uint64_t trim_min_index;       /* floor(trim_min * T as f32)                    (EST:591)                */
  uint64_t trim_max_index;       /* ceil(trim_max * T as f32)                     (EST:592)                */
  uint64_t var_k;                /* lowest depth with a non-zero count            (EST:790-795)            */
  uint64_t var_ex;               /* sum (x-k) n_x      (wrapping u64)             (EST:796-805)            */
  uint64_t var_ex2;              /* sum (x-k)^2 n_x    (wrapping u64)                                      */
  uint64_t hist_offset;          /* CMB_WANT_HIST_CSR: first pair of this contig in the pair array         */
  uint32_t hist_count;           /* number of (depth,count) pairs, ascending depth                         */
  uint32_t reserved;
} cmb_contig_stats;

typedef struct cmb_hist_pair {
  uint32_t depth;
  uint32_t count;
} cmb_hist_pair;

/* Timings of the last sample, measured with CUDA events on the ctx stream. */
typedef struct cmb_sample_timing {
  float ms_zero;      /* K0: arena + row zero fill                     */
  float ms_accumulate;/* K1 launches (sum over batches, incl. H2D waits on the stream) */
  float ms_scan;      /* K2: segmented scan + reductions + histogram emit */
  float ms_finalize;  /* K3: per-contig histogram merge + trimmed/variance walk */
  float ms_total;     /* begin_sample .. end_sample on the stream      */
  uint64_t arena_elems;   /* padded i32 elements scanned by K2        */
  uint64_t n_records;     /* records submitted                         */
  uint64_t n_intervals;   /* intervals submitted                       */
  uint32_t k1_launches, k2_launches, k3_launches, reserved;
} cmb_sample_timing;

int cmb_abi_version(void);

/* Create / destroy a context on one GPU. */
int cmb_create(const cmb_device_cfg* cfg, cmb_ctx** out);
void cmb_destroy(cmb_ctx* ctx);
const char* cmb_last_error(const cmb_ctx* ctx); /* ctx may be NULL: last cmb_create error */

/* Reference layout: `vec![0; header.target_len(tid)]` for every tid at once
 * (contig.rs:144-145).  [tid_begin, tid_end) is the shard this context owns
 * (multi-GPU contig sharding); records on other tids are ignored. */
int cmb_set_reference(cmb_ctx* ctx, uint32_t n_contigs, const uint64_t* contig_len, uint32_t tid_begin,
                      uint32_t tid_end);
int cmb_set_params(cmb_ctx* ctx, const cmb_params* params, cmb_filter_mode* mode_out);

/* Per-gene coverage (`--gff`; gene_coverage, src/genes.rs:182-344): instead of whole contigs the segments are genes --
 * sub-ranges [start, end) of contigs, possibly overlapping.  The reference cuts each gene's delta array out of its contig's
 * with the running depth at `start` as first element (genes.rs:509-514) and assigns reads to the genes containing their
 * leftmost position (genes.rs:516-523); here every aligned block is clipped to each gene it overlaps, which yields the same
 * arrays, and the usual scan / reductions run over the genes.  Call INSTEAD of cmb_set_reference; records keep carrying contig
 * tids.  `genes` must be sorted by (tid, start) with start < end <= contig_len[tid].  Result rows (cmb_end_sample): one per
 * gene, in that order, with n_primary = primaries starting in the gene, sum_edit = sum of NM.saturating_sub(indels)
 * (genes.rs:297; sum_indel stays 0), sum_identity_primary, and the window / histogram statistics of the gene's own length. */
typedef struct cmb_gene {
  uint32_t tid;
  uint32_t start;
  uint32_t end;
} cmb_gene;
int cmb_set_genes(cmb_ctx* ctx, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes);
/* After cmb_end_sample in gene mode: contig_seen[tid] = 1 when a record that passed every filter mapped to contig tid (its
 * genes are reported through the estimators, the others as zero-coverage entries, genes.rs:434-465); *n_kept_primary =
 * primary alignments among those records (ReadsMapped.num_mapped_reads, genes.rs:249-252). */
int cmb_fetch_gene_extras(cmb_ctx* ctx, uint8_t* contig_seen, uint64_t* n_kept_primary);

/* One BAM file ("stoit", contig.rs:22-27). */
int cmb_begin_sample(cmb_ctx* ctx);
int cmb_acquire_batch(cmb_ctx* ctx, cmb_read_batch* batch);                       /* blocks until a staging batch is free */
int cmb_submit_batch(cmb_ctx* ctx, uint32_t n_records, uint32_t n_intervals);     /* async: H2D + filter/delta kernel      */
/* Device-resident input variant (all pointers are DEVICE pointers laid out as cmb_read_batch;
 * used for device-only timing and by hosts that already stage tuples in HBM). */
int cmb_submit_device_batch(cmb_ctx* ctx, const cmb_read_batch* dev_batch, uint32_t n_records, uint32_t n_intervals);
/* Scan + reduce + copy back.  `stats` has n_contigs rows (rows outside the shard are zeroed); NULL leaves the rows on the
 * device (a multi-GPU caller completes the table there with cmb_allgather_stats and copies it back once).
 * `pairs`/`pairs_capacity` receive the CSR histogram when CMB_WANT_HIST_CSR is set (may be NULL otherwise);
 * *n_pairs gets the number of pairs produced. */
int cmb_end_sample(cmb_ctx* ctx, cmb_contig_stats* stats, cmb_hist_pair* pairs, uint64_t pairs_capacity,
                   uint64_t* n_pairs);
/* Copies the CSR histogram pairs of the sample just ended (CMB_WANT_HIST_CSR) into `pairs`
 * (call cmb_end_sample with pairs == NULL first to learn *n_pairs). */
int cmb_fetch_pairs(cmb_ctx* ctx, cmb_hist_pair* pairs, uint64_t n_pairs);
/* Same, but leaves the rows in device memory (no D2H): *dev_stats is a device pointer to n_contigs rows,
 * valid until the next cmb_begin_sample.  For device-only timing and for NCCL all-gather by the caller. */
int cmb_end_sample_device(cmb_ctx* ctx, const cmb_contig_stats** dev_stats);

/* ---- Device-side BAM decode (optional fast path; the step before the path, bam_generator.rs:103-134) ----
 * Instead of tuples, hand the library the BGZF-compressed BAM bytes of the sample plus its block table: the GPU
 * inflates the blocks, finds the record boundaries, extracts the tuples and runs the same filter/delta kernel.
 * Call it between cmb_begin_sample and cmb_end_sample INSTEAD of the acquire/submit loop, and only when
 * cmb_filter_mode.filter_pairs == 0 (mate matching needs read names, which never reach the device).
 * Returns CMB_E_DECLINED -- with nothing accumulated -- when the device path cannot vouch for the stream (malformed
 * deflate data, an inconsistent record chain, an unknown aux type ...): the caller then decodes on the host, which
 * raises the reference's error if there is one.  `data` may be pageable (staged through pinned buffers by
 * `copy_threads` host threads) or pinned / registered memory (copied directly). */
typedef struct cmb_bgzf_input {
  const uint8_t* data;            /* host pointer: the whole BAM file                                  */
  uint64_t size;
  uint32_t n_blocks;
  uint32_t n_ref;                 /* header n_ref, for record plausibility                             */
  const uint64_t* block_coffset;  /* per BGZF block: offset of its deflate payload in `data`           */
  const uint32_t* block_clen;     /* payload length (the 8-byte CRC32/ISIZE footer follows it)         */
  const uint32_t* block_isize;    /* uncompressed size                                                 */
  uint64_t records_at;            /* uncompressed offset of the first alignment record to decode       */
  uint32_t copy_threads;          /* 0 = 4                                                             */
  uint32_t ranged;                /* 0: the whole file.  1: only a block range of it (multi-GPU contig sharding: a
                                     reference-sorted BAM keeps a tid range in a contiguous run of blocks, so each
                                     rank uploads and inflates only its share) -- the fields below apply          */
  uint32_t walk_begin_block;      /* block holding `records_at`                                         */
  uint32_t walk_end_block;        /* records STARTING in blocks [walk_begin_block, walk_end_block) are decoded; the
                                     bytes of a record running past that come from the blocks that follow */
  int32_t own_tid_begin;          /* result counters (n_records, n_primary) and the rank's sortedness summary count  */
  int32_t own_tid_end;            /* only records with own_tid_begin <= tid < own_tid_end ...                        */
  uint32_t own_unplaced;          /* ... plus, when set, records without a reference (tid < 0: the unmapped tail)   */
  uint32_t excl_end_block;        /* neighbouring ranks' walks overlap by a block: records starting before this block are
                                     this rank's EXCLUSIVE share of the stream (cmb_kept_tid_range)                  */
} cmb_bgzf_input;
typedef struct cmb_bgzf_result {
  uint64_t n_records;             /* alignment records in the file                                     */
  uint64_t n_primary;             /* ... neither secondary nor supplementary (bam_generator.rs:113-119) */
  uint64_t n_intervals;           /* interval slots reserved (sum of n_cigar_op)                       */
  uint32_t n_blocks_host;         /* blocks the device declined and the library inflated with zlib     */
  uint32_t chain_repairs;         /* record-chain repair rounds                                        */
  float ms_copy_inflate, ms_chain, ms_extract, ms_total; /* CUDA events on the ctx stream              */
  uint32_t n_launches;            /* decode kernels launched (inflate windows + chain + extract)       */
  uint32_t n_blocks_second_pass;  /* blocks the first inflate pass declined (incl. windows that did not arrive within the bounded
                                     wait, status 31) and the one-stream-per-warp kernel took over      */
  uint64_t h2d_bytes;             /* compressed bytes + block table copied host->device                */
  float ms_copy_enqueue_wall;     /* host wall clock spent enqueueing the window copies (diagnostics)  */
  float ms_host_wall;             /* host wall clock of the whole call                                  */
} cmb_bgzf_result;
int cmb_submit_bgzf(cmb_ctx* ctx, const cmb_bgzf_input* in, cmb_bgzf_result* out);
/* ---- `coverm filter` (src/bin/coverm.rs:408-472): ReferenceSortedBamFilter (src/filter.rs:36-234) as a record sink ----
 * cmb_decode_bgzf is cmb_submit_bgzf without the accumulation: the sample is inflated, its records located and reduced to
 * tuples, mates matched when the pair path of the filter applies -- and everything stays in device memory.  It needs
 * cmb_set_params (thresholds, flag includes; `filtering` = 1) but no reference and no cmb_begin_sample.
 * cmb_filter_plan then decides, per record, whether the filter returns it (inverse = `--inverse`, i.e. filter_out = false)
 * and lays the returned records out in the reference's order -- file order, except that a passing pair comes out as
 * (stored first mate, second mate) at the second mate's position; cmb_filter_fetch copies them (each with its 4-byte
 * block_size, ready to be written into a BAM stream) to the caller.  CMB_E_NM: the reference would have panicked in nm(). */
int cmb_decode_bgzf(cmb_ctx* ctx, const cmb_bgzf_input* in, cmb_bgzf_result* out);
int cmb_filter_plan(cmb_ctx* ctx, int inverse, uint64_t* n_records, uint64_t* n_bytes);
int cmb_filter_fetch(cmb_ctx* ctx, uint8_t* records, uint64_t n_bytes);

/* The tuples the last successful cmb_submit_bgzf extracted, still resident in device memory (valid until the next
 * cmb_submit_bgzf / cmb_destroy): DEVICE pointers laid out as cmb_read_batch, ready for cmb_submit_device_batch.
 * Lets a caller re-run the filter/scan/reduce kernels over an already decoded sample (device-only timing, parameter sweeps). */
int cmb_last_bgzf_batch(cmb_ctx* ctx, cmb_read_batch* dev_batch, uint32_t* n_records, uint32_t* n_intervals);

/* After cmb_end_sample* failed with CMB_E_CAPACITY (a device-side histogram buffer overflowed: very deep coverage over many
 * small contigs): enlarges those buffers (x4).  A caller whose tuples are still in device memory (cmb_last_bgzf_batch) can then
 * run the sample again -- cmb_begin_sample, cmb_submit_device_batch, cmb_end_sample. */
int cmb_grow_buffers(cmb_ctx* ctx);

/* Page-locked host memory for result buffers (cmb_end_sample copies straight into it at PCIe speed).  Plain malloc
 * semantics otherwise; free with cmb_host_free. */
/* ---- Multi-GPU: one sample range-partitioned by contig over several GPUs (SURVEY.md 8e) -------------------------
 * Contigs are independent (contig.rs flushes per tid), so each rank owns a tid range [tid_cuts[r], tid_cuts[r+1])
 * (cmb_set_reference's shard), decodes only the BGZF blocks that hold it, and the per-contig tables are merged by ONE
 * gather over NCCL (NVLink): every rank broadcasts its own row range in place, after which every rank's table is
 * complete -- the global scalars of the printers (contig.rs:70-72, coverage_printer.rs:457-465) are then computed in
 * entry order exactly as on one GPU.  One process per GPU: rank 0 calls cmb_comm_unique_id and shares the id out of
 * band (torch.distributed, MPI, a file); one process driving several GPUs: cmb_comm_init_local. */
#define CMB_COMM_ID_BYTES 128
int cmb_comm_unique_id(uint8_t id[CMB_COMM_ID_BYTES]);
int cmb_comm_init(cmb_ctx* ctx, const uint8_t id[CMB_COMM_ID_BYTES], int rank, int n_ranks);
int cmb_comm_init_local(cmb_ctx* const* ctxs, int n_ranks); /* ctxs[r] becomes rank r */
void cmb_comm_destroy(cmb_ctx* ctx);
/* Small host-to-host all-gather over the communicator (`bytes` per rank, staged through device memory): rank summaries,
 * error status, counters.  Collective: every rank must call it. */
int cmb_comm_allgather(cmb_ctx* ctx, const void* send, void* recv, size_t bytes);
/* The gather of the path.  Call after cmb_end_sample_device on every rank.  tid_cuts has n_ranks + 1 entries.  With
 * CMB_WANT_HIST_CSR, pair_base (n_ranks + 1 entries: exclusive prefix sums of the ranks' pair counts, which the caller
 * exchanged with cmb_comm_allgather) makes the histogram pairs global too: each rank's rows get hist_offset += its
 * base before they travel, and the pair arrays are concatenated in rank order.  On return `stats` (n_contigs rows) and
 * `pairs` (pair_base[n_ranks] entries; may be NULL) hold the complete table on every rank; the device copy of the
 * table is complete as well (cmb_end_sample_device's pointer). */
int cmb_allgather_stats(cmb_ctx* ctx, const uint32_t* tid_cuts, const uint64_t* pair_base, cmb_contig_stats* stats,
                        cmb_hist_pair* pairs);
/* Kept-record tid range of the rank's own part of the stream, for the cross-rank half of the sortedness check
 * (contig.rs:129-132): smallest / largest tid among the records that passed the filters and START in this rank's
 * exclusive share of the blocks; *min_tid > *max_tid when there is none.  Valid after cmb_end_sample*. */
int cmb_kept_tid_range(cmb_ctx* ctx, int32_t* min_tid, int32_t* max_tid);

void* cmb_host_alloc(size_t bytes);
void cmb_host_free(void* p);

int cmb_get_timing(const cmb_ctx* ctx, cmb_sample_timing* out);
/* cudaStream_t of the context (as void*), for callers that order their own work after it. */
void* cmb_stream(cmb_ctx* ctx);

/* NVTX range on the calling thread (nvtxRangePushA / nvtxRangePop): lets the host side (header parse, block index, range probes,
 * estimator replay, printing) show up next to the library's own ranges on a profiler timeline.  No-ops without a tool attached. */
void cmb_nvtx_push(const char* name);
void cmb_nvtx_pop(void);

#ifdef __cplusplus
}
#endif
#endif /* COVERM_B200_H */
