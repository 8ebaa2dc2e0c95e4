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
#define CMB_E_CAPACITY (-7)  /* a device-side buffer (histogram bin pool or pairs) overflowed */
#define CMB_E_DECLINED (-8)  /* cmb_submit_bgzf: the device decoder cannot vouch for this stream; the sample is
                                reset to the state cmb_begin_sample left it in (also when a
                                late slice of a sliced decode declines) -- decode on the host
                                instead                                                      */

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
  uint64_t arena_elems;   /* padded elements (bases) of the reference layout K2 scans */
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
 * (multi-GPU contig sharding); records on other tids are ignored.
 *
 * Device memory: no per-base depth array is kept.  Each owned contig takes whole 32-base spans; the layout costs about
 * 0.0132 B per base (span bitmap and per-word event tables: 12 B per 1024 bases; chunk tables: 12 B per 8192 bases) and about
 * 164 B per owned contig (result row, offsets, histogram bin bases), plus a 144-B result row for every contig of the header.
 * A 137 Gbp reference needs about 1.8 GB.  A sample adds about 20 B per aligned block (event list and its buckets), 4.5 B per
 * record with CMB_WANT_HIST (histogram bins) and 9 B more with CMB_WANT_HIST_CSR (pairs), all grow-only.  One context holds at most CMB_MAX_SPANS spans, about 2^37 bases
 * (137 Gbp): larger references need several contexts on disjoint contig ranges (several GPUs); a larger shard is CMB_E_ARG,
 * with nothing allocated. */
#define CMB_MAX_SPANS 0xfffffff0ull
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
 * (genes.rs:297; sum_indel stays 0), sum_identity_primary, and the window / histogram statistics of the gene's own length.
 * Device memory: the layout of cmb_set_reference over the genes, plus a delta array of 4 B per gene base (each gene padded
 * to whole 32-base spans), so the genes of one context must fit its GPU at 4 B per base. */
typedef struct cmb_gene {
  uint32_t tid;
  uint32_t start;
  uint32_t end;
} cmb_gene;
int cmb_set_genes(cmb_ctx* ctx, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes);
/* Per-gene coverage over a contig shard (multi-GPU): like cmb_set_genes, but this context counts only the records of the
 * contigs [tid_begin, tid_end), and its arena holds only their genes, [gene_first[tid_begin], gene_first[tid_end]) with
 * gene_first[t] = genes on contigs before t (the range that ends at n_contigs also holds the placeholder row of an empty gene
 * set).  Rows keep their global gene numbers; rows outside the range stay zero.  contig_seen and *n_kept_primary
 * (cmb_fetch_gene_extras) cover the owned contigs only, so the ranks' values OR / add up to the whole sample's.  Consecutive
 * contig ranges give consecutive gene ranges: their bounds are the `tid_cuts` of cmb_allgather_stats in gene mode.
 * cmb_set_genes is the same call over [0, n_contigs). */
int cmb_set_genes_range(cmb_ctx* ctx, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes,
                        uint32_t tid_begin, uint32_t tid_end);
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
 * A stream whose whole decode does not fit in device memory is decoded in block slices, each submitted as one batch.
 * Returns CMB_E_DECLINED -- with the sample reset to its empty state -- when the device path cannot vouch for the stream
 * (malformed deflate data, an inconsistent record chain, an unknown aux type, too little device memory even for slices
 * ...): the caller then decodes on the host, which raises the reference's error if there is one.  `data` may be pageable (staged through pinned buffers by
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
 * cmb_decode_bgzf is cmb_submit_bgzf without the accumulation: the sample is inflated and its records located and reduced to
 * tuples -- and everything stays in device memory.  It needs cmb_set_params (thresholds, flag includes; `filtering` = 1) but
 * no reference and no cmb_begin_sample.
 * cmb_filter_plan then matches mates when the pair path of the filter applies (CMB_E_DECLINED when the stream's proper-pair
 * records are not sorted by reference id: the caller runs the filter on the host), decides, per record, whether the filter
 * returns it (inverse = `--inverse`, i.e. filter_out = false)
 * and lays the returned records out in the reference's order -- file order, except that a passing pair comes out as
 * (stored first mate, second mate) at the second mate's position; cmb_filter_fetch copies them (each with its 4-byte
 * block_size, ready to be written into a BAM stream) to the caller.  CMB_E_NM: the reference would have panicked in nm(). */
int cmb_decode_bgzf(cmb_ctx* ctx, const cmb_bgzf_input* in, cmb_bgzf_result* out);
/* ---- Sharded input (`--sharded`; ReadSortedShardedBamReader, src/shard_bam_reader.rs) ----
 * One read set mapped separately against K reference shards: K read-name-sorted BAMs, every one holding every read pair.
 * Pair j is primaries 2j and 2j+1 of every shard (shard_bam_reader.rs:55-129); for each pair the shard with the highest summed
 * AS wins (ties: a deterministic uniform choice, the t-th tied candidate replacing the winner with probability 1/t drawn from a
 * hash of the pair index and the shard), shards whose first mate lies on an excluded contig are not candidates
 * (shard_bam_reader.rs:222-262).  The winners' records, their tids shifted into the concatenated layout, are sorted by tid on
 * the device (counting sort) and accumulated like one reference-sorted sample (cmb_submit_device_batch).  The layout is the
 * shards' headers concatenated in order (cmb_set_reference / cmb_set_genes as usual).  All three calls sit between
 * cmb_begin_sample and cmb_end_sample, and need cmb_filter_mode.filter_pairs == 0 and filtering == 0 (with a read filter the
 * reference ignores --sharded).
 *   cmb_shard_begin: tid_offsets[k] = targets in shards 0..k-1; excluded = n_contigs bytes, or NULL: 1 = a contig of an excluded
 *                    genome, 2 = a contig whose genome cannot be told (its name lacks the separator: the reference panics when a
 *                    candidate's first mate lies there).
 *   cmb_shard_add:   once per shard, in order, with the whole shard file and block table: the shard is inflated and decoded
 *                    on the device (cmb_decode_bgzf's stages) in consecutive block slices sized to the free device memory, each
 *                    slice's primaries appended to a per-shard store (about 41 B per primary + 8 B per CIGAR operation), then
 *                    the running winner of every pair is updated.  `out` sums the slices.  A shard the device decoder declines is
 *                    CMB_E_DECLINED: there is no host route for shards.  CMB_E_NOMEM: the stores, pair state, name hashes, AS
 *                    scratch and sorted winners alone do not fit (the message names the bytes needed and free).
 *   cmb_shard_finish: checks the shards' lengths, sorts and submits the winners, frees nothing (the stores are grow-only).
 * Errors carry the reference's message: CMB_E_SHARD_EXIT where it exits with status 1, CMB_E_SHARD_PANIC where it panics, and
 * CMB_E_NM for an NM tag the reference's clone rejects.  With several errors the one the reference meets first is reported. */
#define CMB_E_SHARD_EXIT (-9)
#define CMB_E_SHARD_PANIC (-10)
typedef struct cmb_shard_result {
  uint64_t n_pairs;        /* read pairs                                                          */
  uint64_t n_records;      /* winners' records, 2 per pair: the sample's primaries (ReadsMapped)   */
  uint64_t n_emitted;      /* mapped winners submitted to K1                                      */
  uint64_t n_intervals;    /* their interval slots                                                */
  uint64_t store_bytes;    /* device bytes of the per-shard stores, pair state and sorted batch    */
  float ms_choose;         /* CUDA events: per-shard compaction + pair updates (summed over shards) */
  float ms_sort;           /* winners, counting sort, gather                                      */
  float ms_decode;         /* cmb_decode_bgzf stages, summed over shards                          */
  uint32_t reserved;
} cmb_shard_result;
int cmb_shard_begin(cmb_ctx* ctx, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded);
int cmb_shard_add(cmb_ctx* ctx, const cmb_bgzf_input* in, cmb_bgzf_result* out);
int cmb_shard_finish(cmb_ctx* ctx, cmb_shard_result* out);
/* ---- Sharded input over a group of ranks (`--sharded --gpus N`, or N processes in one cmbh_session_set_group group) ----
 * Rank r decodes a contiguous run of whole shards [shard_begin, shard_end) (the host cuts the shards by compressed size) and
 * holds only its contigs [tid_offsets[shard_begin], tid_offsets[shard_end]) (cmb_set_reference / cmb_set_genes_range with that
 * range): a winner's records lie on its shard's contigs, so no record moves between GPUs, only every pair's scores do.  Ranks
 * beyond the shards own an empty run and still take part in every call and exchange.  The calls, between cmb_begin_sample and
 * cmb_end_sample, in this order:
 *   cmb_shard_begin_range: cmb_shard_begin plus this rank's run; then cmb_shard_add once per shard of the run, in order (each
 *                    shard's store is built as on one GPU; the pair choice waits).
 *   cmb_shard_score: n_primary[k] = every shard's primaries (cmb_bgzf_result.n_primary of its owner's cmb_shard_add, which the
 *                    ranks exchange).  Writes one int32 column of the [n_shards][n_pairs] score table per owned shard (n_pairs =
 *                    the shortest shard's primaries / 2): the pair's summed AS, or a negative sentinel when the shard is no
 *                    candidate or the pair's records there are in error; the errors are kept like cmb_shard_finish's.
 *   Exchange, either
 *     cmb_shard_exchange: over the NCCL communicator (cmb_comm_init*): each owner broadcasts its columns, and the owner of shard 0
 *                    its 8-byte name hashes of every primary, in place on the device.  shard_cuts[r] = rank r's shard_begin
 *                    (n_ranks + 1 entries).  Collective.
 *     or cmb_shard_export / cmb_shard_import: column `shard` (n_pairs int32) to / from the host, and with shard == 0 and names !=
 *                    NULL shard 0's name hashes (n_primary[0] uint64), for groups whose ranks exchange host buffers.
 *   cmb_shard_choose: checks the owned shards' read names against shard 0's, picks every pair's winner from the table with
 *                    cmb_shard_finish's rule (every rank reaches the same winners), counts and checks the owned winners' records,
 *                    and returns this rank's smallest error key (UINT64_MAX: none).
 *   cmb_shard_finish_group: err_key = the smallest key over the ranks.  Not UINT64_MAX: returns the error cmb_shard_finish returns
 *                    for it (the same on every rank).  Else sorts and submits the winners of the owned shards; `out` counts the
 *                    sample's pairs and primaries (global) and this rank's emitted winners.
 * Device memory per rank: the owned shards' stores, each with its AS columns (5 B per primary) and, after shard 0, its name
 * hashes (8 B per primary), the score
 * table (4 B per pair and shard), shard 0's name hashes (8 B per primary), the choice (16 B per pair) and the owned sorted winners. */
int cmb_shard_begin_range(cmb_ctx* ctx, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded, uint32_t shard_begin,
                          uint32_t shard_end);
int cmb_shard_score(cmb_ctx* ctx, const uint64_t* n_primary);
int cmb_shard_exchange(cmb_ctx* ctx, const uint32_t* shard_cuts);
int cmb_shard_export(cmb_ctx* ctx, uint32_t shard, int32_t* scores, uint64_t* names);
int cmb_shard_import(cmb_ctx* ctx, uint32_t shard, const int32_t* scores, const uint64_t* names);
int cmb_shard_choose(cmb_ctx* ctx, uint64_t* err_key);
int cmb_shard_finish_group(cmb_ctx* ctx, uint64_t err_key, cmb_shard_result* out);
int cmb_filter_plan(cmb_ctx* ctx, int inverse, uint64_t* n_records, uint64_t* n_bytes);
int cmb_filter_fetch(cmb_ctx* ctx, uint8_t* records, uint64_t n_bytes);
/* ---- `coverm filter` over a stream of any size ----
 * cmb_filter_bgzf hands the records the filter returns to `sink`, in the reference's order, as consecutive byte ranges of at
 * most 64 MB (each record with its 4-byte block_size; a range may end inside a record).  When the whole-stream decode fits, it
 * is cmb_decode_bgzf + cmb_filter_plan with what cmb_filter_fetch would copy handed to the sink.  When it does not
 * (CMB_E_NOMEM), the stream is decoded in block slices and filtered slice by slice, each slice's records handed over before the
 * next slice is decoded.  In pair mode a slice that is not the last holds back the trailing run of its last eligible reference
 * id for the next slice, so that every pair lies in one slice.  The bytes of sink call k lie in one of two pinned staging
 * buffers of the context (64 MB each) and stay valid until sink call k + 1 returns -- the last call's until the context's next
 * cmb_filter_bgzf or cmb_destroy: the caller may keep working on them (compressing them) while the device goes on.  A sink
 * returning non-zero stops the call with CMB_E_ARG.
 * CMB_E_DECLINED (the stream is not BGZF, a CG:B placeholder, a corrupt block, proper pairs out of reference-id order, one
 * reference's proper pairs larger than a slice, too little device memory) may come after some sink calls: the caller then
 * discards what it received and runs the filter on the host.  CMB_E_NM (the reference's panic in nm()) is raised in the slice
 * that meets it, before that slice's first sink call.  A sliced call gives its decode buffers back when it ends. */
typedef int (*cmb_filter_sink)(void* user, const uint8_t* bytes, uint64_t n_bytes);
typedef struct cmb_filter_result {
  uint64_t n_records, n_bytes;  /* returned records and their bytes, summed over the sink calls              */
  uint32_t n_slices;            /* block slices decoded (on CMB_E_DECLINED: before it); 0: the whole stream fit */
  uint32_t halvings;            /* slices halved because their buffers did not fit                           */
  uint64_t pair_cut_records;    /* pair mode: records held back at slice ends (each decoded twice)           */
  uint32_t n_sink_calls;
  float ms_decode, ms_filter, ms_d2h; /* device decode (CUDA events), mate matching + filter kernels, staging copies (host clock) */
} cmb_filter_result;
int cmb_filter_bgzf(cmb_ctx* ctx, const cmb_bgzf_input* in, int inverse, cmb_filter_sink sink, void* user, cmb_filter_result* out);

/* ---- BGZF output compressed on the device (`coverm filter --device-deflate`) ----
 * The context holds one output stream.  Everything fed to it is cut into blocks of 0xff00 bytes counted from the stream's
 * start (the last one shorter), each block is deflated alone on the GPU (LZ77 inside the block, dynamic Huffman codes, or a
 * stored block when that is not larger) into one complete BGZF block, and cmb_deflate_finish closes the stream with the
 * 28-byte EOF block.  A block depends only on its own bytes, so the stream's BGZF bytes are the same however it was fed.
 * The BGZF bytes go to `sink` (cmb_filter_sink) in pieces of at most 64 MB, each in one of two pinned staging buffers of the
 * context: the bytes of sink call k stay valid until sink call k + 1 returns (the last call's until the next cmb_deflate_*
 * call or cmb_destroy).  A sink returning non-zero stops the call with CMB_E_ARG, and the stream must be begun again.
 *
 * cmb_deflate_begin starts a new stream and drops whatever the last one held; it allocates the stream's buffers (about
 * 200 MB of device memory and 128 MB of pinned memory, kept for later streams): CMB_E_NOMEM when they do not fit.
 * cmb_deflate_feed appends host bytes (the BAM header, or records filtered on the host); the blocks they complete are
 * handed to the sink before it returns.  cmb_deflate_finish deflates the partial last block and hands it with the EOF block
 * to the sink, fills *stats and ends the stream.  cmb_filter_bgzf_deflate is cmb_filter_bgzf with the returned records fed
 * to the context's stream from device memory (they are not copied to the host raw): the sink receives BGZF bytes, and
 * out->n_bytes counts the raw record bytes fed.  Its CMB_E_DECLINED and CMB_E_NM come as cmb_filter_bgzf's do, possibly
 * after some sink calls: the caller discards what it received and begins the stream again.  All need a begun stream
 * (CMB_E_ARG otherwise). */
typedef struct cmb_deflate_stats {
  uint64_t raw_bytes, bgzf_bytes; /* fed to the stream; handed to the sink, EOF block included           */
  uint64_t blocks, stored_blocks; /* BGZF blocks holding data (EOF block excluded); those stored verbatim  */
  uint32_t sink_calls;
  float ms_deflate, ms_d2h;       /* deflate + pack kernels (CUDA events); BGZF bytes to the host (host clock) */
} cmb_deflate_stats;
int cmb_deflate_begin(cmb_ctx* ctx);
int cmb_deflate_feed(cmb_ctx* ctx, const uint8_t* bytes, uint64_t n_bytes, cmb_filter_sink sink, void* user);
int cmb_deflate_finish(cmb_ctx* ctx, cmb_filter_sink sink, void* user, cmb_deflate_stats* stats);
int cmb_filter_bgzf_deflate(cmb_ctx* ctx, const cmb_bgzf_input* in, int inverse, cmb_filter_sink sink, void* user,
                            cmb_filter_result* out);

/* The tuples the last successful cmb_submit_bgzf extracted, still resident in device memory (valid until the next
 * cmb_submit_bgzf / cmb_destroy): DEVICE pointers laid out as cmb_read_batch, ready for cmb_submit_device_batch.
 * Lets a caller re-run the filter/scan/reduce kernels over an already decoded sample (device-only timing, parameter sweeps). */
int cmb_last_bgzf_batch(cmb_ctx* ctx, cmb_read_batch* dev_batch, uint32_t* n_records, uint32_t* n_intervals);

/* After cmb_end_sample* failed with CMB_E_CAPACITY (a device-side histogram buffer overflowed): grows the histogram bin pool to
 * exactly the size the failed sample needed (one bin per window depth up to each contig's read count; the library sizes it
 * before every sample, so this takes a caller that bypassed that sizing) and the CSR pair buffer x4.  A caller whose tuples
 * are still in device memory (cmb_last_bgzf_batch) can then run the sample again -- cmb_begin_sample,
 * cmb_submit_device_batch, cmb_end_sample. */
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
