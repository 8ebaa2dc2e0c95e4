// libcoverm_b200 — device side: hand-written sm_90a kernels + the C ABI of include/coverm_b200.h.
//
// Data layout in HBM (one cmb_ctx = one GPU = one contig shard):
//   arena        i32[arena_elems]   gene mode only: all segments' `ups_and_downs` (contig.rs:144-145) back to back, 4 B per
//                                   base.  Both modes lay the segments out in these coordinates (element g of the
//                                   layout): every segment starts on a 32-element span boundary (SPAN), the layout is a
//                                   whole number of 8192-element chunks (CHUNK).  Contig mode allocates no arena; its
//                                   events go to the event list, so its device memory does not grow with the bases.
//   span_bits    u32[arena_elems/1024]  one bit per 32-element span: set by K1 for every event it adds, read (and, when
//                                   cleaning as it goes, cleared) by K2, which works only on the spans named there.
//                                   Zero between samples (K2 cleans it, in gene mode together with the arena).
//   events       u64[2 * intervals of the sample]  contig mode, K1: interval k's start / end as (g << 1) | sign
//   word_count   u32[arena_elems/1024]  contig mode, K1: events per bitmap word; K1e counts them back down to zero
//   word_off     u32[arena_elems/1024 + 1]  contig mode, K1b: exclusive scan of word_count
//   buckets      u16[events + 8]    contig mode, K1e: (g % 1024) | sign << 10 of every event, by word (word_off)
//   off_span     u32[n_local+1]     padded contig offsets in span units; len u32[n_local]
//   chunk_first  u32[n_chunks+1]    contig containing the first span of each chunk
//   tail_sum     i32[n_chunks]      K1: sum of the deltas of the contig that continues past the chunk end
//   carry_in     i32[n_chunks]      K1b: running depth at the first element of each chunk
//   rows         cmb_contig_stats[n_contigs]
//   bin_base     u64[n_local+1]     K1b: first bin of each contig in `bins` (read count + 1 bins for a contig with a window)
//   bins         u32[pool]          K2 -> K3 window depth histogram, bins[bin_base[c] + depth]; zero between samples (K3
//                                   re-zeroes what it reads); bin_hi u32[n_local] = highest depth K2 added per contig
//
// Kernels (all HBM-bound integer work, no tensor cores):
//   K1  k1_filter_accumulate  one thread per record: FlagFilter + ReferenceSortedBamFilter predicates
//                             (lib.rs:59-79, filter.rs:243-336), per-contig read counters (contig.rs:157-211),
//                             +1/-1 delta events (contig.rs:166-202): plain stores to the event list (contig mode) or REDs
//                             into the arena (gene mode); span bits, per-word event counts, chunk tail sums.
//   K1b k1b_local/apply       segmented scan of the per-chunk tail sums -> carry_in (so K2 needs no look-back), the
//                             exclusive scans of the contigs' bin counts -> bin_base and of the word counts -> word_off, in
//                             the same two launches.
//   K1e k1e_bucket_events     contig mode: the event list bucketed by bitmap word, 2 B per event.
//   K2  k2_scan_reduce        persistent warps, a warp per chunk, work only for the spans that hold events (slots, 32 per
//                             round): 32-row TMA boxes (cp.async.bulk.tensor, 128B swizzle) + mbarrier for chunks with many
//                             non-empty spans, cp.async of just the non-empty 128-B rows for the others (gene mode); in
//                             contig mode each round's rows are built in shared memory from its word buckets; warp-shuffle
//                             segmented scan of the slot totals, the event-free stretches between slots closed as one run
//                             each, then every O(L) reduction of EST:366-502 in one pass: sum/covered over the end-trimmed window,
//                             covered over the full contig, window depth histogram as REDs into the contig's bins;
//                             optionally re-zeroes the arena (gene mode) and the span bitmap as it goes.
//   K3  k3_finalize           per contig: walk its bins, trimmed-mean walk (EST:598-642) and the variance sums
//                             (EST:790-805) in integers; optional CSR histogram output.
//   KD* kd_inflate ...        device-side BAM decode behind cmb_submit_bgzf (cmb_bgzf.cu, cmb_decode.cuh): BGZF inflate, record
//                             chain, tuple extraction -- the compressed file crosses PCIe instead of tuples.
//
// This unit holds the context, the reference, the sample and K1-K3.  cmb_comm.cu holds the NCCL communicator, cmb_bgzf.cu the
// device decode, and cmb_shard_input.cu sharded input; cmb_context.cuh is what they share.
#include <algorithm>
#include <climits>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "cmb_context.cuh"

namespace {
#include "cmb_common.cuh"
#include "cmb_k1.cuh"
#include "cmb_k1b.cuh"
#include "cmb_k2.cuh"
#include "cmb_k3.cuh"

// ------------------------------------------------------------------------------------------------ host context
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

std::string g_create_error;

}  // namespace

int cmb::fail(cmb_ctx* ctx, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf;
  else g_create_error = buf;
  return code;
}

namespace {

void free_reference(cmb_ctx* c) {
  c->ref = {};
  c->tmap = {};
  c->gene_mode = false;
}

// Gene mode's delta arena (K1 adds its events there, K2 loads the rows that hold them) and its TMA descriptor: the arena as
// [rows][32] i32, box = one K2 round (32 rows x 128 B = four 1024-B swizzle atoms), 128B swizzle.  Contig mode has neither.
int alloc_arena(cmb_ctx* c) {
  auto& r = c->ref;
  if (int rc = r.d_arena.ensure(c, c->arena_elems)) return rc;
  PFN_encodeTiled encode = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CU_TRY(c, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&encode, cudaEnableDefault, &qres));
  if (!encode || qres != cudaDriverEntryPointSuccess) return fail(c, CMB_E_CUDA, "cuTensorMapEncodeTiled not available in this driver");
  cuuint64_t gdim[2] = {ROW_ELEMS, c->arena_elems / ROW_ELEMS};
  cuuint64_t gstride[1] = {ROW_ELEMS * 4};
  cuuint32_t box[2] = {ROW_ELEMS, K2_BOX_ROWS};
  cuuint32_t estr[2] = {1, 1};
  CUresult res = encode(&c->tmap, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, r.d_arena.p, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (res != CUDA_SUCCESS) return fail(c, CMB_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)res);
  return CMB_OK;
}

// CMB_PIPELINE_STATS: the device bytes this context holds for its reference, by part (the sample's event list and buckets,
// sized by the records, are not included)
void print_reference_bytes(const cmb_ctx* c) {
  const auto& r = c->ref;
  const uint64_t arena = r.d_arena.bytes();
  const uint64_t bitmap = r.d_span_bits.bytes() + r.d_word_count.bytes() + r.d_word_off.bytes() + r.d_word_block_sum.bytes();
  const uint64_t chunks = r.d_chunk_first.bytes() + r.d_tail_sum.bytes() + r.d_carry_in.bytes() + r.d_block_agg.bytes();
  const uint64_t rows = r.d_rows.bytes() + r.d_off_span.bytes() + r.d_len.bytes() + r.d_bin_base.bytes() + r.d_bin_block_sum.bytes() +
                        r.d_bin_hi.bytes() + r.d_gene_first.bytes() + r.d_gene_start.bytes() + r.d_gene_end.bytes() +
                        r.d_gene_maxlen.bytes() + r.d_contig_len32.bytes() + r.d_contig_seen.bytes() + r.d_gene_bound.bytes();
  const uint64_t bins = r.d_bins.bytes(), pairs = r.d_pairs.bytes();
  fprintf(stderr, "#reference_bytes\tarena=%llu\tbitmap=%llu\tchunks=%llu\trows=%llu\tbins=%llu\tpairs=%llu\ttotal=%llu\tlayout_elems=%llu\n",
          (unsigned long long)arena, (unsigned long long)bitmap, (unsigned long long)chunks, (unsigned long long)rows,
          (unsigned long long)bins, (unsigned long long)pairs, (unsigned long long)(arena + bitmap + chunks + rows + bins + pairs),
          (unsigned long long)c->arena_elems);
}

}  // namespace

// Whether K1 has work: a context with no local segment has none, except in gene mode, where owned contigs without genes still
// set contig_seen, count kept_primary and take part in the sortedness check.
bool cmb::k1_active(const cmb_ctx* c) { return c->n_local || (c->gene_mode && c->gene_tid_begin < c->gene_tid_end); }

int cmb::launch_k1(cmb_ctx* c, const cmb_read_batch& b, uint32_t n_records, uint32_t n_intervals, uint32_t excl_n, const int32_t* mate) {
  if (n_records == 0) return CMB_OK;
  int rc_ = CMB_OK;
  const uint32_t blocks = (n_records + K1_THREADS - 1) / K1_THREADS;
  if (c->block_minmax_used + blocks > c->d_block_minmax.cap) {
    // grow (rare): allocate larger arrays and copy what is there
    const size_t ncap = std::max<size_t>(c->d_block_minmax.cap * 2, c->block_minmax_used + blocks + 4096);
    if (int rc = c->d_block_minmax.grow_keep(c, c->block_minmax_used, ncap, c->stream)) return rc;
    if (int rc = c->d_block_xrange.grow_keep(c, c->block_minmax_used, ncap, c->stream)) return rc;
  }
  const auto& r = c->ref;
  if (!c->gene_mode) {  // the event list holds the sample's intervals so far: grow it, keeping the earlier batches' entries
    const uint64_t need = c->n_intervals + n_intervals;
    if (2 * need > 0xffffffffull)  // word_off and the buckets count events in u32
      return fail(c, CMB_E_CAPACITY, "more than 2^31 - 1 aligned blocks in one sample; split the input across more GPUs");
    if (c->d_events.cap < need && (rc_ = c->d_events.grow_keep(c, c->n_intervals, with_slack(need), c->stream))) return rc_;
  }
  K1Args a{};
  a.tid = b.tid; a.pos = b.pos; a.flag = b.flag; a.mapq = b.mapq; a.nm_state = b.nm_state; a.nm = b.nm;
  a.l_seq = b.l_seq; a.aligned = b.aligned; a.del = b.del; a.ins = b.ins; a.iv_begin = b.iv_begin;
  a.iv_start = b.iv_start; a.iv_len = b.iv_len;
  a.n = n_records;
  a.off_span = r.d_off_span; a.len = r.d_len;
  a.n_contigs = c->gene_mode ? c->n_ref_contigs : c->n_contigs; a.tid_begin = c->tid_begin; a.tid_end = c->tid_end;
  a.seg_begin = c->tid_begin;
  if (c->gene_mode) {
    a.tid_begin = c->gene_tid_begin; a.tid_end = c->gene_tid_end;
    a.gene_first = r.d_gene_first; a.gene_start = r.d_gene_start; a.gene_end = r.d_gene_end; a.gene_maxlen = r.d_gene_maxlen;
    a.contig_len = r.d_contig_len32; a.contig_seen = r.d_contig_seen; a.kept_primary = (unsigned long long*)(c->d_counters + 8);
    a.gene_bound = r.d_gene_bound;
  }
  a.arena = r.d_arena; a.span_bits = r.d_span_bits; a.tail_sum = r.d_tail_sum; a.rows = r.d_rows;
  if (!c->gene_mode) {
    a.events = c->d_events; a.iv_base = c->n_intervals; a.n_iv = n_intervals; a.word_count = r.d_word_count;
  }
  a.block_minmax = c->d_block_minmax + c->block_minmax_used;
  a.error_flags = c->d_counters + 0;
  a.block_xrange = c->comm_size > 1 || excl_n != 0xffffffffu ? c->d_block_xrange + c->block_minmax_used : nullptr;
  a.excl_n = excl_n;
  if (a.block_xrange) c->have_xrange = true;
  a.mate = mate;
  a.p = c->params;
  a.filter_single = c->mode.filter_single_reads;
  a.filter_pairs = c->mode.filter_pairs;
  if (c->k1_events_used == c->k1_events.size()) {
    cudaEvent_t e0, e1;
    CU_TRY(c, cudaEventCreate(&e0));
    CU_TRY(c, cudaEventCreate(&e1));
    c->k1_events.emplace_back(e0, e1);
  }
  auto& ev = c->k1_events[c->k1_events_used++];
  CU_TRY(c, cudaEventRecord(ev.first, c->stream));
  k1_filter_accumulate<<<blocks, K1_THREADS, 0, c->stream>>>(a);
  CU_TRY(c, cudaGetLastError());
  CU_TRY(c, cudaEventRecord(ev.second, c->stream));
  c->block_minmax_used += blocks;
  c->n_records += n_records;
  c->n_intervals += n_intervals;
  c->timing.k1_launches += 1;
  return CMB_OK;
}

namespace {

// CTAs of k2_scan_reduce<HIST, CLEAN, BUCKETS> that fit on one SM (K2 is persistent: it launches that many per SM)
template <bool HIST, bool CLEAN, bool BUCKETS>
int k2_blocks_per_sm(cmb_ctx* c, int* occ) {
  auto kern = k2_scan_reduce<HIST, CLEAN, BUCKETS>;
  constexpr uint32_t smem = k2_smem_bytes<BUCKETS>();
  CU_TRY(c, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  *occ = 0;
  CU_TRY(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, kern, (int)K2_THREADS, smem));
  if (*occ < 1) return fail(c, CMB_E_CUDA, "k2_scan_reduce does not fit on an SM");
  return CMB_OK;
}

template <bool HIST, bool CLEAN, bool BUCKETS>
int launch_k2_variant(cmb_ctx* c, const K2Args& a) {
  int occ = 0;
  if (int rc = k2_blocks_per_sm<HIST, CLEAN, BUCKETS>(c, &occ)) return rc;
  // a warp per chunk: no more CTAs than it takes to give every chunk its own warp
  const uint32_t grid = std::min<uint32_t>((c->n_chunks + K2_WARPS - 1) / K2_WARPS, (uint32_t)(occ * c->sm_count));
  if (getenv("CMB_PIPELINE_STATS"))
    fprintf(stderr, "#k2_grid\tgrid=%u\tblocks_per_sm=%d\tsms=%d\thist=%d\tclean=%d\tbuckets=%d\twarps=%u\n", grid, occ, c->sm_count,
            (int)HIST, (int)CLEAN, (int)BUCKETS, grid * K2_WARPS);
  k2_scan_reduce<HIST, CLEAN, BUCKETS><<<grid, K2_THREADS, k2_smem_bytes<BUCKETS>(), c->stream>>>(c->tmap, a);
  CU_TRY(c, cudaGetLastError());
  return CMB_OK;
}

// The bin pool holds at least `need` counts.  A new pool is zeroed: K2 only adds to it and K3 re-zeroes what it read.
int ensure_pool(cmb_ctx* c, uint64_t need, uint64_t alloc) {
  auto& r = c->ref;
  if (r.d_bins.cap >= need) return CMB_OK;
  if (int rc = r.d_bins.ensure(c, need, alloc)) return rc;
  CU_TRY(c, cudaMemsetAsync(r.d_bins, 0, 4 * r.d_bins.cap, c->stream));
  return CMB_OK;
}

bool small_hist() { return getenv("CMB_TEST_SMALL_HIST") != nullptr; }  // testing aid: no pre-sizing (cmb_grow_buffers path)

int run_end_of_sample(cmb_ctx* c) {
  const bool hist = c->params.want & (CMB_WANT_HIST | CMB_WANT_HIST_CSR);
  const bool csr = c->params.want & CMB_WANT_HIST_CSR;
  const uint32_t excl = (uint32_t)std::min<uint64_t>(c->params.contig_end_exclusion, 0x7fffffffu);
  auto& r = c->ref;
  CU_TRY(c, cudaEventRecord(c->ev[2], c->stream));
  if (c->block_minmax_used) {
    k1c_check_sorted<<<1, 1024, 0, c->stream>>>(c->d_block_minmax, c->block_minmax_used, c->d_counters + 0,
                                                c->have_xrange ? c->d_block_xrange.p : nullptr, c->d_counters + 6);
    CU_TRY(c, cudaGetLastError());
  }
  {
    K1bBins g{};
    g.len = r.d_len; g.rows = r.d_rows + c->tid_begin; g.gene_bound = c->gene_mode ? r.d_gene_bound.p : nullptr;
    g.n_seg = c->n_local; g.excl = excl; g.bin_base = r.d_bin_base; g.block_sum = r.d_bin_block_sum;
    g.n_blocks = hist ? c->n_local / K1B_BLOCK + 1 : 0;  // n_local + 1 entries
    K1bWords wd{};
    wd.count = r.d_word_count; wd.off = r.d_word_off; wd.block_sum = r.d_word_block_sum; wd.n_words = c->n_chunks * K2_WARPS;
    wd.n_blocks = c->gene_mode ? 0 : wd.n_words / K1B_BLOCK + 1;  // n_words + 1 entries
    const uint32_t blocks = (c->n_chunks + K1B_BLOCK - 1) / K1B_BLOCK + g.n_blocks + wd.n_blocks;
    k1b_local<<<blocks, K1B_THREADS, 0, c->stream>>>(r.d_tail_sum, r.d_chunk_first, r.d_off_span, c->n_chunks, r.d_carry_in, r.d_block_agg, g, wd);
    CU_TRY(c, cudaGetLastError());
    k1b_apply<<<blocks, K1B_THREADS, 0, c->stream>>>(r.d_tail_sum, r.d_block_agg, c->n_chunks, r.d_carry_in, g, wd);
    CU_TRY(c, cudaGetLastError());
  }
  if (!c->gene_mode) {  // K1e: the event list by bitmap word (K2 reads 8 entries past the last event at most)
    const uint64_t n_events = 2 * c->n_intervals;
    if (int rc = c->d_buckets.ensure(c, n_events + 8, with_slack(n_events + 8))) return rc;
    if (c->n_intervals) {
      const uint64_t blocks = (c->n_intervals + K1E_THREADS - 1) / K1E_THREADS;
      k1e_bucket_events<<<(uint32_t)blocks, K1E_THREADS, 0, c->stream>>>(c->d_events, c->n_intervals, r.d_word_off, r.d_word_count, c->d_buckets);
      CU_TRY(c, cudaGetLastError());
      c->timing.k1_launches += 1;
    }
  }
  if (hist && !small_hist()) {
    // Contig mode: a contig's bins are its read count + 1, and the records submitted bound the read counts together.  Gene
    // mode: a read also covers the genes it starts before, so the pool size is read back (one round trip).
    uint64_t need = c->n_records + c->n_local + 1;
    if (c->gene_mode) {
      CU_TRY(c, cudaMemcpyAsync(&need, r.d_bin_base + c->n_local, 8, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaStreamSynchronize(c->stream));
    }
    if (int rc = ensure_pool(c, need, with_slack(need))) return rc;
    // CSR pairs: K3 writes at most one per bin, plus a depth-0 pair per contig
    if (csr)
      if (int rc = r.d_pairs.ensure(c, need + c->n_local, with_slack(need + c->n_local))) return rc;
  }
  K2Args a{};
  a.off_span = r.d_off_span; a.len = r.d_len; a.chunk_first = r.d_chunk_first; a.carry_in = r.d_carry_in;
  a.rows = r.d_rows; a.tid_begin = c->tid_begin; a.n_local = c->n_local; a.n_chunks = c->n_chunks; a.excl = excl;
  a.arena = r.d_arena; a.span_bits = r.d_span_bits; a.load_stats = c->d_counters + 10;
  a.word_off = r.d_word_off; a.buckets = c->d_buckets;
  a.bin_base = r.d_bin_base; a.bins = r.d_bins; a.pool_cap = r.d_bins.cap; a.bin_hi = r.d_bin_hi;
  a.error_flags = c->d_counters + 0;
  CU_TRY(c, cudaEventRecord(c->ev[3], c->stream));
  int rc;
  const bool clean = c->clean_as_you_go;
  if (!c->gene_mode) {  // contig mode: rows from the word buckets
    if (hist) rc = clean ? launch_k2_variant<true, true, true>(c, a) : launch_k2_variant<true, false, true>(c, a);
    else rc = clean ? launch_k2_variant<false, true, true>(c, a) : launch_k2_variant<false, false, true>(c, a);
  } else {  // gene mode: rows from the arena
    if (hist) rc = clean ? launch_k2_variant<true, true, false>(c, a) : launch_k2_variant<true, false, false>(c, a);
    else rc = clean ? launch_k2_variant<false, true, false>(c, a) : launch_k2_variant<false, false, false>(c, a);
  }
  if (rc) return rc;
  c->timing.k2_launches = 1;
  c->arena_dirty = !c->clean_as_you_go;
  CU_TRY(c, cudaEventRecord(c->ev[4], c->stream));
  if (hist) {
    K3Args k{};
    k.len = r.d_len; k.rows = r.d_rows;
    k.tid_begin = c->tid_begin; k.n_local = c->n_local; k.excl = excl;
    k.trim_min = c->params.trim_min; k.trim_max = c->params.trim_max;
    k.bin_base = r.d_bin_base; k.bins = r.d_bins; k.pool_cap = r.d_bins.cap; k.bin_hi = r.d_bin_hi;
    k.pairs = r.d_pairs; k.pair_count = (unsigned long long*)(c->d_counters + 4); k.pair_capacity = r.d_pairs.cap;
    k.want_csr = csr; k.all_rows = c->gene_mode ? 1u : 0u; k.error_flags = c->d_counters + 0;
    const uint32_t per_block = K3_WARPS * K3_CONTIGS_PER_WARP;
    const uint32_t grid = (c->n_local + per_block - 1) / per_block;
    k3_finalize<<<grid, K3_THREADS, 0, c->stream>>>(k);
    CU_TRY(c, cudaGetLastError());
    c->timing.k3_launches = 1;
  }
  CU_TRY(c, cudaEventRecord(c->ev[5], c->stream));
  return CMB_OK;
}

int collect_errors_and_timing(cmb_ctx* c, uint32_t* counters_out) {
  uint32_t h[13];
  CU_TRY(c, cudaMemcpyAsync(h, c->d_counters, sizeof h, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaEventRecord(c->ev[6], c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  memcpy(counters_out, h, 6 * sizeof(uint32_t));
  c->kept_range[0] = h[6];
  c->kept_range[1] = h[7];
  if (c->n_local && getenv("CMB_PIPELINE_STATS"))  // what K2 fetched: 128 B per span loaded + 32 B of bitmap per chunk
    fprintf(stderr, "#k2_load\tspans_loaded=%u\tspans=%llu\tdense_chunks=%u\tchunks=%u\n", h[10],
            (unsigned long long)c->n_chunks * CHUNK_SPANS, h[11], c->n_chunks);
  if (getenv("CMB_PIPELINE_STATS")) print_reference_bytes(c);
  if (c->n_local && !c->gene_mode && getenv("CMB_PIPELINE_STATS")) {  // contig mode: the bucket entries K2 read (2 B each)
    uint32_t events = 0;  // word_off[n_words]: the events of the sample
    CU_TRY(c, cudaMemcpy(&events, c->ref.d_word_off + (size_t)c->n_chunks * K2_WARPS, 4, cudaMemcpyDeviceToHost));
    fprintf(stderr, "#k2_events\tentries_read=%u\tevents=%u\n", h[12], events);
  }
  float ms = 0;
  cudaEventElapsedTime(&ms, c->ev[0], c->ev[1]); c->timing.ms_zero = ms;
  cudaEventElapsedTime(&ms, c->ev[3], c->ev[4]); c->timing.ms_scan = ms;
  cudaEventElapsedTime(&ms, c->ev[4], c->ev[5]); c->timing.ms_finalize = ms;
  cudaEventElapsedTime(&ms, c->ev[0], c->ev[6]); c->timing.ms_total = ms;
  float acc = 0;
  for (uint32_t i = 0; i < c->k1_events_used; ++i) {
    cudaEventElapsedTime(&ms, c->k1_events[i].first, c->k1_events[i].second);
    acc += ms;
  }
  cudaEventElapsedTime(&ms, c->ev[2], c->ev[3]);  // k1c + k1b
  c->timing.ms_accumulate = acc + ms;
  c->timing.arena_elems = c->arena_elems;
  c->timing.n_records = c->n_records;
  c->timing.n_intervals = c->n_intervals;
  const uint32_t e = h[0];
  if (e) c->arena_dirty = true;
  if (e & ERR_UNSORTED)
    return fail(c, CMB_E_UNSORTED, "BAM file appears to be unsorted. Input BAM files must be sorted by reference (i.e. by samtools sort)");
  if (e & ERR_NM)
    return fail(c, CMB_E_NM, "Mapping record encountered that does not have an 'NM' auxiliary tag in the SAM/BAM format. This is required to work out some coverage statistics");
  if (e & (ERR_BOUNDS | ERR_TID)) return fail(c, CMB_E_BOUNDS, "index out of bounds: an aligned block starts beyond the end of its reference sequence");
  if (e & ERR_CAPACITY) return fail(c, CMB_E_CAPACITY, "device histogram bin pool or pair buffer overflowed");
  if (e & ERR_INTERNAL)
    return fail(c, CMB_E_CUDA, "internal error: running depth below 0 or above the read count (inconsistent delta arena, or a "
                "record whose aligned blocks overlap)");
  return CMB_OK;
}

}  // namespace

// ================================================================================================ C ABI
extern "C" {

int cmb_abi_version(void) { return CMB_ABI_VERSION; }

const char* cmb_last_error(const cmb_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int cmb_create(const cmb_device_cfg* cfg, cmb_ctx** out) {
  NvtxRange nvtx_fn("cmb_create");
  if (!cfg || !out) return fail(nullptr, CMB_E_ARG, "cmb_create: null argument");
  *out = nullptr;
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0)
    return fail(nullptr, CMB_E_CUDA, "cmb_create: no usable CUDA device (%s); libcoverm_b200 has no CPU fallback",
                e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  if (cfg->device < 0 || cfg->device >= n_dev) return fail(nullptr, CMB_E_ARG, "cmb_create: device %d out of range", cfg->device);
  cmb_ctx* c = new cmb_ctx();
  c->device = cfg->device;
  c->cfg = *cfg;
  if (c->cfg.batch_records == 0) c->cfg.batch_records = 1u << 20;
  if (c->cfg.batch_intervals == 0) c->cfg.batch_intervals = c->cfg.batch_records + c->cfg.batch_records / 2;
  if (c->cfg.n_staging < 2) c->cfg.n_staging = 2;
  auto bail = [&](int code) {
    g_create_error = c->err;
    cmb_destroy(c);
    return code;
  };
#define CREATE_TRY(expr)                                                                           \
  do {                                                                                             \
    cudaError_t e_ = (expr);                                                                       \
    if (e_ != cudaSuccess) {                                                                       \
      fail(c, CMB_E_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e_));                         \
      return bail(e_ == cudaErrorMemoryAllocation ? CMB_E_NOMEM : CMB_E_CUDA);                     \
    }                                                                                              \
  } while (0)
  CREATE_TRY(cudaSetDevice(c->device));
  cudaDeviceProp prop;
  CREATE_TRY(cudaGetDeviceProperties(&prop, c->device));
  if (prop.major != 9 || prop.minor != 0) {
    fail(c, CMB_E_CUDA, "cmb_create: device %d is sm_%d%d; this library is built for sm_90a only", c->device, prop.major, prop.minor);
    return bail(CMB_E_CUDA);
  }
  c->sm_count = prop.multiProcessorCount;
  CREATE_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  for (auto& ev : c->ev) CREATE_TRY(cudaEventCreate(&ev));
  size_t offs[13];
  const size_t slab = batch_slab_bytes(c->cfg.batch_records, c->cfg.batch_intervals, offs);
  for (uint32_t i = 0; i < c->cfg.n_staging; ++i) {
    PinnedBuf<uint8_t> h;
    if (int rc = h.ensure(c, slab)) return bail(rc);
    cmb_read_batch hb;
    carve_batch(h, c->cfg.batch_records, c->cfg.batch_intervals, &hb);
    c->host_slab.push_back(std::move(h));
    c->host_batch.push_back(hb);
    DevBatch db;
    if (int rc = db.slab.ensure(c, slab)) return bail(rc);
    carve_batch(db.slab, c->cfg.batch_records, c->cfg.batch_intervals, &db.ptr);
    c->dev_batch.push_back(std::move(db));
    cudaEvent_t ev;
    CREATE_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    c->batch_done.push_back(ev);
    c->batch_busy.push_back(false);
  }
  if (int rc = c->d_counters.ensure(c, 16)) return bail(rc);
  CREATE_TRY(cudaMemset(c->d_counters, 0, 64));
  if (int rc = c->d_block_minmax.ensure(c, 1u << 16)) return bail(rc);
  if (int rc = c->d_block_xrange.ensure(c, 1u << 16)) return bail(rc);
  const char* env = getenv("CMB_CLEAN_AS_YOU_GO");
  if (env && env[0] == '0') c->clean_as_you_go = false;
  *out = c;
  return CMB_OK;
}

void cmb_destroy(cmb_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  for (auto e : c->batch_done) cudaEventDestroy(e);
  for (auto e : c->sh.ev)
    if (e) cudaEventDestroy(e);
  for (auto& e : c->k1_events) {
    cudaEventDestroy(e.first);
    cudaEventDestroy(e.second);
  }
  for (auto e : c->ev)
    if (e) cudaEventDestroy(e);
  cmb_comm_destroy(c);
  {
    auto& d = c->dec;
    for (auto st : d.streams) cudaStreamDestroy(st);
    for (auto e : d.slot_events) cudaEventDestroy(e);
    for (auto e : d.done_events) cudaEventDestroy(e);
    if (d.have_events)
      for (auto e : d.ev) cudaEventDestroy(e);
  }
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;  // frees every buffer (the device is still current)
}

// cmb_set_genes (whole = true: every contig, every gene) and cmb_set_genes_range (the contigs [tid_begin, tid_end) and their genes)
static int set_genes(cmb_ctx* c, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes, uint32_t tid_begin,
              uint32_t tid_end, bool whole) {
  if (!c || (!contig_len && n_contigs) || (!genes && n_genes)) return fail(c, CMB_E_ARG, "cmb_set_genes: null argument");
  if (c->in_sample) return fail(c, CMB_E_ARG, "cmb_set_genes: a sample is in progress");
  if (tid_begin > tid_end || tid_end > n_contigs) return fail(c, CMB_E_ARG, "cmb_set_genes_range: bad contig range");
  std::vector<uint64_t> seg_len(std::max<uint32_t>(1, n_genes), 1);
  std::vector<uint32_t> first((size_t)n_contigs + 1, 0), gs(std::max<uint32_t>(1, n_genes)), ge(std::max<uint32_t>(1, n_genes)), maxlen(std::max<uint32_t>(1, n_contigs), 0), clen(std::max<uint32_t>(1, n_contigs), 0);
  for (uint32_t t = 0; t < n_contigs; ++t) {
    if (contig_len[t] > 0x7fffffffull) return fail(c, CMB_E_ARG, "cmb_set_genes: contig %u longer than 2^31-1", t);
    clen[t] = (uint32_t)contig_len[t];
  }
  for (uint32_t g = 0; g < n_genes; ++g) {
    const cmb_gene& x = genes[g];
    if (x.tid >= n_contigs || x.start >= x.end || x.end > contig_len[x.tid]) return fail(c, CMB_E_ARG, "cmb_set_genes: gene %u is not a range of its contig", g);
    if (g && (genes[g - 1].tid > x.tid || (genes[g - 1].tid == x.tid && genes[g - 1].start > x.start)))
      return fail(c, CMB_E_ARG, "cmb_set_genes: genes must be sorted by (tid, start)");
    seg_len[g] = x.end - x.start;
    gs[g] = x.start;
    ge[g] = x.end;
    first[x.tid + 1] += 1;
    maxlen[x.tid] = std::max(maxlen[x.tid], x.end - x.start);
  }
  for (uint32_t t = 0; t < n_contigs; ++t) first[t + 1] += first[t];
  // the arena, rows and histogram buffers are laid out over the genes exactly as over contigs (a placeholder segment keeps an
  // empty gene set well-formed).  A contig range owns the genes of its contigs, [first[tid_begin], first[tid_end]); the range
  // that ends with the last contig also owns the placeholder, so consecutive ranges partition the rows.
  const uint32_t n_seg = std::max<uint32_t>(1, n_genes);
  auto seg_cut = [&](uint32_t t) { return t == n_contigs ? n_seg : first[t]; };
  const uint32_t g_begin = whole || tid_begin == 0 ? 0 : seg_cut(tid_begin), g_end = whole ? n_seg : seg_cut(tid_end);
  int rc = cmb_set_reference(c, n_seg, seg_len.data(), g_begin, g_end);
  if (rc) return rc;
  if (c->n_local && (rc = alloc_arena(c))) {
    free_reference(c);  // no context in gene mode without its arena
    return rc;
  }
  c->gene_mode = true;
  c->n_ref_contigs = n_contigs;
  c->gene_tid_begin = whole ? 0 : tid_begin;
  c->gene_tid_end = whole ? n_contigs : tid_end;
  auto& r = c->ref;
  const size_t n_ctg = std::max<uint32_t>(1, n_contigs);
  if ((rc = r.d_gene_first.ensure(c, (size_t)n_contigs + 1)) || (rc = r.d_gene_start.ensure(c, n_seg)) || (rc = r.d_gene_end.ensure(c, n_seg)) ||
      (rc = r.d_gene_maxlen.ensure(c, n_ctg)) || (rc = r.d_contig_len32.ensure(c, n_ctg)) || (rc = r.d_contig_seen.ensure(c, n_ctg)) ||
      (rc = r.d_gene_bound.ensure(c, std::max<uint32_t>(1, c->n_local))))
    return rc;
  CU_TRY(c, cudaMemcpyAsync(r.d_gene_first, first.data(), 4ull * (n_contigs + 1), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(r.d_gene_start, gs.data(), 4ull * n_seg, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(r.d_gene_end, ge.data(), 4ull * n_seg, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(r.d_gene_maxlen, maxlen.data(), 4 * n_ctg, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(r.d_contig_len32, clen.data(), 4 * n_ctg, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}

int cmb_set_genes(cmb_ctx* c, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes) {
  return set_genes(c, n_contigs, contig_len, n_genes, genes, 0, n_contigs, true);
}

int cmb_set_genes_range(cmb_ctx* c, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes,
                        uint32_t tid_begin, uint32_t tid_end) {
  return set_genes(c, n_contigs, contig_len, n_genes, genes, tid_begin, tid_end, false);
}

int cmb_fetch_gene_extras(cmb_ctx* c, uint8_t* contig_seen, uint64_t* n_kept_primary) {
  if (!c || !contig_seen || !n_kept_primary) return fail(c, CMB_E_ARG, "cmb_fetch_gene_extras: null argument");
  if (!c->gene_mode || !c->ended) return fail(c, CMB_E_ARG, "cmb_fetch_gene_extras: no ended sample in gene mode");
  CU_TRY(c, cudaSetDevice(c->device));
  unsigned long long kp = 0;
  if (c->n_ref_contigs) CU_TRY(c, cudaMemcpyAsync(contig_seen, c->ref.d_contig_seen, c->n_ref_contigs, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(&kp, c->d_counters + 8, 8, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  *n_kept_primary = kp;
  return CMB_OK;
}

int cmb_set_reference(cmb_ctx* c, uint32_t n_contigs, const uint64_t* contig_len, uint32_t tid_begin, uint32_t tid_end) {
  if (!c || !contig_len || tid_begin > tid_end || tid_end > n_contigs) return fail(c, CMB_E_ARG, "cmb_set_reference: bad arguments");
  if (c->in_sample) return fail(c, CMB_E_ARG, "cmb_set_reference: a sample is in progress");
  CU_TRY(c, cudaSetDevice(c->device));
  free_reference(c);
  c->n_contigs = n_contigs;
  c->n_ref_contigs = n_contigs;
  c->tid_begin = tid_begin;
  c->tid_end = tid_end;
  c->n_local = tid_end - tid_begin;
  std::vector<uint32_t> off_span(c->n_local + 1), len(c->n_local);
  uint64_t spans = 0;
  for (uint32_t i = 0; i < c->n_local; ++i) {
    const uint64_t L = contig_len[tid_begin + i];
    if (L > 0x7fffffffull) return fail(c, CMB_E_ARG, "cmb_set_reference: contig %u longer than 2^31-1", tid_begin + i);
    off_span[i] = (uint32_t)spans;
    len[i] = (uint32_t)L;
    spans += std::max<uint64_t>(1, (L + SPAN - 1) / SPAN);
    if (spans > CMB_MAX_SPANS)
      return fail(c, CMB_E_ARG, "cmb_set_reference: contigs [%u, %u) need more than %llu 32-base spans (about 2^37 bases), the limit of "
                  "one context; split them over more GPUs (contig shards)", tid_begin, tid_end, (unsigned long long)CMB_MAX_SPANS);
  }
  off_span[c->n_local] = (uint32_t)spans;
  const uint64_t chunks = std::max<uint64_t>(1, (spans + CHUNK_SPANS - 1) / CHUNK_SPANS);
  c->n_chunks = (uint32_t)chunks;
  c->arena_elems = chunks * CHUNK;
  std::vector<uint32_t> chunk_first(c->n_chunks + 1);
  {
    uint32_t ci = 0;
    for (uint32_t k = 0; k < c->n_chunks; ++k) {
      const uint64_t s = (uint64_t)k * CHUNK_SPANS;
      while (ci + 1 < c->n_local && off_span[ci + 1] <= s) ++ci;
      chunk_first[k] = ci;
    }
    chunk_first[c->n_chunks] = c->n_local ? c->n_local - 1 : 0;
  }
  auto& r = c->ref;
  int rc;
  if (c->n_local == 0)  // empty shard: nothing to allocate beyond the rows
    return r.d_rows.ensure(c, std::max<size_t>(1, n_contigs));
  // no delta arena: contig mode's events go to the sample's event list (K1) and K2 builds its rows in shared memory; gene
  // mode allocates the arena after this layout (set_genes)
  const size_t n_words = c->arena_elems / BITMAP_ELEMS_PER_WORD;
  if ((rc = r.d_span_bits.ensure(c, n_words)) ||
      (rc = r.d_word_count.ensure(c, n_words)) || (rc = r.d_word_off.ensure(c, n_words + 1)) ||
      (rc = r.d_word_block_sum.ensure(c, n_words / K1B_BLOCK + 1)) ||
      (rc = r.d_off_span.ensure(c, (size_t)c->n_local + 1)) || (rc = r.d_len.ensure(c, c->n_local)) ||
      (rc = r.d_chunk_first.ensure(c, (size_t)c->n_chunks + 1)) || (rc = r.d_tail_sum.ensure(c, c->n_chunks)) ||
      (rc = r.d_carry_in.ensure(c, c->n_chunks)) || (rc = r.d_block_agg.ensure(c, (size_t)c->n_chunks / K1B_BLOCK + 1)) ||
      (rc = r.d_rows.ensure(c, n_contigs)))
    return rc;
  CU_TRY(c, cudaMemcpyAsync(r.d_off_span, off_span.data(), 4ull * (c->n_local + 1), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(r.d_len, len.data(), 4ull * c->n_local, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(r.d_chunk_first, chunk_first.data(), 4ull * (c->n_chunks + 1), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  // histogram bin pool: sized before each K2 from the sample (run_end_of_sample); bin_hi starts at zero like the pool
  if ((rc = r.d_bin_base.ensure(c, (size_t)c->n_local + 1)) || (rc = r.d_bin_block_sum.ensure(c, c->n_local / K1B_BLOCK + 1)) ||
      (rc = r.d_bin_hi.ensure(c, c->n_local)))
    return rc;
  CU_TRY(c, cudaMemsetAsync(r.d_bin_hi, 0, 4ull * c->n_local, c->stream));
  CU_TRY(c, cudaMemsetAsync(r.d_bin_base, 0, 8ull * (c->n_local + 1), c->stream));
  if (small_hist() && (rc = ensure_pool(c, 64, 64))) return rc;  // testing aid: a pool that overflows at once
  c->pool_dirty = false;
  c->arena_dirty = true;
  return CMB_OK;
}

int cmb_set_params(cmb_ctx* c, const cmb_params* p, cmb_filter_mode* mode_out) {
  if (!c || !p) return fail(c, CMB_E_ARG, "cmb_set_params: null argument");
  if (c->in_sample) return fail(c, CMB_E_ARG, "cmb_set_params: a sample is in progress");
  c->params = *p;
  // filter.rs:48-61
  const bool single_initial = p->min_aligned_length_single > 0 || p->min_percent_identity_single > 0.0f || p->min_aligned_percent_single > 0.0f;
  const bool pairs_initial = p->min_aligned_length_pair > 0 || p->min_percent_identity_pair > 0.0f || p->min_aligned_percent_pair > 0.0f;
  const bool fs = single_initial || (!pairs_initial && p->min_mapq != 255);
  const bool fp = pairs_initial || ((!fs || !p->include_improper_pairs) && p->min_mapq != 255);
  c->mode.filter_single_reads = p->filtering ? fs : 0;
  c->mode.filter_pairs = p->filtering ? fp : 0;
  if (mode_out) *mode_out = c->mode;
  c->have_params = true;
  return CMB_OK;
}

int cmb_begin_sample(cmb_ctx* c) {
  NvtxRange nvtx_fn("cmb_begin_sample");
  if (!c) return CMB_E_ARG;
  if (!c->ref.d_rows || !c->have_params) return fail(c, CMB_E_ARG, "cmb_begin_sample: set_reference and set_params first");
  if (c->in_sample) return fail(c, CMB_E_ARG, "cmb_begin_sample: previous sample not ended");
  CU_TRY(c, cudaSetDevice(c->device));
  if (int rc = reset_sample(c)) return rc;
  c->in_sample = true;
  c->ended = false;
  c->n_acquired = 0;
  c->sh.active = false;
  return CMB_OK;
}
}  // extern "C"

// The device state of an empty sample: what cmb_begin_sample sets up, and what a declined cmb_submit_bgzf returns to
int cmb::reset_sample(cmb_ctx* c) {
  c->timing = cmb_sample_timing{};
  c->k1_events_used = 0;
  c->block_minmax_used = 0;
  c->have_xrange = false;
  c->n_records = c->n_intervals = 0;
  CU_TRY(c, cudaEventRecord(c->ev[0], c->stream));
  if (c->n_local) {
    if (c->arena_dirty) {  // contig mode adds no event into the arena
      if (c->gene_mode) CU_TRY(c, cudaMemsetAsync(c->ref.d_arena, 0, c->arena_elems * 4, c->stream));
      CU_TRY(c, cudaMemsetAsync(c->ref.d_span_bits, 0, c->arena_elems / BITMAP_ELEMS_PER_WORD * 4, c->stream));
      CU_TRY(c, cudaMemsetAsync(c->ref.d_word_count, 0, c->arena_elems / BITMAP_ELEMS_PER_WORD * 4, c->stream));
    }
    CU_TRY(c, cudaMemsetAsync(c->ref.d_tail_sum, 0, 4ull * c->n_chunks, c->stream));
    if (c->pool_dirty) {
      if (c->ref.d_bins.cap) CU_TRY(c, cudaMemsetAsync(c->ref.d_bins, 0, 4 * c->ref.d_bins.cap, c->stream));
      CU_TRY(c, cudaMemsetAsync(c->ref.d_bin_hi, 0, 4ull * c->n_local, c->stream));
      c->pool_dirty = false;
    }
    if (c->gene_mode) CU_TRY(c, cudaMemsetAsync(c->ref.d_gene_bound, 0, 4ull * c->n_local, c->stream));
  }
  CU_TRY(c, cudaMemsetAsync(c->ref.d_rows, 0, sizeof(cmb_contig_stats) * (size_t)c->n_contigs, c->stream));
  CU_TRY(c, cudaMemsetAsync(c->d_counters, 0, 64, c->stream));
  if (c->gene_mode) CU_TRY(c, cudaMemsetAsync(c->ref.d_contig_seen, 0, std::max<size_t>(1, c->n_ref_contigs), c->stream));
  CU_TRY(c, cudaEventRecord(c->ev[1], c->stream));
  c->arena_dirty = true;  // until K2 has cleaned it
  // The pair buffer is sized from the sample's records before K3 (run_end_of_sample); the testing aid starts it with 64 pairs,
  // which overflow at once (cmb_grow_buffers path)
  if ((c->params.want & CMB_WANT_HIST_CSR) && c->n_local && small_hist())
    if (int rc = c->ref.d_pairs.ensure(c, 64)) return rc;
  return CMB_OK;
}

extern "C" {

int cmb_acquire_batch(cmb_ctx* c, cmb_read_batch* batch) {
  if (!c || !batch) return fail(c, CMB_E_ARG, "cmb_acquire_batch: null argument");
  if (!c->in_sample) return fail(c, CMB_E_ARG, "cmb_acquire_batch: no sample in progress");
  if (c->n_acquired >= c->cfg.n_staging) return fail(c, CMB_E_ARG, "cmb_acquire_batch: every staging batch is already acquired");
  const uint32_t i = c->next_batch;
  if (c->batch_busy[i]) {  // its previous H2D + K1 must have drained
    CU_TRY(c, cudaEventSynchronize(c->batch_done[i]));
    c->batch_busy[i] = false;
  }
  *batch = c->host_batch[i];
  c->next_batch = (i + 1) % c->cfg.n_staging;
  c->n_acquired += 1;
  return CMB_OK;
}

int cmb_submit_batch(cmb_ctx* c, uint32_t n_records, uint32_t n_intervals) {
  NvtxRange nvtx_fn("cmb_submit_batch: H2D + K1");
  if (!c) return CMB_E_ARG;
  if (!c->in_sample || c->n_acquired == 0) return fail(c, CMB_E_ARG, "cmb_submit_batch: no acquired batch");
  if (n_records > c->cfg.batch_records || n_intervals > c->cfg.batch_intervals) return fail(c, CMB_E_ARG, "cmb_submit_batch: batch exceeds capacity");
  const uint32_t i = (c->next_batch + c->cfg.n_staging - c->n_acquired) % c->cfg.n_staging;  // oldest acquired batch
  c->n_acquired -= 1;
  if (n_records == 0) return CMB_OK;
  if (!k1_active(c)) return CMB_OK;
  const cmb_read_batch& h = c->host_batch[i];
  const cmb_read_batch& d = c->dev_batch[i].ptr;
  CU_TRY(c, cudaSetDevice(c->device));
#define H2D(col, bytes) CU_TRY(c, cudaMemcpyAsync(d.col, h.col, (bytes), cudaMemcpyHostToDevice, c->stream))
  H2D(tid, 4ull * n_records);
  H2D(pos, 4ull * n_records);
  H2D(nm, 4ull * n_records);
  H2D(l_seq, 4ull * n_records);
  H2D(aligned, 4ull * n_records);
  H2D(del, 4ull * n_records);
  H2D(ins, 4ull * n_records);
  H2D(iv_begin, 4ull * (n_records + 1));
  if (n_intervals) {
    H2D(iv_start, 4ull * n_intervals);
    H2D(iv_len, 4ull * n_intervals);
  }
  H2D(flag, 2ull * n_records);
  H2D(mapq, 1ull * n_records);
  H2D(nm_state, 1ull * n_records);
#undef H2D
  int rc = launch_k1(c, d, n_records, n_intervals);
  if (rc) return rc;
  CU_TRY(c, cudaEventRecord(c->batch_done[i], c->stream));
  c->batch_busy[i] = true;
  return CMB_OK;
}

int cmb_submit_device_batch(cmb_ctx* c, const cmb_read_batch* dev, uint32_t n_records, uint32_t n_intervals) {
  NvtxRange nvtx_fn("cmb_submit_device_batch: K1");
  if (!c || !dev) return fail(c, CMB_E_ARG, "cmb_submit_device_batch: null argument");
  if (!c->in_sample) return fail(c, CMB_E_ARG, "cmb_submit_device_batch: no sample in progress");
  if (!k1_active(c)) return CMB_OK;
  CU_TRY(c, cudaSetDevice(c->device));
  // re-submitting the tuples of the last device decode (cmb_last_bgzf_batch) in pair mode: its mate table goes with it
  const bool is_last = c->dec.last_valid && (const void*)dev->tid == c->dec.d_tuple_slab;
  if (is_last && c->mode.filter_pairs && (!c->dec.last_mate || c->dec.last_mate_inverse)) {  // decoded by cmb_decode_bgzf
    if (int rc = match_mates(c, c->dec.last_infl_base, c->dec.last_n_rec, true, "cmb_submit_device_batch")) return rc;
  }
  const int32_t* mate = (is_last && c->dec.last_mate && c->mode.filter_pairs) ? c->dec.last_mate : nullptr;
  return launch_k1(c, *dev, n_records, n_intervals, is_last ? c->dec.last_excl_n : 0xffffffffu, mate);
}

int cmb_end_sample_device(cmb_ctx* c, const cmb_contig_stats** dev_stats) {
  NvtxRange nvtx_fn("cmb_end_sample: K1c K1b K2 K3");
  if (!c) return CMB_E_ARG;
  if (!c->in_sample) return fail(c, CMB_E_ARG, "cmb_end_sample: no sample in progress");
  if (c->n_acquired) return fail(c, CMB_E_ARG, "cmb_end_sample: an acquired batch was not submitted");
  CU_TRY(c, cudaSetDevice(c->device));
  c->in_sample = false;
  c->pool_dirty = true;  // until the sample has ended without an error (K3 re-zeroed every bin K2 added)
  if (c->n_local) {
    int rc = run_end_of_sample(c);
    if (rc) return rc;
  } else {
    CU_TRY(c, cudaEventRecord(c->ev[2], c->stream));
    if (c->block_minmax_used) {  // gene mode: owned contigs without genes still ran K1 (k1_active)
      k1c_check_sorted<<<1, 1024, 0, c->stream>>>(c->d_block_minmax, c->block_minmax_used, c->d_counters + 0,
                                                  c->have_xrange ? c->d_block_xrange.p : nullptr, c->d_counters + 6);
      CU_TRY(c, cudaGetLastError());
    }
    for (int i = 3; i <= 5; ++i) CU_TRY(c, cudaEventRecord(c->ev[i], c->stream));
  }
  uint32_t counters[6];
  int rc = collect_errors_and_timing(c, counters);
  if (rc) return rc;
  c->pool_dirty = false;
  c->ended = true;
  if (dev_stats) *dev_stats = c->ref.d_rows;
  return CMB_OK;
}

int cmb_end_sample(cmb_ctx* c, cmb_contig_stats* stats, cmb_hist_pair* pairs, uint64_t pairs_capacity, uint64_t* n_pairs) {
  NvtxRange nvtx_fn("cmb_end_sample: kernels + D2H");
  if (!c) return fail(c, CMB_E_ARG, "cmb_end_sample: null argument");
  int rc = cmb_end_sample_device(c, nullptr);
  if (rc) return rc;
  if (stats) CU_TRY(c, cudaMemcpyAsync(stats, c->ref.d_rows, sizeof(cmb_contig_stats) * (size_t)c->n_contigs, cudaMemcpyDeviceToHost, c->stream));
  uint64_t np = 0;
  if ((c->params.want & CMB_WANT_HIST_CSR) && c->n_local) {
    unsigned long long cnt = 0;
    CU_TRY(c, cudaMemcpyAsync(&cnt, c->d_counters + 4, 8, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    np = cnt;
    if (np > c->ref.d_pairs.cap) return fail(c, CMB_E_CAPACITY, "device histogram pair buffer overflowed");
    if (pairs) {
      if (np > pairs_capacity) return fail(c, CMB_E_CAPACITY, "cmb_end_sample: caller's pair buffer too small (%llu needed)", (unsigned long long)np);
      if (np) CU_TRY(c, cudaMemcpyAsync(pairs, c->ref.d_pairs, sizeof(cmb_hist_pair) * np, cudaMemcpyDeviceToHost, c->stream));
    }
  }
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (n_pairs) *n_pairs = np;
  return CMB_OK;
}

int cmb_fetch_pairs(cmb_ctx* c, cmb_hist_pair* pairs, uint64_t n_pairs) {
  if (!c || (!pairs && n_pairs)) return fail(c, CMB_E_ARG, "cmb_fetch_pairs: null argument");
  if (!c->ended) return fail(c, CMB_E_ARG, "cmb_fetch_pairs: no ended sample");
  if (n_pairs > c->ref.d_pairs.cap) return fail(c, CMB_E_ARG, "cmb_fetch_pairs: more pairs requested than produced");
  if (n_pairs) {
    CU_TRY(c, cudaSetDevice(c->device));
    CU_TRY(c, cudaMemcpyAsync(pairs, c->ref.d_pairs, sizeof(cmb_hist_pair) * n_pairs, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
  }
  return CMB_OK;
}

int cmb_grow_buffers(cmb_ctx* c) {
  if (!c || !c->ref.d_rows) return fail(c, CMB_E_ARG, "cmb_grow_buffers: no reference set");
  if (c->in_sample) return fail(c, CMB_E_ARG, "cmb_grow_buffers: a sample is in progress");
  if (c->n_local == 0) return CMB_OK;
  CU_TRY(c, cudaSetDevice(c->device));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  auto& r = c->ref;  // the next sample rebuilds what these hold
  // the bins the last sample needed: K1b's bin_base[n_local] (it stays in place until the next sample's K1b)
  uint64_t need = 0;
  CU_TRY(c, cudaMemcpyAsync(&need, r.d_bin_base + c->n_local, 8, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  int rc;
  if ((rc = ensure_pool(c, need, need)) || (r.d_pairs && (rc = r.d_pairs.ensure(c, r.d_pairs.cap * 4)))) return rc;
  c->arena_dirty = true;
  return CMB_OK;
}

int cmb_get_timing(const cmb_ctx* c, cmb_sample_timing* out) {
  if (!c || !out) return CMB_E_ARG;
  *out = c->timing;
  return CMB_OK;
}

void* cmb_stream(cmb_ctx* c) { return c ? (void*)c->stream : nullptr; }

void cmb_nvtx_push(const char* name) { nvtxRangePushA(name ? name : "?"); }
void cmb_nvtx_pop(void) { nvtxRangePop(); }

int cmb_kept_tid_range(cmb_ctx* c, int32_t* min_tid, int32_t* max_tid) {
  if (!c || !min_tid || !max_tid) return fail(c, CMB_E_ARG, "cmb_kept_tid_range: null argument");
  if (!c->ended) return fail(c, CMB_E_ARG, "cmb_kept_tid_range: no ended sample");
  if (c->kept_range[0] == 0) {
    *min_tid = INT_MAX;
    *max_tid = INT_MIN;
  } else {
    *max_tid = (int32_t)(c->kept_range[0] - 1);
    *min_tid = INT_MAX - (int32_t)c->kept_range[1];
  }
  return CMB_OK;
}

void* cmb_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
void cmb_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
