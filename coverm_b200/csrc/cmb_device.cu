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
//   KD* kd_inflate ...        device-side BAM decode behind cmb_submit_bgzf (cmb_decode.cuh): BGZF inflate, record chain,
//                             tuple extraction -- the compressed file crosses PCIe instead of tuples.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <nccl.h>
#include <nvtx3/nvToolsExt.h>
#include <strings.h>
#include <unistd.h>
#include <zlib.h>

#include "../../include/coverm_b200.h"

// NVTX ranges around the entry points and the stages of the device decode (visible in Nsight Systems / `ncu --nvtx`; no-ops
// without a tool attached: nvtx3 is header-only and resolves its injection library lazily).
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

namespace {
#include "cmb_common.cuh"
#include "cmb_k1.cuh"
#include "cmb_k1b.cuh"
#include "cmb_k2.cuh"
#include "cmb_k3.cuh"
#include "cmb_decode.cuh"
#include "cmb_decode_g8.cuh"
#include "cmb_decode_t1.cuh"
#include "cmb_pairs.cuh"
#include "cmb_filter.cuh"
#include "cmb_shards.cuh"
#include "cmb_shard_slices.hpp"
#include "cmb_decode_slices.hpp"

// rows[i].hist_offset += base for the rows that carry histogram pairs (cmb_allgather_stats: local -> global pair offsets)
__global__ void __launch_bounds__(256) k_rebase_hist_offsets(cmb_contig_stats* rows, uint32_t n, uint64_t base) {
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i < n && rows[i].hist_count) rows[i].hist_offset += base;
}

// ------------------------------------------------------------------------------------------------ host context
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

std::string g_create_error;

// Ranks that live in ONE process (cmb_comm_init_local) meet here before every collective: a rank must not be inside a CUDA call
// that synchronises across devices (cudaHostAlloc, cudaMalloc, cudaFree ...) while another rank's NCCL kernel is already
// waiting for it -- that is the classic single-process multi-GPU deadlock.  All allocation happens before the barrier, only
// stream-ordered work after it.
struct LocalBarrier {
  std::mutex m;
  std::condition_variable cv;
  int n = 0, waiting = 0;
  uint64_t generation = 0;
  void arrive_and_wait() {
    std::unique_lock<std::mutex> lk(m);
    const uint64_t g = generation;
    if (++waiting == n) {
      waiting = 0;
      ++generation;
      cv.notify_all();
    } else {
      cv.wait(lk, [&] { return generation != g; });
    }
  }
};

// The owner of one device allocation (PINNED: pinned host memory) of `cap` elements of T; it is freed with its owner.
// ensure() only grows and does not keep the contents; the caller decides how much to allocate when it has to grow.
template <class T, bool PINNED = false>
struct Buf {
  T* p = nullptr;
  size_t cap = 0;
  Buf() = default;
  Buf(Buf&& o) noexcept : p(o.p), cap(o.cap) {
    o.p = nullptr;
    o.cap = 0;
  }
  Buf& operator=(Buf&& o) noexcept {
    if (this != &o) {
      release();
      std::swap(p, o.p);
      std::swap(cap, o.cap);
    }
    return *this;
  }
  ~Buf() { release(); }
  operator T*() const { return p; }
  uint64_t bytes() const { return sizeof(T) * (uint64_t)cap; }
  void release() {
    if (p) {
      if (PINNED) cudaFreeHost(p);
      else cudaFree(p);
    }
    p = nullptr;
    cap = 0;
  }
  // room for `need` elements: allocates `alloc` (>= need) when there is less
  int ensure(cmb_ctx* c, size_t need, size_t alloc);
  int ensure(cmb_ctx* c, size_t n) { return ensure(c, n, n); }
  // n elements, keeping the first `used` (copied on `st`, which is synchronised before the old allocation is freed)
  int grow_keep(cmb_ctx* c, size_t used, size_t n, cudaStream_t st);
};
template <class T>
using PinnedBuf = Buf<T, true>;

struct DevBatch {  // device mirror of one staging batch
  Buf<uint8_t> slab;
  cmb_read_batch ptr{};
};

}  // namespace

struct cmb_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  cmb_device_cfg cfg{};
  int sm_count = 0;
  // staging
  std::vector<PinnedBuf<uint8_t>> host_slab;
  std::vector<cmb_read_batch> host_batch;
  std::vector<DevBatch> dev_batch;
  std::vector<cudaEvent_t> batch_done;
  std::vector<bool> batch_busy;
  uint32_t n_acquired = 0;   // staging batches handed out and not yet submitted (FIFO)
  uint32_t next_batch = 0;   // next staging slot to hand out
  // reference
  uint32_t n_contigs = 0, tid_begin = 0, tid_end = 0, n_local = 0;
  uint64_t arena_elems = 0;
  uint32_t n_chunks = 0;
  struct Reference {  // the buffers that live as long as one reference (cmb_set_reference / cmb_set_genes)
    Buf<int32_t> d_arena;
    Buf<uint32_t> d_span_bits;
    Buf<uint32_t> d_word_count, d_word_off, d_word_block_sum;  // contig mode: events per bitmap word, their scan (K1b)
    Buf<uint32_t> d_off_span, d_len, d_chunk_first;
    Buf<int32_t> d_tail_sum, d_carry_in;
    Buf<int2> d_block_agg;
    Buf<cmb_contig_stats> d_rows;
    Buf<uint32_t> d_bins;  // K2 -> K3 histogram bin pool; cap is the capacity K2 is given.  Zero outside a sample
    Buf<uint64_t> d_bin_base, d_bin_block_sum;
    Buf<uint32_t> d_bin_hi;
    Buf<cmb_hist_pair> d_pairs;  // CSR histogram pairs (CMB_WANT_HIST_CSR)
    // gene mode (cmb_set_genes): segments are genes; records carry contig tids
    Buf<uint32_t> d_gene_first, d_gene_start, d_gene_end, d_gene_maxlen, d_contig_len32;
    Buf<uint8_t> d_contig_seen;
    Buf<uint32_t> d_gene_bound;
  } ref;
  Buf<uint32_t> d_counters;  // 16 words: [0] error flags, [4..5] pair_count (u64),
                             // [6..7] kept tid range of the exclusive records (K1Args::kept_range), [8..9] gene mode
                             // kept primaries (u64), [10..12] K2 spans loaded / chunks loaded whole / bucket entries read
  // contig mode: the sample's event list (K1, one entry pair per interval) and its events bucketed by word (K1e); grow-only
  Buf<ulonglong2> d_events;
  Buf<uint16_t> d_buckets;
  uint32_t kept_range[2] = {0, 0};  // host copy after cmb_end_sample*
  // multi-GPU (cmb_comm_*): one NCCL communicator per ctx, collectives on the ctx stream
  ncclComm_t comm = nullptr;
  int comm_rank = 0, comm_size = 1;
  std::shared_ptr<LocalBarrier> local_barrier;  // set when all ranks of the communicator live in this process
  Buf<uint8_t> d_xchg;  // staging of cmb_comm_allgather
  Buf<cmb_hist_pair> d_pairs_all;  // concatenated histogram pairs of all ranks (cmb_allgather_stats)
  Buf<int2> d_block_minmax;
  Buf<int2> d_block_xrange;  // same capacity as d_block_minmax
  bool have_xrange = false;
  uint32_t block_minmax_used = 0;
  bool gene_mode = false;
  uint32_t n_ref_contigs = 0;  // contigs of the BAM header (== n_contigs outside gene mode)
  // gene mode: the contigs whose records this context counts (cmb_set_genes_range); tid_begin / tid_end are then its genes
  uint32_t gene_tid_begin = 0, gene_tid_end = 0;
  CUtensorMap tmap{};
  bool arena_dirty = true;
  bool pool_dirty = false;  // a sample ended with an error: bins / bin_hi may hold counts (cmb_begin_sample zeroes them)
  bool clean_as_you_go = true;
  // params
  cmb_params params{};
  cmb_filter_mode mode{};
  bool have_params = false, in_sample = false, ended = false;
  // timing
  cudaEvent_t ev[8]{};
  cmb_sample_timing timing{};
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> k1_events;
  uint32_t k1_events_used = 0;
  uint64_t n_records = 0, n_intervals = 0;
  // device-side decode (cmb_submit_bgzf); every buffer is grow-only and reused across samples
  struct Decode {
    Buf<uint8_t> d_comp, d_inflated;
    // per BGZF block
    Buf<uint64_t> d_coff, d_ustart, d_guess, d_exit, d_rec_base, d_cig_base;
    Buf<uint32_t> d_clen, d_isize, d_status, d_nrec, d_ncig, d_dirty;
    Buf<uint8_t> d_t1_scratch;  // kd_inflate_t1: code-length scratch, T1_LENS_BYTES per block
    Buf<uint32_t> d_tickets;  // [0] block ticket, [1 + w] window w has arrived
    Buf<uint32_t> d_block_window;
    PinnedBuf<uint32_t> h_ones;  // source of the arrival flags
    Buf<uint32_t> d_cnt;  // 20 words: [0] inflate failures [1] decode error bits [2] chain changed [4..5] n_primary [6..9] totals
                          // [10..11] n_owned; sliced decode: [12..14] pair cut (decode_sliced), [16..19] held-back counts
    Buf<uint64_t> d_rec_off;
    Buf<uint8_t> d_tuple_slab;
    uint32_t last_n_rec = 0, last_n_cig = 0;  // tuples of the last successful cmb_submit_bgzf (cmb_last_bgzf_batch)
    bool last_valid = false;
    // mate matching (cmb_pairs.cuh)
    Buf<uint64_t> d_pair_key;
    Buf<int32_t> d_pair_mate;
    Buf<uint32_t> d_pair_next;
    Buf<unsigned long long> d_pair_tag;
    Buf<uint32_t> d_pair_head;
    Buf<uint2> d_pair_order;  // kd_pair_order: per PAIR_ORDER_CHUNK records, their first and last eligible tid
    const int32_t* last_mate = nullptr;
    bool last_mate_inverse = false;  // last_mate was matched for `coverm filter --inverse` (unmapped records not eligible)
    uint32_t last_excl_n = 0xffffffffu;
    const uint8_t* last_infl_base = nullptr;  // biased base of the inflated stream of the last decode
    // coverm filter
    Buf<unsigned long long> d_filter_anchor;
    Buf<uint8_t> d_filter_role;
    Buf<uint8_t> d_filter_out;
    uint64_t filter_bytes = 0;
    bool filter_planned = false;
    std::vector<PinnedBuf<uint8_t>> pinned;  // two copy slots per copy stream
    std::vector<cudaStream_t> streams;
    std::vector<cudaEvent_t> slot_events, done_events;
    cudaEvent_t ev[6]{};
    bool have_events = false;
  } dec;
  // sharded input (cmb_shard_*; cmb_shards.cuh): per-shard primary stores and the running choice of every pair; grow-only
  struct Shards {
    struct Store {  // one buffer per column, each grown in place (Buf::grow_keep) as the shard's slices append primaries
      Buf<int32_t> tid, pos, iv_start, iv_len;
      Buf<uint32_t> nm, l_seq, aligned, del, ins, iv_begin;
      Buf<uint16_t> flag;
      Buf<uint8_t> mapq, nm_state, info;
      Buf<unsigned long long> names;  // group runs, shards k > 0: name hashes for ks_names
      Buf<int32_t> as_val;            // group runs: the shard's AS values and states, kept until cmb_shard_score
      Buf<uint8_t> as_state;
      ShardStore view{};
      uint64_t n_prim = 0, n_iv = 0;
      uint64_t bytes() const {
        return tid.bytes() + pos.bytes() + iv_start.bytes() + iv_len.bytes() + nm.bytes() + l_seq.bytes() + aligned.bytes() + del.bytes() +
               ins.bytes() + iv_begin.bytes() + flag.bytes() + mapq.bytes() + nm_state.bytes() + info.bytes() + names.bytes() +
               as_val.bytes() + as_state.bytes();
      }
    };
    std::vector<Store> store;
    std::vector<int32_t> tid_offsets;
    uint32_t n_shards = 0, added = 0;
    bool active = false;
    // group runs (cmb_shard_begin_range): this context decodes shards [first, last); the others' scores arrive in d_score
    uint32_t first = 0, last = 0;
    bool group = false;
    Buf<int32_t> d_score;            // [n_shards][n_pairs] score table (ks_score, exchanged, ks_choose)
    std::vector<uint64_t> n_prim;    // every shard's primaries (cmb_shard_score)
    uint64_t n_pairs = 0, n_out = 0;
    unsigned long long len_key = ~0ull;  // the reader's length checks, keyed like the kernels' errors
    int stage = 0;                   // 1 scored, 2 chosen
    Buf<uint8_t> d_excluded;
    bool have_excluded = false;
    Buf<unsigned long long> d_scan, d_hash0, d_err, d_tid_count, d_src, d_slot_iv;
    Buf<int32_t> d_as_val;
    Buf<uint8_t> d_as_state;
    Buf<PairState> d_state;
    Buf<ShardStore> d_stores;
    Buf<int32_t> d_tid_offsets;
    Buf<uint8_t> d_out_slab;
    cudaEvent_t ev[4]{};
    float ms_choose = 0, ms_decode = 0;
  } sh;
};

namespace {

int fail(cmb_ctx* ctx, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf;
  else g_create_error = buf;
  return code;
}

#define CU_TRY(ctx, expr)                                                                                   \
  do {                                                                                                      \
    cudaError_t e_ = (expr);                                                                                \
    if (e_ != cudaSuccess) return fail(ctx, e_ == cudaErrorMemoryAllocation ? CMB_E_NOMEM : CMB_E_CUDA,      \
                                       "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

template <class T, bool PINNED>
int Buf<T, PINNED>::ensure(cmb_ctx* c, size_t need, size_t alloc) {
  if (p && cap >= need) return CMB_OK;
  release();
  if (PINNED) CU_TRY(c, cudaHostAlloc((void**)&p, sizeof(T) * alloc, cudaHostAllocDefault));
  else CU_TRY(c, cudaMalloc((void**)&p, sizeof(T) * alloc));
  cap = alloc;
  return CMB_OK;
}

template <class T, bool PINNED>
int Buf<T, PINNED>::grow_keep(cmb_ctx* c, size_t used, size_t n, cudaStream_t st) {
  Buf b;
  if (int rc = b.ensure(c, n)) return rc;
  if (used) CU_TRY(c, cudaMemcpyAsync(b.p, p, sizeof(T) * used, cudaMemcpyDeviceToDevice, st));
  CU_TRY(c, cudaStreamSynchronize(st));
  *this = std::move(b);
  return CMB_OK;
}

size_t with_slack(size_t n) { return n + n / 8 + 16; }  // grow-only buffers sized by the data

size_t batch_slab_bytes(uint32_t nr, uint32_t ni, size_t* offs) {
  // column order: tid,pos,nm,l_seq,aligned,del,ins,iv_begin(nr+1),iv_start(ni),iv_len(ni),flag(u16),mapq(u8),nm_state(u8)
  size_t o = 0;
  auto take = [&](size_t bytes) {
    size_t r = o;
    o += (bytes + 255) & ~(size_t)255;
    return r;
  };
  offs[0] = take(4ull * nr);        // tid
  offs[1] = take(4ull * nr);        // pos
  offs[2] = take(4ull * nr);        // nm
  offs[3] = take(4ull * nr);        // l_seq
  offs[4] = take(4ull * nr);        // aligned
  offs[5] = take(4ull * nr);        // del
  offs[6] = take(4ull * nr);        // ins
  offs[7] = take(4ull * (nr + 1));  // iv_begin
  offs[8] = take(4ull * ni);        // iv_start
  offs[9] = take(4ull * ni);        // iv_len
  offs[10] = take(2ull * nr);       // flag
  offs[11] = take(1ull * nr);       // mapq
  offs[12] = take(1ull * nr);       // nm_state
  return o;
}

void carve_batch(void* slab, uint32_t nr, uint32_t ni, cmb_read_batch* b) {
  size_t offs[13];
  batch_slab_bytes(nr, ni, offs);
  uint8_t* p = (uint8_t*)slab;
  b->capacity_records = nr;
  b->capacity_intervals = ni;
  b->tid = (int32_t*)(p + offs[0]);
  b->pos = (int32_t*)(p + offs[1]);
  b->nm = (uint32_t*)(p + offs[2]);
  b->l_seq = (uint32_t*)(p + offs[3]);
  b->aligned = (uint32_t*)(p + offs[4]);
  b->del = (uint32_t*)(p + offs[5]);
  b->ins = (uint32_t*)(p + offs[6]);
  b->iv_begin = (uint32_t*)(p + offs[7]);
  b->iv_start = (int32_t*)(p + offs[8]);
  b->iv_len = (int32_t*)(p + offs[9]);
  b->flag = (uint16_t*)(p + offs[10]);
  b->mapq = (uint8_t*)(p + offs[11]);
  b->nm_state = (uint8_t*)(p + offs[12]);
}

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

// Whether K1 has work: a context with no local segment has none, except in gene mode, where owned contigs without genes still
// set contig_seen, count kept_primary and take part in the sortedness check.
bool k1_active(const cmb_ctx* c) { return c->n_local || (c->gene_mode && c->gene_tid_begin < c->gene_tid_end); }

int launch_k1(cmb_ctx* c, const cmb_read_batch& b, uint32_t n_records, uint32_t n_intervals, uint32_t excl_n = 0xffffffffu,
              const int32_t* mate = nullptr) {
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

// Mate matching over the resident inflated stream (cmb_pairs.cuh); sets d.last_mate.  filter_out: ReferenceSortedBamFilter's
// (false only for `coverm filter --inverse`).  Declines when the stream needs the host's file-order walk.  A slice of a sliced
// decode passes the largest eligible tid of the slices before it (`carry`) and gets its own largest in *largest (device).
int match_mates(cmb_ctx* c, const uint8_t* infl_base, uint32_t n_rec, bool filter_out, const char* who, uint32_t carry = 0,
                uint32_t* largest = nullptr) {
  auto& d = c->dec;
  int rc;
  d.last_mate = nullptr;
  d.filter_planned = false;
  if (d.d_pair_key.cap < n_rec) {  // growing: give the filter's buffers back first (cmb_filter_plan sizes them again)
    d.d_filter_anchor.release();
    d.d_filter_role.release();
    d.d_filter_out.release();
  }
  const size_t want = with_slack(n_rec);
  const uint32_t n_chunks = (n_rec + PAIR_ORDER_CHUNK - 1) / PAIR_ORDER_CHUNK;
  if ((rc = d.d_pair_key.ensure(c, n_rec, want)) || (rc = d.d_pair_mate.ensure(c, n_rec, want)) || (rc = d.d_pair_next.ensure(c, n_rec, want)) ||
      (rc = d.d_pair_order.ensure(c, n_chunks, with_slack(n_chunks))))
    return rc;
  size_t table = 1u << 16;
  while (table < 2 * (size_t)n_rec) table <<= 1;
  if ((rc = d.d_pair_tag.ensure(c, table)) || (rc = d.d_pair_head.ensure(c, table))) return rc;
  CU_TRY(c, cudaMemsetAsync(d.d_pair_tag, 0, 8 * table, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_pair_head, 0xff, 4 * table, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_cnt + 1, 0, 4, c->stream));
  PairArgs pa{};
  pa.data = infl_base; pa.rec_off = d.d_rec_off; pa.n_records = n_rec; pa.key = d.d_pair_key; pa.mate = d.d_pair_mate;
  pa.next = d.d_pair_next; pa.slot_tag = d.d_pair_tag; pa.slot_head = d.d_pair_head; pa.table_mask = (uint32_t)(table - 1);
  pa.flags = d.d_cnt + 1; pa.order = d.d_pair_order; pa.filter_out = filter_out ? 1 : 0;
  const uint32_t gr = (n_rec + 255) / 256;
  kd_pair_keys<<<gr, 256, 0, c->stream>>>(pa);
  kd_pair_order<<<(n_chunks + 255) / 256, 256, 0, c->stream>>>(pa);
  kd_pair_order_fold<<<1, 1024, 0, c->stream>>>(d.d_pair_order, n_chunks, pa.flags, carry, largest);
  kd_pair_insert<<<gr, 256, 0, c->stream>>>(pa);
  kd_pair_resolve<<<(uint32_t)((table + 255) / 256), 256, 0, c->stream>>>(pa);
  CU_TRY(c, cudaGetLastError());
  uint32_t flags = 0;
  CU_TRY(c, cudaMemcpyAsync(&flags, d.d_cnt + 1, 4, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (flags)
    return fail(c, CMB_E_DECLINED, "%s: mate matching gave up (flags %u: %s)", who, flags,
                (flags & DEC_ERR_PAIR_ORDER) ? "the proper-pair records' reference ids are not sorted" : "too many records of one name");
  d.last_mate = d.d_pair_mate;
  d.last_mate_inverse = !filter_out;
  return CMB_OK;
}

int reset_sample(cmb_ctx* c);

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

namespace {
// The device state of an empty sample: what cmb_begin_sample sets up, and what a declined cmb_submit_bgzf returns to
int reset_sample(cmb_ctx* c) {
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
}  // namespace

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

// ------------------------------------------------------------------------------------------------ multi-GPU (NCCL)
#define NCCL_TRY(ctx, expr)                                                                                       \
  do {                                                                                                            \
    ncclResult_t r_ = (expr);                                                                                     \
    if (r_ != ncclSuccess) return fail(ctx, CMB_E_CUDA, "%s failed: %s (%s:%d)", #expr, ncclGetErrorString(r_), __FILE__, __LINE__); \
  } while (0)

namespace {
// NCCL writes its banner / debug lines to stdout by default; stdout carries the coverage table.
void nccl_output_to_stderr() {
  static const bool once = [] {
    // NCCL honours NCCL_DEBUG_FILE only above the VERSION level: at NCCL_DEBUG=VERSION the banner goes to stdout regardless
    const char* lvl = getenv("NCCL_DEBUG");
    if (lvl && !strcasecmp(lvl, "VERSION")) setenv("NCCL_DEBUG", "WARN", 1);  // WARN prints the same banner, to the debug file
    if (!getenv("NCCL_DEBUG_FILE")) setenv("NCCL_DEBUG_FILE", "/dev/stderr", 0);
    return true;
  }();
  (void)once;
}
// While a communicator is created, file descriptor 1 points at stderr: whatever NCCL (or a plugin it loads) prints during
// initialisation cannot end up in the coverage table.  Nothing else writes to stdout at that point (tables are printed at the end).
struct StdoutGuard {
  static std::mutex& mu() { static std::mutex m; return m; }
  std::lock_guard<std::mutex> lock{mu()};
  int saved = -1;
  StdoutGuard() {
    fflush(stdout);
    saved = dup(1);
    if (saved >= 0) dup2(2, 1);
  }
  ~StdoutGuard() {
    fflush(stdout);
    if (saved >= 0) {
      dup2(saved, 1);
      close(saved);
    }
  }
};
}  // namespace

int cmb_comm_unique_id(uint8_t id[CMB_COMM_ID_BYTES]) {
  nccl_output_to_stderr();
  static_assert(sizeof(ncclUniqueId) == CMB_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  if (!id) return fail(nullptr, CMB_E_ARG, "cmb_comm_unique_id: null argument");
  ncclUniqueId u;
  StdoutGuard guard;
  NCCL_TRY(nullptr, ncclGetUniqueId(&u));
  memcpy(id, &u, sizeof u);
  return CMB_OK;
}

int cmb_comm_init(cmb_ctx* c, const uint8_t id[CMB_COMM_ID_BYTES], int rank, int n_ranks) {
  if (!c || !id || n_ranks < 1 || rank < 0 || rank >= n_ranks) return fail(c, CMB_E_ARG, "cmb_comm_init: bad arguments");
  if (c->comm) return fail(c, CMB_E_ARG, "cmb_comm_init: the context already has a communicator");
  nccl_output_to_stderr();
  CU_TRY(c, cudaSetDevice(c->device));
  ncclUniqueId u;
  memcpy(&u, id, sizeof u);
  {
    StdoutGuard guard;
    NCCL_TRY(c, ncclCommInitRank(&c->comm, n_ranks, u, rank));
  }
  c->comm_rank = rank;
  c->comm_size = n_ranks;
  return CMB_OK;
}

int cmb_comm_init_local(cmb_ctx* const* ctxs, int n_ranks) {
  if (!ctxs || n_ranks < 1) return fail(nullptr, CMB_E_ARG, "cmb_comm_init_local: bad arguments");
  std::vector<int> devs(n_ranks);
  for (int r = 0; r < n_ranks; ++r) {
    if (!ctxs[r] || ctxs[r]->comm) return fail(ctxs[r], CMB_E_ARG, "cmb_comm_init_local: null context or communicator already set");
    devs[r] = ctxs[r]->device;
  }
  std::vector<ncclComm_t> comms(n_ranks);
  nccl_output_to_stderr();
  {
    StdoutGuard guard;
    NCCL_TRY(ctxs[0], ncclCommInitAll(comms.data(), n_ranks, devs.data()));
  }
  auto barrier = std::make_shared<LocalBarrier>();
  barrier->n = n_ranks;
  for (int r = 0; r < n_ranks; ++r) {
    ctxs[r]->local_barrier = barrier;
    ctxs[r]->comm = comms[r];
    ctxs[r]->comm_rank = r;
    ctxs[r]->comm_size = n_ranks;
  }
  return CMB_OK;
}

void cmb_comm_destroy(cmb_ctx* c) {
  if (!c || !c->comm) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  ncclCommDestroy(c->comm);
  c->comm = nullptr;
  c->local_barrier.reset();
  c->comm_rank = 0;
  c->comm_size = 1;
}

int cmb_comm_allgather(cmb_ctx* c, const void* send, void* recv, size_t bytes) {
  if (!c || !send || !recv || !bytes) return fail(c, CMB_E_ARG, "cmb_comm_allgather: bad arguments");
  if (!c->comm) return fail(c, CMB_E_ARG, "cmb_comm_allgather: no communicator (cmb_comm_init first)");
  CU_TRY(c, cudaSetDevice(c->device));
  const size_t need = bytes * (size_t)(c->comm_size + 1);
  if (int rc = c->d_xchg.ensure(c, need, need + 4096)) return rc;
  uint8_t* d_send = c->d_xchg;
  uint8_t* d_recv = c->d_xchg + bytes;
  if (c->local_barrier) c->local_barrier->arrive_and_wait();
  CU_TRY(c, cudaMemcpyAsync(d_send, send, bytes, cudaMemcpyHostToDevice, c->stream));
  NCCL_TRY(c, ncclAllGather(d_send, d_recv, bytes, ncclChar, c->comm, c->stream));
  CU_TRY(c, cudaMemcpyAsync(recv, d_recv, bytes * (size_t)c->comm_size, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}

int cmb_allgather_stats(cmb_ctx* c, const uint32_t* tid_cuts, const uint64_t* pair_base, cmb_contig_stats* stats, cmb_hist_pair* pairs) {
  NvtxRange nvtx_fn("cmb_allgather_stats: NCCL gather");
  if (!c || !tid_cuts) return fail(c, CMB_E_ARG, "cmb_allgather_stats: null argument");
  if (!c->comm) return fail(c, CMB_E_ARG, "cmb_allgather_stats: no communicator (cmb_comm_init first)");
  if (!c->ended || !c->ref.d_rows) return fail(c, CMB_E_ARG, "cmb_allgather_stats: no ended sample");
  const int N = c->comm_size, me = c->comm_rank;
  if (tid_cuts[0] != 0 || tid_cuts[N] != c->n_contigs || tid_cuts[me] != c->tid_begin || tid_cuts[me + 1] != c->tid_end)
    return fail(c, CMB_E_ARG, "cmb_allgather_stats: tid_cuts do not match this context's shard");
  for (int r = 0; r < N; ++r)
    if (tid_cuts[r] > tid_cuts[r + 1]) return fail(c, CMB_E_ARG, "cmb_allgather_stats: tid_cuts must be non-decreasing");
  CU_TRY(c, cudaSetDevice(c->device));
  const bool csr = pair_base && (c->params.want & CMB_WANT_HIST_CSR);
  if (csr) {
    const uint64_t total = pair_base[N];
    if (pair_base[me + 1] - pair_base[me] > c->ref.d_pairs.cap) return fail(c, CMB_E_ARG, "cmb_allgather_stats: pair_base exceeds this rank's pairs");
    if (int rc = c->d_pairs_all.ensure(c, total, total + total / 8 + 1024)) return rc;
    const uint32_t n_own = c->tid_end - c->tid_begin;
    if (n_own && pair_base[me]) {
      k_rebase_hist_offsets<<<(n_own + 255) / 256, 256, 0, c->stream>>>(c->ref.d_rows + c->tid_begin, n_own, pair_base[me]);
      CU_TRY(c, cudaGetLastError());
    }
  }
  if (c->local_barrier) c->local_barrier->arrive_and_wait();
  // every rank broadcasts its own row range in place: afterwards each rank's table is complete (an all-gather with ragged counts)
  NCCL_TRY(c, ncclGroupStart());
  for (int r = 0; r < N; ++r) {
    const size_t n = (size_t)(tid_cuts[r + 1] - tid_cuts[r]) * sizeof(cmb_contig_stats);
    if (!n) continue;
    cmb_contig_stats* p = c->ref.d_rows + tid_cuts[r];
    NCCL_TRY(c, ncclBroadcast(p, p, n, ncclChar, r, c->comm, c->stream));
  }
  if (csr) {
    for (int r = 0; r < N; ++r) {
      const size_t n = (size_t)(pair_base[r + 1] - pair_base[r]) * sizeof(cmb_hist_pair);
      if (!n) continue;
      NCCL_TRY(c, ncclBroadcast(c->ref.d_pairs, c->d_pairs_all + pair_base[r], n, ncclChar, r, c->comm, c->stream));
    }
  }
  NCCL_TRY(c, ncclGroupEnd());
  if (stats) CU_TRY(c, cudaMemcpyAsync(stats, c->ref.d_rows, sizeof(cmb_contig_stats) * (size_t)c->n_contigs, cudaMemcpyDeviceToHost, c->stream));
  if (csr && pairs && pair_base[N])
    CU_TRY(c, cudaMemcpyAsync(pairs, c->d_pairs_all, sizeof(cmb_hist_pair) * pair_base[N], cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}

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

// ------------------------------------------------------------------------------------------------ device-side decode
namespace {
constexpr size_t DEC_COPY_CHUNK = 8u << 20;    // pinned staging slot
constexpr size_t DEC_WINDOW_BYTES = 32u << 20; // compressed bytes per copy+inflate window
size_t dec_window_bytes() {  // CMB_DECODE_WINDOW_KB: testing aid, lets a small file span many windows
  static const size_t v = [] {
    const char* e = getenv("CMB_DECODE_WINDOW_KB");
    const long kb = e ? atol(e) : 0;
    return kb > 0 ? (size_t)kb << 10 : DEC_WINDOW_BYTES;
  }();
  return v;
}
constexpr size_t DEC_SLACK = 1024;
constexpr size_t DEC_FRONT = 256;              // readable bytes in front of the first uploaded block (the bit readers align down)
constexpr uint64_t DEC_TAIL_BYTES = 4u << 20;  // ranged decode: inflated bytes kept beyond the range for its last straddling record

// First-pass inflate kernel: 0 = kd_inflate_t1 (a thread per block + kd_crc32), 1 = kd_inflate_g8 (four blocks per warp), 2 =
// kd_inflate (a warp per block, also the second pass over declined blocks).  t1 has the higher THROUGHPUT (its sm_count x 5 x 96
// streams, 63 360 on 132 SMs, need that many blocks) but each of its streams is slow, so a short list of blocks finishes sooner
// on g8.  The choice follows the number of blocks: a whole 10 M-read file (46 000 blocks) goes to t1, a rank's share of it on 4
// or 8 GPUs to g8.  CMB_INFLATE=t1|g8|w1 overrides.
constexpr uint32_t T1_MIN_BLOCKS = 28000;
int inflate_kind(uint32_t n_blocks) {
  static const int forced = [] {
    const char* e = getenv("CMB_INFLATE");
    if (e && !strcmp(e, "t1")) return 0;
    if (e && !strcmp(e, "g8")) return 1;
    if (e && !strcmp(e, "w1")) return 2;
    return -1;
  }();
  if (forced >= 0) return forced;
  return n_blocks >= T1_MIN_BLOCKS ? 0 : 1;
}
// Default: ONE persistent launch whose threads poll the windows' arrival flags (bounded wait), so that every SM has work as soon
// as the first window is in.
// Serial mode: copy everything, then ONE inflate launch ordered behind the copies on the context stream -- no flags, nothing on
// the device waits for anything.  Used for files of a single window (nothing to overlap), on request (CMB_INFLATE_SERIAL=1),
// and when a CUDA tool is injected into the process (ncu, compute-sanitizer: they serialise kernels against the other streams,
// so a kernel that polls for copies would only ever see its bounded wait expire).
bool inflate_serial_requested() {
  static const bool v = [] {
    if (const char* e = getenv("CMB_INFLATE_SERIAL")) return e[0] == '1';
    for (const char* name : {"CUDA_INJECTION64_PATH", "NV_NSIGHT_INJECTION_PORT_BASE", "NV_COMPUTE_PROFILER_PERFWORKS_DIR", "NV_SANITIZER_INJECTION_PORT_BASE"})
      if (const char* e = getenv(name))
        if (e[0]) return true;
    return false;
  }();
  return v;
}
// kd_crc32 over the blocks of `a` (the t1 path: its inflate kernel leaves the CRC to a second kernel)
int launch_crc32(cmb_ctx* c, const InflateArgs& a, cudaStream_t st) {
  const uint32_t nb = a.b1 - a.b0;
  kd_crc32<<<std::min<uint32_t>((nb + 7) / 8, (uint32_t)c->sm_count * 8), 256, 0, st>>>(a);
  CU_TRY(c, cudaGetLastError());
  return CMB_OK;
}
// Launch the inflate kernel over blocks [a.b0, a.b1), or over a.block_list[a.b0, a.b1) with kd_inflate (the second pass).
// *crc_pending (when given) is set instead of launching kd_crc32: the caller launches it once nothing else has to get past it
// in the hardware queue (a kernel waiting for its predecessor blocks the queue for every stream that shares it).
int launch_inflate(cmb_ctx* c, const InflateArgs& a, cudaStream_t st, bool* crc_pending = nullptr) {
  const uint32_t nb = a.b1 - a.b0;
  const int k = a.block_list ? 2 : inflate_kind(nb);
  if (k == 0) {
    CU_TRY(c, cudaFuncSetAttribute(kd_inflate_t1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T1_SMEM_BYTES));
    // every resident warp takes part; with fewer blocks than lanes, each warp works with its first `lanes` lanes only
    const uint32_t max_grid = (uint32_t)c->sm_count * 5, warps = max_grid * (T1_THREADS / 32);
    const uint32_t lanes = std::min<uint32_t>(32, std::max<uint32_t>(1, (nb + warps - 1) / warps));
    const uint32_t per_cta = lanes * (T1_THREADS / 32);
    const uint32_t grid = std::min<uint32_t>((nb + per_cta - 1) / per_cta, max_grid);
    InflateArgs at = a;
    at.lane_limit = lanes;
    kd_inflate_t1<<<grid, T1_THREADS, T1_SMEM_BYTES, st>>>(at);
    CU_TRY(c, cudaGetLastError());
    if (crc_pending) *crc_pending = true;
    else if (int rc = launch_crc32(c, a, st)) return rc;
  } else if (k == 1) {
    CU_TRY(c, cudaFuncSetAttribute(kd_inflate_g8, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G8_SMEM_BYTES));
    const uint32_t per_cta = G8_WARPS * G8_STREAMS;
    const uint32_t grid = std::min<uint32_t>((nb + per_cta - 1) / per_cta, (uint32_t)c->sm_count * 2);
    kd_inflate_g8<<<grid, G8_WARPS * 32, G8_SMEM_BYTES, st>>>(a);
  } else {
    CU_TRY(c, cudaFuncSetAttribute(kd_inflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)INF_SMEM_BYTES));
    const uint32_t grid = std::min<uint32_t>((nb + INF_WARPS - 1) / INF_WARPS, (uint32_t)c->sm_count * 2);
    kd_inflate<<<grid, INF_WARPS * 32, INF_SMEM_BYTES, st>>>(a);
  }
  CU_TRY(c, cudaGetLastError());
  return CMB_OK;
}

// zlib's inflate of BGZF block b into buf[0, isize), checked against the block's length and CRC-32 footer
bool host_inflate_block(const cmb_bgzf_input* in, uint32_t b, std::vector<uint8_t>& buf) {
  const uint32_t isz = in->block_isize[b];
  if (buf.size() < (size_t)isz + 64) buf.resize((size_t)isz + 64);
  z_stream zs;
  memset(&zs, 0, sizeof zs);
  if (inflateInit2(&zs, -15) != Z_OK) return false;
  zs.next_in = const_cast<Bytef*>(in->data + in->block_coffset[b]);
  zs.avail_in = in->block_clen[b];
  zs.next_out = buf.data();
  zs.avail_out = isz;
  const bool ok = inflate(&zs, Z_FINISH) == Z_STREAM_END && zs.avail_out == 0;
  inflateEnd(&zs);
  uint32_t want_crc;
  memcpy(&want_crc, in->data + in->block_coffset[b] + in->block_clen[b], 4);
  return ok && (uint32_t)crc32(0, buf.data(), isz) == want_crc;
}

// One cmb_submit_bgzf / cmb_decode_bgzf call, handed from stage to stage.
struct BgzfCall {
  cmb_ctx* c;
  cmb_ctx::Decode& d;
  const cmb_bgzf_input* in;
  cmb_bgzf_result* out;
  bool decode_only;
  uint32_t nb;
  bool nothing_to_decode = true;  // header only, or an empty share of a ranged decode
  std::vector<uint64_t> ustart;   // offset of every block in the inflated stream; [nb] = its length
  // Blocks: records starting in [first_block, walk_end) are decoded; [first_block, data_end) are uploaded and inflated (the tail
  // beyond walk_end only supplies the bytes of a record that straddles out of the range).  Whole file: walk_end = data_end = nb.
  // Blocks before first_block are header text the host has already read: not inflated here.
  uint32_t first_block = 0, walk_end = 0, data_end = 0;
  // Device buffers hold only [byte_lo, byte_hi) of the file and [u_lo, total) of the inflated stream; the kernels index both
  // with absolute offsets through biased base pointers.
  uint64_t byte_lo = 0, byte_hi = 0, u_lo = 0, total = 0;
  uint8_t* comp_base = nullptr;
  uint8_t* infl_base = nullptr;
  struct Window { uint32_t b0, b1; uint64_t byte0, byte1; };
  std::vector<Window> windows;  // whole blocks, ~DEC_WINDOW_BYTES of file each
  uint32_t n_copy_threads = 0;
  bool src_pinned = false;
  uint64_t n_rec = 0, n_cig = 0;
  uint64_t tail_bytes = DEC_TAIL_BYTES;  // ranged: inflated bytes uploaded beyond walk_end
  bool tail_short = false;               // ranged: a record runs past the tail (a longer tail may decode it)
  uint64_t exit_off = 0;                 // end of the last record that starts in the range: the next range's records_at

  InflateArgs inflate_args(uint32_t b0, uint32_t b1) const;
  int prepare();
  int copy_inflate();
  int declined();
  int chain();
  int extract();
  int excl_n(uint32_t* n);
};

// The inflate kernels' arguments over blocks [b0, b1) of the call
InflateArgs BgzfCall::inflate_args(uint32_t b0, uint32_t b1) const {
  InflateArgs a{};
  a.comp = comp_base; a.coff = d.d_coff; a.clen = d.d_clen; a.isize = d.d_isize; a.uoff = d.d_ustart; a.scratch = d.d_t1_scratch;
  a.b0 = b0; a.b1 = b1; a.out = infl_base; a.status = d.d_status; a.ticket = d.d_tickets; a.fail_count = d.d_cnt + 0;
  return a;
}

// Stage 1: the block table, the blocks this call decodes, its copy windows, and every buffer, stream and copy slot it needs.
int BgzfCall::prepare() {
  ustart.assign((size_t)nb + 1, 0);
  for (uint32_t b = 0; b < nb; ++b) {
    if (in->block_coffset[b] + in->block_clen[b] + 8 > in->size) return fail(c, CMB_E_ARG, "cmb_submit_bgzf: block %u lies outside the data", b);
    ustart[b + 1] = ustart[b] + in->block_isize[b];
  }
  const uint64_t stream_total = ustart[nb];
  if (in->records_at > stream_total) return fail(c, CMB_E_ARG, "cmb_submit_bgzf: records_at beyond the end of the stream");
  if (in->records_at == stream_total) return CMB_OK;  // header only
  first_block = (uint32_t)(std::upper_bound(ustart.begin(), ustart.end(), in->records_at) - ustart.begin()) - 1;
  walk_end = data_end = nb;
  if (in->ranged) {
    if (in->walk_begin_block != first_block || in->walk_end_block > nb || in->walk_end_block < in->walk_begin_block)
      return fail(c, CMB_E_ARG, "cmb_submit_bgzf: inconsistent block range");
    walk_end = in->walk_end_block;
    if (walk_end == first_block) return CMB_OK;  // an empty share
    data_end = walk_end;
    uint64_t tail = 0;
    while (data_end < nb && tail < tail_bytes) tail += in->block_isize[data_end++];
  }
  nothing_to_decode = false;
  byte_lo = in->block_coffset[first_block];
  byte_hi = data_end == nb ? in->size : in->block_coffset[data_end - 1] + in->block_clen[data_end - 1] + 8;
  u_lo = ustart[first_block];
  total = ustart[data_end];  // end of the inflated bytes available to this call
  // ---- buffers
  if (const char* lim = getenv("CMB_DECODE_MEM_LIMIT_MB")) {  // testing aid: behave as if the device had this much room
    if (((byte_hi - byte_lo) + (total - u_lo)) >> 20 > strtoull(lim, nullptr, 10)) return CMB_E_NOMEM;
  }
  int rc;
  const size_t comp_need = (size_t)(byte_hi - byte_lo) + DEC_FRONT + DEC_SLACK, infl_need = (size_t)(total - u_lo) + DEC_SLACK;
  if ((rc = d.d_comp.ensure(c, comp_need, with_slack(comp_need))) || (rc = d.d_inflated.ensure(c, infl_need, with_slack(infl_need))))
    return rc;
  comp_base = reinterpret_cast<uint8_t*>(reinterpret_cast<uintptr_t>(d.d_comp.p) + DEC_FRONT - byte_lo);
  infl_base = reinterpret_cast<uint8_t*>(reinterpret_cast<uintptr_t>(d.d_inflated.p) - u_lo);
  const size_t blocks_need = (size_t)nb + 1, blocks_want = (size_t)nb + nb / 8 + 64;
  for (auto* b : {&d.d_coff, &d.d_ustart, &d.d_guess, &d.d_exit, &d.d_rec_base, &d.d_cig_base})
    if ((rc = b->ensure(c, blocks_need, blocks_want))) return rc;
  for (auto* b : {&d.d_clen, &d.d_isize, &d.d_status, &d.d_nrec, &d.d_ncig, &d.d_dirty})
    if ((rc = b->ensure(c, blocks_need, blocks_want))) return rc;
  if ((rc = d.d_t1_scratch.ensure(c, blocks_need * T1_LENS_BYTES, blocks_want * T1_LENS_BYTES))) return rc;
  if ((rc = d.d_cnt.ensure(c, 20))) return rc;  // [16..19]: a sliced decode's held-back counts (decode_sliced)
  if (!d.have_events) {
    for (auto& e : d.ev) CU_TRY(c, cudaEventCreate(&e));
    d.have_events = true;
  }
  // ---- windows
  {
    uint32_t b = first_block;
    uint64_t byte0 = byte_lo;
    while (b < data_end) {
      uint32_t e = b;
      uint64_t byte1 = byte0;
      while (e < data_end && (e == b || in->block_coffset[e] + in->block_clen[e] + 8 - byte0 <= dec_window_bytes())) {
        byte1 = in->block_coffset[e] + in->block_clen[e] + 8;
        ++e;
      }
      if (e == data_end) byte1 = byte_hi;
      windows.push_back({b, e, byte0, byte1});
      b = e;
      byte0 = byte1;
    }
  }
  const size_t n_windows = windows.size();
  if ((rc = d.d_tickets.ensure(c, n_windows + 8, n_windows * 3 + 64))) return rc;  // [0] block ticket, [1, 1 + W) arrival flags
  if ((rc = d.d_block_window.ensure(c, nb, with_slack(nb)))) return rc;
  if (!d.h_ones) {
    if ((rc = d.h_ones.ensure(c, 16))) return rc;
    for (int k = 0; k < 16; ++k) d.h_ones.p[k] = 1;
  }
  // ---- copy threads, their streams and pinned slots
  cudaPointerAttributes attr{};
  src_pinned = cudaPointerGetAttributes(&attr, in->data) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();  // cudaPointerGetAttributes on pageable memory may leave a sticky-free error code
  const uint32_t T = std::min<uint32_t>(std::min<uint32_t>(in->copy_threads ? in->copy_threads : 4, 16), (uint32_t)n_windows);
  n_copy_threads = T;
  while (d.streams.size() < T) {
    cudaStream_t st;
    CU_TRY(c, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    d.streams.push_back(st);
    cudaEvent_t e;
    CU_TRY(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    d.done_events.push_back(e);
    for (int k = 0; k < 2; ++k) {
      CU_TRY(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      d.slot_events.push_back(e);
      PinnedBuf<uint8_t> slot;
      if ((rc = slot.ensure(c, DEC_COPY_CHUNK))) return rc;
      d.pinned.push_back(std::move(slot));
    }
  }
  return CMB_OK;
}

// Stage 2: the block table goes up on the context stream, the windows on the copy streams (one host thread each, a 4-byte
// arrival flag after each window), and the inflate kernel runs: one persistent launch before the copies whose threads wait for
// their window's flag, or (serial) one launch behind all the copies.
int BgzfCall::copy_inflate() {
  NvtxRange nvtx("bgzf: H2D copy + inflate");
  const uint32_t T = n_copy_threads;
  std::vector<uint32_t> block_window(nb, 0);
  for (size_t w = 0; w < windows.size(); ++w)
    for (uint32_t b = windows[w].b0; b < windows[w].b1; ++b) block_window[b] = (uint32_t)w;
  // ---- upload the block table, reset counters (ctx stream), then let the copy streams start after it
  CU_TRY(c, cudaEventRecord(d.ev[0], c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_coff, in->block_coffset, 8ull * nb, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_clen, in->block_clen, 4ull * nb, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_isize, in->block_isize, 4ull * nb, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_ustart, ustart.data(), 8ull * (nb + 1), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_cnt, 0, 64, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_status, 0, 4ull * nb, c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_block_window, block_window.data(), 4ull * nb, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_tickets, 0, 4 * (windows.size() + 1), c->stream));
  CU_TRY(c, cudaMemsetAsync(infl_base + total, 0, DEC_SLACK, c->stream));
  CU_TRY(c, cudaMemsetAsync(comp_base + byte_hi, 0, DEC_SLACK, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_comp, 0, DEC_FRONT, c->stream));
  CU_TRY(c, cudaEventRecord(d.ev[1], c->stream));
  for (uint32_t t = 0; t < T; ++t) CU_TRY(c, cudaStreamWaitEvent(d.streams[t], d.ev[1], 0));
  const bool serial = windows.size() <= 1 || inflate_serial_requested();
  bool crc_pending = false;
  InflateArgs persistent = inflate_args(first_block, data_end);
  int rc;
  if (!serial) {  // one persistent launch over every block; its warps wait for their block's window to arrive
    persistent.block_window = d.d_block_window;
    persistent.ready = d.d_tickets + 1;
    if ((rc = launch_inflate(c, persistent, c->stream, &crc_pending))) return rc;
  }
  std::atomic<size_t> next_window{0};
  std::atomic<int> first_err{0};
  auto worker = [&](uint32_t t) {
    cudaSetDevice(c->device);
    cudaStream_t st = d.streams[t];
    int slot = 0;
    bool used[2] = {false, false};
    auto check = [&](cudaError_t e) {
      if (e != cudaSuccess) {
        int z = 0;
        first_err.compare_exchange_strong(z, (int)e);
      }
      return e == cudaSuccess;
    };
    for (;;) {
      const size_t w = next_window.fetch_add(1);
      if (w >= windows.size() || first_err.load()) break;
      const Window& win = windows[w];
      if (src_pinned) {
        if (!check(cudaMemcpyAsync(comp_base + win.byte0, in->data + win.byte0, win.byte1 - win.byte0, cudaMemcpyHostToDevice, st))) break;
      } else {
        for (uint64_t o = win.byte0; o < win.byte1; o += DEC_COPY_CHUNK) {
          const size_t n = (size_t)std::min<uint64_t>(DEC_COPY_CHUNK, win.byte1 - o);
          const size_t si = (size_t)t * 2 + slot;
          if (used[slot] && !check(cudaEventSynchronize(d.slot_events[si]))) return;
          memcpy(d.pinned[si], in->data + o, n);
          if (!check(cudaMemcpyAsync(comp_base + o, d.pinned[si], n, cudaMemcpyHostToDevice, st))) return;
          if (!check(cudaEventRecord(d.slot_events[si], st))) return;
          used[slot] = true;
          slot ^= 1;
        }
      }
      if (!check(cudaMemcpyAsync(d.d_tickets + 1 + w, d.h_ones, 4, cudaMemcpyHostToDevice, st))) break;  // window w has arrived
    }
    check(cudaEventRecord(d.done_events[t], st));
  };
  const auto copy_t0 = std::chrono::steady_clock::now();
  {
    std::vector<std::thread> threads;
    for (uint32_t t = 1; t < T; ++t) threads.emplace_back(worker, t);
    worker(0);
    for (auto& th : threads) th.join();
  }
  const double copy_wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - copy_t0).count();
  out->ms_copy_enqueue_wall = (float)copy_wall_ms;
  if (crc_pending && (rc = launch_crc32(c, persistent, c->stream))) return rc;  // every copy is enqueued: nothing left to hold up
  if (serial && !first_err.load()) {
    for (uint32_t t = 0; t < T; ++t) CU_TRY(c, cudaStreamWaitEvent(c->stream, d.done_events[t], 0));
    if ((rc = launch_inflate(c, inflate_args(first_block, data_end), c->stream))) return rc;
  }
  if (first_err.load()) {  // release the warps still waiting for windows that will never arrive
    cudaMemsetAsync(d.d_tickets + 1, 1, 4 * windows.size(), d.streams[0]);
    cudaStreamSynchronize(d.streams[0]);
    cudaStreamSynchronize(c->stream);
  }
  out->n_launches = 1;
  out->h2d_bytes = (byte_hi - byte_lo) + 24ull * nb + 8;
  if (first_err.load()) return fail(c, CMB_E_CUDA, "cmb_submit_bgzf: copy/inflate stage failed: %s", cudaGetErrorString((cudaError_t)first_err.load()));
  for (uint32_t t = 0; t < T; ++t) CU_TRY(c, cudaStreamWaitEvent(c->stream, d.done_events[t], 0));
  if (getenv("CMB_PIPELINE_STATS")) {  // how long the window copies alone took (the done events carry no timing: time them on the host)
    const auto h0 = std::chrono::steady_clock::now();
    for (uint32_t t = 0; t < T; ++t) cudaEventSynchronize(d.done_events[t]);
    const double wait_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - h0).count();
    fprintf(stderr, "#decode_h2d\twindows=%zu\tbytes=%llu\tcopy_streams_done_after_ms=%.1f (host clock from the end of the enqueue; enqueue took %.1f ms)\n",
            windows.size(), (unsigned long long)(byte_hi - byte_lo), wait_ms, copy_wall_ms);
  }
  CU_TRY(c, cudaEventRecord(d.ev[2], c->stream));
  if (getenv("CMB_DECODE_PROFILE")) {  // debugging aid: the inflate kernel alone, all blocks resident, one launch
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    cudaEvent_t p0, p1;
    cudaEventCreate(&p0);
    cudaEventCreate(&p1);
    CU_TRY(c, cudaMemsetAsync(d.d_tickets, 0, 4, c->stream));
    InflateArgs a = inflate_args(first_block, data_end);
    a.fail_count = d.d_cnt + 8;
    cudaEventRecord(p0, c->stream);
    if ((rc = launch_inflate(c, a, c->stream))) return rc;
    cudaEventRecord(p1, c->stream);
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, p0, p1);
    fprintf(stderr, "#decode_profile\tinflate_only_ms=%.3f\tblocks=%u\tcompressed=%llu\tinflated=%llu\tinflated_GBps=%.2f\tcopy_threads=%u\tsrc_pinned=%d\tcopy_enqueue_wall_ms=%.2f\n", ms, data_end - first_block,
            (unsigned long long)(byte_hi - byte_lo), (unsigned long long)(total - u_lo), (total - u_lo) / ms * 1e-6, T, (int)src_pinned, copy_wall_ms);
    cudaEventDestroy(p0);
    cudaEventDestroy(p1);
  }
  return CMB_OK;
}

// Stage 3: blocks the first pass declined get a second device pass, then zlib on the host, patched into the inflated stream.
int BgzfCall::declined() {
  NvtxRange nvtx("bgzf: declined blocks (second pass, host zlib)");
  uint32_t h_cnt[16];
  CU_TRY(c, cudaMemcpyAsync(h_cnt, d.d_cnt, 64, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  std::vector<uint8_t> tmp;
  if (h_cnt[0] || getenv("CMB_DECODE_RETRY_TEST")) {
    std::vector<uint32_t> status(nb);
    CU_TRY(c, cudaMemcpy(status.data(), d.d_status, 4ull * nb, cudaMemcpyDeviceToHost));
    if (getenv("CMB_DECODE_RETRY_TEST"))  // testing aid: pretend every 7th block was declined by the first pass (code 29)
      for (uint32_t b = first_block; b < data_end; b += 7) status[b] = 29;
    if (getenv("CMB_DECODE_VERIFY") || getenv("CMB_PIPELINE_STATS")) {
      uint32_t hist[32] = {0};
      for (uint32_t b = 0; b < nb; ++b) hist[std::min<uint32_t>(status[b], 31)]++;
      fprintf(stderr, "#decode_status");
      for (int k = 0; k < 32; ++k)
        if (hist[k]) fprintf(stderr, "\t%d:%u", k, hist[k]);
      fprintf(stderr, "\n");
    }
    // Second chance on the device: the one-stream-per-warp kernel has larger Huffman tables (10-bit roots, 128 long-code
    // prefixes) than the four-streams-per-warp one, so most blocks the first pass declined for table space fit there.
    std::vector<uint32_t> again;
    for (uint32_t b = first_block; b < data_end; ++b)
      if (status[b] != INF_OK) again.push_back(b);
    out->n_blocks_second_pass = (uint32_t)again.size();
    if (!again.empty()) {
      uint32_t* d_list = d.d_dirty;  // free until the record chain starts (nb entries)
      CU_TRY(c, cudaMemcpyAsync(d_list, again.data(), 4ull * again.size(), cudaMemcpyHostToDevice, c->stream));
      CU_TRY(c, cudaMemsetAsync(d.d_tickets, 0, 4, c->stream));
      CU_TRY(c, cudaMemsetAsync(d.d_cnt, 0, 4, c->stream));
      InflateArgs a = inflate_args(0, (uint32_t)again.size());
      a.block_list = d_list;
      if (int rc = launch_inflate(c, a, c->stream)) return rc;
      out->n_launches += 1;
      std::vector<uint32_t> st2(nb);
      CU_TRY(c, cudaMemcpyAsync(st2.data(), d.d_status, 4ull * nb, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaStreamSynchronize(c->stream));
      for (uint32_t b : again) status[b] = st2[b];
    }
    for (uint32_t b = first_block; b < data_end; ++b) {
      if (status[b] == INF_OK) continue;
      if (!host_inflate_block(in, b, tmp)) return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: BGZF block %u does not inflate", b);
      CU_TRY(c, cudaMemcpy(infl_base + ustart[b], tmp.data(), in->block_isize[b], cudaMemcpyHostToDevice));
      out->n_blocks_host += 1;
    }
  }
  if (getenv("CMB_DECODE_VERIFY")) {  // debugging aid: compare every device-inflated block with zlib's output
    std::vector<uint8_t> dev(total - u_lo);
    CU_TRY(c, cudaMemcpy(dev.data(), d.d_inflated, total - u_lo, cudaMemcpyDeviceToHost));
    uint32_t bad = 0;
    for (uint32_t b = first_block; b < data_end; ++b) {
      const uint32_t isz = in->block_isize[b];
      if (!isz) continue;
      const uint8_t* got = dev.data() + (ustart[b] - u_lo);
      const bool zlib_ok = host_inflate_block(in, b, tmp);
      if (!zlib_ok || memcmp(tmp.data(), got, isz) != 0) {
        uint32_t k = 0;
        while (k < isz && tmp[k] == got[k]) ++k;
        if (bad < 8) fprintf(stderr, "#decode_verify\tblock %u (clen %u isize %u): zlib %s, first difference at byte %u\n", b, in->block_clen[b], isz, zlib_ok ? "ok" : "failed", k);
        ++bad;
      }
    }
    fprintf(stderr, "#decode_verify\t%u of %u blocks differ from zlib; %u inflated on the host\n", bad, data_end - first_block, out->n_blocks_host);
  }
  return CMB_OK;
}

// Stage 4: the record chain -- a guessed first record per block, walked to the block's end, verified against the neighbour's
// guess (repaired and re-walked until it settles), then the record and CIGAR bases of every block.
int BgzfCall::chain() {
  NvtxRange nvtx("bgzf: record chain (guess, walk, verify, offsets)");
  WalkArgs wa{};
  // The chain is walked over [first_block, walk_hi): one block past the range when there is one, so that the range's last
  // record boundary is also checked against an independent guess.
  const uint32_t walk_hi = std::min<uint32_t>(walk_end + 1, data_end);
  wa.data = infl_base; wa.total = total; wa.ustart = d.d_ustart; wa.first_block = first_block; wa.n_blocks = walk_hi;
  wa.records_at = in->records_at; wa.n_ref = (int32_t)in->n_ref; wa.guess = d.d_guess; wa.exit_off = d.d_exit; wa.n_rec = d.d_nrec;
  wa.n_cig = d.d_ncig; wa.dirty = d.d_dirty; wa.flags = d.d_cnt + 1; wa.only_dirty = 0;
  const uint32_t nwb = walk_hi - first_block;
  CU_TRY(c, cudaMemsetAsync(d.d_dirty, 0, 4ull * nb, c->stream));
  kd_guess<<<(nwb * 32 + 255) / 256, 256, 0, c->stream>>>(wa);
  kd_walk<<<(nwb + 127) / 128, 128, 0, c->stream>>>(wa);
  CU_TRY(c, cudaGetLastError());
  out->n_launches += 2;
  uint32_t h_cnt[16];
  uint64_t h_exit = 0;
  for (uint32_t round = 0;; ++round) {
    if (nwb > 1) {
      CU_TRY(c, cudaMemsetAsync(d.d_cnt + 2, 0, 4, c->stream));
      kd_verify<<<(nwb - 1 + 255) / 256, 256, 0, c->stream>>>(wa);
      CU_TRY(c, cudaGetLastError());
      out->n_launches += 1;
    }
    CU_TRY(c, cudaMemcpyAsync(h_cnt, d.d_cnt, 64, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaMemcpyAsync(&h_exit, d.d_exit + (walk_end - 1), 8, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    if (nwb <= 1 || !h_cnt[2]) break;
    if (round >= 256) return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: record chain did not settle");
    out->chain_repairs += 1;
    out->n_launches += 1;
    wa.only_dirty = 1;
    kd_walk<<<(nwb + 127) / 128, 128, 0, c->stream>>>(wa);
    CU_TRY(c, cudaGetLastError());
  }
  if (walk_end == nb ? h_exit != ustart[nb] : (h_exit == WALK_UNKNOWN || h_exit > total)) {
    tail_short = walk_end != nb && data_end < nb;
    return fail(c, CMB_E_DECLINED, walk_end == nb ? "cmb_submit_bgzf: record chain does not end at the end of the stream"
                                                  : "cmb_submit_bgzf: a record runs past the inflated tail of the block range");
  }
  exit_off = h_exit;
  kd_scan_items<<<1, 1024, 0, c->stream>>>(d.d_nrec, d.d_ncig, first_block, walk_end, d.d_rec_base, d.d_cig_base, (uint64_t*)(d.d_cnt + 6));
  CU_TRY(c, cudaGetLastError());
  out->n_launches += 1;
  uint64_t totals[2] = {0, 0};
  CU_TRY(c, cudaMemcpyAsync(totals, d.d_cnt + 6, 16, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  CU_TRY(c, cudaEventRecord(d.ev[3], c->stream));
  n_rec = totals[0];
  n_cig = totals[1];
  return CMB_OK;
}

// Stage 5: the per-record tuples, mate matching when a pair filter needs it, and K1 over the tuples (not for cmb_decode_bgzf).
int BgzfCall::extract() {
  NvtxRange nvtx("bgzf: extract, mate matching, K1");
  if (n_rec >= 0xffffff00ull || n_cig >= 0xffffff00ull) return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: more than 2^32 records or cigar operations");
  out->n_records = n_rec;
  out->n_intervals = n_cig;
  if (!n_rec) {
    CU_TRY(c, cudaEventRecord(d.ev[4], c->stream));
    CU_TRY(c, cudaEventRecord(d.ev[5], c->stream));
    return CMB_OK;
  }
  int rc;
  size_t offs[13];
  const size_t slab_need = batch_slab_bytes((uint32_t)n_rec, (uint32_t)n_cig, offs);
  if ((rc = d.d_rec_off.ensure(c, n_rec, with_slack(n_rec))) || (rc = d.d_tuple_slab.ensure(c, slab_need, slab_need + slab_need / 8)))
    return rc;
  cmb_read_batch tb;
  carve_batch(d.d_tuple_slab, (uint32_t)n_rec, (uint32_t)n_cig, &tb);
  d.last_n_rec = (uint32_t)n_rec;
  d.last_n_cig = (uint32_t)n_cig;
  OffsetArgs oa{};
  oa.data = infl_base; oa.ustart = d.d_ustart; oa.guess = d.d_guess; oa.rec_base = d.d_rec_base; oa.cig_base = d.d_cig_base;
  oa.first_block = first_block; oa.n_blocks = walk_end; oa.rec_off = d.d_rec_off; oa.iv_begin = tb.iv_begin; oa.n_records = n_rec; oa.n_cig_total = n_cig;
  kd_offsets<<<(walk_end - first_block + 127) / 128, 128, 0, c->stream>>>(oa);
  CU_TRY(c, cudaGetLastError());
  ExtractArgs ea{};
  ea.data = infl_base; ea.rec_off = d.d_rec_off; ea.n_records = n_rec;
  ea.own_lo = in->ranged ? in->own_tid_begin : INT_MIN; ea.own_hi = in->ranged ? in->own_tid_end : INT_MAX;
  ea.own_unplaced = in->ranged ? in->own_unplaced : 1u; ea.n_owned = (unsigned long long*)(d.d_cnt + 10);
  ea.tid = tb.tid; ea.pos = tb.pos; ea.flag = tb.flag; ea.mapq = tb.mapq; ea.nm_state = tb.nm_state; ea.nm = tb.nm; ea.l_seq = tb.l_seq;
  ea.aligned = tb.aligned; ea.del = tb.del; ea.ins = tb.ins; ea.iv_begin = tb.iv_begin; ea.iv_start = tb.iv_start; ea.iv_len = tb.iv_len;
  ea.n_primary = (unsigned long long*)(d.d_cnt + 4); ea.flags = d.d_cnt + 1;
  kd_extract<<<(uint32_t)((n_rec + 255) / 256), 256, 0, c->stream>>>(ea);
  CU_TRY(c, cudaGetLastError());
  out->n_launches += 2;
  uint32_t h_cnt[16];
  CU_TRY(c, cudaMemcpyAsync(h_cnt, d.d_cnt, 64, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (h_cnt[1]) return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: malformed alignment record (flags %u)", h_cnt[1]);
  memcpy(&out->n_primary, h_cnt + 4, 8);
  memcpy(&out->n_records, h_cnt + 10, 8);  // records this call owns (all of them unless ranged)
  d.last_valid = true;
  d.last_mate = nullptr;
  d.last_infl_base = infl_base;
  // mate matching on the device (filter.rs:117-233; cmb_pairs.cuh) for coverage when the pair thresholds apply; `coverm
  // filter` matches in cmb_filter_plan, where --inverse (which decides the eligible records) is known
  if (!decode_only && c->mode.filter_pairs) {
    if ((rc = match_mates(c, infl_base, (uint32_t)n_rec, true, "cmb_submit_bgzf"))) return rc;
    out->n_launches += 5;
  }
  CU_TRY(c, cudaEventRecord(d.ev[4], c->stream));
  if (k1_active(c) && !decode_only) {
    uint32_t excl = 0;
    if ((rc = excl_n(&excl))) return rc;
    d.last_excl_n = excl;
    if ((rc = launch_k1(c, tb, (uint32_t)n_rec, (uint32_t)n_cig, excl, d.last_mate))) return rc;
  }
  CU_TRY(c, cudaEventRecord(d.ev[5], c->stream));
  return CMB_OK;
}

// K1's excl_n for the call's records: those that start before excl_end_block are this rank's exclusive share of the stream
// (cmb_kept_tid_range) -- none when the block lies before the range, all when it lies after it
int BgzfCall::excl_n(uint32_t* n) {
  *n = 0xffffffffu;
  if (in->ranged && in->excl_end_block < walk_end) {
    if (in->excl_end_block <= first_block) *n = 0;
    else {
      uint64_t base = 0;
      CU_TRY(c, cudaMemcpyAsync(&base, d.d_rec_base + in->excl_end_block, 8, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaStreamSynchronize(c->stream));
      *n = (uint32_t)base;
    }
  }
  return CMB_OK;
}

int submit_bgzf_impl(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out, bool decode_only) {
  NvtxRange nvtx_fn("cmb_submit_bgzf");
  if (!c || !in || !out || !in->data || !in->block_coffset || !in->block_clen || !in->block_isize)
    return fail(c, CMB_E_ARG, "cmb_submit_bgzf: null argument");
  if (!decode_only && !c->in_sample) return fail(c, CMB_E_ARG, "cmb_submit_bgzf: no sample in progress");
  if (decode_only && (c->in_sample || !c->have_params)) return fail(c, CMB_E_ARG, "cmb_decode_bgzf: set the parameters first; not inside a sample");
  if (c->n_acquired) return fail(c, CMB_E_ARG, "cmb_submit_bgzf: a staging batch is still acquired");
  *out = cmb_bgzf_result{};
  if (in->n_blocks == 0) return CMB_OK;
  CU_TRY(c, cudaSetDevice(c->device));
  BgzfCall j{c, c->dec, in, out, decode_only, in->n_blocks};
  int rc;
  if ((rc = j.prepare()) || j.nothing_to_decode) return rc;
  if ((rc = j.copy_inflate()) || (rc = j.declined()) || (rc = j.chain()) || (rc = j.extract())) return rc;
  auto& d = c->dec;
  CU_TRY(c, cudaEventSynchronize(d.ev[4]));
  cudaEventElapsedTime(&out->ms_copy_inflate, d.ev[0], d.ev[2]);
  cudaEventElapsedTime(&out->ms_chain, d.ev[2], d.ev[3]);
  cudaEventElapsedTime(&out->ms_extract, d.ev[3], d.ev[4]);
  cudaEventElapsedTime(&out->ms_total, d.ev[0], d.ev[4]);
  return CMB_OK;
}

int decode_sliced(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out);

int bgzf_entry(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out, bool decode_only) {
  if (c) {
    c->dec.last_valid = false;
    c->dec.filter_planned = false;
  }
  const auto t_call0 = std::chrono::steady_clock::now();
  int rc = submit_bgzf_impl(c, in, out, decode_only);
  if (rc == CMB_E_NOMEM) {
    cudaGetLastError();
    auto& d = c->dec;  // give the big buffers back so that the rest of the sample has room
    d.d_comp.release();
    d.d_inflated.release();
    d.d_tuple_slab.release();
    d.d_rec_off.release();
    // nothing was accumulated: the whole-stream call allocates every buffer before K1
    rc = decode_only ? fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: not enough device memory for device-side decode") : decode_sliced(c, in, out);
  }
  if (out) out->ms_host_wall = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_call0).count();
  return rc;
}
}  // namespace

// Device memory for the whole-stream decode buffers (compressed file + inflated stream + tuples) is requested before anything
// is accumulated; when it runs out, the stream is decoded in block slices (decode_sliced), and a sample that declines there is
// reset to its empty state first, so that the host decoder can take it over with only the staging batches.
extern "C" int cmb_last_bgzf_batch(cmb_ctx* c, cmb_read_batch* dev_batch, uint32_t* n_records, uint32_t* n_intervals) {
  if (!c || !dev_batch || !n_records || !n_intervals) return fail(c, CMB_E_ARG, "cmb_last_bgzf_batch: null argument");
  if (!c->dec.last_valid || !c->dec.d_tuple_slab) return fail(c, CMB_E_ARG, "cmb_last_bgzf_batch: no device-decoded sample is resident");
  carve_batch(c->dec.d_tuple_slab, c->dec.last_n_rec, c->dec.last_n_cig, dev_batch);
  *n_records = c->dec.last_n_rec;
  *n_intervals = c->dec.last_n_cig;
  return CMB_OK;
}

extern "C" int cmb_submit_bgzf(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out) { return bgzf_entry(c, in, out, false); }
extern "C" int cmb_decode_bgzf(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out) { return bgzf_entry(c, in, out, true); }

extern "C" int cmb_filter_plan(cmb_ctx* c, int inverse, uint64_t* n_records, uint64_t* n_bytes) {
  if (!c || !n_records || !n_bytes) return fail(c, CMB_E_ARG, "cmb_filter_plan: null argument");
  auto& d = c->dec;
  if (!d.last_valid || !d.d_tuple_slab || !c->have_params) return fail(c, CMB_E_ARG, "cmb_filter_plan: no device-decoded sample is resident (cmb_decode_bgzf first)");
  CU_TRY(c, cudaSetDevice(c->device));
  *n_records = 0;
  *n_bytes = 0;
  d.filter_planned = false;
  const uint32_t n = d.last_n_rec;
  if (n == 0) {
    d.filter_bytes = 0;
    d.filter_planned = true;
    return CMB_OK;
  }
  const bool pair_path = !(c->mode.filter_single_reads && !c->mode.filter_pairs);
  int rc;
  if (pair_path && (rc = match_mates(c, d.last_infl_base, n, !inverse, "cmb_filter_plan"))) return rc;
  if ((rc = d.d_filter_anchor.ensure(c, (size_t)n + 1, with_slack(n))) || (rc = d.d_filter_role.ensure(c, (size_t)n + 1, with_slack(n))))
    return rc;
  cmb_read_batch tb;
  carve_batch(d.d_tuple_slab, d.last_n_rec, d.last_n_cig, &tb);
  FilterArgs a{};
  a.data = d.last_infl_base; a.rec_off = d.d_rec_off; a.n = n; a.flag = tb.flag; a.mapq = tb.mapq; a.nm_state = tb.nm_state; a.nm = tb.nm;
  a.l_seq = tb.l_seq; a.aligned = tb.aligned; a.del = tb.del; a.mate = pair_path ? d.last_mate : nullptr; a.p = c->params;
  a.filter_single = c->mode.filter_single_reads; a.pair_path = pair_path; a.filter_out = inverse ? 0 : 1;
  a.anchor_bytes = d.d_filter_anchor; a.role = d.d_filter_role; a.error_flags = d.d_cnt + 12; a.n_emit = (unsigned long long*)(d.d_cnt + 14);
  CU_TRY(c, cudaMemsetAsync(d.d_cnt + 12, 0, 16, c->stream));
  kf_decide<<<(n + 255) / 256, 256, 0, c->stream>>>(a);
  kf_scan<<<1, 1024, 0, c->stream>>>(d.d_filter_anchor, n);
  CU_TRY(c, cudaGetLastError());
  uint32_t h[4];
  unsigned long long total = 0;
  CU_TRY(c, cudaMemcpyAsync(h, d.d_cnt + 12, 16, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(&total, d.d_filter_anchor + n, 8, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (h[0] & ERR_NM)
    return fail(c, CMB_E_NM, "Mapping record encountered that does not have an 'NM' auxiliary tag in the SAM/BAM format. This is required to work out some coverage statistics");
  unsigned long long n_emit;
  memcpy(&n_emit, h + 2, 8);
  if ((rc = d.d_filter_out.ensure(c, total, (size_t)total + (size_t)total / 8 + 4096))) return rc;
  a.out = d.d_filter_out;
  kf_gather<<<(n + 7) / 8, 256, 0, c->stream>>>(a);
  CU_TRY(c, cudaGetLastError());
  d.filter_bytes = total;
  d.filter_planned = true;
  *n_records = n_emit;
  *n_bytes = total;
  return CMB_OK;
}

extern "C" int cmb_filter_fetch(cmb_ctx* c, uint8_t* records, uint64_t n_bytes) {
  if (!c || (!records && n_bytes)) return fail(c, CMB_E_ARG, "cmb_filter_fetch: null argument");
  auto& d = c->dec;
  if (!d.filter_planned || n_bytes != d.filter_bytes) return fail(c, CMB_E_ARG, "cmb_filter_fetch: call cmb_filter_plan first and pass the size it reported");
  CU_TRY(c, cudaSetDevice(c->device));
  if (n_bytes) CU_TRY(c, cudaMemcpyAsync(records, d.d_filter_out, n_bytes, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}


// ---- sharded input (cmb_shards.cuh) ---------------------------------------------------------------------------------------
namespace {

// The reference's message for the smallest error key of ks_* (see cmb_shards.cuh), or CMB_OK
int shard_error(cmb_ctx* c, unsigned long long key) {
  if (key == ~0ull) return CMB_OK;
  const uint32_t kind = (uint32_t)(key >> 8) & 0xf, detail = (uint32_t)key & 0xff;
  const unsigned long long set = key >> 24;
  switch (kind) {
    case SHE_UNPAIRED:
      return fail(c, CMB_E_SHARD_EXIT, "This code can only handle paired-end input (at the moment), sorry. Found an unpaired record before primary %llu", set);
    case SHE_NAME:
      return fail(c, CMB_E_SHARD_EXIT, "BAM files do not appear to be properly sorted by read name. The read names of primary alignment %llu differ between the shards", set);
    case SHE_AS_MISSING:
      return fail(c, CMB_E_SHARD_PANIC, "Mapping record encountered that does not have an 'AS' auxiliary tag in the SAM/BAM format. This is required for ranking pairs of alignments.");
    case SHE_AS_TYPE: {
      const char* name = detail == 'c' ? "I8" : detail == 's' ? "I16" : detail == 'i' ? "I32" : detail == 'I' ? "U32" : detail == 'f' ? "Float"
                         : detail == 'A' ? "Char" : detail == 'Z' ? "String" : detail == 'H' ? "HexByteArray" : "Array";
      return fail(c, CMB_E_SHARD_PANIC, "Unexpected data type of AS aux tag, found %s", name);
    }
    case SHE_NO_SEPARATOR:
      return fail(c, CMB_E_SHARD_PANIC, "Contig name does not contain split symbol, so cannot determine which genome it belongs to");
    case SHE_EXCLUDED:
      return fail(c, CMB_E_SHARD_EXIT, "CoverM cannot currently deal with reads that only map to excluded genomes");
    case SHE_NM_TYPE:
      return fail(c, CMB_E_NM, "Unexpected data type of NM aux tag");
    case SHE_NM_MISSING:
      return fail(c, CMB_E_NM, "record with name at primary alignment %llu had no NM tag", set);
  }
  return fail(c, CMB_E_CUDA, "sharded input: unknown error key %llx", key);
}

int shard_event(cmb_ctx* c, int i) {
  if (!c->sh.ev[i]) CU_TRY(c, cudaEventCreate(&c->sh.ev[i]));
  return CMB_OK;
}

uint64_t shard_bytes(const cmb_ctx* c);

constexpr uint64_t SLICE_TAIL_BYTES = 64u << 10;  // a slice's first tail: one BGZF block; doubled for a longer record
constexpr int SLICE_HALVINGS = 8;                 // a slice whose buffers fail to allocate is halved this often before giving up
constexpr uint64_t SLICE_MIN_BYTES = 64u << 20;   // budget floor: below it a failed allocation, not the estimate, shrinks a slice

// CMB_DECODE_MEM_LIMIT_MB (testing aid): behave as if the device had this much room for the sharded sample -- its stores and
// one slice's compressed and inflated bytes; a fraction of a megabyte slices small files -- or, for an ordinary sliced stream,
// for the slices' decode buffers and the sample's event list (decode_sliced).  0 when unset.
uint64_t shard_mem_limit() {
  const char* lim = getenv("CMB_DECODE_MEM_LIMIT_MB");
  return lim ? (uint64_t)(std::max(0.0, strtod(lim, nullptr)) * 1048576.0) : 0;
}

// The decode buffers a slice fills (d_scan included); released when a store cannot grow beside them
uint64_t decode_bytes(const cmb_ctx* c) {
  const auto& d = c->dec;
  return d.d_comp.bytes() + d.d_inflated.bytes() + d.d_tuple_slab.bytes() + d.d_rec_off.bytes() + c->sh.d_scan.bytes();
}
// The buffers shard_need counts: stores, AS scratch, name hashes, pair state
uint64_t store_bytes_held(const cmb_ctx* c) {
  const auto& s = c->sh;
  uint64_t b = s.d_as_val.bytes() + s.d_as_state.bytes() + s.d_hash0.bytes() + s.d_state.bytes();
  for (const auto& st : s.store) b += st.bytes();
  return b;
}
void release_decode(cmb_ctx* c) {
  cudaGetLastError();
  auto& d = c->dec;
  d.d_comp.release();
  d.d_inflated.release();
  d.d_tuple_slab.release();
  d.d_rec_off.release();
  c->sh.d_scan.release();
}

// Bytes the sharded sample needs beyond its decode buffers when shard k holds n_prim primaries and n_iv interval slots: the
// stores (37 B per primary, 8 B per interval slot), AS scratch (5 B per primary of the largest shard), shard 0's name hashes
// and the pair state (8 + 8 B per primary), and the n_out sorted winners with their n_out_iv slots (52 B and 8 B)
uint64_t shard_need(const cmb_ctx* c, uint32_t k, uint64_t n_prim, uint64_t n_iv, uint64_t n_out = 0, uint64_t n_out_iv = 0) {
  const auto& s = c->sh;
  // a group rank holds the stores of its own shards [first, k] only, each with its AS columns (5 B per primary) and, after
  // shard 0, its name hashes (8 B)
  auto per_prim = [&](uint32_t i) -> uint64_t { return s.group ? (i ? 50 : 42) : 37; };
  uint64_t b = per_prim(k) * n_prim + 8 * n_iv, as = s.group ? 0 : n_prim;
  for (uint32_t i = s.first; i < k; ++i) {
    b += per_prim(i) * s.store[i].n_prim + 8 * s.store[i].n_iv;
    if (!s.group) as = std::max(as, s.store[i].n_prim);
  }
  return b + 5 * as + 16 * (k > s.first ? s.store[s.first].n_prim : n_prim) + 52 * n_out + 8 * n_out_iv;
}

// Bytes the device has for them and a slice: the limit under CMB_DECODE_MEM_LIMIT_MB, else what is free plus the stores and
// decode buffers the sample holds (the sorted winners' buffers of an earlier sample are not counted: they stay allocated)
uint64_t shard_room(const cmb_ctx* c) {
  if (const uint64_t lim = shard_mem_limit()) return lim;
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  cudaGetLastError();
  return free_b + store_bytes_held(c) + decode_bytes(c);
}

int shard_nomem(cmb_ctx* c, uint64_t need) {
  return fail(c, CMB_E_NOMEM, "sharded input needs %llu bytes of device memory for its shard stores, pair state, name hashes, AS scratch and "
              "sorted winners; the device has %llu bytes free for them", (unsigned long long)need, (unsigned long long)shard_room(c));
}

// `alloc` once, and again after the decode buffers are released; CMB_E_NOMEM with the sample's need when it still fails
template <class F>
int shard_alloc(cmb_ctx* c, uint64_t need, F alloc) {
  if (const uint64_t lim = shard_mem_limit(); lim && need > lim) return shard_nomem(c, need);
  int rc = alloc();
  if (rc != CMB_E_NOMEM) return rc;
  release_decode(c);
  rc = alloc();
  if (rc == CMB_E_NOMEM) {
    cudaGetLastError();
    return shard_nomem(c, need);
  }
  return rc;
}

// Room for `need` elements keeping the first `used`; `hint` (the shard's expected total) is allocated at once when it fits, so
// that a sliced shard grows each column about once instead of once per slice
template <class T>
int grow_col(cmb_ctx* c, Buf<T>& b, uint64_t used, uint64_t need, uint64_t hint = 0) {
  if (b.p && b.cap >= need) return CMB_OK;
  if (hint > need && b.grow_keep(c, used, with_slack(hint), c->stream) == CMB_OK) return CMB_OK;
  cudaGetLastError();
  return b.grow_keep(c, used, with_slack(need), c->stream);
}

// Room in the store for n_prim primaries and n_iv interval slots, keeping what it holds; the view follows the columns
int store_grow(cmb_ctx* c, cmb_ctx::Shards::Store& st, uint64_t n_prim, uint64_t n_iv, uint64_t hint_prim = 0, uint64_t hint_iv = 0) {
  const uint64_t r = st.n_prim, v = st.n_iv, h = hint_prim;
  int rc;
  if ((rc = grow_col(c, st.tid, r, n_prim, h)) || (rc = grow_col(c, st.pos, r, n_prim, h)) || (rc = grow_col(c, st.nm, r, n_prim, h)) ||
      (rc = grow_col(c, st.l_seq, r, n_prim, h)) || (rc = grow_col(c, st.aligned, r, n_prim, h)) || (rc = grow_col(c, st.del, r, n_prim, h)) ||
      (rc = grow_col(c, st.ins, r, n_prim, h)) || (rc = grow_col(c, st.iv_begin, r, n_prim + 1, h + 1)) || (rc = grow_col(c, st.flag, r, n_prim, h)) ||
      (rc = grow_col(c, st.mapq, r, n_prim, h)) || (rc = grow_col(c, st.nm_state, r, n_prim, h)) || (rc = grow_col(c, st.info, r, n_prim, h)) ||
      (rc = grow_col(c, st.iv_start, v, n_iv, hint_iv)) || (rc = grow_col(c, st.iv_len, v, n_iv, hint_iv)))
    return rc;
  cmb_read_batch& b = st.view.b;
  b.capacity_records = (uint32_t)std::min<size_t>(st.tid.cap, UINT32_MAX);
  b.capacity_intervals = (uint32_t)std::min<size_t>(st.iv_start.cap, UINT32_MAX);
  b.tid = st.tid; b.pos = st.pos; b.nm = st.nm; b.l_seq = st.l_seq; b.aligned = st.aligned; b.del = st.del; b.ins = st.ins;
  b.iv_begin = st.iv_begin; b.iv_start = st.iv_start; b.iv_len = st.iv_len; b.flag = st.flag; b.mapq = st.mapq; b.nm_state = st.nm_state;
  st.view.info = st.info;
  return CMB_OK;
}

// Statistics of one sliced decode
struct SliceStats {
  uint32_t n_slices = 0;
  uint32_t halvings = 0;  // over the whole decode
  uint64_t max_slice = 0;  // compressed + inflated bytes of the largest slice
  float ms_inflate = 0, ms_chain = 0, ms_extract = 0;
};
constexpr int SLICE_HALVE = 1;  // a slice step's verdict: a buffer of the slice did not fit, halve it
constexpr int SLICE_AGAIN = 2;  // a slice step's verdict: decode the same slice again (the step released the decode buffers)

// The records of `in` (the whole stream, or its block range when ranged) in consecutive block slices, each a ranged
// cmb_decode_bgzf call over blocks [b0, b1) that owns every record starting there.  A slice starts at the exact offset where
// the previous slice's record walk stopped, or where its step cut it.  budget(at): the compressed and inflated bytes the slice
// from `at` may take (slice_end).  A slice whose buffers fail to allocate, in the call or in its step, is halved up to
// SLICE_HALVINGS times, after which nomem(blocks, b0, b1, tail) is the error; its tail starts at SLICE_TAIL_BYTES and doubles when a
// record runs past it.  step(j, r, &next) does the caller's part with the slice's records and may lower `next` (the exit
// offset): CMB_OK, SLICE_HALVE, SLICE_AGAIN or an error.  `out` sums the slices' results.
template <class Budget, class Step, class Nomem>
int decode_in_slices(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out, SliceStats& ss, Budget budget, Step step, Nomem nomem) {
  auto& d = c->dec;
  const uint32_t nb = in->n_blocks;
  std::vector<uint64_t> ustart((size_t)nb + 1, 0);
  for (uint32_t b = 0; b < nb; ++b) ustart[b + 1] = ustart[b] + in->block_isize[b];
  const ShardBlocks blocks{nb, in->size, in->block_coffset, in->block_clen, ustart.data()};
  const uint32_t walk_end = in->ranged ? std::min(in->walk_end_block, nb) : nb;
  uint64_t at = in->records_at, tail = SLICE_TAIL_BYTES;
  uint32_t halvings = 0;
  uint32_t cap_end = nb;  // a slice end forced lower by a failed allocation (cleared once a slice decodes)
  while (at < ustart[walk_end]) {
    // ---- the slice: from the block holding `at`, as many blocks as the budget allows
    const uint32_t b0 = (uint32_t)(std::upper_bound(ustart.begin(), ustart.end(), at) - ustart.begin()) - 1;
    bool over = false;
    const uint32_t b1 = std::min({slice_end(blocks, b0, budget(at), tail, &over), std::max(cap_end, b0 + 1), walk_end});
    // ---- decode it: halved when its buffers do not fit, the tail doubled when a record runs past it
    cmb_bgzf_input si = *in;
    si.ranged = 1; si.records_at = at; si.walk_begin_block = b0; si.walk_end_block = b1;
    if (!in->ranged) {
      si.own_tid_begin = INT_MIN; si.own_tid_end = INT_MAX; si.own_unplaced = 1; si.excl_end_block = b1;
    }
    cmb_bgzf_result r{};
    BgzfCall j{c, d, &si, &r, true, nb};
    j.tail_bytes = tail;
    int rc = j.prepare();
    if (!rc && !j.nothing_to_decode && !(rc = j.copy_inflate()) && !(rc = j.declined()) && !(rc = j.chain())) rc = j.extract();
    if (rc == CMB_E_NOMEM) rc = SLICE_HALVE;
    uint64_t next = j.exit_off;
    if (!rc && !j.nothing_to_decode) {
      CU_TRY(c, cudaEventSynchronize(d.ev[4]));
      cudaEventElapsedTime(&r.ms_total, d.ev[0], d.ev[4]);
      cudaEventElapsedTime(&r.ms_copy_inflate, d.ev[0], d.ev[2]);
      cudaEventElapsedTime(&r.ms_chain, d.ev[2], d.ev[3]);
      cudaEventElapsedTime(&r.ms_extract, d.ev[3], d.ev[4]);
      if (!j.n_rec || j.exit_off <= at) return fail(c, CMB_E_DECLINED, "the slice from block %u decoded no record", b0);
      rc = step(j, r, &next);
    }
    if (rc == SLICE_HALVE) {
      release_decode(c);
      if (b1 - b0 > 1 && halvings < SLICE_HALVINGS) {
        ++halvings;
        ++ss.halvings;
        cap_end = b0 + (b1 - b0) / 2;
        continue;
      }
      return nomem(blocks, b0, b1, tail);
    }
    if (rc == CMB_E_DECLINED && j.tail_short) {
      tail *= 2;
      continue;
    }
    if (rc == SLICE_AGAIN) continue;
    if (rc) return rc;
    if (j.nothing_to_decode) break;
    // ---- the slice's result into the call's
    out->n_records += r.n_records; out->n_primary += r.n_primary; out->n_intervals += r.n_intervals;
    out->n_blocks_host += r.n_blocks_host; out->chain_repairs += r.chain_repairs; out->n_launches += r.n_launches;
    out->n_blocks_second_pass += r.n_blocks_second_pass; out->h2d_bytes += r.h2d_bytes;
    out->ms_copy_enqueue_wall += r.ms_copy_enqueue_wall; out->ms_total += r.ms_total;
    ss.ms_inflate += r.ms_copy_inflate; ss.ms_chain += r.ms_chain; ss.ms_extract += r.ms_extract;
    ss.max_slice = std::max(ss.max_slice, (j.byte_hi - j.byte_lo) + (j.total - j.u_lo));
    ++ss.n_slices;
    at = next;
    cap_end = nb;
    halvings = 0;
  }
  c->dec.last_valid = false;  // the tuples are a slice's, not the stream's: cmb_last_bgzf_batch must not hand them out
  return CMB_OK;
}

// Shard k's slices: every slice's primaries appended to the store, AS scratch and (shard 0) name hashes; `out` sums the
// slices' results
int decode_shard(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out, uint32_t k) {
  auto& s = c->sh;
  auto& d = c->dec;
  auto& st = s.store[k];
  c->dec.last_valid = false;
  c->dec.filter_planned = false;
  *out = cmb_bgzf_result{};
  st.n_prim = st.n_iv = 0;
  if (in->n_blocks == 0 || in->ranged) return fail(c, CMB_E_ARG, "cmb_shard_add: shard %u: a whole BGZF file is needed", k);
  const uint32_t nb = in->n_blocks;
  uint64_t stream_total = 0;
  for (uint32_t b = 0; b < nb; ++b) stream_total += in->block_isize[b];
  const uint64_t lim = shard_mem_limit();
  // shards after this context's first are expected to be sized like it (on one GPU: like shard 0)
  const bool later = k > s.first;
  const uint64_t n0 = later ? s.store[s.first].n_prim : 0, iv0 = later ? s.store[s.first].n_iv : 0;
  float ms_grow = 0;
  auto budget = [&](uint64_t at) -> uint64_t {
    const uint64_t need_now = shard_need(c, k, st.n_prim, st.n_iv);
    // What the sample is still expected to need: this shard's rest, the later shards' stores like shard 0's, and the sorted
    // winners (at most one record per primary of a shard, 60 B each with an interval slot).  Shard 0's first slice has no
    // estimate: like a whole-shard decode it takes what is free, and a failed allocation halves it.
    uint64_t expect = 0;
    if (later) {
      expect = 37 * (n0 > st.n_prim ? n0 - st.n_prim : 0) + 8 * (iv0 > st.n_iv ? iv0 - st.n_iv : 0) + (s.last - 1 - k) * (37 * n0 + 8 * iv0) +
               60 * n0;
    } else if (at > in->records_at) {  // the first shard: scaled by the inflated bytes its slices so far held
      const double scale = (double)(stream_total - in->records_at) / (double)(at - in->records_at);
      const double total = need_now * scale, store = (37.0 * st.n_prim + 8.0 * st.n_iv) * scale, winners = 60.0 * st.n_prim * scale;
      expect = (uint64_t)(total - need_now + store * (s.last - 1 - k) + winners);
    }
    const uint64_t room = shard_room(c), held = need_now + expect;
    const uint64_t budget = room > held ? room - held : 0;
    return std::max(budget, lim ? lim / 64 : SLICE_MIN_BYTES);
  };
  auto step = [&](BgzfCall& j, cmb_bgzf_result&, uint64_t*) -> int {
    const uint64_t n_rec = j.n_rec;
    // ---- which records are primaries, and where their tuples and intervals go
    CU_TRY(c, cudaEventRecord(s.ev[0], c->stream));
    int rc = s.d_scan.ensure(c, n_rec + 1, with_slack(n_rec + 1));
    if (rc == CMB_E_NOMEM) return SLICE_HALVE;  // part of the slice: halve it like its other buffers
    if (rc) return rc;
    ShardScanArgs a{};
    a.data = d.last_infl_base; a.rec_off = d.d_rec_off; a.n_records = n_rec; a.scan = s.d_scan;
    a.shard = k; a.tid_offset = s.tid_offsets[k]; a.err = s.d_err;
    carve_batch(d.d_tuple_slab, (uint32_t)n_rec, (uint32_t)j.n_cig, &a.tb);
    ks_mark<<<(uint32_t)((n_rec + 255) / 256), 256, 0, c->stream>>>(a);
    kf_scan<<<1, 1024, 0, c->stream>>>(s.d_scan, (uint32_t)n_rec);
    CU_TRY(c, cudaGetLastError());
    unsigned long long packed = 0;
    CU_TRY(c, cudaMemcpyAsync(&packed, s.d_scan + n_rec, 8, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    const uint64_t n_prim = st.n_prim + (packed >> 32), n_iv = st.n_iv + (uint32_t)packed;
    if (n_iv >= 0xffffff00ull) return fail(c, CMB_E_ARG, "cmb_shard_add: shard %u: more than 2^32 CIGAR operations in its primaries", k);
    // ---- room for them in the store, the AS scratch and (shard 0) the name hashes; without the decode buffers the slice is
    // decoded again
    // The expected totals: shard 0's, for shard k > 0; for shard 0, its slices so far scaled by the inflated bytes they cover
    const double scale = (double)(stream_total - in->records_at) / (double)(j.exit_off - in->records_at);
    const uint64_t hint_prim = later ? n0 : (uint64_t)(n_prim * scale), hint_iv = later ? iv0 : (uint64_t)(n_iv * scale);
    bool released = false;
    const auto g0 = std::chrono::steady_clock::now();
    auto grow = [&]() -> int {
      int e;
      auto& as_val = s.group ? st.as_val : s.d_as_val;
      auto& as_state = s.group ? st.as_state : s.d_as_state;
      if ((e = store_grow(c, st, n_prim, n_iv, hint_prim, hint_iv)) || (e = grow_col(c, as_val, st.n_prim, n_prim + 1, hint_prim + 1)) ||
          (e = grow_col(c, as_state, st.n_prim, n_prim + 1, hint_prim + 1)) ||
          (k == 0 && (e = grow_col(c, s.d_hash0, st.n_prim, n_prim + 1, hint_prim + 1))) ||
          (k && s.group && (e = grow_col(c, st.names, st.n_prim, n_prim + 1, hint_prim + 1))))
        released = released || e == CMB_E_NOMEM;
      return e;
    };
    if ((rc = shard_alloc(c, shard_need(c, k, n_prim, n_iv), grow))) return rc;
    ms_grow += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - g0).count();
    if (released) return SLICE_AGAIN;
    a.st = st.view; a.prim_base = st.n_prim; a.iv_base = (uint32_t)st.n_iv;
    a.as_val = s.group ? st.as_val.p : s.d_as_val.p; a.as_state = s.group ? st.as_state.p : s.d_as_state.p; a.hash0 = s.d_hash0; a.n0 = k ? s.store[0].n_prim : 0;
    if (k && s.group) a.names = st.names;
    ks_compact<<<(uint32_t)((n_rec + 255) / 256), 256, 0, c->stream>>>(a);
    CU_TRY(c, cudaGetLastError());
    CU_TRY(c, cudaEventRecord(s.ev[1], c->stream));
    CU_TRY(c, cudaEventSynchronize(s.ev[1]));
    float ms = 0;
    cudaEventElapsedTime(&ms, s.ev[0], s.ev[1]);
    s.ms_choose += ms;
    st.n_prim = n_prim;
    st.n_iv = n_iv;
    return CMB_OK;
  };
  auto nomem = [&](const ShardBlocks& blocks, uint32_t b0, uint32_t b1, uint64_t tail) {
    return fail(c, CMB_E_NOMEM, "shard %u: not enough device memory to decode blocks %u..%u (%llu bytes); the sharded sample holds %llu bytes", k, b0, b1,
                (unsigned long long)slice_bytes(blocks, b0, b1, tail), (unsigned long long)shard_need(c, k, st.n_prim, st.n_iv));
  };
  SliceStats ss;
  const int rc = decode_in_slices(c, in, out, ss, budget, step, nomem);
  if (rc == CMB_E_DECLINED) return fail(c, CMB_E_DECLINED, "shard %u: the device decoder declined it (%s); sharded input is decoded on the device only", k, c->err.c_str());
  if (rc) return rc;
  if (getenv("CMB_PIPELINE_STATS"))
    fprintf(stderr, "#shard_slices\tshard=%u\tslices=%u\tmax_slice_bytes=%llu\tcopy_inflate_ms=%.1f\tchain_ms=%.1f\textract_ms=%.1f\tgrow_ms=%.1f\n", k,
            ss.n_slices, (unsigned long long)ss.max_slice, ss.ms_inflate, ss.ms_chain, ss.ms_extract, ms_grow);
  return CMB_OK;
}

// cmb_submit_bgzf when the whole-stream buffers do not fit: the stream (a rank's block range in a group) in block slices, each
// submitted to K1 as one batch at the sample's running interval base -- in pair mode after its mates are matched, and only
// up to its cut (cmb_decode_slices.hpp).  A decline leaves the sample as cmb_begin_sample left it, for the host decoder.
int decode_sliced(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out) {
  auto& d = c->dec;
  *out = cmb_bgzf_result{};
  auto decline = [&](int rc) {
    cudaGetLastError();
    release_decode(c);
    if (int e = reset_sample(c)) return e;
    return rc;
  };
  // Room for the decode buffers and the sample's event list: the limit under CMB_DECODE_MEM_LIMIT_MB, else free memory plus
  // the decode buffers held
  auto room = [&]() -> uint64_t {
    if (const uint64_t lim = shard_mem_limit()) return lim;
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    cudaGetLastError();
    return free_b + decode_bytes(c);
  };
  if (room() < SLICE_MIN_BYTES) return decline(fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: not enough device memory for device-side decode"));
  uint64_t stream_end = 0;  // end of the inflated bytes whose records are walked
  const uint32_t walk_end = in->ranged ? std::min(in->walk_end_block, in->n_blocks) : in->n_blocks;
  for (uint32_t b = 0; b < walk_end; ++b) stream_end += in->block_isize[b];
  const uint64_t iv0 = c->n_intervals;
  double side = 0;       // the last slice's other buffers per compressed + inflated byte
  uint32_t carry = 0;    // pair mode: the largest eligible tid of the slices so far
  uint64_t cut_records = 0;
  auto budget = [&](uint64_t at) -> uint64_t {
    const uint64_t done = at > in->records_at ? at - in->records_at : 0;
    const uint64_t total = stream_end > in->records_at ? stream_end - in->records_at : 0;
    return decode_slice_budget(room(), !c->gene_mode, c->d_events.bytes(), done, total, c->n_intervals - iv0, side);
  };
  auto step = [&](BgzfCall& j, cmb_bgzf_result& r, uint64_t* next) -> int {
    const uint32_t n = (uint32_t)j.n_rec;
    uint32_t n_sub = n, iv_sub = (uint32_t)j.n_cig;
    cmb_read_batch tb;
    carve_batch(d.d_tuple_slab, n, (uint32_t)j.n_cig, &tb);
    const int32_t* mate = nullptr;
    uint32_t largest = carry;
    int rc;
    if (c->mode.filter_pairs) {
      // words 12..14 of d_cnt: the slice's largest eligible tid, then the cut's `after` and n - cut (zeroed by copy_inflate)
      uint32_t* w = d.d_cnt + 12;
      rc = match_mates(c, d.last_infl_base, n, true, "cmb_submit_bgzf", carry, w);
      if (rc == CMB_E_NOMEM) return SLICE_HALVE;
      if (rc) return rc;
      r.n_launches += 5;
      if (j.walk_end < walk_end) {  // not the last slice: hold the trailing run of its last eligible tid back for the next one
        const uint32_t g = (n + 255) / 256;
        kd_pair_cut_after<<<g, 256, 0, c->stream>>>(d.d_pair_key, tb.tid, n, w, w + 1);
        kd_pair_cut_at<<<g, 256, 0, c->stream>>>(d.d_pair_key, tb.tid, n, w, w + 1, w + 2);
        CU_TRY(c, cudaGetLastError());
        r.n_launches += 2;
      }
      uint32_t h[3] = {0, 0, 0};
      CU_TRY(c, cudaMemcpyAsync(h, w, 12, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaStreamSynchronize(c->stream));
      largest = h[0];
      const uint32_t cut = n - h[2];
      if (cut == 0)
        return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: the proper-pair records of reference %d do not fit in one decode slice; mates are "
                    "matched on the host", (int32_t)largest);
      if (cut < n) {  // the next slice starts at record `cut`; its records leave this slice's counters
        uint64_t off = 0;
        CU_TRY(c, cudaMemcpyAsync(&off, d.d_rec_off + cut, 8, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaMemcpyAsync(&iv_sub, tb.iv_begin + cut, 4, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaMemsetAsync(d.d_cnt + 16, 0, 16, c->stream));
        kd_count_held<<<(n - cut + 255) / 256, 256, 0, c->stream>>>(tb.tid, tb.flag, cut, n, j.in->own_tid_begin, j.in->own_tid_end, j.in->own_unplaced,
                                                                   (unsigned long long*)(d.d_cnt + 16), (unsigned long long*)(d.d_cnt + 18));
        CU_TRY(c, cudaGetLastError());
        uint64_t held[2] = {0, 0};
        CU_TRY(c, cudaMemcpyAsync(held, d.d_cnt + 16, 16, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaStreamSynchronize(c->stream));
        r.n_primary -= held[0];
        r.n_records -= held[1];
        r.n_intervals = iv_sub;
        r.n_launches += 1;
        *next = off;
        n_sub = cut;
        cut_records += n - cut;
      }
      mate = d.d_pair_mate;
    }
    if (k1_active(c)) {
      uint32_t excl = 0;
      if ((rc = j.excl_n(&excl))) return rc;
      rc = launch_k1(c, tb, n_sub, iv_sub, excl, mate);
      if (rc == CMB_E_NOMEM) return SLICE_HALVE;  // the event list did not grow: nothing of the slice was accumulated
      if (rc) return rc;
    }
    carry = largest;
    uint64_t other = d.d_tuple_slab.bytes() + d.d_rec_off.bytes();
    if (c->mode.filter_pairs)
      other += d.d_pair_key.bytes() + d.d_pair_mate.bytes() + d.d_pair_next.bytes() + d.d_pair_tag.bytes() + d.d_pair_head.bytes();
    side = (double)other / (double)std::max<uint64_t>(1, (j.byte_hi - j.byte_lo) + (j.total - j.u_lo));
    return CMB_OK;
  };
  auto nomem = [&](const ShardBlocks&, uint32_t, uint32_t, uint64_t) {
    return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: not enough device memory for device-side decode");
  };
  SliceStats ss;
  const int rc = decode_in_slices(c, in, out, ss, budget, step, nomem);
  if (rc == CMB_E_DECLINED) return decline(rc);
  if (rc) return rc;
  release_decode(c);  // the end of the sample needs the room; a sliced sample has no resident tuples to hand out
  out->ms_copy_inflate = ss.ms_inflate;
  out->ms_chain = ss.ms_chain;
  out->ms_extract = ss.ms_extract;
  if (getenv("CMB_PIPELINE_STATS"))
    fprintf(stderr, "#decode_slices\tslices=%u\tmax_slice_bytes=%llu\thalvings=%u\tpair_cut_records=%llu\n", ss.n_slices,
            (unsigned long long)ss.max_slice, ss.halvings, (unsigned long long)cut_records);
  return CMB_OK;
}

uint64_t shard_bytes(const cmb_ctx* c) {
  const auto& s = c->sh;
  uint64_t b = s.d_scan.bytes() + s.d_hash0.bytes() + s.d_tid_count.bytes() + s.d_src.bytes() + s.d_slot_iv.bytes() + s.d_as_val.bytes() +
               s.d_as_state.bytes() + s.d_state.bytes() + s.d_out_slab.bytes() + s.d_excluded.bytes();
  for (const auto& st : s.store) b += st.bytes();
  return b;
}

}  // namespace

namespace {
int begin_shards(cmb_ctx* c, const char* fn, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded, uint32_t first, uint32_t last,
                bool group) {
  if (!c || !tid_offsets || n_shards == 0) return fail(c, CMB_E_ARG, "%s: null argument or no shards", fn);
  if (!c->in_sample) return fail(c, CMB_E_ARG, "%s: no sample in progress", fn);
  if (c->mode.filter_pairs || c->params.filtering) return fail(c, CMB_E_ARG, "%s: sharded input takes no read filter", fn);
  if (n_shards > 255) return fail(c, CMB_E_ARG, "%s: at most 255 shards", fn);
  if (first > last || last > n_shards) return fail(c, CMB_E_ARG, "%s: shard range [%u, %u) outside the %u shards", fn, first, last, n_shards);
  const uint32_t n_ref = c->gene_mode ? c->n_ref_contigs : c->n_contigs;
  for (uint32_t k = 0; k < n_shards; ++k)
    if (tid_offsets[k] > n_ref || (k && tid_offsets[k] < tid_offsets[k - 1])) return fail(c, CMB_E_ARG, "%s: tid offsets outside the reference", fn);
  CU_TRY(c, cudaSetDevice(c->device));
  auto& s = c->sh;
  s.n_shards = n_shards;
  s.first = first;
  s.last = last;
  s.group = group;
  s.added = first;
  s.stage = 0;
  s.tid_offsets.assign(tid_offsets, tid_offsets + n_shards);
  if (s.store.size() < n_shards) s.store.resize(n_shards);
  for (auto& st : s.store) st.n_prim = st.n_iv = 0;
  s.have_excluded = excluded != nullptr;
  if (excluded) {
    if (int rc = s.d_excluded.ensure(c, std::max<uint32_t>(1, n_ref))) return rc;
    CU_TRY(c, cudaMemcpyAsync(s.d_excluded, excluded, n_ref, cudaMemcpyHostToDevice, c->stream));
  }
  if (int rc = s.d_err.ensure(c, 1)) return rc;
  CU_TRY(c, cudaMemsetAsync(s.d_err, 0xff, 8, c->stream));
  for (int i = 0; i < 4; ++i)
    if (int rc = shard_event(c, i)) return rc;
  s.ms_choose = s.ms_decode = 0;
  s.active = true;
  return CMB_OK;
}
}  // namespace

extern "C" int cmb_shard_begin(cmb_ctx* c, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded) {
  NvtxRange nvtx_fn("cmb_shard_begin");
  return begin_shards(c, "cmb_shard_begin", n_shards, tid_offsets, excluded, 0, n_shards, false);
}

extern "C" int cmb_shard_begin_range(cmb_ctx* c, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded, uint32_t shard_begin,
                                     uint32_t shard_end) {
  NvtxRange nvtx_fn("cmb_shard_begin_range");
  return begin_shards(c, "cmb_shard_begin_range", n_shards, tid_offsets, excluded, shard_begin, shard_end, true);
}

extern "C" int cmb_shard_add(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out) {
  NvtxRange nvtx_fn("cmb_shard_add");
  if (!c || !in || !out || !in->data || !in->block_coffset || !in->block_clen || !in->block_isize)
    return fail(c, CMB_E_ARG, "cmb_shard_add: null argument");
  auto& s = c->sh;
  if (!c->in_sample || !s.active || s.added >= s.last) return fail(c, CMB_E_ARG, "cmb_shard_add: call cmb_shard_begin first, once per shard");
  CU_TRY(c, cudaSetDevice(c->device));
  const uint32_t k = s.added;
  if (int rc = decode_shard(c, in, out, k)) return rc;
  s.ms_decode += out->ms_total;
  auto& st = s.store[k];
  CU_TRY(c, cudaEventRecord(s.ev[0], c->stream));
  // ---- the store's closing interval offset; shard 0 sizes every pair's running winner
  const uint64_t n0 = s.store[0].n_prim;
  if (int rc = shard_alloc(c, shard_need(c, k, st.n_prim, st.n_iv), [&] {
        int e = store_grow(c, st, st.n_prim, st.n_iv);
        if (!e && k == 0 && !s.group) e = s.d_state.ensure(c, n0 / 2 + 1, with_slack(n0 / 2 + 1));
        return e;
      }))
    return rc;
  const uint32_t iv_total = (uint32_t)st.n_iv;
  CU_TRY(c, cudaMemcpyAsync(st.view.b.iv_begin + st.n_prim, &iv_total, 4, cudaMemcpyHostToDevice, c->stream));
  if (s.group) {  // a group run scores every pair once all shards' lengths are known (cmb_shard_score)
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    s.added += 1;
    return CMB_OK;
  }
  if (k == 0) CU_TRY(c, cudaMemsetAsync(s.d_state, 0xff, sizeof(PairState) * (n0 / 2 + 1), c->stream));
  // ---- every pair's running winner, over the whole store: a pair whose primaries fell in different slices is whole here
  ShardPairArgs p{};
  p.st = st.view; p.as_val = s.d_as_val; p.as_state = s.d_as_state; p.excluded = s.have_excluded ? s.d_excluded.p : nullptr;
  p.state = s.d_state; p.n_pairs = std::min(st.n_prim, n0) / 2; p.shard = k; p.tid_offset = s.tid_offsets[k]; p.err = s.d_err;
  if (p.n_pairs) ks_pairs<<<(uint32_t)((p.n_pairs + 255) / 256), 256, 0, c->stream>>>(p);
  CU_TRY(c, cudaGetLastError());
  CU_TRY(c, cudaEventRecord(s.ev[1], c->stream));
  CU_TRY(c, cudaEventSynchronize(s.ev[1]));
  float ms = 0;
  cudaEventElapsedTime(&ms, s.ev[0], s.ev[1]);
  s.ms_choose += ms;
  s.added += 1;
  return CMB_OK;
}

namespace {
// The reader's own checks (shard_bam_reader.rs:117-121, 187-190), keyed like the kernels' errors: after every kernel-found error
// of the same set
unsigned long long shard_length_key(const std::vector<uint64_t>& n_prim) {
  const uint64_t n0 = n_prim[0];
  uint64_t n_min = n0;
  bool equal = true;
  for (uint64_t n : n_prim) {
    n_min = std::min(n_min, n);
    equal = equal && n == n0;
  }
  const unsigned long long phase_end = 0xfff;
  if (!equal) return (n_min << 24) | (phase_end << 12) | (3ull << 8);
  if (n0 % 2) return (n0 << 24) | (phase_end << 12) | (4ull << 8);
  return ~0ull;
}

// The error of the smallest key, or CMB_OK
int shard_key_error(cmb_ctx* c, unsigned long long key) {
  if (key != ~0ull && ((key >> 8) & 0xf) == 3)
    return fail(c, CMB_E_SHARD_EXIT, "Unexpectedly one BAM file input finished while another had further reads");
  if (key != ~0ull && ((key >> 8) & 0xf) == 4)
    return fail(c, CMB_E_SHARD_PANIC, "Unexpectedly was able to read a first read set, but not a second. Hmm.");
  return shard_error(c, key);
}

// The store views and tid offsets on the device, the winners counted per tid (ks_count after s.d_state holds the choice); the
// error key and the mapped winners' count come back to the host
int shard_count(cmb_ctx* c, ShardSortArgs& a, unsigned long long* key) {
  auto& s = c->sh;
  const uint32_t n_ref = c->gene_mode ? c->n_ref_contigs : c->n_contigs;
  if (int rc = s.d_tid_count.ensure(c, (size_t)n_ref + 1, (size_t)n_ref + 1)) return rc;
  if (int rc = s.d_stores.ensure(c, s.n_shards)) return rc;
  if (int rc = s.d_tid_offsets.ensure(c, s.n_shards)) return rc;
  std::vector<ShardStore> views(s.n_shards);
  for (uint32_t k = s.first; k < s.last; ++k) views[k] = s.store[k].view;
  CU_TRY(c, cudaMemcpyAsync(s.d_stores, views.data(), sizeof(ShardStore) * s.n_shards, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(s.d_tid_offsets, s.tid_offsets.data(), 4ull * s.n_shards, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(s.d_tid_count, 0, 8ull * ((size_t)n_ref + 1), c->stream));
  a = ShardSortArgs{};
  a.stores = s.d_stores; a.tid_offsets = s.d_tid_offsets; a.state = s.d_state; a.n_pairs = s.n_pairs; a.n_contigs = n_ref;
  a.tid_count = s.d_tid_count; a.err = s.d_err; a.own_begin = s.first; a.own_end = s.last;
  if (s.n_pairs) ks_count<<<(uint32_t)((s.n_pairs + 255) / 256), 256, 0, c->stream>>>(a);
  kf_scan<<<1, 1024, 0, c->stream>>>(s.d_tid_count, n_ref);
  CU_TRY(c, cudaGetLastError());
  unsigned long long h[2] = {~0ull, 0};
  CU_TRY(c, cudaMemcpyAsync(&h[0], s.d_err, 8, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(&h[1], s.d_tid_count + n_ref, 8, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  *key = std::min(h[0], s.len_key);
  s.n_out = h[1];
  return CMB_OK;
}

// The counted winners, sorted by tid, into one device batch that is submitted; `out` reports the sample
int shard_sort_submit(cmb_ctx* c, ShardSortArgs& a, cmb_shard_result* out) {
  auto& s = c->sh;
  const uint64_t n_out = s.n_out, n_pairs = s.n_pairs;
  if (n_out >= 0xffffff00ull) return fail(c, CMB_E_ARG, "cmb_shard_finish: more than 2^32 mapped winners");
  if (int rc = shard_alloc(c, shard_need(c, s.last, 0, 0, n_out), [&] {
        int e = s.d_src.ensure(c, n_out + 1, with_slack(n_out + 1));
        return e ? e : s.d_slot_iv.ensure(c, n_out + 1, with_slack(n_out + 1));
      }))
    return rc;
  a.src = s.d_src; a.slot_iv = s.d_slot_iv; a.n_out = n_out;
  if (n_pairs) ks_scatter<<<(uint32_t)((n_pairs + 255) / 256), 256, 0, c->stream>>>(a);
  kf_scan<<<1, 1024, 0, c->stream>>>(s.d_slot_iv, (uint32_t)n_out);
  unsigned long long n_iv = 0;
  CU_TRY(c, cudaMemcpyAsync(&n_iv, s.d_slot_iv + n_out, 8, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  size_t offs[13];
  const size_t slab = batch_slab_bytes((uint32_t)n_out, (uint32_t)n_iv, offs);
  if (int rc = shard_alloc(c, shard_need(c, s.last, 0, 0, n_out, n_iv), [&] { return s.d_out_slab.ensure(c, slab, slab + slab / 8); }))
    return rc;
  carve_batch(s.d_out_slab, (uint32_t)n_out, (uint32_t)n_iv, &a.out);
  if (n_out) ks_gather<<<(uint32_t)((n_out + 255) / 256), 256, 0, c->stream>>>(a);
  CU_TRY(c, cudaGetLastError());
  CU_TRY(c, cudaEventRecord(s.ev[3], c->stream));
  out->n_pairs = n_pairs;
  out->n_records = 2 * n_pairs;
  out->n_emitted = n_out;
  out->n_intervals = n_iv;
  out->store_bytes = shard_bytes(c);
  out->ms_choose = s.ms_choose;
  out->ms_decode = s.ms_decode;
  CU_TRY(c, cudaEventSynchronize(s.ev[3]));
  cudaEventElapsedTime(&out->ms_sort, s.ev[2], s.ev[3]);
  if (!n_out) return CMB_OK;
  return cmb_submit_device_batch(c, &a.out, (uint32_t)n_out, (uint32_t)n_iv);
}
}  // namespace

extern "C" int cmb_shard_finish(cmb_ctx* c, cmb_shard_result* out) {
  NvtxRange nvtx_fn("cmb_shard_finish");
  if (!c || !out) return fail(c, CMB_E_ARG, "cmb_shard_finish: null argument");
  auto& s = c->sh;
  if (!c->in_sample || !s.active || s.group || s.added != s.n_shards) return fail(c, CMB_E_ARG, "cmb_shard_finish: every shard must be added first");
  s.active = false;
  CU_TRY(c, cudaSetDevice(c->device));
  *out = cmb_shard_result{};
  s.n_prim.resize(s.n_shards);
  for (uint32_t k = 0; k < s.n_shards; ++k) s.n_prim[k] = s.store[k].n_prim;
  s.n_pairs = *std::min_element(s.n_prim.begin(), s.n_prim.end()) / 2;
  s.len_key = shard_length_key(s.n_prim);
  CU_TRY(c, cudaEventRecord(s.ev[2], c->stream));
  ShardSortArgs a{};
  unsigned long long key;
  if (int rc = shard_count(c, a, &key)) return rc;
  if (int rc = shard_key_error(c, key)) return rc;
  // ---- the winners, sorted by tid, into one device batch
  return shard_sort_submit(c, a, out);
}

// ---- group runs -------------------------------------------------------------------------------------------------------------
extern "C" int cmb_shard_score(cmb_ctx* c, const uint64_t* n_primary) {
  NvtxRange nvtx_fn("cmb_shard_score");
  if (!c || !n_primary) return fail(c, CMB_E_ARG, "cmb_shard_score: null argument");
  auto& s = c->sh;
  if (!c->in_sample || !s.active || !s.group || s.added != s.last || s.stage != 0)
    return fail(c, CMB_E_ARG, "cmb_shard_score: call cmb_shard_begin_range and add this context's shards first");
  for (uint32_t k = s.first; k < s.last; ++k)
    if (n_primary[k] != s.store[k].n_prim)
      return fail(c, CMB_E_ARG, "cmb_shard_score: shard %u holds %llu primaries, not %llu", k, (unsigned long long)s.store[k].n_prim,
                  (unsigned long long)n_primary[k]);
  CU_TRY(c, cudaSetDevice(c->device));
  s.n_prim.assign(n_primary, n_primary + s.n_shards);
  const uint64_t n0 = s.n_prim[0];
  s.n_pairs = *std::min_element(s.n_prim.begin(), s.n_prim.end()) / 2;
  s.len_key = shard_length_key(s.n_prim);
  const uint64_t cells = (uint64_t)s.n_shards * s.n_pairs;
  // the score table, shard 0's name hashes where shard 0 is decoded elsewhere, and the choice
  if (int rc = shard_alloc(c, shard_need(c, s.last, 0, 0) + 4 * cells + 8 * n0, [&] {
        int e = s.d_score.ensure(c, std::max<uint64_t>(1, cells), with_slack(std::max<uint64_t>(1, cells)));
        if (!e && !(s.first == 0 && s.last > 0)) e = s.d_hash0.ensure(c, n0 + 1, with_slack(n0 + 1));
        if (!e) e = s.d_state.ensure(c, s.n_pairs + 1, with_slack(s.n_pairs + 1));
        return e;
      }))
    return rc;
  CU_TRY(c, cudaEventRecord(s.ev[0], c->stream));
  for (uint32_t k = s.first; k < s.last; ++k) {
    const auto& st = s.store[k];
    ShardPairArgs p{};
    p.st = st.view; p.as_val = st.as_val; p.as_state = st.as_state; p.excluded = s.have_excluded ? s.d_excluded.p : nullptr;
    p.n_pairs = std::min(st.n_prim, n0) / 2; p.shard = k; p.tid_offset = s.tid_offsets[k]; p.err = s.d_err;
    p.score = s.d_score.p + (uint64_t)k * s.n_pairs; p.n_score = s.n_pairs;
    if (p.n_pairs) ks_score<<<(uint32_t)((p.n_pairs + 255) / 256), 256, 0, c->stream>>>(p);
  }
  CU_TRY(c, cudaGetLastError());
  CU_TRY(c, cudaEventRecord(s.ev[1], c->stream));
  CU_TRY(c, cudaEventSynchronize(s.ev[1]));
  float ms = 0;
  cudaEventElapsedTime(&ms, s.ev[0], s.ev[1]);
  s.ms_choose += ms;
  s.stage = 1;
  return CMB_OK;
}

namespace {
int shard_io(cmb_ctx* c, const char* fn, uint32_t shard, void* scores, void* names, cudaMemcpyKind dir) {
  if (!c || !scores) return fail(c, CMB_E_ARG, "%s: null argument", fn);
  auto& s = c->sh;
  if (!s.active || !s.group || s.stage != 1 || shard >= s.n_shards) return fail(c, CMB_E_ARG, "%s: no scored shard %u (cmb_shard_score first)", fn, shard);
  CU_TRY(c, cudaSetDevice(c->device));
  const bool h2d = dir == cudaMemcpyHostToDevice;
  int32_t* col = s.d_score.p + (uint64_t)shard * s.n_pairs;
  if (s.n_pairs) CU_TRY(c, cudaMemcpyAsync(h2d ? (void*)col : scores, h2d ? scores : (const void*)col, 4 * s.n_pairs, dir, c->stream));
  if (shard == 0 && names && s.n_prim[0])
    CU_TRY(c, cudaMemcpyAsync(h2d ? (void*)s.d_hash0.p : names, h2d ? names : (const void*)s.d_hash0.p, 8 * s.n_prim[0], dir, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}
}  // namespace

extern "C" int cmb_shard_export(cmb_ctx* c, uint32_t shard, int32_t* scores, uint64_t* names) {
  return shard_io(c, "cmb_shard_export", shard, scores, names, cudaMemcpyDeviceToHost);
}

extern "C" int cmb_shard_import(cmb_ctx* c, uint32_t shard, const int32_t* scores, const uint64_t* names) {
  return shard_io(c, "cmb_shard_import", shard, const_cast<int32_t*>(scores), const_cast<uint64_t*>(names), cudaMemcpyHostToDevice);
}

extern "C" int cmb_shard_exchange(cmb_ctx* c, const uint32_t* shard_cuts) {
  NvtxRange nvtx_fn("cmb_shard_exchange: NCCL broadcasts");
  if (!c || !shard_cuts) return fail(c, CMB_E_ARG, "cmb_shard_exchange: null argument");
  if (!c->comm) return fail(c, CMB_E_ARG, "cmb_shard_exchange: no communicator (cmb_comm_init first)");
  auto& s = c->sh;
  if (!s.active || !s.group || s.stage != 1) return fail(c, CMB_E_ARG, "cmb_shard_exchange: call cmb_shard_score first");
  const int N = c->comm_size, me = c->comm_rank;
  if (shard_cuts[0] != 0 || shard_cuts[N] != s.n_shards || shard_cuts[me] != s.first || shard_cuts[me + 1] != s.last)
    return fail(c, CMB_E_ARG, "cmb_shard_exchange: shard_cuts do not match this context's shards");
  for (int r = 0; r < N; ++r)
    if (shard_cuts[r] > shard_cuts[r + 1]) return fail(c, CMB_E_ARG, "cmb_shard_exchange: shard_cuts must be non-decreasing");
  CU_TRY(c, cudaSetDevice(c->device));
  if (c->local_barrier) c->local_barrier->arrive_and_wait();
  // each owner broadcasts its columns in place (shard k's column sits at k * n_pairs on every rank), the owner of shard 0 its names
  NCCL_TRY(c, ncclGroupStart());
  for (int r = 0; r < N; ++r) {
    const size_t n = (size_t)(shard_cuts[r + 1] - shard_cuts[r]) * s.n_pairs * 4;
    int32_t* p = s.d_score.p + (uint64_t)shard_cuts[r] * s.n_pairs;
    if (n) NCCL_TRY(c, ncclBroadcast(p, p, n, ncclChar, r, c->comm, c->stream));
    if (shard_cuts[r] == 0 && shard_cuts[r + 1] > 0 && s.n_prim[0])
      NCCL_TRY(c, ncclBroadcast(s.d_hash0.p, s.d_hash0.p, 8 * s.n_prim[0], ncclChar, r, c->comm, c->stream));
  }
  NCCL_TRY(c, ncclGroupEnd());
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}

extern "C" int cmb_shard_choose(cmb_ctx* c, uint64_t* err_key) {
  NvtxRange nvtx_fn("cmb_shard_choose");
  if (!c || !err_key) return fail(c, CMB_E_ARG, "cmb_shard_choose: null argument");
  auto& s = c->sh;
  if (!c->in_sample || !s.active || !s.group || s.stage != 1) return fail(c, CMB_E_ARG, "cmb_shard_choose: call cmb_shard_score (and exchange the scores) first");
  CU_TRY(c, cudaSetDevice(c->device));
  CU_TRY(c, cudaEventRecord(s.ev[0], c->stream));
  const uint64_t n0 = s.n_prim[0];
  for (uint32_t k = std::max<uint32_t>(1, s.first); k < s.last; ++k) {
    const uint64_t n = std::min(s.store[k].n_prim, n0);
    if (n) ks_names<<<(uint32_t)((n + 255) / 256), 256, 0, c->stream>>>(s.store[k].names.p, s.d_hash0.p, n, k, s.d_err);
  }
  if (s.n_pairs) ks_choose<<<(uint32_t)((s.n_pairs + 255) / 256), 256, 0, c->stream>>>(s.d_score.p, s.n_pairs, s.n_shards, s.d_state.p);
  CU_TRY(c, cudaGetLastError());
  CU_TRY(c, cudaEventRecord(s.ev[1], c->stream));
  CU_TRY(c, cudaEventSynchronize(s.ev[1]));
  float ms = 0;
  cudaEventElapsedTime(&ms, s.ev[0], s.ev[1]);
  s.ms_choose += ms;
  CU_TRY(c, cudaEventRecord(s.ev[2], c->stream));
  ShardSortArgs a{};
  unsigned long long key;
  if (int rc = shard_count(c, a, &key)) return rc;
  *err_key = key;
  s.stage = 2;
  return CMB_OK;
}

extern "C" int cmb_shard_finish_group(cmb_ctx* c, uint64_t err_key, cmb_shard_result* out) {
  NvtxRange nvtx_fn("cmb_shard_finish_group");
  if (!c || !out) return fail(c, CMB_E_ARG, "cmb_shard_finish_group: null argument");
  auto& s = c->sh;
  if (!c->in_sample || !s.active || !s.group || s.stage != 2) return fail(c, CMB_E_ARG, "cmb_shard_finish_group: call cmb_shard_choose first");
  s.active = false;
  CU_TRY(c, cudaSetDevice(c->device));
  *out = cmb_shard_result{};
  if (int rc = shard_key_error(c, err_key)) return rc;
  // shard_count's view of the device buffers, rebuilt (the choice and the counts are on the device)
  ShardSortArgs a{};
  a.stores = s.d_stores; a.tid_offsets = s.d_tid_offsets; a.state = s.d_state; a.n_pairs = s.n_pairs;
  a.n_contigs = c->gene_mode ? c->n_ref_contigs : c->n_contigs; a.tid_count = s.d_tid_count; a.err = s.d_err;
  a.own_begin = s.first; a.own_end = s.last;
  return shard_sort_submit(c, a, out);
}
