// The device library's context (cmb_ctx) and what its translation units share: cmb_device.cu (context, reference, sample,
// K1-K3), cmb_comm.cu (NCCL), cmb_bgzf.cu (device decode, mate matching, `coverm filter`) and cmb_shard_input.cu (sharded
// input).  Private to the library; no kernel is declared here.  Every kernel is compiled in exactly one of those units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include <nccl.h>
#include <nvtx3/nvToolsExt.h>

#include "../../include/coverm_b200.h"

// Hidden: the shared helpers link across the library's units but are not part of its ABI.
namespace cmb __attribute__((visibility("hidden"))) {

// NVTX ranges around the entry points and the stages of the device decode (visible in Nsight Systems / `ncu --nvtx`; no-ops
// without a tool attached: nvtx3 is header-only and resolves its injection library lazily).
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

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

// Sharded input (cmb_shards.cuh): a shard's primary store as the kernels see it
struct ShardStore {
  cmb_read_batch b;  // device pointers; tids already shifted into the concatenated layout
  uint8_t* info;
};

// Running choice of every pair (shard_bam_reader.rs:210-262).  best = highest score so far, winner = its shard, ties = how many
// candidates share it.
struct PairState {
  long long best;
  uint32_t winner;
  uint32_t ties;
};

}  // namespace cmb

using namespace cmb;  // every unit that includes this header works with these names

// The ABI's opaque handle keeps default visibility (every entry point takes it), while its members' types stay hidden
#pragma GCC diagnostic push
#pragma GCC diagnostic ignored "-Wattributes"
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
                          // [10..11] n_owned; sliced decode: [12..14] pair cut (pair_cut), [16..19] held-back counts
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
    PinnedBuf<uint8_t> filter_stage[2];  // cmb_filter_bgzf: sink call k's bytes are in filter_stage[k & 1]; 64 MB each
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
  // the BGZF output stream deflated on the device (cmb_deflate_*; cmb_deflate.cu); buffers allocated by cmb_deflate_begin
  struct Deflate {
    Buf<uint8_t> d_raw;     // the stream's bytes not yet deflated: the carry (< one block) first, then what a feed appends
    Buf<uint8_t> d_blocks;  // one DFL_MAX_OUT slot per block of the piece
    Buf<uint32_t> d_size;   // per block: its BGZF size | DFL_STORED_FLAG when stored
    Buf<uint8_t> d_packed;  // the piece's blocks back to back
    PinnedBuf<uint8_t> stage[2];  // sink call k's bytes are in stage[k & 1]
    PinnedBuf<uint32_t> h_size;
    uint64_t carry = 0;
    bool active = false;
    cmb_deflate_stats stats{};
    cudaEvent_t ev[2]{};
    ~Deflate() {
      for (auto e : ev)
        if (e) cudaEventDestroy(e);
    }
  } dfl;
};
#pragma GCC diagnostic pop

namespace cmb __attribute__((visibility("hidden"))) {

// `code`, with its message as the error of `ctx` (of cmb_create when null)
int fail(cmb_ctx* ctx, int code, const char* fmt, ...);

#define CU_TRY(ctx, expr)                                                                                   \
  do {                                                                                                      \
    cudaError_t e_ = (expr);                                                                                \
    if (e_ != cudaSuccess) return fail(ctx, e_ == cudaErrorMemoryAllocation ? CMB_E_NOMEM : CMB_E_CUDA,      \
                                       "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

#define NCCL_TRY(ctx, expr)                                                                                       \
  do {                                                                                                            \
    ncclResult_t r_ = (expr);                                                                                     \
    if (r_ != ncclSuccess) return fail(ctx, CMB_E_CUDA, "%s failed: %s (%s:%d)", #expr, ncclGetErrorString(r_), __FILE__, __LINE__); \
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

inline size_t with_slack(size_t n) { return n + n / 8 + 16; }  // grow-only buffers sized by the data

inline size_t batch_slab_bytes(uint32_t nr, uint32_t ni, size_t* offs) {
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

inline void carve_batch(void* slab, uint32_t nr, uint32_t ni, cmb_read_batch* b) {
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

// ---- host functions one unit calls in another
// cmb_device.cu
bool k1_active(const cmb_ctx* c);
int launch_k1(cmb_ctx* c, const cmb_read_batch& b, uint32_t n_records, uint32_t n_intervals, uint32_t excl_n = 0xffffffffu,
              const int32_t* mate = nullptr);
int reset_sample(cmb_ctx* c);
// cmb_bgzf.cu
// Mate matching over the resident inflated stream (cmb_pairs.cuh); sets d.last_mate.  filter_out: ReferenceSortedBamFilter's
// (false only for `coverm filter --inverse`).  Declines when the stream needs the host's file-order walk.  A slice of a sliced
// decode passes the largest eligible tid of the slices before it (`carry`) and gets its own largest in *largest (device).
int match_mates(cmb_ctx* c, const uint8_t* infl_base, uint32_t n_rec, bool filter_out, const char* who, uint32_t carry = 0,
                uint32_t* largest = nullptr);
// cmb_deflate.cu: d_src[0, n) (device memory) fed to the context's deflate stream, as cmb_deflate_feed feeds host bytes;
// *n_calls counts the sink calls made
int deflate_feed_device(cmb_ctx* c, const uint8_t* d_src, uint64_t n, cmb_filter_sink sink, void* user, uint32_t* n_calls);
// kf_scan (cmb_filter.cuh) on the context stream: v[0, n) exclusively scanned in place, v[n] = the total
void launch_scan(cmb_ctx* c, unsigned long long* v, uint32_t n);

}  // namespace cmb
