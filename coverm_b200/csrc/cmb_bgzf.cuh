// The device decode as the rest of the library drives it (cmb_bgzf.cu): one staged decode call (BgzfCall), the memory its
// buffers take, and the loop that decodes a stream in block slices.  An ordinary stream that does not fit goes through that
// loop by one driver in cmb_bgzf.cu (stream_in_slices), decoded for K1 (decode_sliced) or filtered for `coverm filter`
// (cmb_filter_bgzf); the shards of sharded input (decode_shard, cmb_shard_input.cu) drive it with their own budget and step.
#pragma once
#include <algorithm>
#include <climits>
#include <optional>
#include <vector>

#include "cmb_context.cuh"
#include "cmb_slices.hpp"

namespace cmb __attribute__((visibility("hidden"))) {

constexpr uint64_t DEC_TAIL_BYTES = 4u << 20;  // ranged decode: inflated bytes kept beyond the range for its last straddling record

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

  int run();  // prepare, then the four stages unless there is nothing to decode
  int prepare();
  int copy_inflate();
  int declined();
  int chain();
  int extract();
  int stage_times();  // waits for the extract; out's ms_copy_inflate, ms_chain, ms_extract and ms_total from the stage events
  int excl_n(uint32_t* n);
};

// ---- the decode's device memory

// CMB_DECODE_MEM_LIMIT_MB (testing aid): behave as if the device had this much room, in bytes; a fraction of a megabyte slices
// small files.  A call whose compressed and inflated bytes exceed its whole megabytes fails as if out of memory
// (BgzfCall::prepare).  A sliced decode gives it to its slices' decode buffers and the sample's event list (decode_sliced), or
// to a sharded sample's stores and one slice's compressed and inflated bytes (decode_shard).
std::optional<uint64_t> decode_mem_limit();
// The decode buffers a slice fills (d_scan included); released when a store cannot grow beside them
uint64_t decode_bytes(const cmb_ctx* c);
void release_decode(cmb_ctx* c);
// Bytes the device has room for: the limit under CMB_DECODE_MEM_LIMIT_MB, else what is free plus `held`, what the caller
// holds and may give back
uint64_t device_room(uint64_t held);

// ---- the decode in block slices

constexpr uint64_t SLICE_TAIL_BYTES = 64u << 10;  // a slice's first tail: one BGZF block; doubled for a longer record
constexpr int SLICE_HALVINGS = 8;                 // a slice whose buffers fail to allocate is halved this often before giving up
constexpr uint64_t SLICE_MIN_BYTES = 64u << 20;   // budget floor: below it a failed allocation, not the estimate, shrinks a slice

// Statistics of one sliced decode
struct SliceStats {
  uint32_t n_slices = 0;
  uint32_t halvings = 0;  // over the whole decode
  uint64_t max_slice = 0;  // compressed + inflated bytes of the largest slice
  float ms_inflate = 0, ms_chain = 0, ms_extract = 0;
  uint64_t pair_cut_records = 0;  // pair mode (stream_in_slices): records held back at the ends of the slices
  float ms_mates = 0;             // pair mode (stream_in_slices): host clock of mate matching and the cuts
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
  const SliceBlocks blocks{nb, in->size, in->block_coffset, in->block_clen, ustart.data()};
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
    int rc = j.run();
    if (rc == CMB_E_NOMEM) rc = SLICE_HALVE;
    uint64_t next = j.exit_off;
    if (!rc && !j.nothing_to_decode) {
      if (int e = j.stage_times()) return e;
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

}  // namespace cmb
