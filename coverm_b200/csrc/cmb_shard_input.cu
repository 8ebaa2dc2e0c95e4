// libcoverm_b200 -- sharded input (cmb_shard_*; kernels in cmb_shards.cuh): every shard decoded in block slices into its
// primary store, the choice of each pair's shard (running winner on one GPU, score table in a group), and the winners sorted
// by tid into one device batch.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdio>
#include <cstdlib>

#include "cmb_context.cuh"
#include "cmb_bgzf.cuh"

namespace {
#include "cmb_common.cuh"
#include "cmb_shards.cuh"

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

// The buffers shard_need counts: stores, AS scratch, name hashes, pair state
uint64_t store_bytes_held(const cmb_ctx* c) {
  const auto& s = c->sh;
  uint64_t b = s.d_as_val.bytes() + s.d_as_state.bytes() + s.d_hash0.bytes() + s.d_state.bytes();
  for (const auto& st : s.store) b += st.bytes();
  return b;
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
uint64_t shard_room(const cmb_ctx* c) { return device_room(store_bytes_held(c) + decode_bytes(c)); }

int shard_nomem(cmb_ctx* c, uint64_t need) {
  return fail(c, CMB_E_NOMEM, "sharded input needs %llu bytes of device memory for its shard stores, pair state, name hashes, AS scratch and "
              "sorted winners; the device has %llu bytes free for them", (unsigned long long)need, (unsigned long long)shard_room(c));
}

// `alloc` once, and again after the decode buffers are released; CMB_E_NOMEM with the sample's need when it still fails
template <class F>
int shard_alloc(cmb_ctx* c, uint64_t need, F alloc) {
  if (const uint64_t lim = decode_mem_limit().value_or(0); lim && need > lim) return shard_nomem(c, need);
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
  const uint64_t lim = decode_mem_limit().value_or(0);
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
    launch_scan(c, s.d_scan, (uint32_t)n_rec);
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
  auto nomem = [&](const SliceBlocks& blocks, uint32_t b0, uint32_t b1, uint64_t tail) {
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
  launch_scan(c, s.d_tid_count, n_ref);
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
  launch_scan(c, s.d_slot_iv, (uint32_t)n_out);
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
