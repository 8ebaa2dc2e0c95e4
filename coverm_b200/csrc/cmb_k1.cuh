// K1: filter + delta accumulation, K1c: cross-block sortedness check (see cmb_device.cu header).
#pragma once
#include "cmb_filter_preds.cuh"
// ------------------------------------------------------------------------------------------------ K1
struct K1Args {
  // batch (device pointers)
  const int32_t* tid;
  const int32_t* pos;
  const uint16_t* flag;
  const uint8_t* mapq;
  const uint8_t* nm_state;
  const uint32_t* nm;
  const uint32_t* l_seq;
  const uint32_t* aligned;
  const uint32_t* del;
  const uint32_t* ins;
  const uint32_t* iv_begin;
  const int32_t* iv_start;
  const int32_t* iv_len;
  uint32_t n;
  // reference
  const uint32_t* off_span;  // [n_local+1]
  const uint32_t* len;       // [n_local]
  // the contigs [tid_begin, tid_end) this context owns; in gene mode seg_begin is the global number of its first local segment
  // (gene), as the arena, gene_bound and the bin pool are laid out over the genes [seg_begin, seg_begin + n_local) only
  uint32_t n_contigs, tid_begin, tid_end, seg_begin;
  // outputs
  int32_t* arena;       // gene mode: the events are added here
  // contig mode: the sample's event list, entry 2k / 2k + 1 = interval k's start / end as (arena element << 1) | sign (1 for
  // the -1 at the end), K1_NO_EVENT where there is none; interval k counts from the sample's first (iv_base is the batch's
  // first, n_iv its interval slots).  K1e buckets the entries by bitmap word, in the order word_count (+1 per event) gives.
  ulonglong2* events;
  uint64_t iv_base;
  uint32_t n_iv;
  uint32_t* word_count;
  uint32_t* span_bits;  // span occupancy bitmap: the bit of every span an event is added to (K2 works only on those spans)
  int32_t* tail_sum;
  cmb_contig_stats* rows;
  int2* block_minmax;  // per block {min kept tid, max kept tid} for the cross-block sortedness check
  uint32_t* error_flags;
  // cross-RANK half of the sortedness check (multi-GPU contig sharding only, else NULL): per block {min, max} kept tid of
  // the records with index < excl_n (INT_MAX / INT_MIN = none); k1c_check_sorted folds them into the rank's kept range
  int2* block_xrange;
  uint32_t excl_n;
  // per-gene coverage (genes.rs): the arena's segments are genes, records carry contig tids.  NULL = contig mode.
  const uint32_t* gene_first;   // [n_contigs + 1] first gene of each contig (genes sorted by (tid, start))
  const uint32_t* gene_start;   // [n_genes] gene range on its contig, clamped to the contig
  const uint32_t* gene_end;
  const uint32_t* gene_maxlen;  // [n_contigs] longest gene of the contig (bounds the backward search for overlaps)
  const uint32_t* contig_len;   // [n_contigs]
  uint8_t* contig_seen;         // [n_contigs] a kept record of an owned contig mapped here (genes.rs:220-246)
  unsigned long long* kept_primary;  // primaries among the kept records of owned contigs (ReadsMapped, genes.rs:249-252)
  uint32_t* gene_bound;         // [n_local] records that may add events to the gene: bounds its depth (K1b's bin pool layout)
  // pair path: partner of each record (cmb_pairs.cuh, records in file order) or NULL = the host layout (completed pairs
  // only, stored first mate at the even index, its partner right after)
  const int32_t* mate;
  // params
  cmb_params p;
  uint8_t filter_single, filter_pairs;
};

constexpr unsigned long long K1_NO_EVENT = ~0ull;

#ifndef CMB_K1_MINBLOCKS
#define CMB_K1_MINBLOCKS 6
#endif
#ifndef CMB_K1_PREFETCH
#define CMB_K1_PREFETCH 1  // issue the segment and first-interval loads right behind the column loads (one DRAM round trip less)
#endif
__global__ void __launch_bounds__(K1_THREADS, CMB_K1_MINBLOCKS) k1_filter_accumulate(const K1Args a) {
  const uint32_t i = blockIdx.x * K1_THREADS + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool valid = i < a.n;
  const cmb_params& p = a.p;

  RecView r = {};
  int32_t tid = -1, pos = 0;
  uint32_t ins = 0, ivb = 0, ive = 0;
  if (valid) {
    tid = a.tid[i];
    pos = a.pos[i];
    r.flag = a.flag[i];
    r.mapq = a.mapq[i];
    r.nm_state = a.nm_state[i];
    r.nm = a.nm[i];
    r.l_seq = a.l_seq[i];
    r.aligned = a.aligned[i];
    r.del = a.del[i];
    ins = a.ins[i];
    ivb = a.iv_begin[i];
    ive = a.iv_begin[i + 1];
  }
#if CMB_K1_PREFETCH
  // A thread's loads form the chain columns -> intervals -> segment table -> REDs.  The segment of a
  // record depends on its tid only and its first aligned block on iv_begin only, so both are requested here, before the
  // filter arithmetic and the block-wide sortedness scan, and are in registers by the time the events are added.
  uint32_t pre_L = 0, pre_off0 = 0, pre_off1 = 0;
  int32_t pre_s = INT_MIN, pre_n = 0;
  const bool pre_seg = valid && !a.gene_first && tid >= 0 && (uint32_t)tid >= a.tid_begin && (uint32_t)tid < a.tid_end &&
                       (uint32_t)tid < a.n_contigs;
  if (pre_seg) {
    const uint32_t lc = (uint32_t)tid - a.tid_begin;
    pre_L = __ldg(a.len + lc);
    pre_off0 = __ldg(a.off_span + lc);
    pre_off1 = __ldg(a.off_span + lc + 1);
  }
  if (valid && ivb < ive) {
    pre_s = __ldg(a.iv_start + ivb);
    pre_n = __ldg(a.iv_len + ivb);
  }
#endif
  const bool unmapped = r.flag & 0x4, secondary = r.flag & 0x100, supplementary = r.flag & 0x800, proper = r.flag & 0x2;
  // FlagFilter::passes, lib.rs:67-78
  const bool flag_pass = !(secondary && !p.include_secondary) && !(supplementary && !p.include_supplementary) &&
                         !(!proper && !p.include_improper_pairs);
  bool keep = valid && flag_pass && !unmapped;  // contig.rs:119-125
  bool nm_err = false;
  if (valid && p.filtering) {
    bool passes;
    if (a.filter_single && !a.filter_pairs) {  // filter.rs:88-116
      const bool passes_filter1 = !unmapped && (p.include_supplementary || !supplementary) && (p.include_secondary || !secondary);
      passes = passes_filter1 && single_read_passes(r, p, &nm_err);
    } else {  // filter.rs:117-233: the host submits completed pairs only; stored first mate at the even index
      const int32_t mi = a.mate ? a.mate[i] : (int32_t)(i ^ 1u);
      const uint32_t m = (uint32_t)mi;
      RecView o = {};
      const bool have_mate = mi >= 0 && m < a.n;
      const bool i_is_second = a.mate ? m < i : (i & 1u);  // the stored first mate is the earlier record
      if (have_mate) {
        o.flag = a.flag[m];
        o.mapq = a.mapq[m];
        o.nm_state = a.nm_state[m];
        o.nm = a.nm[m];
        o.l_seq = a.l_seq[m];
        o.aligned = a.aligned[m];
        o.del = a.del[m];
      }
      const RecView& first = i_is_second ? o : r;   // record1 (stored)
      const RecView& second = i_is_second ? r : o;  // record (just read)
      bool ok = have_mate;
      if (ok && a.filter_single) ok = single_read_passes(first, p, &nm_err) && single_read_passes(second, p, &nm_err);
      if (ok) ok = read_pair_passes(second, first, p, &nm_err);
      passes = ok;
    }
    keep = keep && passes;
  }
  uint32_t err = 0;
  if (keep && r.nm_state != 1) nm_err = true;  // nm(&record), contig.rs:206
  if (nm_err) err |= ERR_NM;
  if (keep && (tid < 0 || (uint32_t)tid >= a.n_contigs)) {
    err |= ERR_TID;
    keep = false;
  }

  // ---- sortedness of the kept stream (contig.rs:128-132): prefix max over the block
  __shared__ int s_wmax[K1_THREADS / 32];
  __shared__ int s_wmin[K1_THREADS / 32];
  {
    const int key = keep ? tid : INT_MIN;
    int pm = key;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(FULL, pm, d);
      if ((int)lane >= d) pm = max(pm, o);
    }
    int excl = __shfl_up_sync(FULL, pm, 1);
    if (lane == 0) excl = INT_MIN;
    int kmin = keep ? tid : INT_MAX;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) kmin = min(kmin, __shfl_xor_sync(FULL, kmin, d));
    if (lane == 31) s_wmax[warp] = pm;
    if (lane == 0) s_wmin[warp] = kmin;
    __shared__ int s_xmax[K1_THREADS / 32];
    __shared__ int s_xmin[K1_THREADS / 32];
    if (a.block_xrange) {
      const bool xk = keep && i < a.excl_n;
      const int xmax = __reduce_max_sync(FULL, xk ? tid : INT_MIN);
      const int xmin = __reduce_min_sync(FULL, xk ? tid : INT_MAX);
      if (lane == 0) {
        s_xmax[warp] = xmax;
        s_xmin[warp] = xmin;
      }
    }
    __syncthreads();
    if (a.block_xrange && threadIdx.x == 0) {
      int xmax = INT_MIN, xmin = INT_MAX;
      for (uint32_t w = 0; w < K1_THREADS / 32; ++w) {
        xmax = max(xmax, s_xmax[w]);
        xmin = min(xmin, s_xmin[w]);
      }
      a.block_xrange[blockIdx.x] = make_int2(xmin, xmax);
    }
    int before = INT_MIN;
    for (uint32_t w = 0; w < warp; ++w) before = max(before, s_wmax[w]);
    if (keep && tid < max(before, excl)) err |= ERR_UNSORTED;
    if (threadIdx.x == 0) {
      int bmax = INT_MIN, bmin = INT_MAX;
      for (uint32_t w = 0; w < K1_THREADS / 32; ++w) {
        bmax = max(bmax, s_wmax[w]);
        bmin = min(bmin, s_wmin[w]);
      }
      a.block_minmax[blockIdx.x] = make_int2(bmin, bmax);
    }
  }

  // +1 at `s` and -1 at `e` (when e lies inside the segment) of segment `lc`, the bits of their spans, plus the chunk tail
  // sums K1b scans.  Gene mode adds the events into the arena; contig mode returns them as event list entries.
  // Records are sorted, so neighbouring lanes mostly mark the same bitmap word: one RED per distinct word of the warp.  Plain
  // per-lane REDs took K1 from 6.7 to 14.2 ms on `bench.py --config ns` (H100 80GB HBM3, 400 W); aggregated: 7.0 ms.  The
  // same group adds its event count to the word's count (contig mode).
  auto mark_span = [&](uint64_t g) {
    const uint32_t w = (uint32_t)(g / BITMAP_ELEMS_PER_WORD);
    const uint32_t peers = __match_any_sync(__activemask(), w);
    const uint32_t bits = __reduce_or_sync(peers, 1u << ((uint32_t)(g / SPAN) % BITMAP_SPANS_PER_WORD));
    if (lane == (uint32_t)__ffs(peers) - 1) {
      atomicOr(a.span_bits + w, bits);
      if (a.word_count) atomicAdd(a.word_count + w, (uint32_t)__popc(peers));
    }
  };
  // Returns the events as event list entries; only gene mode (add_gene_events) also adds them into the arena, which contig
  // mode does not have
  auto add_events_in = [&](uint32_t L, uint32_t off0, uint32_t off1, uint32_t s, uint64_t e) -> ulonglong2 {
    const uint64_t base = (uint64_t)off0 * SPAN;
    const uint64_t end_padded = (uint64_t)off1 * SPAN;  // first element of the next segment
    const uint64_t gs = base + s;
    const bool has_end = e < L;  // "True unless the read hits the contig end"
    ulonglong2 out = make_ulonglong2(gs << 1, K1_NO_EVENT);
    mark_span(gs);
    const uint64_t ks = gs / CHUNK;
    const bool cont_s = end_padded > (ks + 1) * (uint64_t)CHUNK;  // this segment continues past chunk ks
    if (has_end) {
      const uint64_t ge = base + e;
      out.y = ge << 1 | 1u;
      mark_span(ge);
      const uint64_t ke = ge / CHUNK;
      if (ke != ks) {
        if (cont_s) atomicAdd(a.tail_sum + ks, 1);
        if (end_padded > (ke + 1) * (uint64_t)CHUNK) atomicAdd(a.tail_sum + ke, -1);
      }
    } else if (cont_s) {
      atomicAdd(a.tail_sum + ks, 1);
    }
    return out;
  };
  auto add_gene_events = [&](uint32_t lc, uint32_t s, uint64_t e) {
    const ulonglong2 ev = add_events_in(a.len[lc], a.off_span[lc], a.off_span[lc + 1], s, e);
    atomicAdd(a.arena + (ev.x >> 1), 1);
    if (ev.y != K1_NO_EVENT) atomicAdd(a.arena + (ev.y >> 1), -1);
  };

  if (a.gene_first) {
    // ---- per-gene coverage (genes.rs:182-344, 467-552).  A gene's delta array is the contig's, cut to [start, end) with the
    //      running depth at `start` as its first element: exactly what clipping every aligned block to the gene gives.  Reads
    //      are assigned to the genes that contain their leftmost position.  Under a contig shard (cmb_set_genes_range) only
    //      records of the owned contigs count: all of their genes are local segments, rows keep the global gene number.
    //      keep implies 0 <= tid < n_contigs, so one unsigned compare tests the range.
    if (keep && (uint32_t)tid - a.tid_begin < a.tid_end - a.tid_begin) {
      const bool primary = !secondary && !supplementary;
      a.contig_seen[tid] = 1;
      if (primary) atomicAdd(a.kept_primary, 1ull);
      const uint32_t CL = a.contig_len[tid];
      uint64_t ref_end = (uint32_t)pos;  // end of the last aligned block
      for (uint32_t k = ivb; k < ive; ++k) {
        const int32_t s = a.iv_start[k];
        if (s == INT_MIN) continue;
        if (s < 0 || (uint32_t)s >= CL) {  // `ups_and_downs[cursor] += 1` would panic
          err |= ERR_BOUNDS;
          continue;
        }
        ref_end = max(ref_end, (uint64_t)(uint32_t)s + (uint32_t)a.iv_len[k]);
      }
      const uint32_t g0 = a.gene_first[tid], g1 = a.gene_first[tid + 1];
      if (g0 < g1 && !(err & ERR_BOUNDS)) {
        const uint32_t maxlen = a.gene_maxlen[tid];
        const uint32_t from = (uint32_t)pos >= maxlen ? (uint32_t)pos - maxlen + 1 : 0;  // a gene starting earlier ends at or before pos
        uint32_t lo = g0, hi = g1;  // first gene with start >= from
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (a.gene_start[mid] < from) lo = mid + 1;
          else hi = mid;
        }
        const uint64_t indels = (uint64_t)ins + r.del;
        for (uint32_t g = lo; g < g1; ++g) {
          const uint32_t gsx = a.gene_start[g], gex = a.gene_end[g];
          if ((uint64_t)gsx >= max(ref_end, (uint64_t)(uint32_t)pos + 1)) break;  // genes are sorted by start
          const uint32_t lg = g - a.seg_begin;
          atomicAdd(a.gene_bound + lg, 1u);  // every gene the record may add events to: bounds the gene's depth
          if ((uint32_t)pos >= gsx && (uint32_t)pos < gex) {  // read_starts.partition_point range (genes.rs:518-523)
            cmb_contig_stats* row = a.rows + g;
            atomicAdd((unsigned long long*)&row->n_records, 1ull);
            if (primary) atomicAdd((unsigned long long*)&row->n_primary, 1ull);
            const uint64_t mis = r.nm >= indels ? r.nm - indels : 0;  // edit.saturating_sub(indels), genes.rs:297
            if (mis) atomicAdd((unsigned long long*)&row->sum_edit, (unsigned long long)mis);
            if (primary && r.aligned > 0) atomicAdd(&row->sum_identity_primary, ((double)r.aligned - (double)r.nm) / (double)r.aligned);
          }
          for (uint32_t k = ivb; k < ive; ++k) {
            const int32_t s = a.iv_start[k];
            if (s == INT_MIN) continue;
            const uint64_t e = (uint64_t)(uint32_t)s + (uint32_t)a.iv_len[k];
            if (e <= gsx || (uint32_t)s >= gex) continue;  // no overlap
            const uint32_t cs = max((uint32_t)s, gsx) - gsx;
            add_gene_events(lg, cs, e - gsx);  // e - gsx >= gene length: the block runs past the gene, no -1
          }
        }
      }
    }
    err = __reduce_or_sync(FULL, err);
    if (err && lane == 0) atomicOr(a.error_flags, err);
    return;
  }

  const bool mine = keep && (uint32_t)tid >= a.tid_begin && (uint32_t)tid < a.tid_end;
  // ---- per-contig read counters (contig.rs:157-159, 204-211; genome.rs:173-174, 220-223, 677-682, 724-727)
  //      One set of REDs per run of a warp's counted records with the same contig: records are sorted, so a warp's 32 records
  //      fall in a few runs, and per-lane REDs would queue up in L2 on the same row.  Records that are not counted (filtered
  //      out, other ranks' contigs) do not break a run.  A run starts at a counted lane whose contig differs from the previous
  //      counted lane's, so unsorted input (ERR_UNSORTED) only splits a contig into more runs; the adds commute.
  {
    const uint32_t mine_mask = __ballot_sync(FULL, mine);
    if (mine_mask) {
      const bool primary = !secondary && !supplementary;
      const uint32_t below = mine_mask & ((1u << lane) - 1);
      const int prev_tid = __shfl_sync(FULL, tid, below ? 31 - __clz(below) : lane);  // the previous counted lane's
      const uint32_t heads = __ballot_sync(FULL, mine && (!below || prev_tid != tid)) | 1u;  // lane 0 ends uncounted lanes
      const uint32_t after = heads & ~((2u << lane) - 1);  // heads above this lane (2u << 31 == 0: none above lane 31)
      const uint32_t run_end = after ? __ffs(after) - 1 : 32;  // one past the last lane of this lane's run
      const uint32_t run = (run_end == 32 ? FULL : (1u << run_end) - 1) & ~((1u << lane) - 1);  // the run, seen from its head
      uint64_t s_edit = mine ? r.nm : 0, s_indel = mine ? (uint64_t)ins + r.del : 0;  // a warp's sum may pass 2^32
      double idn = 0.0;
      if (mine && r.aligned > 0) idn = ((double)r.aligned - (double)r.nm) / (double)r.aligned;
      double s_idp = primary ? idn : 0.0, s_idn = !supplementary ? idn : 0.0;
#pragma unroll
      for (uint32_t d = 1; d < 32; d <<= 1) {  // segmented: lane l ends up with the sums of lanes l .. run_end-1
        const uint64_t oe = __shfl_down_sync(FULL, s_edit, d), oi = __shfl_down_sync(FULL, s_indel, d);
        const double op = __shfl_down_sync(FULL, s_idp, d), on = __shfl_down_sync(FULL, s_idn, d);
        if (lane + d < run_end) {
          s_edit += oe;
          s_indel += oi;
          s_idp += op;
          s_idn += on;
        }
      }
      const uint32_t s_rec = __popc(mine_mask & run), s_pri = __popc(__ballot_sync(FULL, mine && primary) & run),
                     s_ns = __popc(__ballot_sync(FULL, mine && !supplementary) & run);
      if (mine && (heads >> lane & 1)) {
        cmb_contig_stats* row = a.rows + tid;
        atomicAdd((unsigned long long*)&row->n_records, (unsigned long long)s_rec);
        if (s_pri) atomicAdd((unsigned long long*)&row->n_primary, (unsigned long long)s_pri);
        if (s_ns) atomicAdd((unsigned long long*)&row->n_nonsupp, (unsigned long long)s_ns);
        if (s_edit) atomicAdd((unsigned long long*)&row->sum_edit, (unsigned long long)s_edit);
        if (s_indel) atomicAdd((unsigned long long*)&row->sum_indel, (unsigned long long)s_indel);
        if (s_idp != 0.0) atomicAdd(&row->sum_identity_primary, s_idp);
        if (s_idn != 0.0) atomicAdd(&row->sum_identity_nonsupp, s_idn);
      }
    }
  }

  // ---- delta events (contig.rs:171-186) into the event list: plain coalesced stores, one 16-B entry pair per interval slot.
  //      Every slot of the batch is written: K1_NO_EVENT for the slots of records that add no event (filtered out, another
  //      shard's contig), for CMB_IV_PAD and for an interval out of bounds.  Threads 0 and n - 1 also fill the slots before
  //      the first record's and after the last record's, which belong to no record.
  if (valid) {
    const ulonglong2 none = make_ulonglong2(K1_NO_EVENT, K1_NO_EVENT);
    ulonglong2* ev = a.events + a.iv_base;
    if (i == 0)
      for (uint32_t k = 0; k < min(ivb, a.n_iv); ++k) __stcs(ev + k, none);
    if (i + 1 == a.n)
      for (uint32_t k = ive; k < a.n_iv; ++k) __stcs(ev + k, none);
    const uint32_t lc = (uint32_t)tid - a.tid_begin;
    (void)lc;
#if CMB_K1_PREFETCH
    const uint32_t L = pre_L, off0 = pre_off0, off1 = pre_off1;
#else
    uint32_t L = 0, off0 = 0, off1 = 0;
    if (mine) L = a.len[lc], off0 = a.off_span[lc], off1 = a.off_span[lc + 1];
#endif
    for (uint32_t k = ivb; k < min(ive, a.n_iv); ++k) {
      ulonglong2 out = none;
      if (mine) {
#if CMB_K1_PREFETCH
        const int32_t s = k == ivb ? pre_s : a.iv_start[k];
        const uint32_t n = (uint32_t)(k == ivb ? pre_n : a.iv_len[k]);
#else
        const int32_t s = a.iv_start[k];
        const uint32_t n = (uint32_t)a.iv_len[k];
#endif
        if (s == INT_MIN) {
          // CMB_IV_PAD: unused slot of the interval pool
        } else if (s < 0 || (uint32_t)s >= L) {  // `ups_and_downs[cursor] += 1` would panic
          err |= ERR_BOUNDS;
        } else {
          out = add_events_in(L, off0, off1, (uint32_t)s, (uint64_t)(uint32_t)s + n);
        }
      }
      __stcs(ev + k, out);
    }
  }
  err = __reduce_or_sync(FULL, err);
  if (err && lane == 0) atomicOr(a.error_flags, err);
}

// Cross-block sortedness: block b's smallest kept tid must be >= every earlier block's largest.
// With block_xrange (multi-GPU): also folds the blocks' exclusive kept tid ranges into kept_range[0] = max tid + 1 (0 = none),
// kept_range[1] = INT_MAX - min tid.
__global__ void __launch_bounds__(1024) k1c_check_sorted(const int2* block_minmax, uint32_t n_blocks, uint32_t* error_flags,
                                                         const int2* block_xrange, uint32_t* kept_range) {
  __shared__ int s_max[1024];
  const uint32_t t = threadIdx.x;
  const uint32_t per = (n_blocks + 1023) / 1024;
  const uint32_t b0 = t * per, b1 = min(n_blocks, b0 + per);
  if (block_xrange) {
    int xmin = INT_MAX, xmax = INT_MIN;
    for (uint32_t b = b0; b < b1; ++b) {
      const int2 x = block_xrange[b];
      xmin = min(xmin, x.x);
      xmax = max(xmax, x.y);
    }
    xmin = __reduce_min_sync(FULL, xmin);
    xmax = __reduce_max_sync(FULL, xmax);
    if ((t & 31) == 0 && xmax != INT_MIN) {
      atomicMax(kept_range + 0, (uint32_t)xmax + 1u);
      atomicMax(kept_range + 1, (uint32_t)(INT_MAX - xmin));
    }
  }
  int lmax = INT_MIN;
  bool bad = false;
  for (uint32_t b = b0; b < b1; ++b) {
    const int2 mm = block_minmax[b];
    if (mm.x != INT_MAX && mm.x < lmax) bad = true;
    lmax = max(lmax, mm.y);
  }
  s_max[t] = lmax;
  __syncthreads();
  int before = INT_MIN;
  for (uint32_t k = 0; k < t; ++k) before = max(before, s_max[k]);
  for (uint32_t b = b0; b < b1 && !bad; ++b) {
    const int2 mm = block_minmax[b];
    if (mm.x != INT_MAX && mm.x < before) bad = true;
  }
  if (bad) atomicOr(error_flags, ERR_UNSORTED);
}

// ------------------------------------------------------------------------------------------------ K1e
// Contig mode: the sample's event list bucketed by bitmap word (1024 arena elements), one thread per interval slot.  An event
// at element g goes to buckets[word_off[w] + r] of its word w = g / 1024 as the u16 code (g % 1024) | sign << 10.  The slots
// r of a word are handed out by counting word_count[w] down from K1's count, one RED per distinct word of a warp (records are
// sorted, so a warp's events fall in a few words), which leaves every count at zero for the next sample.  Order inside a
// bucket is arbitrary: K2 only adds the deltas up.
constexpr uint32_t K1E_THREADS = 256;
__global__ void __launch_bounds__(K1E_THREADS) k1e_bucket_events(const ulonglong2* events, uint64_t n_iv, const uint32_t* word_off,
                                                                uint32_t* word_count, uint16_t* buckets) {
  const uint64_t k = (uint64_t)blockIdx.x * K1E_THREADS + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  const ulonglong2 e = k < n_iv ? __ldcs(events + k) : make_ulonglong2(K1_NO_EVENT, K1_NO_EVENT);
  auto place = [&](unsigned long long x) {
    const bool has = x != K1_NO_EVENT;
    const uint32_t active = __ballot_sync(FULL, has);
    if (!has) return;
    const uint64_t g = x >> 1;
    const uint32_t w = (uint32_t)(g / BITMAP_ELEMS_PER_WORD);
    const uint32_t off = __ldg(word_off + w);
    const uint32_t peers = __match_any_sync(active, w), n = __popc(peers), head = __ffs(peers) - 1;
    uint32_t top = 0;
    if (lane == head) top = atomicSub(word_count + w, n);
    top = __shfl_sync(peers, top, head);
    const uint32_t r = top - n + __popc(peers & ((1u << lane) - 1));
    buckets[off + r] =(uint16_t)((uint32_t)(g % BITMAP_ELEMS_PER_WORD) | (uint32_t)(x & 1) << 10);
  };
  place(e.x);
  place(e.y);
}

