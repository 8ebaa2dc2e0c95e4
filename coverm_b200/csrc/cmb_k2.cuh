// K2: segmented prefix sum of the delta arena + every O(L) reduction of EST::add_contig, one pass, HBM-bound.
//
// Persistent CTAs (2 or 3 per SM, 256 threads).  Iteration i of CTA b works on the 8192-element chunk b + i * gridDim.x and
// keeps a ring of K2_STAGES 32 KB tiles in flight.  Which of a chunk's 256 spans hold any event is known from the span
// occupancy bitmap K1 sets (8 words per chunk): a chunk with at least K2_DENSE_SPANS such spans is fetched whole with TMA
// (cp.async.bulk.tensor.2d, 128B swizzle, mbarrier complete_tx); in any other chunk each warp copies only its non-empty
// 128-byte rows with cp.async into the same swizzled tile positions, and the spans it does not fetch are zero by
// construction.  A thread owns one 32-element span (8 x LDS.128, conflict-free through the swizzle); contigs start on span
// boundaries, so a span never straddles two contigs.  Running depth at a span = chunk carry (K1b) + segmented warp/CTA scan
// of the span totals.  Depth is piecewise constant and deltas are sparse (~1-2 % of positions), so a thread only keeps the
// span total and a 32-bit mask of its non-zero positions; covered bases, sum of depth and the depth histogram of the
// end-trimmed window are then accumulated per RUN in a short loop over the set bits (the deltas are re-read from the
// shared-memory tile, which stays resident until the next iteration's barrier).  The window depth histogram is a dense
// array of u32 counts per contig in global memory, bins[bin_base[c] + depth] (K1b laid it out: every window depth of c is at
// most its read count), so a run's count is one fire-and-forget RED; K3 reads the bins in depth order and re-zeroes them.
// Depth 0 is not added: K3 derives its count from the window length and covered_window.  At config 2's coverage about half
// of the runs are at depth 0, all of them on one address per contig.
#pragma once

struct K2Args {
  const uint32_t* off_span;
  const uint32_t* len;
  const uint32_t* chunk_first;
  const int32_t* carry_in;
  cmb_contig_stats* rows;
  uint32_t tid_begin, n_local, n_chunks, excl;
  int32_t* arena;
  uint32_t* span_bits;   // [n_chunks * K2_WARPS] span occupancy bitmap (K1); word w of a chunk = the spans of its warp w
  uint32_t* load_stats;  // [0] += spans loaded, [1] += chunks loaded whole (CMB_PIPELINE_STATS)
  const uint64_t* bin_base;  // [n_local + 1] first bin of each contig (K1b); bin_base[n_local] = bins needed
  uint32_t* bins;            // the bin pool: pool_cap u32 counts, zero outside a sample
  uint64_t pool_cap;
  uint32_t* bin_hi;          // [n_local] highest depth added per contig (atomicMax)
  uint32_t* error_flags;
};

// A chunk with at least this many non-empty spans (of 256) is loaded whole with one TMA tile; sparser chunks row by row.
// On an H100 80GB HBM3 at 400 W, K2 time moved by under 2 % for thresholds from 96 to 257 (never whole) on both `bench.py
// --config 2` and `--config ns` (DESIGN.md §4, K2): row copies are not what limits K2 there.  160 sends chunks above ~60 %
// occupancy down the TMA path.
#ifndef CMB_K2_DENSE_SPANS
#define CMB_K2_DENSE_SPANS 160
#endif
constexpr uint32_t K2_DENSE_SPANS = CMB_K2_DENSE_SPANS;
static_assert(K2_STAGES >= 2, "the refill of a stage is issued one iteration after it was read");

constexpr uint32_t K2_SMEM_STAGE_BYTES = K2_STAGES * CHUNK_BYTES;
constexpr uint32_t K2_SMEM_MISC = 64 /*barriers*/ + 2 * K2_WARPS * 8 /*warp aggregates, double-buffered*/;
constexpr uint32_t K2_SMEM_BYTES = K2_SMEM_STAGE_BYTES + K2_SMEM_MISC;

template <bool HIST, bool CLEAN>
__global__ void __launch_bounds__(K2_THREADS, CMB_K2_MINBLOCKS) k2_scan_reduce(const __grid_constant__ CUtensorMap tmap, const K2Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];  // stage tiles need the 1024 B swizzle-atom alignment
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + K2_SMEM_STAGE_BYTES);
  int2* wagg2 = reinterpret_cast<int2*>(smem + K2_SMEM_STAGE_BYTES + 64);

  const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
  // The pool is sized before the launch from a bound of bin_base[n_local]; when it is still too small (cmb_grow_buffers
  // then grows it to exactly that) no bin is added and K3 reads none.
  const bool hist = HIST && __ldg(a.bin_base + a.n_local) <= a.pool_cap;
  if (HIST && !hist && blockIdx.x == 0 && t == 0) atomicOr(a.error_flags, ERR_CAPACITY);

  // Static schedule: iteration i of CTA b works on chunk b + i * gridDim.x.  Every thread knows its next chunk, so the chunk's
  // metadata (first / last contig, carry-in, bitmap words) is requested ahead and the dependent lookups (contig of the span,
  // its start and length) can start before the tile has even arrived.
  auto chunk_of = [&](uint32_t i) -> uint32_t { return blockIdx.x + i * gridDim.x; };
  // word `lane` (lanes 0..7) of chunk ck's span bitmap
  auto load_bits = [&](uint32_t ck) -> uint32_t {
    return ck < a.n_chunks && lane < K2_WARPS ? a.span_bits[ck * K2_WARPS + lane] : 0u;
  };
  uint32_t n_loaded = 0, n_dense = 0;  // thread 0: what this CTA fetched (load_stats)
  // All threads: start loading chunk ck into stage s.  `bits` is load_bits(ck).  Every thread commits one cp.async group per
  // call, so that cp.async.wait_group counts the same way everywhere.  Returns the warp's spans that the stage will hold.
  auto fill = [&](uint32_t s, uint32_t ck, uint32_t bits) -> uint32_t {
    uint32_t have = 0;
    if (ck < a.n_chunks) {
      const uint32_t pop = __reduce_add_sync(FULL, __popc(bits));  // the same on every thread: a CTA-uniform decision
      const uint32_t own = __shfl_sync(FULL, bits, warp);
      const bool dense = pop >= K2_DENSE_SPANS;
      uint8_t* tile = smem + s * CHUNK_BYTES;
      if (t == 0) {
        const uint32_t bar = smem_u32(full + s);
        if (dense) {
          fence_proxy_async_smem();  // the stage's previous reads and cp.async writes (ordered by the CTA barrier) come first
          mbar_arrive_expect_tx(bar, CHUNK_BYTES);
          tma_load_2d(smem_u32(tile), &tmap, 0, (int32_t)(ck * CHUNK_ROWS), bar);
        } else {
          mbar_arrive(bar);  // keeps the barrier's phase in step with the whole-tile stages
        }
        n_loaded += dense ? CHUNK_SPANS : pop;
        n_dense += dense;
      }
      if (dense) {
        have = FULL;
      } else {
        // The warp copies its own non-empty rows, four per instruction: lanes 8q..8q+7 take the eight 16-byte units of the
        // q-th row of the round, so every instruction moves four whole 128-byte lines.  The rows land where the TMA box would
        // put them (unit j of row r at r * 128 + (j ^ (r & 7)) * 16).  A thread lets other lanes write only its own row and
        // reads no other row, so a stage needs no CTA-wide completion; the warp waits for its group and syncs before reading.
        have = own;
        uint32_t m = own;
        const uint32_t q = lane >> 3, unit = lane & 7;
        const int4* src = reinterpret_cast<const int4*>(a.arena + (uint64_t)ck * CHUNK + (uint64_t)warp * 32 * SPAN) + unit;
        while (m) {
          uint32_t r = 32;
#pragma unroll
          for (uint32_t k = 0; k < 4; ++k) {
            if (k == q && m) r = (uint32_t)__ffs(m) - 1;
            m &= m - 1;
          }
          if (r < 32) {
            const uint32_t row = warp * 32 + r;
            cp_async_16(smem_u32(tile + row * 128 + ((unit ^ (row & 7)) << 4)), src + r * (SPAN / 4));
          }
        }
      }
    }
    cp_async_commit();
    return have;
  };

  if (t == 0) {
    for (uint32_t s = 0; s < K2_STAGES; ++s) mbar_init(smem_u32(full + s), 1);
    fence_barrier_init();
  }
  __syncthreads();
  // have[k] / own[k]: the spans of this warp that stage k holds / the bitmap word of this warp for the chunk in stage k
  uint32_t have[K2_STAGES], own[K2_STAGES];
#pragma unroll
  for (uint32_t s = 0; s < K2_STAGES; ++s) {
    const uint32_t bits = load_bits(chunk_of(s));
    own[s] = __shfl_sync(FULL, bits, warp);
    have[s] = fill(s, chunk_of(s), bits);
  }
  uint32_t n_bits = load_bits(chunk_of(K2_STAGES));  // the bitmap of the next chunk to fill, requested an iteration ahead
  __syncthreads();

  constexpr uint32_t UNITS = SPAN / 4;  // 16-byte units per span
  const uint32_t row = t;               // this thread's span is tile row t
  // byte offset inside a stage tile of element e of this thread's span
  auto elem_off = [&](uint32_t e) -> uint32_t { return row * 128 + (((e >> 2) ^ (row & 7)) << 4) + ((e & 3) << 2); };
  const uint32_t E = a.excl;
  uint32_t n_cf = 0, n_cl = 0;  // metadata of the NEXT iteration's chunk, requested an iteration ahead
  int n_cin = 0;
  if (chunk_of(0) < a.n_chunks) {
    n_cf = __ldg(a.chunk_first + chunk_of(0));
    n_cl = __ldg(a.chunk_first + chunk_of(0) + 1);
    n_cin = __ldg(a.carry_in + chunk_of(0));
  }
  uint32_t it = 0;

  for (;; ++it) {
    const uint32_t s = it % K2_STAGES;
    const uint32_t chunk = chunk_of(it);
    if (chunk >= a.n_chunks) break;
    const uint32_t cf = n_cf, cl = n_cl;
    const int cin = n_cin;
    {
      const uint32_t nx = chunk_of(it + 1);
      if (nx < a.n_chunks) {
        n_cf = __ldg(a.chunk_first + nx);
        n_cl = __ldg(a.chunk_first + nx + 1);
        n_cin = __ldg(a.carry_in + nx);
      }
    }
    // ---- which contig owns this thread's span (needs no tile data: these loads fly while the tile arrives and is scanned)
    const uint32_t span = chunk * CHUNK_SPANS + t;
    uint32_t c;
    {
      uint32_t lo = cf, hi = cl;
      while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (__ldg(a.off_span + mid) <= span) lo = mid;
        else hi = mid - 1;
      }
      c = lo;
    }
    const uint32_t cstart = __ldg(a.off_span + c);
    const uint32_t L = __ldg(a.len + c);
    uint64_t bin0 = 0, bin1 = 0;  // this contig's bins
    if (hist) {
      bin0 = __ldg(a.bin_base + c);
      bin1 = __ldg(a.bin_base + c + 1);
    }
    uint32_t s_have = 0, s_own = 0;
#pragma unroll
    for (uint32_t k = 0; k < K2_STAGES; ++k)
      if (k == s) {
        s_have = have[k];
        s_own = own[k];
      }
    mbar_wait(smem_u32(full + s), (it / K2_STAGES) & 1);
    cp_async_wait<K2_STAGES - 2>();  // this thread's copies into stage s (only later fills may still be in flight)
    __syncwarp();                    // ... and those of the other lanes of its warp
    if (CLEAN && lane == 0 && s_own) a.span_bits[chunk * K2_WARPS + warp] = 0;
    int2* wagg = wagg2 + (it & 1) * K2_WARPS;

    // ---- SPAN consecutive deltas per thread: LDS.128s through the 128B swizzle (conflict-free).
    //      Only their sum and the mask of non-zero positions stay in registers.  A span the stage does not hold is all zero.
    const uint8_t* tilep = smem + s * CHUNK_BYTES;
    int total = 0;
    uint32_t ev = 0;
    if ((s_have >> lane) & 1u) {
      int4* g = reinterpret_cast<int4*>(a.arena + (uint64_t)span * SPAN);
#pragma unroll
      for (uint32_t j = 0; j < UNITS; ++j) {
        const int4 q = *reinterpret_cast<const int4*>(tilep + row * 128 + ((j ^ (row & 7)) << 4));
        const uint32_t e4 = (q.x != 0 ? 1u : 0u) | (q.y != 0 ? 2u : 0u) | (q.z != 0 ? 4u : 0u) | (q.w != 0 ? 8u : 0u);
        total += (q.x + q.y) + (q.z + q.w);
        ev |= e4 << (4 * j);
        if (CLEAN && e4) g[j] = make_int4(0, 0, 0, 0);  // re-zero only the 16 B units that hold an event
      }
    }

    const bool is_head = span == cstart;
    const uint32_t rel = (span - cstart) * SPAN;  // position in the contig of the span's first element
    const uint32_t n_in = rel >= L ? 0u : min(SPAN, L - rel);
    uint32_t w0 = 0, w1 = 0;
    if (2ull * E < L) {
      const uint32_t ws = E, we = L - E;
      w0 = rel >= ws ? 0u : min(SPAN, ws - rel);
      w1 = rel >= we ? 0u : min(SPAN, we - rel);
      if (w1 < w0) w1 = w0;
    }

    // ---- segmented (by contig head) inclusive scan of span totals across the warp
    int val = total;
    int flg = is_head;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int ov = __shfl_up_sync(FULL, val, d);
      const int of = __shfl_up_sync(FULL, flg, d);
      if ((int)lane >= d) {
        if (!flg) val += ov;
        flg |= of;
      }
    }
    int pval = __shfl_up_sync(FULL, val, 1), pflg = __shfl_up_sync(FULL, flg, 1);
    if (lane == 0) {
      pval = 0;
      pflg = 0;
    }
    if (lane == 31) wagg[warp] = make_int2(val, flg);
    __syncthreads();  // warp aggregates visible; the previous iteration's tile reads are complete
    if (it > 0) {
      // refill the stage of the previous iteration (read until this barrier)
      const uint32_t rs = (it - 1) % K2_STAGES, rk = chunk_of(it - 1 + K2_STAGES);
      const uint32_t r_own = __shfl_sync(FULL, n_bits, warp);
      const uint32_t r_have = fill(rs, rk, n_bits);
#pragma unroll
      for (uint32_t k = 0; k < K2_STAGES; ++k)
        if (k == rs) {
          have[k] = r_have;
          own[k] = r_own;
        }
      n_bits = load_bits(chunk_of(it + K2_STAGES));
    }

    int wv, wf;
    {
      const int2 wa = lane < K2_WARPS ? wagg[lane] : make_int2(0, 0);
      wv = wa.x;
      wf = wa.y;
#pragma unroll
      for (int d = 1; d < (int)K2_WARPS; d <<= 1) {
        const int ov = __shfl_up_sync(FULL, wv, d);
        const int of = __shfl_up_sync(FULL, wf, d);
        if ((int)lane >= d) {
          if (!wf) wv += ov;
          wf |= of;
        }
      }
      const int src = warp ? (int)warp - 1 : 0;
      wv = __shfl_sync(FULL, wv, src);
      wf = __shfl_sync(FULL, wf, src);
      if (warp == 0) {
        wv = 0;
        wf = 0;
      }
    }
    int carry;
    if (is_head) carry = 0;
    else if (pflg) carry = pval;
    else if (wf) carry = wv + pval;
    else carry = cin + wv + pval;

    // ---- reductions over this span (EST:393-404, 447-465, 494-501), run by run
    uint32_t cov_full = 0, cov_win = 0;
    uint64_t sum_win = 0;
    uint32_t bin_top = 0;  // highest depth this thread added to contig c's bins
    auto hist_add = [&](int depth, uint32_t cnt) {
      // 0 <= depth <= bound = bin1 - bin0 - 1 for a consistent arena (every -1 follows its +1 within the contig, and a
      // record adds at most 1 at any position)
      if (depth < 0 || (uint64_t)depth >= bin1 - bin0) {
        atomicOr(a.error_flags, ERR_INTERNAL);
        return;
      }
      atomicAdd(a.bins + bin0 + (uint32_t)depth, cnt);
      bin_top = max(bin_top, (uint32_t)depth);
    };
    // a run [from, to) of the span at one depth, clipped to the contig and to its end-trimmed window
    auto close_run = [&](int depth, uint32_t from, uint32_t to) {
      const uint32_t nc = min(to, n_in) - min(from, n_in);
      const uint32_t nw = min(max(to, w0), w1) - min(max(from, w0), w1);
      if (depth > 0) {
        cov_full += nc;
        cov_win += nw;
      }
      if (nw) {
        sum_win += (uint64_t)(int64_t)depth * nw;
        if (hist && depth != 0) hist_add(depth, nw);
      }
    };
    if (ev) {
      int depth = carry;
      uint32_t from = 0;
      uint32_t m = ev;
      while (m) {
        const uint32_t j = (uint32_t)__ffs((int)m) - 1;
        m &= m - 1;
        close_run(depth, from, j);
        depth += *reinterpret_cast<const int*>(tilep + elem_off(j));  // the delta at position j
        from = j;
      }
      close_run(depth, from, SPAN);
    } else {  // no event in the span: constant depth
      const uint32_t nc = n_in, nw = w1 - w0;
      if (carry > 0) {
        cov_full += nc;
        cov_win += nw;
      }
      sum_win += (uint64_t)(int64_t)carry * nw;
    }
    if (hist) {
      // event-free spans: one RED per distinct (contig, depth) of the warp, added by the group's first lane (usually 1-3 groups)
      const uint32_t nw = w1 - w0;
      uint32_t cm = __ballot_sync(FULL, ev == 0 && nw > 0 && carry != 0);
      while (cm) {
        const int leader = __ffs(cm) - 1;
        const int d0 = __shfl_sync(FULL, carry, leader);
        const uint32_t c0 = __shfl_sync(FULL, c, leader);
        const bool same = ((cm >> lane) & 1u) && carry == d0 && c == c0;
        const uint32_t m = __ballot_sync(FULL, same);
        if (same) {
          const uint32_t tot = __reduce_add_sync(m, nw);
          if ((int)lane == leader) hist_add(carry, tot);
        }
        cm &= ~m;
      }
    }

    // ---- per-contig accumulation: one RED triple (and the bin_hi max) per (warp, contig)
    {
      const uint32_t c0 = __shfl_sync(FULL, c, 0);
      if (__all_sync(FULL, c == c0)) {
        const uint32_t sf = __reduce_add_sync(FULL, cov_full), sw = __reduce_add_sync(FULL, cov_win);
        const uint64_t sd = warp_sum_u64(sum_win);
        const uint32_t top = hist ? __reduce_max_sync(FULL, bin_top) : 0u;
        if (lane == 0) {
          cmb_contig_stats* rowp2 = a.rows + a.tid_begin + c0;
          if (sf) atomicAdd((unsigned long long*)&rowp2->covered_full, (unsigned long long)sf);
          if (sw) atomicAdd((unsigned long long*)&rowp2->covered_window, (unsigned long long)sw);
          if (sd) atomicAdd((unsigned long long*)&rowp2->sum_depth_window, (unsigned long long)sd);
          if (top) atomicMax(a.bin_hi + c0, top);
        }
      } else {
        cmb_contig_stats* rowp2 = a.rows + a.tid_begin + c;
        if (cov_full) atomicAdd((unsigned long long*)&rowp2->covered_full, (unsigned long long)cov_full);
        if (cov_win) atomicAdd((unsigned long long*)&rowp2->covered_window, (unsigned long long)cov_win);
        if (sum_win) atomicAdd((unsigned long long*)&rowp2->sum_depth_window, (unsigned long long)sum_win);
        if (bin_top) atomicMax(a.bin_hi + c, bin_top);
      }
    }
  }
  if (t == 0 && n_loaded) {
    atomicAdd(a.load_stats + 0, n_loaded);
    atomicAdd(a.load_stats + 1, n_dense);
  }
}
