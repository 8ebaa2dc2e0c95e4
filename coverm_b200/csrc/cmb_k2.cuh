// K2: segmented prefix sum of the delta events + every O(L) reduction of EST::add_contig, one pass over the spans that hold
// events.
//
// Persistent warps: warp g of W (8 per CTA) reduces the 8192-element chunks g, g + W, g + 2W, ...  Which of a chunk's 256
// spans hold any event is known from the span occupancy bitmap K1 sets (8 words per chunk).  Depth is piecewise constant
// between events, so only those spans need work: a chunk's SLOTS are its occupied spans in order (all 256 spans when it has
// at least K2_DENSE_SPANS occupied ones), and slot j covers the positions from its span up to the next slot's span, the
// chunk's end for the last one (cmb_k2_slots.cuh).  The event-free stretch after a slot's last event has that event's depth,
// so it is closed as one run; positions past the slot's contig's end are padding or contigs without events so far (depth 0).
// The stretch before the first slot has the chunk's carry-in (K1b) as its depth in the chunk's first contig.
//
// Slots go 32 per round, one per lane.  A lane reads its slot's span from the chunk's slot -> span table (built when the warp
// enters the chunk), its contig from the chunk's contig table (contig mode; by bisection in global memory in gene mode and in
// chunks with more contigs than the table holds), and reads the span's 32 deltas (8 x LDS.128 through the 128-B swizzle), keeping their sum and the mask of
// non-zero positions.  The depth entering a slot is a segmented (by contig) warp scan of the slot totals, seeded with the
// previous round's last slot (the chunk's first contig at its carry-in for round 0); no CTA barrier is involved.  Covered
// bases, sum of depth and the depth histogram of the end-trimmed window are accumulated per run.  The histogram is a dense
// array of u32 counts per contig in global memory, bins[bin_base[c] + depth] (K1b laid it out: every window depth of c is at
// most its read count), so a run's count is one fire-and-forget RED; K3 reads the bins in depth order and re-zeroes them.
// Depth 0 is not added: K3 derives its count from the window length and covered_window.
//
// Loads (gene mode, from the arena): each warp has a ring of K2_STAGES buffers of 32 rows x 128 B laid out as a TMA box with
// the 128-B swizzle writes them.  A dense chunk's rounds are one 32-row TMA box each (completion on the stage's mbarrier); a sparse round copies its
// occupied rows with cp.async into rows 0..n-1, four whole 128-B lines per instruction.  The next round's rows, possibly of
// the next chunk, are requested before the current round is reduced.
//
// Contig mode (BUCKETS) reads no arena: K1 wrote the sample's events to a list and K1e bucketed them by bitmap word
// (cmb_k1.cuh), so a round's events are the contiguous bucket range of the words its slots lie in.  The fetch stage copies
// that range into the round's stage of bucket entries with cp.async (16-B units, up to K2_STAGE_CODES entries; a round with
// more reads the rest straight from global memory), and right before the reduction the warp adds each entry into the one row
// buffer in shared memory, at its slot's row (cmb_k2_slots.cuh, k2_round_events), with a shared-memory atomic.  The
// reduction reads the rows exactly as it reads an arena round, then re-zeroes the units that held an event.
#pragma once
#include "cmb_k2_slots.cuh"

struct K2Args {
  const uint32_t* off_span;
  const uint32_t* len;
  const uint32_t* chunk_first;
  const int32_t* carry_in;
  cmb_contig_stats* rows;
  uint32_t tid_begin, n_local, n_chunks, excl;
  int32_t* arena;               // gene mode (null in contig mode, whose tensor map is all zero)
  const uint32_t* word_off;     // contig mode: [n_chunks * 8 + 1] first bucket entry of each bitmap word (K1b)
  const uint16_t* buckets;      // contig mode: the events bucketed by word (K1e), 8 entries of padding at the end
  uint32_t* span_bits;   // [n_chunks * 8] span occupancy bitmap (K1); bit b of word w of a chunk = its span 32 w + b
  uint32_t* load_stats;  // [0] += spans loaded, [1] += chunks loaded whole, [2] += bucket entries read (CMB_PIPELINE_STATS)
  const uint64_t* bin_base;  // [n_local + 1] first bin of each contig (K1b); bin_base[n_local] = bins needed
  uint32_t* bins;            // the bin pool: pool_cap u32 counts, zero outside a sample
  uint64_t pool_cap;
  uint32_t* bin_hi;          // [n_local] highest depth added per contig (atomicMax)
  uint32_t* error_flags;
};

// A chunk with at least this many non-empty spans (of 256) is reduced whole, all 256 spans as slots (gene mode: loaded 32 rows
// per TMA box); sparser chunks only their occupied spans.
// On an H100 80GB HBM3 at 400 W, K2 time moved by under 2 % for thresholds from 96 to 257 (never whole) on both `bench.py
// --config 2` and `--config ns` (DESIGN.md §4, K2): row copies are not what limits K2 there.  160 sends chunks above ~60 %
// occupancy down the TMA path.
#ifndef CMB_K2_DENSE_SPANS
#define CMB_K2_DENSE_SPANS 160
#endif
constexpr uint32_t K2_DENSE_SPANS = CMB_K2_DENSE_SPANS;
static_assert(K2_STAGES >= 2, "a round's rows are requested one round before it is reduced");
static_assert(K2_CHUNK_SPANS == CHUNK_SPANS && K2_WARPS == 8, "a chunk is 8 bitmap words of 32 spans");

constexpr uint32_t K2_ROUND = 32;                     // slots per round, one per lane
constexpr uint32_t K2_BUF_BYTES = K2_ROUND * 128;     // one round's rows: 4 KB, whole 1024-B swizzle atoms
constexpr uint32_t K2_BOX_ROWS = K2_ROUND;            // rows of the TMA box (cmb_set_reference encodes it)
constexpr uint32_t K2_STAGE_CODES = 1024;             // bucket entries one stage holds (contig mode): 2 KB
constexpr uint32_t K2_STAGE_BYTES = K2_STAGE_CODES * 2;
// a warp's buffers: a ring of K2_STAGES round buffers (arena), or one round buffer and K2_STAGES stages of bucket entries
template <bool BUCKETS>
__host__ __device__ constexpr uint32_t k2_warp_bytes() { return BUCKETS ? K2_BUF_BYTES + K2_STAGES * K2_STAGE_BYTES : K2_STAGES * K2_BUF_BYTES; }
// Contig mode: the contigs of a chunk, [chunk_first[k], chunk_first[k + 1]], when there are at most K2_CHUNK_CONTIGS of them:
// entry t is contig chunk_first[k] + t.  A contig is at least one span, so a chunk with more has contigs shorter than ~500
// bases; such chunks, and gene mode (where the table pushed K2 into spills), find their contigs in global memory.
constexpr uint32_t K2_CHUNK_CONTIGS = 16;
struct K2ChunkContigs {
  uint64_t bin[K2_CHUNK_CONTIGS + 1];  // bin_base (HIST only)
  uint32_t start[K2_CHUNK_CONTIGS];    // off_span
  uint32_t len[K2_CHUNK_CONTIGS];
};
// A warp's per-chunk tables: the contigs of the chunk being reduced, and the slot -> span tables (k2_span_table_lane) of the
// fetch cursor's chunk [0] and of the one being reduced [1].
struct K2WarpTables {
  K2ChunkContigs ct;
  uint8_t span[2][K2_CHUNK_SPANS];
  uint8_t pre[2][8];
};
static_assert(sizeof(K2WarpTables) % 8 == 0, "the contig tables hold u64 bins");
constexpr uint32_t K2_SMEM_MISC = K2_WARPS * K2_STAGES * 8 /*an mbarrier per (warp, stage)*/ +
                                  K2_WARPS * 128 /*a chunk's bitmap words and bucket offsets*/ +
                                  K2_WARPS * sizeof(K2WarpTables);
template <bool BUCKETS>
__host__ __device__ constexpr uint32_t k2_smem_bytes() { return K2_WARPS * k2_warp_bytes<BUCKETS>() + K2_SMEM_MISC; }
static_assert(k2_warp_bytes<true>() % 1024 == 0 && k2_warp_bytes<false>() % 1024 == 0, "round buffers are whole swizzle atoms");

__device__ __forceinline__ uint32_t k2_rounds(uint32_t pop, bool dense) { return dense ? CHUNK_SPANS / K2_ROUND : (pop + K2_ROUND - 1) / K2_ROUND; }

template <bool HIST, bool CLEAN, bool BUCKETS>
__global__ void __launch_bounds__(K2_THREADS, CMB_K2_MINBLOCKS) k2_scan_reduce(const __grid_constant__ CUtensorMap tmap, const K2Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];  // the buffers need the 1024 B swizzle-atom alignment
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr uint32_t RING = K2_WARPS * k2_warp_bytes<BUCKETS>();
  uint8_t* ring = smem + warp * k2_warp_bytes<BUCKETS>();
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + RING) + warp * K2_STAGES;
  // the 8 bitmap words of the chunk being reduced and (BUCKETS) the 9 bucket offsets of its words (in shared memory rather
  // than registers: K2 runs at the 80-register cap); the fetch cursor needs only its chunk's slot -> span table
  uint32_t* words = reinterpret_cast<uint32_t*>(smem + RING + K2_WARPS * K2_STAGES * 8) + warp * 32;
  uint32_t(&w)[8] = *reinterpret_cast<uint32_t(*)[8]>(words + 8);
  uint32_t* wo = words + 16;
  K2WarpTables& tb = reinterpret_cast<K2WarpTables*>(smem + RING + K2_WARPS * K2_STAGES * 8 + K2_WARPS * 128)[warp];

  // The pool is sized before the launch from a bound of bin_base[n_local]; when it is still too small (cmb_grow_buffers
  // then grows it to exactly that) no bin is added and K3 reads none.
  const bool hist = HIST && __ldg(a.bin_base + a.n_local) <= a.pool_cap;
  if (HIST && !hist && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(a.error_flags, ERR_CAPACITY);

  const uint32_t W = gridDim.x * K2_WARPS, g = blockIdx.x * K2_WARPS + warp;
  // word `lane` (lanes 0..7) of chunk ck's span bitmap
  auto load_word = [&](uint32_t ck) -> uint32_t { return ck < a.n_chunks && lane < K2_WARPS ? a.span_bits[ck * K2_WARPS + lane] : 0u; };
  // BUCKETS: the first bucket entry of word `lane` (lanes 0..8, 8 = the next chunk's first) of chunk ck
  auto load_off = [&](uint32_t ck) -> uint32_t { return BUCKETS && ck < a.n_chunks && lane <= K2_WARPS ? __ldg(a.word_off + ck * K2_WARPS + lane) : 0u; };
  // lanes 0..7 put their words of a chunk into `to` for the whole warp (and lanes 0..8 their bucket offsets into `to_off`),
  // and the warp writes the chunk's slot -> span table t; returns the chunk's popcount
  auto spread = [&](uint32_t word, uint32_t* to, uint32_t t, uint32_t off = 0, uint32_t* to_off = nullptr) -> uint32_t {
    __syncwarp();  // every lane is done with the previous chunk's words and table
    if (to && lane < K2_WARPS) to[lane] = word;
    if (to_off && lane <= K2_WARPS) to_off[lane] = off;
    const uint32_t pop = __reduce_add_sync(FULL, __popc(word));
    const uint32_t mw = pop >= K2_DENSE_SPANS && lane < K2_WARPS ? ~0u : word;  // a dense chunk's slots are all its spans
    uint32_t before = __popc(mw);  // lanes 0..7: slots of the words up to `lane`, then before it
#pragma unroll
    for (uint32_t d = 1; d < K2_WARPS; d <<= 1) {
      const uint32_t o = __shfl_up_sync(FULL, before, d);
      if (lane >= d) before += o;
    }
    before -= __popc(mw);
    if (lane < K2_WARPS) tb.pre[t][lane] = (uint8_t)before;
    k2_span_table_lane(__shfl_sync(FULL, mw, lane / 4), __shfl_sync(FULL, before, lane / 4), lane, tb.span[t]);
    __syncwarp();
    return pop;
  };

  if (lane == 0) {
    for (uint32_t s = 0; s < K2_STAGES; ++s) mbar_init(smem_u32(bars + s), 1);
    fence_barrier_init();
  }
  if (BUCKETS)  // the round buffer starts at zero; every round leaves it so
    for (uint32_t u = lane; u < K2_BUF_BYTES / 16; u += 32) reinterpret_cast<int4*>(ring)[u] = make_int4(0, 0, 0, 0);
  __syncwarp();

  // ---- the fetch cursor: round fr of chunk fk is the next one whose rows are requested.  It runs K2_STAGES - 1
  //      rounds ahead of the reduction, through the same chunks and rounds, skipping the chunks that have none.
  uint32_t fk = g, fr = 0, fns = 0;  // fns: the slots of chunk fk (CHUNK_SPANS when dense, so dense = fns >= K2_DENSE_SPANS)
  uint32_t f_word = load_word(fk);      // bitmap word of chunk fk, requested a chunk ahead
  uint32_t f_off = load_off(fk), fo = 0;  // BUCKETS: bucket offsets of chunk fk, requested a chunk ahead; of the cursor's chunk
  uint32_t n_loaded = 0, n_dense = 0, n_events = 0;  // what this warp fetched (load_stats)
  auto f_enter = [&]() {
    for (; fk < a.n_chunks; fk += W) {
      const uint32_t word = f_word;
      f_word = load_word(fk + W);
      fo = f_off;
      f_off = load_off(fk + W);
      const uint32_t pop = spread(word, nullptr, 0);
      fns = pop >= K2_DENSE_SPANS ? CHUNK_SPANS : pop;
      fr = 0;
      if (fns) {
        n_loaded += fns;
        n_dense += pop >= K2_DENSE_SPANS;
        return;
      }
    }
  };
  // Request the fetch cursor's round, the warp's fi-th, into stage fi % K2_STAGES and advance the cursor.  Every lane commits
  // one cp.async group per call (empty past the last round), so that cp.async.wait_group counts the same way on every lane.
  auto fill = [&](uint32_t fi) {
    if (fk < a.n_chunks) {
      uint8_t* buf = ring + (fi % K2_STAGES) * K2_BUF_BYTES;
      const uint32_t bar = smem_u32(bars + fi % K2_STAGES);
      if constexpr (BUCKETS) {  // contig mode has no arena and no tensor map: only the gene-mode branches name them
        // the round's bucket entries, 16-B units from the one holding its first entry, as many as the stage holds
        uint32_t wf, wl;
        k2_round_words(tb.span[0], fns, fr, wf, wl);
        const uint32_t b0 = __shfl_sync(FULL, fo, wf), b1 = __shfl_sync(FULL, fo, wl + 1);
        const uint32_t base = b0 & ~7u, units = min((b1 - base + 7) / 8, K2_STAGE_CODES / 8);
        uint8_t* stg = ring + K2_BUF_BYTES + (fi % K2_STAGES) * K2_STAGE_BYTES;
        const int4* src = reinterpret_cast<const int4*>(a.buckets + base);
        for (uint32_t u = lane; u < units; u += 32) cp_async_16(smem_u32(stg + u * 16), src + u);
        n_events += b1 - b0;
      } else if (fns >= K2_DENSE_SPANS) {
        if (lane == 0) {
          fence_proxy_async_smem();  // the stage's earlier reads and cp.async writes (ordered by __syncwarp) come first
          mbar_arrive_expect_tx(bar, K2_BUF_BYTES);
          tma_load_2d(smem_u32(buf), &tmap, 0, (int32_t)(fk * CHUNK_ROWS + fr * K2_BOX_ROWS), bar);
        }
      } else {
        // lanes 8q..8q+7 take the eight 16-byte units of row r0 + q, so every instruction moves four whole 128-byte lines;
        // unit u of row r lands at r * 128 + (u ^ (r & 7)) * 16, where the TMA box would put it
        const uint32_t n = min(K2_ROUND, fns - fr * K2_ROUND);
        const uint32_t jf = fr * K2_ROUND + lane, sp = jf < fns ? tb.span[0][jf] : 0u;
        const uint32_t q = lane >> 3, unit = lane & 7;
        const int4* src = reinterpret_cast<const int4*>(a.arena + (uint64_t)fk * CHUNK) + unit;
        for (uint32_t r0 = 0; r0 < n; r0 += 4) {
          const uint32_t row = r0 + q;
          const uint32_t rsp = __shfl_sync(FULL, sp, row & 31);
          if (row < n) cp_async_16(smem_u32(buf + row * 128 + ((unit ^ (row & 7)) << 4)), src + rsp * (SPAN / 4));
        }
        if (lane == 0) mbar_arrive(bar);  // keeps the barrier's phase in step with the TMA stages
      }
      if (++fr == (fns + K2_ROUND - 1) / K2_ROUND) {
        fk += W;
        f_enter();
      }
    }
    cp_async_commit();
  };
  f_enter();
  for (uint32_t p = 0; p + 1 < K2_STAGES; ++p) fill(p);

  const uint32_t E = a.excl;
  // one contig's share of a warp's runs: the REDs into its row and its bin_hi
  auto flush = [&](uint32_t c, uint32_t sf, uint32_t sw, uint64_t sd, uint32_t top) {
    cmb_contig_stats* rowp = a.rows + a.tid_begin + c;
    if (sf) atomicAdd((unsigned long long*)&rowp->covered_full, (unsigned long long)sf);
    if (sw) atomicAdd((unsigned long long*)&rowp->covered_window, (unsigned long long)sw);
    if (sd) atomicAdd((unsigned long long*)&rowp->sum_depth_window, (unsigned long long)sd);
    if (top) atomicMax(a.bin_hi + c, top);
  };
  // a run's window count into bin `depth` of the contig whose bins are [bin0, bin1)
  auto bin_add = [&](uint64_t bin0, uint64_t bin1, int depth, uint32_t cnt, uint32_t& top) {
    // 0 <= depth <= bound = bin1 - bin0 - 1 for a consistent arena (every -1 follows its +1 within the contig, and a record
    // adds at most 1 at any position)
    if (depth < 0 || (uint64_t)depth >= bin1 - bin0) {
      atomicOr(a.error_flags, ERR_INTERNAL);
      return;
    }
    atomicAdd(a.bins + bin0 + (uint32_t)depth, cnt);
    top = max(top, (uint32_t)depth);
  };

  uint32_t c_word = load_word(g), c_off = load_off(g);  // the next chunk's bitmap word and metadata, requested a chunk ahead
  uint32_t n_cf = 0, n_cl = 0;
  int n_cin = 0;
  if (g < a.n_chunks) {
    n_cf = __ldg(a.chunk_first + g);
    n_cl = __ldg(a.chunk_first + g + 1);
    n_cin = __ldg(a.carry_in + g);
  }
  uint32_t i = 0;  // rounds reduced by this warp
  for (uint32_t k = g; k < a.n_chunks; k += W) {
    const uint32_t word = c_word, off = c_off, cf = n_cf, cl = n_cl;
    const int cin = n_cin;
    c_word = load_word(k + W);
    c_off = load_off(k + W);
    if (k + W < a.n_chunks) {
      n_cf = __ldg(a.chunk_first + k + W);
      n_cl = __ldg(a.chunk_first + k + W + 1);
      n_cin = __ldg(a.carry_in + k + W);
    }
    // ---- the chunk's contigs cf..cl into the warp's table, entry `lane` (bins: lanes 0..cl - cf + 1), when they fit
    const bool tabled = BUCKETS && cl - cf < K2_CHUNK_CONTIGS;
    uint32_t t_start = 0, t_len = 0;
    uint64_t t_bin = 0;
    if (tabled && lane <= cl - cf) {
      t_start = __ldg(a.off_span + cf + lane);
      t_len = __ldg(a.len + cf + lane);
    }
    if (HIST && tabled && lane <= cl - cf + 1) t_bin = __ldg(a.bin_base + cf + lane);
    const uint32_t pop = spread(word, w, 1, off, BUCKETS ? wo : nullptr);
    if (tabled && lane <= cl - cf) {
      tb.ct.start[lane] = t_start;
      tb.ct.len[lane] = t_len;
    }
    if (HIST && tabled && lane <= cl - cf + 1) tb.ct.bin[lane] = t_bin;
    __syncwarp();
    const bool dense = pop >= K2_DENSE_SPANS;
    const uint32_t nr = k2_rounds(pop, dense), nslots = dense ? CHUNK_SPANS : pop;
    const uint32_t span0 = k * CHUNK_SPANS;
    uint32_t pc = cf, c_first = 0xffffffffu;  // contig of the previous round's last slot; of the chunk's first slot
    int pd = cin;                             // depth leaving the previous round's last slot
    for (uint32_t r = 0; r < nr; ++r, ++i) {
      __syncwarp();  // every lane is done with the stage that the fill below overwrites
      fill(i + K2_STAGES - 1);
      const uint32_t j = r * K2_ROUND + lane;
      const bool valid = j < nslots;
      const uint32_t s = valid ? tb.span[1][j] : CHUNK_SPANS, sn = j + 1 < nslots ? tb.span[1][j + 1] : CHUNK_SPANS;
      // ---- the slot's contig, start, window and bins: from the chunk's table, else by bisection in global memory (no tile
      //      data needed: those loads fly while the rows arrive)
      uint32_t c = 0xffffffffu, cstart = 0;
      K2Win win{0u, 0u, 0u};
      uint64_t bin0 = 0, bin1 = 0;
      if (valid && tabled) {
        uint32_t t = 0;  // the last entry that starts at or before the slot's span (entry 0 starts before the chunk)
#pragma unroll
        for (uint32_t h = K2_CHUNK_CONTIGS / 2; h; h >>= 1)
          if (t + h <= cl - cf && tb.ct.start[t + h] <= span0 + s) t += h;
        c = cf + t;
        cstart = tb.ct.start[t];
        win = k2_window(tb.ct.len[t], E);
        if (hist) {
          bin0 = tb.ct.bin[t];
          bin1 = tb.ct.bin[t + 1];
        }
      } else if (valid) {
        uint32_t lo = cf, hi = cl;
        while (lo < hi) {
          const uint32_t mid = (lo + hi + 1) >> 1;
          if (__ldg(a.off_span + mid) <= span0 + s) lo = mid;
          else hi = mid - 1;
        }
        c = lo;
        cstart = __ldg(a.off_span + c);
        win = k2_window(__ldg(a.len + c), E);
        if (hist) {
          bin0 = __ldg(a.bin_base + c);
          bin1 = __ldg(a.bin_base + c + 1);
        }
      }
      const uint32_t st = i % K2_STAGES;
      if (!BUCKETS) mbar_wait(smem_u32(bars + st), (i / K2_STAGES) & 1);
      cp_async_wait<K2_STAGES - 1>();  // this lane's copies into stage st (only the fill above may still be in flight)
      __syncwarp();                    // ... and those of the other lanes
      uint8_t* rows = BUCKETS ? ring : ring + st * K2_BUF_BYTES;
      if (BUCKETS) {
        // ---- the round's rows from its bucket entries: staged ones from the stage, the rest from global memory
        // the words of its first and last slot (k2_round_words, from the spans the lanes already hold)
        const uint32_t wf = __shfl_sync(FULL, s, 0) / 32, wl = __shfl_sync(FULL, s, min(nslots - r * K2_ROUND, K2_ROUND) - 1) / 32;
        const uint32_t base = wo[wf] & ~7u;
        const uint16_t* stg = reinterpret_cast<const uint16_t*>(ring + K2_BUF_BYTES + st * K2_STAGE_BYTES);
        k2_round_events(
            w, tb.pre[1], wo, dense, r, wf, wl, lane, 32,
            [&](uint32_t p) { return p - base < K2_STAGE_CODES ? (uint32_t)stg[p - base] : (uint32_t)__ldg(a.buckets + p); },
            [&](uint32_t rw, uint32_t e, int d) {
              atomicAdd(reinterpret_cast<int*>(rows + rw * 128 + (((e >> 2) ^ (rw & 7)) << 4) + ((e & 3) << 2)), d);
            });
        __syncwarp();
      }
      // ---- the slot's 32 deltas (row `lane`): only their sum and the mask of non-zero positions stay in registers
      uint8_t* row = rows + lane * 128;
      int total = 0;
      uint32_t ev = 0;
      if (valid) {
#pragma unroll
        for (uint32_t u = 0; u < SPAN / 4; ++u) {
          const int4 v = *reinterpret_cast<const int4*>(row + ((u ^ (lane & 7)) << 4));
          const uint32_t e4 = (v.x != 0 ? 1u : 0u) | (v.y != 0 ? 2u : 0u) | (v.z != 0 ? 4u : 0u) | (v.w != 0 ? 8u : 0u);
          total += (v.x + v.y) + (v.z + v.w);
          ev |= e4 << (4 * u);
          if constexpr (!BUCKETS && CLEAN)  // gene mode: re-zero only the arena's 16 B units that hold an event
            if (e4) reinterpret_cast<int4*>(a.arena + (uint64_t)(span0 + s) * SPAN)[u] = make_int4(0, 0, 0, 0);
        }
      }
      // ---- depth entering the slot: segmented (by contig) exclusive scan of the slot totals, seeded from the previous slot
      int incl = total;
#pragma unroll
      for (uint32_t d = 1; d < 32; d <<= 1) {
        const int ov = __shfl_up_sync(FULL, incl, d);
        const uint32_t oc = __shfl_up_sync(FULL, c, d);
        if (lane >= d && oc == c) incl += ov;
      }
      const int depth = incl - total + (c == pc ? pd : 0);
      // ---- the slot's runs; the chunk's first slot also takes the chunk's head when it is in the head's contig
      const uint32_t rel = (span0 + s - cstart) * SPAN;
      const uint32_t from = j == 0 && c == cf ? (span0 - cstart) * SPAN : rel;
      const uint32_t to = rel + (sn - s) * SPAN;
      K2Acc acc{0u, 0u, 0ull};
      uint32_t top = 0;
      int out = 0;
      if (valid)
        out = k2_slot_runs(
            acc, win, depth, ev, rel, from, to,
            [&](uint32_t e) { return *reinterpret_cast<const int*>(row + (((e >> 2) ^ (lane & 7)) << 4) + ((e & 3) << 2)); },
            [&](int d, uint32_t n) {
              if (hist) bin_add(bin0, bin1, d, n, top);
            });
      if (BUCKETS)  // the row buffer is zero again for the next round
#pragma unroll
        for (uint32_t u = 0; u < SPAN / 4; ++u)
          if (ev >> (4 * u) & 15u) *reinterpret_cast<int4*>(row + ((u ^ (lane & 7)) << 4)) = make_int4(0, 0, 0, 0);
      pc = __shfl_sync(FULL, c, 31);
      pd = __shfl_sync(FULL, out, 31);
      if (r == 0) c_first = __shfl_sync(FULL, c, 0);
      // ---- per-contig REDs: lanes are in contig order; the first lane of each contig's lanes adds their sums
      uint32_t sf = acc.cov_full, sw = acc.cov_win;
      uint64_t sd = acc.sum_win;
#pragma unroll
      for (uint32_t d = 1; d < 32; d <<= 1) {
        const uint32_t of = __shfl_down_sync(FULL, sf, d), ow = __shfl_down_sync(FULL, sw, d);
        const uint64_t od = __shfl_down_sync(FULL, sd, d);
        const uint32_t ot = HIST ? __shfl_down_sync(FULL, top, d) : 0u;
        const uint32_t oc = __shfl_down_sync(FULL, c, d);
        if (lane + d < 32 && oc == c) {
          sf += of;
          sw += ow;
          sd += od;
          top = max(top, ot);
        }
      }
      const uint32_t prev_c = __shfl_up_sync(FULL, c, 1);
      if (valid && (lane == 0 || prev_c != c)) flush(c, sf, sw, sd, top);
    }
    // ---- the chunk's head when no slot took it: from the chunk start to the first slot (the whole chunk if it has none),
    //      at the carry-in, in the chunk's first contig
    if (lane == 0 && cin != 0 && c_first != cf) {
      const uint32_t cstart = tabled ? tb.ct.start[0] : __ldg(a.off_span + cf);
      const K2Win win = k2_window(tabled ? tb.ct.len[0] : __ldg(a.len + cf), E);
      const uint32_t s0 = nslots ? tb.span[1][0] : CHUNK_SPANS;
      K2Acc acc{0u, 0u, 0ull};
      uint32_t top = 0;
      const uint32_t nw = k2_close_run(acc, win, cin, (span0 - cstart) * SPAN, (span0 + s0 - cstart) * SPAN);
      if (hist && nw)
        bin_add(tabled ? tb.ct.bin[0] : __ldg(a.bin_base + cf), tabled ? tb.ct.bin[1] : __ldg(a.bin_base + cf + 1), cin, nw, top);
      flush(cf, acc.cov_full, acc.cov_win, acc.sum_win, top);
    }
    if (CLEAN && word) a.span_bits[k * K2_WARPS + lane] = 0;  // lanes 0..7 (the others hold no word)
  }
  if (lane == 0 && n_loaded) {
    atomicAdd(a.load_stats + 0, n_loaded);
    atomicAdd(a.load_stats + 1, n_dense);
    if (BUCKETS) atomicAdd(a.load_stats + 2, n_events);
  }
}
