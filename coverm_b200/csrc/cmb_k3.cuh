// K3: per-contig histogram finalisation, four contigs per WARP.
//
// K2 left the window depth histogram of contig c in bins[bin_base[c] .. bin_base[c] + bin_hi[c]] (one u32 count per depth),
// except depth 0, which it never adds: that count is the window length minus covered_window (the window positions of depth
// > 0, which K2 counts anyway).  The contig's lanes walk the bins in depth order, one per lane per step, with segmented
// scans:
//   * trimmed-mean `total` exactly as the reference's ascending walk (EST:598-642),
//   * S0 = sum n, S1 = sum x n, S2 = sum x^2 n (wrapping u64) and k = lowest depth -> variance sums (EST:790-805),
//   * optionally the (depth,count) pairs (CSR) for the host-side per-genome merge / coverage_histogram,
// and re-zeroes every bin it read and bin_hi[c], so that the pool is zero again for the next sample.
// Most contigs are shallow (a contig's depth is bounded by its read count): when all four of a warp's contigs have bin_hi < 8,
// each takes 8 lanes and one step; otherwise the whole warp walks them one after another, 32 bins per step.
#pragma once

constexpr uint32_t K3_WARPS = 8;
constexpr uint32_t K3_THREADS = K3_WARPS * 32;
constexpr uint32_t K3_GROUP = 8;                        // lanes per contig when the warp's four contigs are shallow
constexpr uint32_t K3_CONTIGS_PER_WARP = 32 / K3_GROUP;

struct K3Args {
  const uint32_t* len;
  cmb_contig_stats* rows;
  uint32_t tid_begin, n_local, excl;
  float trim_min, trim_max;
  const uint64_t* bin_base;
  uint32_t* bins;
  uint64_t pool_cap;
  uint32_t* bin_hi;
  cmb_hist_pair* pairs;
  unsigned long long* pair_count;
  uint64_t pair_capacity;
  uint32_t want_csr;
  uint32_t all_rows;  // gene mode: a gene is covered by reads that start before it, so "no record counted here" does not mean "empty"
  uint32_t* error_flags;
};

struct K3Contig {
  bool active;  // has a histogram to finalise
  uint32_t lc, hi, n_zero;
  uint32_t* bins;
  uint64_t min_index, max_index;
};

// K3 is latency-bound per contig (little work each): every per-contig value is requested at once, before any branch
__device__ __forceinline__ K3Contig k3_contig(const K3Args& a, uint32_t lc) {
  K3Contig c{false, lc, 0u, 0u, nullptr, 0ull, 0ull};
  if (lc >= a.n_local) return c;
  const cmb_contig_stats* row = a.rows + a.tid_begin + lc;
  const uint64_t pool_need = __ldg(a.bin_base + a.n_local), b_first = __ldg(a.bin_base + lc), b_end = __ldg(a.bin_base + lc + 1);
  const uint32_t hi = a.bin_hi[lc];  // K3 re-zeroes it: not a read-only load
  const uint32_t L = __ldg(a.len + lc);
  const uint64_t n_records = row->n_records, covered_window = row->covered_window;
  if (pool_need > a.pool_cap) return c;  // K2 added no bin (ERR_CAPACITY)
  if (b_end == b_first) return c;        // no window (EST:436-445), no bins
  // unseen contig: the host never consults its histogram, and with no read every depth is 0, so K2 added no bin
  if (n_records == 0 && !a.all_rows) return c;
  const uint64_t T = (uint64_t)L - 2ull * a.excl;
  const float Tf = __ull2float_rn(T);  // EST:591-592: f32 products, `as usize` saturating casts
  c.active = true;
  c.hi = hi;
  c.n_zero = (uint32_t)(T - covered_window);  // window positions at depth 0
  c.bins = a.bins + b_first;
  c.min_index = (uint64_t)floorf(__fmul_rn(a.trim_min, Tf));
  c.max_index = (uint64_t)ceilf(__fmul_rn(a.trim_max, Tf));
  return c;
}

// Walks contig c with the W lanes of its group (gl: lane in the group, gshift: the group's first lane).  All 32 lanes of the
// warp call it together and take the same number of steps; an inactive contig's lanes only take part in the shuffles.
template <uint32_t W>
__device__ __forceinline__ void k3_walk(const K3Args& a, const K3Contig& c, uint32_t gl, uint32_t gshift) {
  const uint32_t gmask = W == 32 ? FULL : (1u << (W % 32)) - 1;
  cmb_contig_stats* row = a.rows + a.tid_begin + c.lc;
  unsigned long long ltot = 0, l0 = 0, l1 = 0, l2 = 0;  // per-lane partial sums
  uint32_t n_pairs = 0, k = 0xffffffffu;                // k: lowest depth with a non-zero count
  unsigned long long pair_base = 0;
  const int n_rounds = a.want_csr ? 2 : 1;  // round 0: statistics (+ count the pairs); round 1: write the pairs
  for (int round = 0; round < n_rounds; ++round) {
    const bool last = round == n_rounds - 1;
    unsigned long long cum = 0;  // counts below the current step
    uint32_t written = 0;
    for (uint32_t b0 = 0; b0 <= c.hi; b0 += W) {
      const uint32_t b = b0 + gl;
      const uint32_t got = c.active && b <= c.hi ? c.bins[b] : 0u;
      if (last && got) c.bins[b] = 0;
      const uint32_t n = b == 0 ? c.n_zero : got;
      uint32_t incl = n;  // inclusive scan of the W bins (a contig holds < 2^31 bases: fits u32)
#pragma unroll
      for (uint32_t d = 1; d < W; d <<= 1) {
        const uint32_t o = __shfl_up_sync(FULL, incl, d, W);
        if (gl >= d) incl += o;
      }
      const uint32_t nzmask = (__ballot_sync(FULL, n != 0) >> gshift) & gmask;
      if (round == 0) {
        if (nzmask && k == 0xffffffffu) k = b0 + __ffs(nzmask) - 1;
        if (n) {
          const unsigned long long depth = b;
          const unsigned long long cprev = cum + (incl - n), ccur = cum + incl;
          unsigned long long w;
          if (ccur < c.min_index) w = 0;
          else if (cprev < c.min_index) w = ccur > c.max_index ? c.max_index - c.min_index + 1 : ccur - c.min_index + 1;
          else w = cprev > c.max_index ? 0 : (ccur > c.max_index ? c.max_index - cprev + 1 : (unsigned long long)n);
          ltot += w * depth;
          l0 += n;
          l1 += depth * n;
          l2 += depth * depth * n;
        }
        n_pairs += __popc(nzmask);
      } else if (n) {
        const unsigned long long idx = pair_base + written + __popc(nzmask & ((1u << gl) - 1));
        if (idx < a.pair_capacity) {
          cmb_hist_pair pr;
          pr.depth = b;
          pr.count = n;
          a.pairs[idx] = pr;
        }
      }
      written += __popc(nzmask);
      cum += __shfl_sync(FULL, incl, W - 1, W);
    }
    if (round == 0) {
#pragma unroll
      for (uint32_t d = W / 2; d > 0; d >>= 1) {
        ltot += __shfl_xor_sync(FULL, ltot, d, W);
        l0 += __shfl_xor_sync(FULL, l0, d, W);
        l1 += __shfl_xor_sync(FULL, l1, d, W);
        l2 += __shfl_xor_sync(FULL, l2, d, W);
      }
      // k unset: no count at all (cannot happen for a contig with a window); the row is left as it is and no pair is written
      if (gl == 0 && k != 0xffffffffu) {
        const unsigned long long kk = k, S0 = l0, S1 = l1, S2 = l2;
        row->trimmed_total = ltot;
        row->trim_min_index = c.min_index;
        row->trim_max_index = c.max_index;
        row->var_k = kk;
        row->var_ex = S1 - kk * S0;                     // sum (x-k) n    (mod 2^64, as the reference's usize)
        row->var_ex2 = S2 - 2 * kk * S1 + kk * kk * S0;  // sum (x-k)^2 n
        row->hist_count = n_pairs;
        if (a.want_csr) {
          pair_base = atomicAdd(a.pair_count, (unsigned long long)n_pairs);
          row->hist_offset = pair_base;
          if (pair_base + n_pairs > a.pair_capacity) atomicOr(a.error_flags, ERR_CAPACITY);
        }
      }
      pair_base = __shfl_sync(FULL, pair_base, 0, W);
    }
  }
  if (gl == 0 && c.active) a.bin_hi[c.lc] = 0;
}

__global__ void __launch_bounds__(K3_THREADS) k3_finalize(const K3Args a) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t first = (blockIdx.x * K3_WARPS + warp) * K3_CONTIGS_PER_WARP;
  if (first >= a.n_local) return;
  const uint32_t g = lane / K3_GROUP;
  const K3Contig c = k3_contig(a, first + g);
  if (__reduce_max_sync(FULL, c.active ? c.hi : 0u) < K3_GROUP) {
    k3_walk<K3_GROUP>(a, c, lane % K3_GROUP, g * K3_GROUP);
  } else {
    for (uint32_t j = 0; j < K3_CONTIGS_PER_WARP; ++j) {
      const K3Contig cj = k3_contig(a, first + j);
      if (cj.active) k3_walk<32>(a, cj, lane, 0);
    }
  }
}
