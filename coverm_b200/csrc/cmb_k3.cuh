// K3: per-contig histogram finalisation, one WARP per contig.
//
// K2 left the window depth histogram of contig c in bins[bin_base[c] .. bin_base[c] + bin_hi[c]] (one u32 count per depth),
// except depth 0, which it never adds: that count is the window length minus covered_window (the window positions of depth
// > 0, which K2 counts anyway).  The warp walks the bins in depth order, 32 per step, with warp scans:
//   * trimmed-mean `total` exactly as the reference's ascending walk (EST:598-642),
//   * S0 = sum n, S1 = sum x n, S2 = sum x^2 n (wrapping u64) and k = lowest depth -> variance sums (EST:790-805),
//   * optionally the (depth,count) pairs (CSR) for the host-side per-genome merge / coverage_histogram,
// and re-zeroes every bin it read and bin_hi[c], so that the pool is zero again for the next sample.
#pragma once

constexpr uint32_t K3_WARPS = 8;
constexpr uint32_t K3_THREADS = K3_WARPS * 32;

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

__global__ void __launch_bounds__(K3_THREADS) k3_finalize(const K3Args a) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lc = blockIdx.x * K3_WARPS + warp;
  if (lc >= a.n_local) return;
  // K3 is latency-bound (a warp per contig, little work each): every per-contig value is requested at once, before any branch
  cmb_contig_stats* row = a.rows + a.tid_begin + lc;
  const uint64_t pool_need = __ldg(a.bin_base + a.n_local), b_first = __ldg(a.bin_base + lc), b_end = __ldg(a.bin_base + lc + 1);
  const uint32_t hi = a.bin_hi[lc];  // K3 re-zeroes it below: not a read-only load
  const uint32_t L = __ldg(a.len + lc);
  const uint64_t n_records = row->n_records, covered_window = row->covered_window;
  if (pool_need > a.pool_cap) return;  // K2 added no bin (ERR_CAPACITY)
  if (b_end == b_first) return;        // no window (EST:436-445), no bins
  // unseen contig: the host never consults its histogram, and with no read every depth is 0, so K2 added no bin
  if (n_records == 0 && !a.all_rows) return;
  uint32_t* bins = a.bins + b_first;
  const uint64_t T = (uint64_t)L - 2ull * a.excl;
  const uint32_t n_zero = (uint32_t)(T - covered_window);  // window positions at depth 0
  const float Tf = __ull2float_rn(T);  // EST:591-592: f32 products, `as usize` saturating casts
  const uint64_t min_index = (uint64_t)floorf(__fmul_rn(a.trim_min, Tf));
  const uint64_t max_index = (uint64_t)ceilf(__fmul_rn(a.trim_max, Tf));

  unsigned long long ltot = 0, l0 = 0, l1 = 0, l2 = 0;  // per-lane partial sums
  uint32_t n_pairs = 0, k = 0xffffffffu;                // k: lowest depth with a non-zero count
  unsigned long long pair_base = 0;
  const int n_rounds = a.want_csr ? 2 : 1;  // round 0: statistics (+ count the pairs); round 1: write the pairs
  for (int round = 0; round < n_rounds; ++round) {
    const bool last = round == n_rounds - 1;
    unsigned long long cum = 0;  // counts below the current step
    uint32_t written = 0;
    for (uint32_t b0 = 0; b0 <= hi; b0 += 32) {
      const uint32_t b = b0 + lane;
      const uint32_t got = b <= hi ? bins[b] : 0u;
      if (last && got) bins[b] = 0;
      const uint32_t n = b == 0 ? n_zero : got;
      uint32_t incl = n;  // inclusive scan of the 32 bins (a contig holds < 2^31 bases: fits u32)
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(FULL, incl, d);
        if ((int)lane >= d) incl += o;
      }
      const uint32_t nzmask = __ballot_sync(FULL, n != 0);
      if (round == 0) {
        if (nzmask && k == 0xffffffffu) k = b0 + __ffs(nzmask) - 1;
        if (n) {
          const unsigned long long depth = b;
          const unsigned long long cprev = cum + (incl - n), ccur = cum + incl;
          unsigned long long w;
          if (ccur < min_index) w = 0;
          else if (cprev < min_index) w = ccur > max_index ? max_index - min_index + 1 : ccur - min_index + 1;
          else w = cprev > max_index ? 0 : (ccur > max_index ? max_index - cprev + 1 : (unsigned long long)n);
          ltot += w * depth;
          l0 += n;
          l1 += depth * n;
          l2 += depth * depth * n;
        }
        n_pairs += __popc(nzmask);
      } else if (n) {
        const unsigned long long idx = pair_base + written + __popc(nzmask & ((1u << lane) - 1));
        if (idx < a.pair_capacity) {
          cmb_hist_pair pr;
          pr.depth = b;
          pr.count = n;
          a.pairs[idx] = pr;
        }
      }
      written += __popc(nzmask);
      cum += __shfl_sync(FULL, incl, 31);
    }
    if (round == 0) {
      if (k == 0xffffffffu) break;  // no count at all (cannot happen for a contig with a window)
      const unsigned long long total = warp_sum_u64(ltot), S0 = warp_sum_u64(l0), S1 = warp_sum_u64(l1), S2 = warp_sum_u64(l2);
      if (lane == 0) {
        const unsigned long long kk = k;
        row->trimmed_total = total;
        row->trim_min_index = min_index;
        row->trim_max_index = max_index;
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
      pair_base = __shfl_sync(FULL, pair_base, 0);
    }
  }
  if (lane == 0) a.bin_hi[lc] = 0;
}
