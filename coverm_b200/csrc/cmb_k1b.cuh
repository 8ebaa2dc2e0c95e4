// K1b: running depth at the first element of every chunk (carry_in), from the per-chunk tail sums K1 accumulated, and the
// layout of the histogram bin pool (bin_base).
//
//   x_0 = 0;   x_{k+1} = mid_k ? ((same_k ? x_k : 0) + tail_sum[k]) : 0
//   mid_k  = chunk k+1 starts in the middle of a contig,  same_k = that contig also owns the first span of chunk k.
// A segmented scan over ~L/8192 elements, done in two tiny launches: k1b_local scans 1024-chunk blocks (thread = 4
// consecutive chunks, warp shuffles, one shared-memory step) and leaves a "needs the block carry" flag in tail_sum;
// k1b_apply folds in the block carries.  With the carries known up front K2 needs no inter-CTA look-back at all.
//
// The blocks after the chunk blocks (K1bBins) scan the segments instead: bin_base[c] = sum over c' < c of the bins of c',
// (bound[c'] + 1) for a segment with an end-trimmed window (2E < L) and 0 otherwise, bin_base[n_seg] = the pool size.  bound
// is the number of records that add an event to the segment (contig mode: rows[c].n_records; gene mode: gene_bound[c],
// counted by K1).  A record's aligned blocks are disjoint, so it adds at most 1 to the depth at any position: every window
// depth of c lies in [0, bound[c]] and K2 can add it straight into bin bin_base[c] + depth.
#pragma once

constexpr uint32_t K1B_THREADS = 256;
constexpr uint32_t K1B_PER = 4;
constexpr uint32_t K1B_BLOCK = K1B_THREADS * K1B_PER;  // chunks (or segments) per block

struct K1bBins {
  const uint32_t* len;            // [n_seg]
  const cmb_contig_stats* rows;   // rows of the local segments (contig mode)
  const uint32_t* gene_bound;     // [n_seg] gene mode, else NULL
  uint32_t n_seg, excl;
  uint64_t* bin_base;             // [n_seg + 1]
  uint64_t* block_sum;            // [n_blocks]: bins of each block of K1B_BLOCK segments
  uint32_t n_blocks;              // 0 = no histogram wanted
};

// Contig mode: the exclusive scan of K1's per-bitmap-word event counts, word_off[w] = events of the words before w (the
// first of w's bucket, K1e), word_off[n_words] = events of the sample.  The host keeps a sample under 2^32 events.
struct K1bWords {
  const uint32_t* count;  // [n_words]
  uint32_t* off;          // [n_words + 1]
  uint32_t* block_sum;    // [n_blocks]: events of each block of K1B_BLOCK words
  uint32_t n_words, n_blocks;  // n_blocks = 0: gene mode, no scan
};

// Word block `b` of k1b_local: local exclusive scan of its K1B_BLOCK counts (entry n_words gets the total) and its sum.
__device__ __forceinline__ void k1b_words_local(const K1bWords& g, uint32_t b) {
  __shared__ uint32_t s_w[K1B_THREADS / 32];
  const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint32_t i0 = b * K1B_BLOCK + t * K1B_PER;
  uint32_t n[K1B_PER], sum = 0;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    n[i] = i0 + i < g.n_words ? g.count[i0 + i] : 0u;
    sum += n[i];
  }
  uint32_t incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(FULL, incl, d);
    if ((int)lane >= d) incl += o;
  }
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  uint32_t x = incl - sum;
  for (uint32_t w = 0; w < warp; ++w) x += s_w[w];
  if (t == K1B_THREADS - 1) g.block_sum[b] = x + sum;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    if (i0 + i <= g.n_words) g.off[i0 + i] = x;
    x += n[i];
  }
}

// Word block `b` of k1b_apply: adds the events of the blocks before it.
__device__ __forceinline__ void k1b_words_apply(const K1bWords& g, uint32_t b) {
  __shared__ uint32_t s_w[K1B_THREADS / 32];
  const uint32_t t = threadIdx.x;
  uint32_t acc = 0;
  for (uint32_t j = t; j < b; j += K1B_THREADS) acc += g.block_sum[j];
  acc = __reduce_add_sync(FULL, acc);
  if ((t & 31) == 0) s_w[t >> 5] = acc;
  __syncthreads();
  uint32_t before = 0;
#pragma unroll
  for (uint32_t w = 0; w < K1B_THREADS / 32; ++w) before += s_w[w];
  if (before == 0) return;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    const uint32_t s = b * K1B_BLOCK + t * K1B_PER + i;
    if (s <= g.n_words) g.off[s] += before;
  }
}

struct K1bElem {
  bool reset;
  int add;
};
__device__ __forceinline__ K1bElem k1b_elem(uint32_t k, uint32_t n_chunks, const int32_t* tail_sum, const uint32_t* chunk_first,
                                           const uint32_t* off_span) {
  K1bElem e;
  if (k + 1 >= n_chunks) {
    e.reset = true;
    e.add = 0;
    return e;
  }
  const uint32_t cn = chunk_first[k + 1];
  const bool mid = off_span[cn] < (k + 1) * CHUNK_SPANS;
  const bool same = chunk_first[k] == cn;
  e.reset = !(mid && same);
  e.add = mid ? tail_sum[k] : 0;
  return e;
}

// Bin block `b` of k1b_local: local exclusive scan of the bins of its K1B_BLOCK segments (entry n_seg, with no bins, gets the
// total) and the block's sum.
__device__ __forceinline__ void k1b_bins_local(const K1bBins& g, uint32_t b) {
  __shared__ unsigned long long s_w[K1B_THREADS / 32];
  const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint32_t i0 = b * K1B_BLOCK + t * K1B_PER;
  uint64_t nb[K1B_PER], sum = 0;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    const uint32_t s = i0 + i;
    nb[i] = 0;
    if (s < g.n_seg && 2ull * g.excl < g.len[s]) nb[i] = (g.gene_bound ? (uint64_t)g.gene_bound[s] : (uint64_t)g.rows[s].n_records) + 1;
    sum += nb[i];
  }
  uint64_t incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t o = __shfl_up_sync(FULL, incl, d);
    if ((int)lane >= d) incl += o;
  }
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  uint64_t x = incl - sum;
  for (uint32_t w = 0; w < warp; ++w) x += s_w[w];
  if (t == K1B_THREADS - 1) g.block_sum[b] = x + sum;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    if (i0 + i <= g.n_seg) g.bin_base[i0 + i] = x;
    x += nb[i];
  }
}

// Bin block `b` of k1b_apply: adds the bins of the blocks before it.
__device__ __forceinline__ void k1b_bins_apply(const K1bBins& g, uint32_t b) {
  __shared__ unsigned long long s_w[K1B_THREADS / 32];
  const uint32_t t = threadIdx.x;
  uint64_t acc = 0;
  for (uint32_t j = t; j < b; j += K1B_THREADS) acc += g.block_sum[j];
  acc = warp_sum_u64(acc);
  if ((t & 31) == 0) s_w[t >> 5] = acc;
  __syncthreads();
  uint64_t before = 0;
#pragma unroll
  for (uint32_t w = 0; w < K1B_THREADS / 32; ++w) before += s_w[w];
  if (before == 0) return;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    const uint32_t s = b * K1B_BLOCK + t * K1B_PER + i;
    if (s <= g.n_seg) g.bin_base[s] += before;
  }
}

// Blocks [0, ceil(n_chunks / K1B_BLOCK)) scan the chunks, the g.n_blocks after them the segments, the wd.n_blocks after
// those the bitmap words.
__global__ void __launch_bounds__(K1B_THREADS) k1b_local(int32_t* tail_sum, const uint32_t* chunk_first, const uint32_t* off_span,
                                                        uint32_t n_chunks, int32_t* carry_in, int2* block_agg, const K1bBins g,
                                                        const K1bWords wd) {
  const uint32_t chunk_blocks = gridDim.x - g.n_blocks - wd.n_blocks;
  if (blockIdx.x >= chunk_blocks + g.n_blocks) {
    k1b_words_local(wd, blockIdx.x - chunk_blocks - g.n_blocks);
    return;
  }
  if (blockIdx.x >= chunk_blocks) {
    k1b_bins_local(g, blockIdx.x - chunk_blocks);
    return;
  }
  __shared__ int2 s_w[K1B_THREADS / 32];
  const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint32_t k0 = blockIdx.x * K1B_BLOCK + t * K1B_PER;
  K1bElem el[K1B_PER];
  int val = 0, flg = 0;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    const uint32_t k = k0 + i;
    if (k < n_chunks) {
      el[i] = k1b_elem(k, n_chunks, tail_sum, chunk_first, off_span);
    } else {
      el[i].reset = false;
      el[i].add = 0;
    }
    if (el[i].reset) {
      val = el[i].add;
      flg = 1;
    } else {
      val += el[i].add;
    }
  }
  // inclusive segmented scan of (flg, val) over the threads of the block
  int v = val, f = flg;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int ov = __shfl_up_sync(FULL, v, d), of = __shfl_up_sync(FULL, f, d);
    if ((int)lane >= d) {
      if (!f) v += ov;
      f |= of;
    }
  }
  int pv = __shfl_up_sync(FULL, v, 1), pf = __shfl_up_sync(FULL, f, 1);
  if (lane == 0) {
    pv = 0;
    pf = 0;
  }
  if (lane == 31) s_w[warp] = make_int2(v, f);
  __syncthreads();
  int wv = 0, wf = 0;  // exclusive over the preceding warps
  for (uint32_t w = 0; w < warp; ++w) {
    const int2 x = s_w[w];
    wv = x.y ? x.x : wv + x.x;
    wf |= x.y;
  }
  // exclusive prefix for this thread: preceding warps, then preceding lanes of this warp
  int ev = pf ? pv : wv + pv, ef = pf | wf;
  if (t == K1B_THREADS - 1) {
    const int bv = f ? v : wv + v, bf = f | wf;
    block_agg[blockIdx.x] = make_int2(bv, bf);
  }
  int x = ev, xf = ef;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    const uint32_t k = k0 + i;
    if (k < n_chunks) {
      carry_in[k] = x;         // exact if a reset precedes it inside the block, else missing the block carry
      tail_sum[k] = xf ? 0 : 1;  // 1 = "add the block carry"
    }
    if (el[i].reset) {
      x = el[i].add;
      xf = 1;
    } else {
      x += el[i].add;
    }
  }
}

__global__ void __launch_bounds__(K1B_THREADS) k1b_apply(const int32_t* needs, const int2* block_agg, uint32_t n_chunks, int32_t* carry_in,
                                                        const K1bBins g, const K1bWords wd) {
  const uint32_t chunk_blocks = gridDim.x - g.n_blocks - wd.n_blocks;
  if (blockIdx.x >= chunk_blocks + g.n_blocks) {
    k1b_words_apply(wd, blockIdx.x - chunk_blocks - g.n_blocks);
    return;
  }
  if (blockIdx.x >= chunk_blocks) {
    k1b_bins_apply(g, blockIdx.x - chunk_blocks);
    return;
  }
  __shared__ int s_carry;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int j = (int)blockIdx.x - 1; j >= 0; --j) {  // walk back to the nearest block that contains a reset
      const int2 a = block_agg[j];
      acc += a.x;
      if (a.y) break;
    }
    s_carry = acc;
  }
  __syncthreads();
  const int bc = s_carry;
  if (bc == 0) return;
#pragma unroll
  for (uint32_t i = 0; i < K1B_PER; ++i) {
    const uint32_t k = blockIdx.x * K1B_BLOCK + threadIdx.x * K1B_PER + i;
    if (k < n_chunks && needs[k]) carry_in[k] += bc;
  }
}
