// BGZF deflate encoder: one block of at most DFL_BLOCK raw bytes -> one complete BGZF block (18-byte header with the BC extra
// field and BSIZE, a raw DEFLATE payload of one final block, CRC32 and ISIZE).  On the device one CTA of DFL_THREADS threads
// encodes one block (kz_deflate, cmb_deflate.cu); compiled as plain C++ (no __CUDACC__) the same code runs every phase's
// threads one after the other, which gives the same bytes because no phase depends on the order of its threads: every
// shared result is a plain store to a slot only one thread writes, an integer sum, an OR, or "the largest wins" (max).
//
//   match finding  rounds of DFL_ROUND positions: each position reads the hash head (the largest earlier position with the
//                  same 3-byte hash, from the rounds before), then the round raises the heads to its own positions (max)
//   parse          DFL_SEGS segments of DFL_SEG positions, one thread each: greedy with one step of lazy evaluation; a match
//                  stays inside its segment and reaches at most 32 KiB back inside the block.  Tokens are written in place
//                  over the segment's candidates and counted into the symbol histograms
//   code           one thread: Huffman code lengths (15-bit literal/length and distance codes, 7-bit code-length code), the
//                  dynamic block's size, and a stored block instead when that is not larger
//   emission       each segment's bits at the prefix sum of the segments' bit counts, ORed into the payload words
#pragma once
#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#define DFL_HD __device__ __forceinline__
#define DFL_FOR_THREADS(...)             \
  do {                                   \
    {                                    \
      const uint32_t tid = threadIdx.x;  \
      __VA_ARGS__                        \
    }                                    \
    __syncthreads();                     \
  } while (0)
#else
#include <zlib.h>
#define DFL_HD inline
#define DFL_FOR_THREADS(...)                                         \
  do {                                                               \
    for (uint32_t tid = 0; tid < cmb_dfl::DFL_THREADS; ++tid) {      \
      __VA_ARGS__                                                    \
    }                                                                \
  } while (0)
#endif

namespace cmb_dfl {

constexpr uint32_t DFL_BLOCK = 0xff00;   // raw bytes per BGZF block (htslib's BGZF_BLOCK_SIZE)
constexpr uint32_t DFL_MAX_OUT = 65536;  // largest BGZF block
constexpr uint32_t DFL_THREADS = 512;
constexpr uint32_t DFL_ROUND = DFL_THREADS;  // positions per match-finding round
constexpr uint32_t DFL_SEG = 512;            // positions per parse segment
constexpr uint32_t DFL_SEGS = (DFL_BLOCK + DFL_SEG - 1) / DFL_SEG;
constexpr uint32_t DFL_HASH_BITS = 12;
constexpr uint32_t DFL_WINDOW = 32768;
constexpr uint32_t DFL_MAX_MATCH = 258;
constexpr uint32_t DFL_LAZY = 32;  // a match at least this long is taken without looking one position further
constexpr uint32_t DFL_STORED_FLAG = 1u << 31;  // kz_deflate's size word: the block was stored

struct DflTables {  // the code phase's state; lives where the hash heads were
  uint32_t lfreq[288], dfreq[32], cfreq[20];
  uint16_t lcode[288], dcode[32], ccode[20];  // bit-reversed canonical codes
  uint8_t llen[288], dlen[32], clen[20];
  uint16_t rle[320];  // code-length symbols: symbol | extra value << 5
  uint32_t key[288];  // Huffman build: (freq << 9 | symbol), sorted; then the lengths in that order
  uint16_t hsym[288];  // Huffman build: the symbols in that order
  uint8_t all[320];    // the concatenated code lengths
  uint32_t n_rle, hlit, hdist, hclen;
  uint32_t crcT[1024];
};

struct DflSmem {
  union {
    uint8_t in[DFL_MAX_OUT];           // the block's bytes
    uint32_t out[DFL_MAX_OUT / 4];     // after the parse: the DEFLATE payload
  };
  uint16_t tok[DFL_BLOCK];  // per position: candidate + 1 (0: none); then each segment's tokens from its first position on
  union {
    uint32_t head[1u << DFL_HASH_BITS];
    DflTables t;
  };
  uint32_t seg_ntok[DFL_SEGS], seg_off[DFL_SEGS + 1];
  uint32_t n, hdr_bits, total_bits, stored, size, crc;
};

DFL_HD uint32_t dfl_log2(uint32_t v) {
#ifdef __CUDACC__
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}
DFL_HD void dfl_atomic_max(uint32_t* p, uint32_t v) {
#ifdef __CUDACC__
  atomicMax(p, v);
#else
  if (v > *p) *p = v;
#endif
}
DFL_HD void dfl_atomic_add(uint32_t* p, uint32_t v) {
#ifdef __CUDACC__
  atomicAdd(p, v);
#else
  *p += v;
#endif
}
DFL_HD void dfl_atomic_or(uint32_t* p, uint32_t v) {
#ifdef __CUDACC__
  atomicOr(p, v);
#else
  *p |= v;
#endif
}

// length 3..258 -> symbol - 257, extra bits, extra value (RFC 1951 3.2.5)
DFL_HD void dfl_len_code(uint32_t len, uint32_t& code, uint32_t& nx, uint32_t& x) {
  const uint32_t v = len - 3;
  if (len == 258) code = 28, nx = 0, x = 0;
  else if (v < 8) code = v, nx = 0, x = 0;
  else {
    nx = dfl_log2(v) - 2;
    code = 4 * nx + 4 + ((v >> nx) & 3);
    x = v & ((1u << nx) - 1);
  }
}
// distance 1..32768 -> code, extra bits, extra value
DFL_HD void dfl_dist_code(uint32_t dist, uint32_t& code, uint32_t& nx, uint32_t& x) {
  const uint32_t v = dist - 1;
  if (v < 4) code = v, nx = 0, x = 0;
  else {
    nx = dfl_log2(v) - 1;
    code = 2 * nx + 2 + ((v >> nx) & 1);
    x = v & ((1u << nx) - 1);
  }
}
DFL_HD uint32_t dfl_len_extra(uint32_t sym) { return sym < 265 || sym == 285 ? 0 : (sym - 261) / 4; }
DFL_HD uint32_t dfl_dist_extra(uint32_t code) { return code < 4 ? 0 : code / 2 - 1; }

DFL_HD uint32_t dfl_hash(const uint8_t* p) {
  const uint32_t v = (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16;
  return (v * 2654435761u) >> (32 - DFL_HASH_BITS);
}

// Longest match at p against its candidate, inside [.., end) and at most DFL_MAX_MATCH; 0 when shorter than 3
DFL_HD uint32_t dfl_match(const DflSmem& S, uint32_t p, uint32_t end, uint32_t& dist) {
  const uint32_t c = S.tok[p];
  if (!c || p - (c - 1) > DFL_WINDOW) return 0;
  const uint32_t j = c - 1, lim = end - p < DFL_MAX_MATCH ? end - p : DFL_MAX_MATCH;
  uint32_t l = 0;
  while (l < lim && S.in[j + l] == S.in[p + l]) ++l;
  dist = p - j;
  return l >= 3 ? l : 0;
}

// Code lengths limited to `maxlen` for freq[0, n), at least two codes, so that the code is complete (as zlib's trees are).
// One thread.
DFL_HD void dfl_huffman(const uint32_t* freq, uint32_t n, uint32_t maxlen, uint8_t* len, uint32_t* A, uint16_t* sym) {
  uint32_t m = 0;
  for (uint32_t s = 0; s < n; ++s) {
    len[s] = 0;
    if (freq[s]) A[m++] = freq[s] << 9 | s;
  }
  for (uint32_t s = 0; m < 2; ++s)  // pad with the lowest unused symbols
    if (!freq[s]) A[m++] = s;
  // Shell sort by (freq, symbol): keys are distinct, so the order is fixed
  const uint32_t gaps[6] = {132, 57, 23, 10, 4, 1};
  for (uint32_t g : gaps)
    for (uint32_t i = g; i < m; ++i) {
      const uint32_t v = A[i];
      uint32_t j = i;
      for (; j >= g && A[j - g] > v; j -= g) A[j] = A[j - g];
      A[j] = v;
    }
  for (uint32_t i = 0; i < m; ++i) sym[i] = (uint16_t)(A[i] & 511), A[i] >>= 9;
  if (A[0] == 0) A[0] = 1;  // a padding symbol
  if (A[1] == 0) A[1] = 1;
  // in-place minimum-redundancy code lengths over the sorted weights (Moffat and Katajainen, 1995)
  {
    A[0] += A[1];
    uint32_t root = 0, leaf = 2;
    for (uint32_t next = 1; next < m - 1; ++next) {
      if (leaf >= m || A[root] < A[leaf]) A[next] = A[root], A[root++] = next;
      else A[next] = A[leaf++];
      if (leaf >= m || (root < next && A[root] < A[leaf])) A[next] += A[root], A[root++] = next;
      else A[next] += A[leaf++];
    }
    A[m - 2] = 0;
    for (int next = (int)m - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
    int avbl = 1, used = 0, dpth = 0, r = (int)m - 2, nx = (int)m - 1;
    while (avbl > 0) {
      while (r >= 0 && (int)A[r] == dpth) ++used, --r;
      while (avbl > used) A[nx--] = dpth, --avbl;
      avbl = 2 * used, ++dpth, used = 0;
    }
  }
  // limit to maxlen: fold the longer codes into maxlen, then lengthen codes until the Kraft sum is exact again
  uint32_t count[33] = {0};
  for (uint32_t i = 0; i < m; ++i) count[A[i]]++;
  for (uint32_t l = maxlen + 1; l <= 32; ++l) count[maxlen] += count[l], count[l] = 0;
  uint32_t total = 0;
  for (uint32_t l = maxlen; l > 0; --l) total += count[l] << (maxlen - l);
  while (total != (1u << maxlen)) {
    count[maxlen]--;
    for (uint32_t l = maxlen - 1; l > 0; --l)
      if (count[l]) {
        count[l]--;
        count[l + 1] += 2;
        break;
      }
    total--;
  }
  // the shortest lengths to the most frequent symbols (the end of the sorted order)
  int k = (int)m - 1;
  for (uint32_t l = 1; l <= maxlen; ++l)
    for (uint32_t c = count[l]; c; --c) len[sym[k--]] = (uint8_t)l;
}

// Canonical codes, bit-reversed for LSB-first output
DFL_HD void dfl_codes(const uint8_t* len, uint32_t n, uint16_t* code) {
  uint32_t count[16] = {0}, next[16];
  for (uint32_t s = 0; s < n; ++s) count[len[s]]++;
  count[0] = 0;
  uint32_t c = 0;
  for (uint32_t l = 1; l < 16; ++l) c = (c + count[l - 1]) << 1, next[l] = c;
  for (uint32_t s = 0; s < n; ++s) {
    const uint32_t l = len[s];
    if (!l) {
      code[s] = 0;
      continue;
    }
    uint32_t v = next[l]++, r = 0;
    for (uint32_t b = 0; b < l; ++b) r = r << 1 | ((v >> b) & 1);
    code[s] = (uint16_t)r;
  }
}

struct DflBits {  // LSB-first bit writer into S.out from bit `pos` on, merging with neighbours' words by OR
  uint32_t* w;
  uint32_t word, cnt;
  uint64_t acc;
  DFL_HD DflBits(uint32_t* out, uint32_t pos) : w(out), word(pos >> 5), cnt(pos & 31), acc(0) {}
  DFL_HD void put(uint32_t v, uint32_t nb) {  // nb <= 32
    acc |= (uint64_t)v << cnt;
    cnt += nb;
    while (cnt >= 32) {
      dfl_atomic_or(&w[word++], (uint32_t)acc);
      acc >>= 32;
      cnt -= 32;
    }
  }
  DFL_HD void flush() {
    if (cnt) dfl_atomic_or(&w[word], (uint32_t)acc);
  }
};

// k-th entry of the code-length code's transmission order (RFC 1951 3.2.7)
DFL_HD uint32_t dfl_clen_order(uint32_t k) {
  const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  return order[k];
}

// The CRC: warp_crc32 (cmb_crc32.cuh) on the device, over the block's bytes in global memory; zlib's in the host build
DFL_HD void dfl_crc_tables(DflSmem& S, uint32_t i) {
#ifdef __CUDACC__
  if (i < 256) crc32_fill_tables(S.t.crcT, i);
#else
  (void)S, (void)i;
#endif
}
DFL_HD void dfl_crc(DflSmem& S, const uint8_t* src, uint32_t n, uint32_t tid) {
#ifdef __CUDACC__
  if (tid < 32) {
    const uint32_t c = warp_crc32(src, n, S.t.crcT, tid);
    if (tid == 0) S.crc = c;
  }
#else
  if (tid == 0) S.crc = (uint32_t)crc32(0, src, n);
#endif
}

// The code phase (one thread): trees, header, sizes, and the stored / dynamic choice
DFL_HD void dfl_plan(DflSmem& S) {
  DflTables& T = S.t;
  const uint32_t n = S.n;
  T.lfreq[256] += 1;  // end of block
  dfl_huffman(T.lfreq, 286, 15, T.llen, T.key, T.hsym);
  dfl_huffman(T.dfreq, 30, 15, T.dlen, T.key, T.hsym);
  uint32_t hlit = 286, hdist = 30;
  while (hlit > 257 && !T.llen[hlit - 1]) --hlit;
  while (hdist > 1 && !T.dlen[hdist - 1]) --hdist;
  // run-length code of the concatenated code lengths (RFC 1951 3.2.7)
  uint8_t* all = T.all;
  for (uint32_t i = 0; i < hlit; ++i) all[i] = T.llen[i];
  for (uint32_t i = 0; i < hdist; ++i) all[hlit + i] = T.dlen[i];
  const uint32_t n_all = hlit + hdist;
  uint32_t nr = 0;
  for (uint32_t s = 0; s < 19; ++s) T.cfreq[s] = 0;
  auto emit = [&](uint32_t sym, uint32_t x) {
    T.rle[nr++] = (uint16_t)(sym | x << 5);
    T.cfreq[sym]++;
  };
  for (uint32_t i = 0; i < n_all;) {
    const uint32_t l = all[i];
    uint32_t run = 1;
    while (i + run < n_all && all[i + run] == l) ++run;
    i += run;
    if (l == 0) {
      while (run >= 11) {
        const uint32_t r = run < 138 ? run : 138;
        emit(18, r - 11);
        run -= r;
      }
      if (run >= 3) emit(17, run - 3), run = 0;
    } else {
      emit(l, 0);
      --run;
      while (run >= 3) {
        const uint32_t r = run < 6 ? run : 6;
        emit(16, r - 3);
        run -= r;
      }
    }
    while (run) emit(l, 0), --run;
  }
  dfl_huffman(T.cfreq, 19, 7, T.clen, T.key, T.hsym);
  uint32_t hclen = 19;
  while (hclen > 4 && !T.clen[dfl_clen_order(hclen - 1)]) --hclen;
  uint64_t bits = 3 + 5 + 5 + 4 + 3 * hclen;
  for (uint32_t k = 0; k < nr; ++k) {
    const uint32_t sym = T.rle[k] & 31;
    bits += T.clen[sym] + (sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0);
  }
  S.hdr_bits = (uint32_t)bits;
  for (uint32_t s = 0; s < 286; ++s) bits += (uint64_t)T.lfreq[s] * (T.llen[s] + dfl_len_extra(s));
  for (uint32_t d = 0; d < 30; ++d) bits += (uint64_t)T.dfreq[d] * (T.dlen[d] + dfl_dist_extra(d));
  S.total_bits = (uint32_t)bits;
  const uint32_t dyn_bytes = (uint32_t)((bits + 7) / 8), stored_bytes = n + 5;
  S.stored = stored_bytes <= dyn_bytes;
  S.size = 18 + (S.stored ? stored_bytes : dyn_bytes) + 8;
  T.n_rle = nr, T.hlit = hlit, T.hdist = hdist, T.hclen = hclen;
  dfl_codes(T.llen, 286, T.lcode);
  dfl_codes(T.dlen, 30, T.dcode);
  dfl_codes(T.clen, 19, T.ccode);
}

DFL_HD void dfl_put_token(DflBits& b, const DflTables& T, const uint16_t* t, uint32_t& k) {
  const uint32_t v = t[k++];
  if (!(v & 0x8000)) {
    b.put(T.lcode[v], T.llen[v]);
    return;
  }
  const uint32_t dist = t[k++];
  uint32_t code, nx, x;
  dfl_len_code((v & 0x7fff) + 3, code, nx, x);
  b.put(T.lcode[257 + code], T.llen[257 + code]);
  if (nx) b.put(x, nx);
  dfl_dist_code(dist, code, nx, x);
  b.put(T.dcode[code], T.dlen[code]);
  if (nx) b.put(x, nx);
}

DFL_HD uint32_t dfl_token_bits(const DflTables& T, const uint16_t* t, uint32_t& k) {
  const uint32_t v = t[k++];
  if (!(v & 0x8000)) return T.llen[v];
  const uint32_t dist = t[k++];
  uint32_t code, nx, x, bits;
  dfl_len_code((v & 0x7fff) + 3, code, nx, x);
  bits = T.llen[257 + code] + nx;
  dfl_dist_code(dist, code, nx, x);
  return bits + T.dlen[code] + nx;
}

// Encodes src[0, n) (n <= DFL_BLOCK) into dst (room for DFL_MAX_OUT bytes) as one BGZF block; its size is S.size, and
// S.stored tells whether the payload is a stored block.  On the device every thread of the CTA calls it.
DFL_HD void dfl_encode_block(DflSmem& S, const uint8_t* src, uint32_t n, uint8_t* dst) {
  DFL_FOR_THREADS({
    if (tid == 0) S.n = n;
    for (uint32_t k = tid; k < n; k += DFL_THREADS) S.in[k] = src[k];
    for (uint32_t k = tid; k < (1u << DFL_HASH_BITS); k += DFL_THREADS) S.head[k] = 0;
  });
  // ---- match candidates: the largest earlier position with the same hash, from the rounds before
  for (uint32_t r0 = 0; r0 < n; r0 += DFL_ROUND) {
    DFL_FOR_THREADS({
      const uint32_t i = r0 + tid;
      if (tid < DFL_ROUND && i < n) S.tok[i] = i + 2 < n ? (uint16_t)S.head[dfl_hash(S.in + i)] : 0;
    });
    DFL_FOR_THREADS({
      const uint32_t i = r0 + tid;
      if (tid < DFL_ROUND && i + 2 < n) dfl_atomic_max(&S.head[dfl_hash(S.in + i)], i + 1);
    });
  }
  DFL_FOR_THREADS({
    for (uint32_t k = tid; k < 288; k += DFL_THREADS) S.t.lfreq[k] = 0;
    if (tid < 32) S.t.dfreq[tid] = 0;
  });
  // ---- parse, one segment per thread; tokens in place: literal byte, or 0x8000 | (length - 3) then the distance
  DFL_FOR_THREADS({
    if (tid < DFL_SEGS) {
      const uint32_t s0 = tid * DFL_SEG, s1 = s0 + DFL_SEG < n ? s0 + DFL_SEG : n;
      uint32_t i = s0, w = s0;
      while (i < s1) {
        uint32_t dist = 0, dist2 = 0;
        const uint32_t l = dfl_match(S, i, s1, dist);
        const uint32_t l2 = l && l < DFL_LAZY && i + 1 < s1 ? dfl_match(S, i + 1, s1, dist2) : 0;
        if (!l || l2 > l) {
          const uint8_t b = S.in[i];
          S.tok[w++] = b;
          dfl_atomic_add(&S.t.lfreq[b], 1);
          ++i;
          continue;
        }
        uint32_t code, nx, x;
        dfl_len_code(l, code, nx, x);
        dfl_atomic_add(&S.t.lfreq[257 + code], 1);
        dfl_dist_code(dist, code, nx, x);
        dfl_atomic_add(&S.t.dfreq[code], 1);
        S.tok[w++] = (uint16_t)(0x8000 | (l - 3));
        S.tok[w++] = (uint16_t)dist;
        i += l;
      }
      S.seg_ntok[tid] = w - s0;
    }
  });
  DFL_FOR_THREADS({
    if (tid == 0) dfl_plan(S);
  });
  // ---- bit counts per segment, their prefix sum, and the payload words zeroed (dynamic) ; the CRC
  DFL_FOR_THREADS({
    if (tid < DFL_SEGS) {
      uint32_t bits = 0;
      if (!S.stored) {
        const uint32_t s0 = tid * DFL_SEG;
        for (uint32_t k = 0; k < S.seg_ntok[tid];) bits += dfl_token_bits(S.t, S.tok + s0, k);
      }
      S.seg_off[tid + 1] = bits;
    }
    if (tid >= 256) dfl_crc_tables(S, tid - 256);
  });
  DFL_FOR_THREADS({
    if (tid == 0) {
      uint32_t o = S.hdr_bits;
      S.seg_off[0] = o;
      for (uint32_t s = 0; s < DFL_SEGS; ++s) {
        const uint32_t b = S.seg_off[s + 1];
        S.seg_off[s + 1] = o + b;
        o += b;
      }
    }
    if (!S.stored)
      for (uint32_t k = tid; k < DFL_MAX_OUT / 4; k += DFL_THREADS) S.out[k] = 0;
  });
  DFL_FOR_THREADS({
    if (!S.stored) {
      const DflTables& T = S.t;
      if (tid < DFL_SEGS && S.seg_ntok[tid]) {
        DflBits b(S.out, S.seg_off[tid]);
        const uint16_t* t = S.tok + tid * DFL_SEG;
        for (uint32_t k = 0; k < S.seg_ntok[tid];) dfl_put_token(b, T, t, k);
        b.flush();
      }
      if (tid == DFL_THREADS - 1) {  // block header, tables, end of block
        DflBits b(S.out, 0);
        b.put(1, 1);  // BFINAL
        b.put(2, 2);  // dynamic Huffman
        b.put(T.hlit - 257, 5);
        b.put(T.hdist - 1, 5);
        b.put(T.hclen - 4, 4);
        for (uint32_t k = 0; k < T.hclen; ++k) b.put(T.clen[dfl_clen_order(k)], 3);
        for (uint32_t k = 0; k < T.n_rle; ++k) {
          const uint32_t sym = T.rle[k] & 31, x = T.rle[k] >> 5;
          b.put(T.ccode[sym], T.clen[sym]);
          if (sym >= 16) b.put(x, sym == 16 ? 2 : sym == 17 ? 3 : 7);
        }
        b.flush();
        DflBits e(S.out, S.seg_off[DFL_SEGS]);
        e.put(T.lcode[256], T.llen[256]);
        e.flush();
      }
    }
    dfl_crc(S, src, n, tid);
  });
  // ---- the BGZF block
  DFL_FOR_THREADS({
    const uint32_t size = S.size, payload = size - 26;
    if (tid < 18) {
      const uint8_t hdr[18] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, (uint8_t)((size - 1) & 0xff), (uint8_t)((size - 1) >> 8)};
      dst[tid] = hdr[tid];
    } else if (tid < 26) {
      const uint32_t k = tid - 18, v = k < 4 ? S.crc : n;
      dst[18 + payload + k] = (uint8_t)(v >> (8 * (k & 3)));
    }
    if (S.stored) {
      if (tid == 26) {
        dst[18] = 1;  // BFINAL, stored
        dst[19] = (uint8_t)(n & 0xff), dst[20] = (uint8_t)(n >> 8);
        dst[21] = (uint8_t)(~n & 0xff), dst[22] = (uint8_t)((~n >> 8) & 0xff);
      }
      for (uint32_t k = tid; k < n; k += DFL_THREADS) dst[23 + k] = S.in[k];
    } else {
      for (uint32_t k = tid; k < payload; k += DFL_THREADS) dst[18 + k] = S.in[k];
    }
  });
}

}  // namespace cmb_dfl
