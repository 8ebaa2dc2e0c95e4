// CRC-32 of a byte range by one warp (warp_crc32), shared by the inflate kernels (cmb_decode.cuh, cmb_decode_t1.cuh) and the
// BGZF deflate encoder (cmb_deflate.cu).  Needs FULL (cmb_common.cuh).
#pragma once
#include <cstdint>

// ---- CRC-32 (ISO-HDLC, the gzip/BGZF checksum; reflected polynomial 0xEDB88320) of a block's output, by the whole warp:
// every lane checksums a 2 KB slice with slicing-by-4 tables, then the slices are combined through the linearity of the
// CRC: crc(A||B) = crc(A) * x^(8|B|) mod P  xor  crc(B)  (polynomial arithmetic over GF(2), bit 31 = x^0).
constexpr uint32_t CRC_POLY = 0xedb88320u;
constexpr uint32_t CRC_SLICE = 2048;
constexpr uint32_t INF_CRC_TABLE_BYTES = 4 * 256 * 4;

__device__ __forceinline__ uint32_t gf2_mulmod(uint32_t a, uint32_t b) {  // a(x) * b(x) mod P(x)
  uint32_t p = 0;
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
  }
  return p;
}
__device__ uint32_t gf2_x_pow_8n(uint32_t n_bytes) {  // x^(8 n) mod P by square and multiply
  uint32_t sq = 0x00800000u;  // x^8: x^0 is bit 31, x^k is bit 31-k
  uint32_t r = 1u << 31;
  while (n_bytes) {
    if (n_bytes & 1) r = gf2_mulmod(sq, r);
    sq = gf2_mulmod(sq, sq);
    n_bytes >>= 1;
  }
  return r;
}
__device__ uint32_t warp_crc32(const uint8_t* data, uint32_t n, const uint32_t* T, uint32_t lane) {
  const uint32_t b0 = min(n, lane * CRC_SLICE), b1 = min(n, (lane + 1) * CRC_SLICE);
  uint32_t c = 0;
  if (b1 > b0) {
    const uint8_t* p = data + b0;
    const uint8_t* e = data + b1;
    c = 0xffffffffu;
    while (p < e && ((uintptr_t)p & 3)) c = T[(c ^ __ldcg(p++)) & 0xff] ^ (c >> 8);
    for (; p + 4 <= e; p += 4) {
      c ^= __ldcg(reinterpret_cast<const uint32_t*>(p));
      c = T[768 + (c & 0xff)] ^ T[512 + ((c >> 8) & 0xff)] ^ T[256 + ((c >> 16) & 0xff)] ^ T[c >> 24];
    }
    while (p < e) c = T[(c ^ __ldcg(p++)) & 0xff] ^ (c >> 8);
    c = ~c;
    c = gf2_mulmod(gf2_x_pow_8n(n - b1), c);
  }
  return __reduce_xor_sync(FULL, c);
}

// The four slicing-by-4 tables warp_crc32 reads (T[k * 256 + i]), entry i of each filled by thread i < 256
__device__ __forceinline__ void crc32_fill_tables(uint32_t* T, uint32_t i) {
  auto step = [](uint32_t c) {
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ CRC_POLY : c >> 1;
    return c;
  };
  uint32_t c = step(i);
  T[i] = c;
  for (int k = 1; k < 4; ++k) {
    c = step(c & 0xff) ^ (c >> 8);
    T[k * 256 + i] = c;
  }
}
