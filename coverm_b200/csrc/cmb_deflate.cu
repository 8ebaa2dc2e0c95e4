// The BGZF output stream deflated on the device (cmb_deflate_*, cmb_filter_bgzf_deflate's output): the stream's bytes are
// gathered in d_raw (the carry of the last feed first), every full block of a piece is deflated by kz_deflate (one CTA per
// block, cmb_deflate.cuh) into a fixed slot, kz_pack moves the blocks back to back at the prefix sum of their sizes, and the
// piece crosses to a pinned staging buffer and on to the sink.  What is left past the last full block is the next carry.
#include <algorithm>
#include <chrono>
#include <cstring>

#include "cmb_context.cuh"
#include "cmb_common.cuh"
#include "cmb_crc32.cuh"
#include "cmb_deflate.cuh"

using namespace cmb_dfl;

namespace {

constexpr uint32_t PIECE_BLOCKS = 1024;  // blocks per piece: at most 64 MB of BGZF bytes, one staging buffer
constexpr uint64_t PIECE_RAW = (uint64_t)PIECE_BLOCKS * DFL_BLOCK;
constexpr uint8_t EOF_BLOCK[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};

// blocks [0, gridDim.x) of raw[0, n): block b is raw[b * DFL_BLOCK, min(n, (b + 1) * DFL_BLOCK))
__global__ void __launch_bounds__(DFL_THREADS, 1) kz_deflate(const uint8_t* raw, uint64_t n, uint8_t* slots, uint32_t* size) {
  extern __shared__ __align__(16) uint8_t dfl_smem[];
  DflSmem& S = *reinterpret_cast<DflSmem*>(dfl_smem);
  const uint64_t b0 = (uint64_t)blockIdx.x * DFL_BLOCK;
  const uint32_t len = n - b0 < DFL_BLOCK ? (uint32_t)(n - b0) : DFL_BLOCK;
  dfl_encode_block(S, raw + b0, len, slots + (uint64_t)blockIdx.x * DFL_MAX_OUT);
  if (threadIdx.x == 0) size[blockIdx.x] = S.size | (S.stored ? DFL_STORED_FLAG : 0);
}

// block b's bytes to packed + (sum of the sizes of blocks 0 .. b-1)
__global__ void __launch_bounds__(256) kz_pack(const uint8_t* slots, const uint32_t* size, uint8_t* packed) {
  __shared__ uint32_t part[8];
  const uint32_t b = blockIdx.x;
  uint64_t s = 0;
  for (uint32_t k = threadIdx.x; k < b; k += 256) s += size[k] & ~DFL_STORED_FLAG;
  s = warp_sum_u64(s);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = (uint32_t)s;
  __syncthreads();
  uint64_t off = 0;
  for (int w = 0; w < 8; ++w) off += part[w];
  const uint32_t n = size[b] & ~DFL_STORED_FLAG;
  const uint8_t* src = slots + (uint64_t)b * DFL_MAX_OUT;
  for (uint32_t k = threadIdx.x; k < n; k += 256) packed[off + k] = src[k];
}

double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// The first k blocks of d_raw (raw_bytes of it; the last block may be partial) deflated and handed to the sink, followed by
// `tail` (the EOF block) when given
int deflate_piece(cmb_ctx* c, uint32_t k, uint64_t raw_bytes, cmb_filter_sink sink, void* user, uint32_t* n_calls,
                  const uint8_t* tail = nullptr, uint32_t tail_len = 0) {
  auto& z = c->dfl;
  uint64_t total = 0;
  if (k) {
    CU_TRY(c, cudaEventRecord(z.ev[0], c->stream));
    kz_deflate<<<k, DFL_THREADS, sizeof(DflSmem), c->stream>>>(z.d_raw, raw_bytes, z.d_blocks, z.d_size);
    kz_pack<<<k, 256, 0, c->stream>>>(z.d_blocks, z.d_size, z.d_packed);
    CU_TRY(c, cudaGetLastError());
    CU_TRY(c, cudaEventRecord(z.ev[1], c->stream));
    CU_TRY(c, cudaMemcpyAsync(z.h_size, z.d_size, 4ull * k, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    float ms = 0;
    CU_TRY(c, cudaEventElapsedTime(&ms, z.ev[0], z.ev[1]));
    z.stats.ms_deflate += ms;
    for (uint32_t b = 0; b < k; ++b) {
      total += z.h_size[b] & ~DFL_STORED_FLAG;
      z.stats.stored_blocks += (z.h_size[b] & DFL_STORED_FLAG) ? 1 : 0;
    }
    z.stats.blocks += k;
    z.stats.raw_bytes += raw_bytes;
  }
  uint8_t* stage = z.stage[z.stats.sink_calls & 1];
  const auto t0 = std::chrono::steady_clock::now();
  if (total) {
    CU_TRY(c, cudaMemcpyAsync(stage, z.d_packed, total, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
  }
  z.stats.ms_d2h += (float)ms_since(t0);
  if (tail_len) memcpy(stage + total, tail, tail_len);
  total += tail_len;
  if (!total) return CMB_OK;
  if (const int s = sink(user, stage, total)) {
    z.active = false;
    return fail(c, CMB_E_ARG, "cmb_deflate: the sink returned %d", s);
  }
  z.stats.sink_calls += 1;
  z.stats.bgzf_bytes += total;
  if (n_calls) *n_calls += 1;
  return CMB_OK;
}

// src[0, n) (host or device memory, per `kind`) appended to the stream; every piece of full blocks it completes deflated
int feed(cmb_ctx* c, const uint8_t* src, uint64_t n, cudaMemcpyKind kind, cmb_filter_sink sink, void* user, uint32_t* n_calls) {
  auto& z = c->dfl;
  if (!z.active) return fail(c, CMB_E_ARG, "cmb_deflate: no stream begun (cmb_deflate_begin first)");
  if (!sink || (!src && n)) return fail(c, CMB_E_ARG, "cmb_deflate: null argument");
  while (n) {
    const uint64_t take = std::min<uint64_t>(n, PIECE_RAW - z.carry);
    CU_TRY(c, cudaMemcpyAsync(z.d_raw + z.carry, src, take, kind, c->stream));
    z.carry += take;
    src += take;
    n -= take;
    const uint32_t k = (uint32_t)(z.carry / DFL_BLOCK);
    if (!k) break;
    if (int rc = deflate_piece(c, k, (uint64_t)k * DFL_BLOCK, sink, user, n_calls)) return rc;
    const uint64_t rest = z.carry - (uint64_t)k * DFL_BLOCK;  // < one block, so it does not overlap its new place
    if (rest) CU_TRY(c, cudaMemcpyAsync(z.d_raw, z.d_raw + (uint64_t)k * DFL_BLOCK, rest, cudaMemcpyDeviceToDevice, c->stream));
    z.carry = rest;
  }
  CU_TRY(c, cudaStreamSynchronize(c->stream));  // a host source may be reused once the call returns
  return CMB_OK;
}

}  // namespace

int cmb::deflate_feed_device(cmb_ctx* c, const uint8_t* d_src, uint64_t n, cmb_filter_sink sink, void* user, uint32_t* n_calls) {
  return feed(c, d_src, n, cudaMemcpyDeviceToDevice, sink, user, n_calls);
}

extern "C" int cmb_deflate_begin(cmb_ctx* c) {
  if (!c) return fail(c, CMB_E_ARG, "cmb_deflate_begin: null argument");
  CU_TRY(c, cudaSetDevice(c->device));
  auto& z = c->dfl;
  z.active = false;
  z.carry = 0;
  z.stats = cmb_deflate_stats{};
  int rc;
  if ((rc = z.d_raw.ensure(c, PIECE_RAW)) || (rc = z.d_blocks.ensure(c, (size_t)PIECE_BLOCKS * DFL_MAX_OUT)) ||
      (rc = z.d_size.ensure(c, PIECE_BLOCKS)) || (rc = z.d_packed.ensure(c, (size_t)PIECE_BLOCKS * DFL_MAX_OUT)) ||
      (rc = z.h_size.ensure(c, PIECE_BLOCKS)))
    return rc;
  for (auto& s : z.stage)  // room for a full piece and the EOF block
    if ((rc = s.ensure(c, (size_t)PIECE_BLOCKS * DFL_MAX_OUT + sizeof EOF_BLOCK))) return rc;
  for (auto& e : z.ev)
    if (!e) CU_TRY(c, cudaEventCreate(&e));
  CU_TRY(c, cudaFuncSetAttribute(kz_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DflSmem)));
  z.active = true;
  return CMB_OK;
}

extern "C" int cmb_deflate_feed(cmb_ctx* c, const uint8_t* bytes, uint64_t n_bytes, cmb_filter_sink sink, void* user) {
  NvtxRange nvtx("cmb_deflate_feed");
  if (!c) return fail(c, CMB_E_ARG, "cmb_deflate_feed: null argument");
  CU_TRY(c, cudaSetDevice(c->device));
  return feed(c, bytes, n_bytes, cudaMemcpyHostToDevice, sink, user, nullptr);
}

extern "C" int cmb_deflate_finish(cmb_ctx* c, cmb_filter_sink sink, void* user, cmb_deflate_stats* stats) {
  NvtxRange nvtx("cmb_deflate_finish");
  if (!c || !sink || !stats) return fail(c, CMB_E_ARG, "cmb_deflate_finish: null argument");
  auto& z = c->dfl;
  if (!z.active) return fail(c, CMB_E_ARG, "cmb_deflate_finish: no stream begun (cmb_deflate_begin first)");
  CU_TRY(c, cudaSetDevice(c->device));
  if (int rc = deflate_piece(c, z.carry ? 1 : 0, z.carry, sink, user, nullptr, EOF_BLOCK, sizeof EOF_BLOCK)) return rc;
  z.carry = 0;
  z.active = false;
  *stats = z.stats;
  return CMB_OK;
}
