// libcoverm_b200 -- device-side BAM decode behind cmb_submit_bgzf / cmb_decode_bgzf (cmb_decode*.cuh): the staged call
// (BgzfCall), the decode in block slices when the whole stream does not fit (decode_sliced), mate matching (cmb_pairs.cuh)
// and `coverm filter` (cmb_filter.cuh) over the resident sample or, through cmb_filter_bgzf, slice by slice.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>

#include <zlib.h>

#include "cmb_context.cuh"
#include "cmb_bgzf.cuh"

namespace {
#include "cmb_common.cuh"
#include "cmb_decode.cuh"
#include "cmb_decode_g8.cuh"
#include "cmb_decode_t1.cuh"
#include "cmb_pairs.cuh"
#include "cmb_filter.cuh"
}  // namespace

// ------------------------------------------------------------------------------------------------ device-side decode
namespace {
constexpr size_t DEC_COPY_CHUNK = 8u << 20;    // pinned staging slot
constexpr size_t DEC_WINDOW_BYTES = 32u << 20; // compressed bytes per copy+inflate window
size_t dec_window_bytes() {  // CMB_DECODE_WINDOW_KB: testing aid, lets a small file span many windows
  static const size_t v = [] {
    const char* e = getenv("CMB_DECODE_WINDOW_KB");
    const long kb = e ? atol(e) : 0;
    return kb > 0 ? (size_t)kb << 10 : DEC_WINDOW_BYTES;
  }();
  return v;
}
constexpr size_t DEC_SLACK = 1024;
// the reference's panic in nm() (CMB_E_NM)
constexpr const char* NM_PANIC = "Mapping record encountered that does not have an 'NM' auxiliary tag in the SAM/BAM format. This is "
                                 "required to work out some coverage statistics";
constexpr size_t DEC_FRONT = 256;              // readable bytes in front of the first uploaded block (the bit readers align down)

// First-pass inflate kernel: 0 = kd_inflate_t1 (a thread per block + kd_crc32), 1 = kd_inflate_g8 (four blocks per warp), 2 =
// kd_inflate (a warp per block, also the second pass over declined blocks).  t1 has the higher THROUGHPUT (its sm_count x 5 x 96
// streams, 63 360 on 132 SMs, need that many blocks) but each of its streams is slow, so a short list of blocks finishes sooner
// on g8.  The choice follows the number of blocks: a whole 10 M-read file (46 000 blocks) goes to t1, a rank's share of it on 4
// or 8 GPUs to g8.  CMB_INFLATE=t1|g8|w1 overrides.
constexpr uint32_t T1_MIN_BLOCKS = 28000;
int inflate_kind(uint32_t n_blocks) {
  static const int forced = [] {
    const char* e = getenv("CMB_INFLATE");
    if (e && !strcmp(e, "t1")) return 0;
    if (e && !strcmp(e, "g8")) return 1;
    if (e && !strcmp(e, "w1")) return 2;
    return -1;
  }();
  if (forced >= 0) return forced;
  return n_blocks >= T1_MIN_BLOCKS ? 0 : 1;
}
// Default: ONE persistent launch whose threads poll the windows' arrival flags (bounded wait), so that every SM has work as soon
// as the first window is in.
// Serial mode: copy everything, then ONE inflate launch ordered behind the copies on the context stream -- no flags, nothing on
// the device waits for anything.  Used for files of a single window (nothing to overlap), on request (CMB_INFLATE_SERIAL=1),
// and when a CUDA tool is injected into the process (ncu, compute-sanitizer: they serialise kernels against the other streams,
// so a kernel that polls for copies would only ever see its bounded wait expire).
bool inflate_serial_requested() {
  static const bool v = [] {
    if (const char* e = getenv("CMB_INFLATE_SERIAL")) return e[0] == '1';
    for (const char* name : {"CUDA_INJECTION64_PATH", "NV_NSIGHT_INJECTION_PORT_BASE", "NV_COMPUTE_PROFILER_PERFWORKS_DIR", "NV_SANITIZER_INJECTION_PORT_BASE"})
      if (const char* e = getenv(name))
        if (e[0]) return true;
    return false;
  }();
  return v;
}
// kd_crc32 over the blocks of `a` (the t1 path: its inflate kernel leaves the CRC to a second kernel)
int launch_crc32(cmb_ctx* c, const InflateArgs& a, cudaStream_t st) {
  const uint32_t nb = a.b1 - a.b0;
  kd_crc32<<<std::min<uint32_t>((nb + 7) / 8, (uint32_t)c->sm_count * 8), 256, 0, st>>>(a);
  CU_TRY(c, cudaGetLastError());
  return CMB_OK;
}
// Launch the inflate kernel over blocks [a.b0, a.b1), or over a.block_list[a.b0, a.b1) with kd_inflate (the second pass).
// *crc_pending (when given) is set instead of launching kd_crc32: the caller launches it once nothing else has to get past it
// in the hardware queue (a kernel waiting for its predecessor blocks the queue for every stream that shares it).
int launch_inflate(cmb_ctx* c, const InflateArgs& a, cudaStream_t st, bool* crc_pending = nullptr) {
  const uint32_t nb = a.b1 - a.b0;
  const int k = a.block_list ? 2 : inflate_kind(nb);
  if (k == 0) {
    CU_TRY(c, cudaFuncSetAttribute(kd_inflate_t1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T1_SMEM_BYTES));
    // every resident warp takes part; with fewer blocks than lanes, each warp works with its first `lanes` lanes only
    const uint32_t max_grid = (uint32_t)c->sm_count * 5, warps = max_grid * (T1_THREADS / 32);
    const uint32_t lanes = std::min<uint32_t>(32, std::max<uint32_t>(1, (nb + warps - 1) / warps));
    const uint32_t per_cta = lanes * (T1_THREADS / 32);
    const uint32_t grid = std::min<uint32_t>((nb + per_cta - 1) / per_cta, max_grid);
    InflateArgs at = a;
    at.lane_limit = lanes;
    kd_inflate_t1<<<grid, T1_THREADS, T1_SMEM_BYTES, st>>>(at);
    CU_TRY(c, cudaGetLastError());
    if (crc_pending) *crc_pending = true;
    else if (int rc = launch_crc32(c, a, st)) return rc;
  } else if (k == 1) {
    CU_TRY(c, cudaFuncSetAttribute(kd_inflate_g8, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G8_SMEM_BYTES));
    const uint32_t per_cta = G8_WARPS * G8_STREAMS;
    const uint32_t grid = std::min<uint32_t>((nb + per_cta - 1) / per_cta, (uint32_t)c->sm_count * 2);
    kd_inflate_g8<<<grid, G8_WARPS * 32, G8_SMEM_BYTES, st>>>(a);
  } else {
    CU_TRY(c, cudaFuncSetAttribute(kd_inflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)INF_SMEM_BYTES));
    const uint32_t grid = std::min<uint32_t>((nb + INF_WARPS - 1) / INF_WARPS, (uint32_t)c->sm_count * 2);
    kd_inflate<<<grid, INF_WARPS * 32, INF_SMEM_BYTES, st>>>(a);
  }
  CU_TRY(c, cudaGetLastError());
  return CMB_OK;
}

// zlib's inflate of BGZF block b into buf[0, isize), checked against the block's length and CRC-32 footer
bool host_inflate_block(const cmb_bgzf_input* in, uint32_t b, std::vector<uint8_t>& buf) {
  const uint32_t isz = in->block_isize[b];
  if (buf.size() < (size_t)isz + 64) buf.resize((size_t)isz + 64);
  z_stream zs;
  memset(&zs, 0, sizeof zs);
  if (inflateInit2(&zs, -15) != Z_OK) return false;
  zs.next_in = const_cast<Bytef*>(in->data + in->block_coffset[b]);
  zs.avail_in = in->block_clen[b];
  zs.next_out = buf.data();
  zs.avail_out = isz;
  const bool ok = inflate(&zs, Z_FINISH) == Z_STREAM_END && zs.avail_out == 0;
  inflateEnd(&zs);
  uint32_t want_crc;
  memcpy(&want_crc, in->data + in->block_coffset[b] + in->block_clen[b], 4);
  return ok && (uint32_t)crc32(0, buf.data(), isz) == want_crc;
}

// The inflate kernels' arguments over blocks [b0, b1) of call j
InflateArgs inflate_args(const BgzfCall& j, uint32_t b0, uint32_t b1) {
  const auto& d = j.d;
  InflateArgs a{};
  a.comp = j.comp_base; a.coff = d.d_coff; a.clen = d.d_clen; a.isize = d.d_isize; a.uoff = d.d_ustart; a.scratch = d.d_t1_scratch;
  a.b0 = b0; a.b1 = b1; a.out = j.infl_base; a.status = d.d_status; a.ticket = d.d_tickets; a.fail_count = d.d_cnt + 0;
  return a;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ device memory
std::optional<uint64_t> cmb::decode_mem_limit() {
  const char* lim = getenv("CMB_DECODE_MEM_LIMIT_MB");
  if (!lim) return std::nullopt;
  return (uint64_t)(std::max(0.0, strtod(lim, nullptr)) * 1048576.0);
}

uint64_t cmb::decode_bytes(const cmb_ctx* c) {
  const auto& d = c->dec;
  return d.d_comp.bytes() + d.d_inflated.bytes() + d.d_tuple_slab.bytes() + d.d_rec_off.bytes() + c->sh.d_scan.bytes();
}

void cmb::release_decode(cmb_ctx* c) {
  cudaGetLastError();
  auto& d = c->dec;
  d.d_comp.release();
  d.d_inflated.release();
  d.d_tuple_slab.release();
  d.d_rec_off.release();
  c->sh.d_scan.release();
}

uint64_t cmb::device_room(uint64_t held) {
  if (const uint64_t lim = decode_mem_limit().value_or(0)) return lim;
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  cudaGetLastError();
  return free_b + held;
}

// ------------------------------------------------------------------------------------------------ the stages of one call

int BgzfCall::run() {
  int rc = prepare();
  if (!rc && !nothing_to_decode && !(rc = copy_inflate()) && !(rc = declined()) && !(rc = chain())) rc = extract();
  return rc;
}

// Stage 1: the block table, the blocks this call decodes, its copy windows, and every buffer, stream and copy slot it needs.
int BgzfCall::prepare() {
  ustart.assign((size_t)nb + 1, 0);
  for (uint32_t b = 0; b < nb; ++b) {
    if (in->block_coffset[b] + in->block_clen[b] + 8 > in->size) return fail(c, CMB_E_ARG, "cmb_submit_bgzf: block %u lies outside the data", b);
    ustart[b + 1] = ustart[b] + in->block_isize[b];
  }
  const uint64_t stream_total = ustart[nb];
  if (in->records_at > stream_total) return fail(c, CMB_E_ARG, "cmb_submit_bgzf: records_at beyond the end of the stream");
  if (in->records_at == stream_total) return CMB_OK;  // header only
  first_block = (uint32_t)(std::upper_bound(ustart.begin(), ustart.end(), in->records_at) - ustart.begin()) - 1;
  walk_end = data_end = nb;
  if (in->ranged) {
    if (in->walk_begin_block != first_block || in->walk_end_block > nb || in->walk_end_block < in->walk_begin_block)
      return fail(c, CMB_E_ARG, "cmb_submit_bgzf: inconsistent block range");
    walk_end = in->walk_end_block;
    if (walk_end == first_block) return CMB_OK;  // an empty share
    data_end = walk_end;
    uint64_t tail = 0;
    while (data_end < nb && tail < tail_bytes) tail += in->block_isize[data_end++];
  }
  nothing_to_decode = false;
  byte_lo = in->block_coffset[first_block];
  byte_hi = data_end == nb ? in->size : in->block_coffset[data_end - 1] + in->block_clen[data_end - 1] + 8;
  u_lo = ustart[first_block];
  total = ustart[data_end];  // end of the inflated bytes available to this call
  // ---- buffers
  if (const auto lim = decode_mem_limit())  // testing aid: behave as if the device had this much room
    if (((byte_hi - byte_lo) + (total - u_lo)) >> 20 > *lim >> 20) return CMB_E_NOMEM;
  int rc;
  const size_t comp_need = (size_t)(byte_hi - byte_lo) + DEC_FRONT + DEC_SLACK, infl_need = (size_t)(total - u_lo) + DEC_SLACK;
  if ((rc = d.d_comp.ensure(c, comp_need, with_slack(comp_need))) || (rc = d.d_inflated.ensure(c, infl_need, with_slack(infl_need))))
    return rc;
  comp_base = reinterpret_cast<uint8_t*>(reinterpret_cast<uintptr_t>(d.d_comp.p) + DEC_FRONT - byte_lo);
  infl_base = reinterpret_cast<uint8_t*>(reinterpret_cast<uintptr_t>(d.d_inflated.p) - u_lo);
  const size_t blocks_need = (size_t)nb + 1, blocks_want = (size_t)nb + nb / 8 + 64;
  for (auto* b : {&d.d_coff, &d.d_ustart, &d.d_guess, &d.d_exit, &d.d_rec_base, &d.d_cig_base})
    if ((rc = b->ensure(c, blocks_need, blocks_want))) return rc;
  for (auto* b : {&d.d_clen, &d.d_isize, &d.d_status, &d.d_nrec, &d.d_ncig, &d.d_dirty})
    if ((rc = b->ensure(c, blocks_need, blocks_want))) return rc;
  if ((rc = d.d_t1_scratch.ensure(c, blocks_need * T1_LENS_BYTES, blocks_want * T1_LENS_BYTES))) return rc;
  if ((rc = d.d_cnt.ensure(c, 20))) return rc;  // [16..19]: a sliced decode's held-back counts (decode_sliced)
  if (!d.have_events) {
    for (auto& e : d.ev) CU_TRY(c, cudaEventCreate(&e));
    d.have_events = true;
  }
  // ---- windows
  {
    uint32_t b = first_block;
    uint64_t byte0 = byte_lo;
    while (b < data_end) {
      uint32_t e = b;
      uint64_t byte1 = byte0;
      while (e < data_end && (e == b || in->block_coffset[e] + in->block_clen[e] + 8 - byte0 <= dec_window_bytes())) {
        byte1 = in->block_coffset[e] + in->block_clen[e] + 8;
        ++e;
      }
      if (e == data_end) byte1 = byte_hi;
      windows.push_back({b, e, byte0, byte1});
      b = e;
      byte0 = byte1;
    }
  }
  const size_t n_windows = windows.size();
  if ((rc = d.d_tickets.ensure(c, n_windows + 8, n_windows * 3 + 64))) return rc;  // [0] block ticket, [1, 1 + W) arrival flags
  if ((rc = d.d_block_window.ensure(c, nb, with_slack(nb)))) return rc;
  if (!d.h_ones) {
    if ((rc = d.h_ones.ensure(c, 16))) return rc;
    for (int k = 0; k < 16; ++k) d.h_ones.p[k] = 1;
  }
  // ---- copy threads, their streams and pinned slots
  cudaPointerAttributes attr{};
  src_pinned = cudaPointerGetAttributes(&attr, in->data) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();  // cudaPointerGetAttributes on pageable memory may leave a sticky-free error code
  const uint32_t T = std::min<uint32_t>(std::min<uint32_t>(in->copy_threads ? in->copy_threads : 4, 16), (uint32_t)n_windows);
  n_copy_threads = T;
  while (d.streams.size() < T) {
    cudaStream_t st;
    CU_TRY(c, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    d.streams.push_back(st);
    cudaEvent_t e;
    CU_TRY(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    d.done_events.push_back(e);
    for (int k = 0; k < 2; ++k) {
      CU_TRY(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      d.slot_events.push_back(e);
      PinnedBuf<uint8_t> slot;
      if ((rc = slot.ensure(c, DEC_COPY_CHUNK))) return rc;
      d.pinned.push_back(std::move(slot));
    }
  }
  return CMB_OK;
}

// Stage 2: the block table goes up on the context stream, the windows on the copy streams (one host thread each, a 4-byte
// arrival flag after each window), and the inflate kernel runs: one persistent launch before the copies whose threads wait for
// their window's flag, or (serial) one launch behind all the copies.
int BgzfCall::copy_inflate() {
  NvtxRange nvtx("bgzf: H2D copy + inflate");
  const uint32_t T = n_copy_threads;
  std::vector<uint32_t> block_window(nb, 0);
  for (size_t w = 0; w < windows.size(); ++w)
    for (uint32_t b = windows[w].b0; b < windows[w].b1; ++b) block_window[b] = (uint32_t)w;
  // ---- upload the block table, reset counters (ctx stream), then let the copy streams start after it
  CU_TRY(c, cudaEventRecord(d.ev[0], c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_coff, in->block_coffset, 8ull * nb, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_clen, in->block_clen, 4ull * nb, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_isize, in->block_isize, 4ull * nb, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_ustart, ustart.data(), 8ull * (nb + 1), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_cnt, 0, 64, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_status, 0, 4ull * nb, c->stream));
  CU_TRY(c, cudaMemcpyAsync(d.d_block_window, block_window.data(), 4ull * nb, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_tickets, 0, 4 * (windows.size() + 1), c->stream));
  CU_TRY(c, cudaMemsetAsync(infl_base + total, 0, DEC_SLACK, c->stream));
  CU_TRY(c, cudaMemsetAsync(comp_base + byte_hi, 0, DEC_SLACK, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_comp, 0, DEC_FRONT, c->stream));
  CU_TRY(c, cudaEventRecord(d.ev[1], c->stream));
  for (uint32_t t = 0; t < T; ++t) CU_TRY(c, cudaStreamWaitEvent(d.streams[t], d.ev[1], 0));
  const bool serial = windows.size() <= 1 || inflate_serial_requested();
  bool crc_pending = false;
  InflateArgs persistent = inflate_args(*this, first_block, data_end);
  int rc;
  if (!serial) {  // one persistent launch over every block; its warps wait for their block's window to arrive
    persistent.block_window = d.d_block_window;
    persistent.ready = d.d_tickets + 1;
    if ((rc = launch_inflate(c, persistent, c->stream, &crc_pending))) return rc;
  }
  std::atomic<size_t> next_window{0};
  std::atomic<int> first_err{0};
  auto worker = [&](uint32_t t) {
    cudaSetDevice(c->device);
    cudaStream_t st = d.streams[t];
    int slot = 0;
    bool used[2] = {false, false};
    auto check = [&](cudaError_t e) {
      if (e != cudaSuccess) {
        int z = 0;
        first_err.compare_exchange_strong(z, (int)e);
      }
      return e == cudaSuccess;
    };
    for (;;) {
      const size_t w = next_window.fetch_add(1);
      if (w >= windows.size() || first_err.load()) break;
      const Window& win = windows[w];
      if (src_pinned) {
        if (!check(cudaMemcpyAsync(comp_base + win.byte0, in->data + win.byte0, win.byte1 - win.byte0, cudaMemcpyHostToDevice, st))) break;
      } else {
        for (uint64_t o = win.byte0; o < win.byte1; o += DEC_COPY_CHUNK) {
          const size_t n = (size_t)std::min<uint64_t>(DEC_COPY_CHUNK, win.byte1 - o);
          const size_t si = (size_t)t * 2 + slot;
          if (used[slot] && !check(cudaEventSynchronize(d.slot_events[si]))) return;
          memcpy(d.pinned[si], in->data + o, n);
          if (!check(cudaMemcpyAsync(comp_base + o, d.pinned[si], n, cudaMemcpyHostToDevice, st))) return;
          if (!check(cudaEventRecord(d.slot_events[si], st))) return;
          used[slot] = true;
          slot ^= 1;
        }
      }
      if (!check(cudaMemcpyAsync(d.d_tickets + 1 + w, d.h_ones, 4, cudaMemcpyHostToDevice, st))) break;  // window w has arrived
    }
    check(cudaEventRecord(d.done_events[t], st));
  };
  const auto copy_t0 = std::chrono::steady_clock::now();
  {
    std::vector<std::thread> threads;
    for (uint32_t t = 1; t < T; ++t) threads.emplace_back(worker, t);
    worker(0);
    for (auto& th : threads) th.join();
  }
  const double copy_wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - copy_t0).count();
  out->ms_copy_enqueue_wall = (float)copy_wall_ms;
  if (crc_pending && (rc = launch_crc32(c, persistent, c->stream))) return rc;  // every copy is enqueued: nothing left to hold up
  if (serial && !first_err.load()) {
    for (uint32_t t = 0; t < T; ++t) CU_TRY(c, cudaStreamWaitEvent(c->stream, d.done_events[t], 0));
    if ((rc = launch_inflate(c, inflate_args(*this, first_block, data_end), c->stream))) return rc;
  }
  if (first_err.load()) {  // release the warps still waiting for windows that will never arrive
    cudaMemsetAsync(d.d_tickets + 1, 1, 4 * windows.size(), d.streams[0]);
    cudaStreamSynchronize(d.streams[0]);
    cudaStreamSynchronize(c->stream);
  }
  out->n_launches = 1;
  out->h2d_bytes = (byte_hi - byte_lo) + 24ull * nb + 8;
  if (first_err.load()) return fail(c, CMB_E_CUDA, "cmb_submit_bgzf: copy/inflate stage failed: %s", cudaGetErrorString((cudaError_t)first_err.load()));
  for (uint32_t t = 0; t < T; ++t) CU_TRY(c, cudaStreamWaitEvent(c->stream, d.done_events[t], 0));
  if (getenv("CMB_PIPELINE_STATS")) {  // how long the window copies alone took (the done events carry no timing: time them on the host)
    const auto h0 = std::chrono::steady_clock::now();
    for (uint32_t t = 0; t < T; ++t) cudaEventSynchronize(d.done_events[t]);
    const double wait_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - h0).count();
    fprintf(stderr, "#decode_h2d\twindows=%zu\tbytes=%llu\tcopy_streams_done_after_ms=%.1f (host clock from the end of the enqueue; enqueue took %.1f ms)\n",
            windows.size(), (unsigned long long)(byte_hi - byte_lo), wait_ms, copy_wall_ms);
  }
  CU_TRY(c, cudaEventRecord(d.ev[2], c->stream));
  if (getenv("CMB_DECODE_PROFILE")) {  // debugging aid: the inflate kernel alone, all blocks resident, one launch
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    cudaEvent_t p0, p1;
    cudaEventCreate(&p0);
    cudaEventCreate(&p1);
    CU_TRY(c, cudaMemsetAsync(d.d_tickets, 0, 4, c->stream));
    InflateArgs a = inflate_args(*this, first_block, data_end);
    a.fail_count = d.d_cnt + 8;
    cudaEventRecord(p0, c->stream);
    if ((rc = launch_inflate(c, a, c->stream))) return rc;
    cudaEventRecord(p1, c->stream);
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, p0, p1);
    fprintf(stderr, "#decode_profile\tinflate_only_ms=%.3f\tblocks=%u\tcompressed=%llu\tinflated=%llu\tinflated_GBps=%.2f\tcopy_threads=%u\tsrc_pinned=%d\tcopy_enqueue_wall_ms=%.2f\n", ms, data_end - first_block,
            (unsigned long long)(byte_hi - byte_lo), (unsigned long long)(total - u_lo), (total - u_lo) / ms * 1e-6, T, (int)src_pinned, copy_wall_ms);
    cudaEventDestroy(p0);
    cudaEventDestroy(p1);
  }
  return CMB_OK;
}

// Stage 3: blocks the first pass declined get a second device pass, then zlib on the host, patched into the inflated stream.
int BgzfCall::declined() {
  NvtxRange nvtx("bgzf: declined blocks (second pass, host zlib)");
  uint32_t h_cnt[16];
  CU_TRY(c, cudaMemcpyAsync(h_cnt, d.d_cnt, 64, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  std::vector<uint8_t> tmp;
  if (h_cnt[0] || getenv("CMB_DECODE_RETRY_TEST")) {
    std::vector<uint32_t> status(nb);
    CU_TRY(c, cudaMemcpy(status.data(), d.d_status, 4ull * nb, cudaMemcpyDeviceToHost));
    if (getenv("CMB_DECODE_RETRY_TEST"))  // testing aid: pretend every 7th block was declined by the first pass (code 29)
      for (uint32_t b = first_block; b < data_end; b += 7) status[b] = 29;
    if (getenv("CMB_DECODE_VERIFY") || getenv("CMB_PIPELINE_STATS")) {
      uint32_t hist[32] = {0};
      for (uint32_t b = 0; b < nb; ++b) hist[std::min<uint32_t>(status[b], 31)]++;
      fprintf(stderr, "#decode_status");
      for (int k = 0; k < 32; ++k)
        if (hist[k]) fprintf(stderr, "\t%d:%u", k, hist[k]);
      fprintf(stderr, "\n");
    }
    // Second chance on the device: the one-stream-per-warp kernel has larger Huffman tables (10-bit roots, 128 long-code
    // prefixes) than the four-streams-per-warp one, so most blocks the first pass declined for table space fit there.
    std::vector<uint32_t> again;
    for (uint32_t b = first_block; b < data_end; ++b)
      if (status[b] != INF_OK) again.push_back(b);
    out->n_blocks_second_pass = (uint32_t)again.size();
    if (!again.empty()) {
      uint32_t* d_list = d.d_dirty;  // free until the record chain starts (nb entries)
      CU_TRY(c, cudaMemcpyAsync(d_list, again.data(), 4ull * again.size(), cudaMemcpyHostToDevice, c->stream));
      CU_TRY(c, cudaMemsetAsync(d.d_tickets, 0, 4, c->stream));
      CU_TRY(c, cudaMemsetAsync(d.d_cnt, 0, 4, c->stream));
      InflateArgs a = inflate_args(*this, 0, (uint32_t)again.size());
      a.block_list = d_list;
      if (int rc = launch_inflate(c, a, c->stream)) return rc;
      out->n_launches += 1;
      std::vector<uint32_t> st2(nb);
      CU_TRY(c, cudaMemcpyAsync(st2.data(), d.d_status, 4ull * nb, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaStreamSynchronize(c->stream));
      for (uint32_t b : again) status[b] = st2[b];
    }
    for (uint32_t b = first_block; b < data_end; ++b) {
      if (status[b] == INF_OK) continue;
      if (!host_inflate_block(in, b, tmp)) return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: BGZF block %u does not inflate", b);
      CU_TRY(c, cudaMemcpy(infl_base + ustart[b], tmp.data(), in->block_isize[b], cudaMemcpyHostToDevice));
      out->n_blocks_host += 1;
    }
  }
  if (getenv("CMB_DECODE_VERIFY")) {  // debugging aid: compare every device-inflated block with zlib's output
    std::vector<uint8_t> dev(total - u_lo);
    CU_TRY(c, cudaMemcpy(dev.data(), d.d_inflated, total - u_lo, cudaMemcpyDeviceToHost));
    uint32_t bad = 0;
    for (uint32_t b = first_block; b < data_end; ++b) {
      const uint32_t isz = in->block_isize[b];
      if (!isz) continue;
      const uint8_t* got = dev.data() + (ustart[b] - u_lo);
      const bool zlib_ok = host_inflate_block(in, b, tmp);
      if (!zlib_ok || memcmp(tmp.data(), got, isz) != 0) {
        uint32_t k = 0;
        while (k < isz && tmp[k] == got[k]) ++k;
        if (bad < 8) fprintf(stderr, "#decode_verify\tblock %u (clen %u isize %u): zlib %s, first difference at byte %u\n", b, in->block_clen[b], isz, zlib_ok ? "ok" : "failed", k);
        ++bad;
      }
    }
    fprintf(stderr, "#decode_verify\t%u of %u blocks differ from zlib; %u inflated on the host\n", bad, data_end - first_block, out->n_blocks_host);
  }
  return CMB_OK;
}

// Stage 4: the record chain -- a guessed first record per block, walked to the block's end, verified against the neighbour's
// guess (repaired and re-walked until it settles), then the record and CIGAR bases of every block.
int BgzfCall::chain() {
  NvtxRange nvtx("bgzf: record chain (guess, walk, verify, offsets)");
  WalkArgs wa{};
  // The chain is walked over [first_block, walk_hi): one block past the range when there is one, so that the range's last
  // record boundary is also checked against an independent guess.
  const uint32_t walk_hi = std::min<uint32_t>(walk_end + 1, data_end);
  wa.data = infl_base; wa.total = total; wa.ustart = d.d_ustart; wa.first_block = first_block; wa.n_blocks = walk_hi;
  wa.records_at = in->records_at; wa.n_ref = (int32_t)in->n_ref; wa.guess = d.d_guess; wa.exit_off = d.d_exit; wa.n_rec = d.d_nrec;
  wa.n_cig = d.d_ncig; wa.dirty = d.d_dirty; wa.flags = d.d_cnt + 1; wa.only_dirty = 0;
  const uint32_t nwb = walk_hi - first_block;
  CU_TRY(c, cudaMemsetAsync(d.d_dirty, 0, 4ull * nb, c->stream));
  kd_guess<<<(nwb * 32 + 255) / 256, 256, 0, c->stream>>>(wa);
  kd_walk<<<(nwb + 127) / 128, 128, 0, c->stream>>>(wa);
  CU_TRY(c, cudaGetLastError());
  out->n_launches += 2;
  uint32_t h_cnt[16];
  uint64_t h_exit = 0;
  for (uint32_t round = 0;; ++round) {
    if (nwb > 1) {
      CU_TRY(c, cudaMemsetAsync(d.d_cnt + 2, 0, 4, c->stream));
      kd_verify<<<(nwb - 1 + 255) / 256, 256, 0, c->stream>>>(wa);
      CU_TRY(c, cudaGetLastError());
      out->n_launches += 1;
    }
    CU_TRY(c, cudaMemcpyAsync(h_cnt, d.d_cnt, 64, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaMemcpyAsync(&h_exit, d.d_exit + (walk_end - 1), 8, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    if (nwb <= 1 || !h_cnt[2]) break;
    if (round >= 256) return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: record chain did not settle");
    out->chain_repairs += 1;
    out->n_launches += 1;
    wa.only_dirty = 1;
    kd_walk<<<(nwb + 127) / 128, 128, 0, c->stream>>>(wa);
    CU_TRY(c, cudaGetLastError());
  }
  if (walk_end == nb ? h_exit != ustart[nb] : (h_exit == WALK_UNKNOWN || h_exit > total)) {
    tail_short = walk_end != nb && data_end < nb;
    return fail(c, CMB_E_DECLINED, walk_end == nb ? "cmb_submit_bgzf: record chain does not end at the end of the stream"
                                                  : "cmb_submit_bgzf: a record runs past the inflated tail of the block range");
  }
  exit_off = h_exit;
  kd_scan_items<<<1, 1024, 0, c->stream>>>(d.d_nrec, d.d_ncig, first_block, walk_end, d.d_rec_base, d.d_cig_base, (uint64_t*)(d.d_cnt + 6));
  CU_TRY(c, cudaGetLastError());
  out->n_launches += 1;
  uint64_t totals[2] = {0, 0};
  CU_TRY(c, cudaMemcpyAsync(totals, d.d_cnt + 6, 16, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  CU_TRY(c, cudaEventRecord(d.ev[3], c->stream));
  n_rec = totals[0];
  n_cig = totals[1];
  return CMB_OK;
}

// Stage 5: the per-record tuples, mate matching when a pair filter needs it, and K1 over the tuples (not for cmb_decode_bgzf).
int BgzfCall::extract() {
  NvtxRange nvtx("bgzf: extract, mate matching, K1");
  if (n_rec >= 0xffffff00ull || n_cig >= 0xffffff00ull) return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: more than 2^32 records or cigar operations");
  out->n_records = n_rec;
  out->n_intervals = n_cig;
  if (!n_rec) {
    CU_TRY(c, cudaEventRecord(d.ev[4], c->stream));
    CU_TRY(c, cudaEventRecord(d.ev[5], c->stream));
    return CMB_OK;
  }
  int rc;
  size_t offs[13];
  const size_t slab_need = batch_slab_bytes((uint32_t)n_rec, (uint32_t)n_cig, offs);
  if ((rc = d.d_rec_off.ensure(c, n_rec, with_slack(n_rec))) || (rc = d.d_tuple_slab.ensure(c, slab_need, slab_need + slab_need / 8)))
    return rc;
  cmb_read_batch tb;
  carve_batch(d.d_tuple_slab, (uint32_t)n_rec, (uint32_t)n_cig, &tb);
  d.last_n_rec = (uint32_t)n_rec;
  d.last_n_cig = (uint32_t)n_cig;
  OffsetArgs oa{};
  oa.data = infl_base; oa.ustart = d.d_ustart; oa.guess = d.d_guess; oa.rec_base = d.d_rec_base; oa.cig_base = d.d_cig_base;
  oa.first_block = first_block; oa.n_blocks = walk_end; oa.rec_off = d.d_rec_off; oa.iv_begin = tb.iv_begin; oa.n_records = n_rec; oa.n_cig_total = n_cig;
  kd_offsets<<<(walk_end - first_block + 127) / 128, 128, 0, c->stream>>>(oa);
  CU_TRY(c, cudaGetLastError());
  ExtractArgs ea{};
  ea.data = infl_base; ea.rec_off = d.d_rec_off; ea.n_records = n_rec;
  ea.own_lo = in->ranged ? in->own_tid_begin : INT_MIN; ea.own_hi = in->ranged ? in->own_tid_end : INT_MAX;
  ea.own_unplaced = in->ranged ? in->own_unplaced : 1u; ea.n_owned = (unsigned long long*)(d.d_cnt + 10);
  ea.tid = tb.tid; ea.pos = tb.pos; ea.flag = tb.flag; ea.mapq = tb.mapq; ea.nm_state = tb.nm_state; ea.nm = tb.nm; ea.l_seq = tb.l_seq;
  ea.aligned = tb.aligned; ea.del = tb.del; ea.ins = tb.ins; ea.iv_begin = tb.iv_begin; ea.iv_start = tb.iv_start; ea.iv_len = tb.iv_len;
  ea.n_primary = (unsigned long long*)(d.d_cnt + 4); ea.flags = d.d_cnt + 1;
  kd_extract<<<(uint32_t)((n_rec + 255) / 256), 256, 0, c->stream>>>(ea);
  CU_TRY(c, cudaGetLastError());
  out->n_launches += 2;
  uint32_t h_cnt[16];
  CU_TRY(c, cudaMemcpyAsync(h_cnt, d.d_cnt, 64, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (h_cnt[1]) return fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: malformed alignment record (flags %u)", h_cnt[1]);
  memcpy(&out->n_primary, h_cnt + 4, 8);
  memcpy(&out->n_records, h_cnt + 10, 8);  // records this call owns (all of them unless ranged)
  d.last_valid = true;
  d.last_mate = nullptr;
  d.last_infl_base = infl_base;
  // mate matching on the device (filter.rs:117-233; cmb_pairs.cuh) for coverage when the pair thresholds apply; `coverm
  // filter` matches in cmb_filter_plan, where --inverse (which decides the eligible records) is known
  if (!decode_only && c->mode.filter_pairs) {
    if ((rc = match_mates(c, infl_base, (uint32_t)n_rec, true, "cmb_submit_bgzf"))) return rc;
    out->n_launches += 5;
  }
  CU_TRY(c, cudaEventRecord(d.ev[4], c->stream));
  if (k1_active(c) && !decode_only) {
    uint32_t excl = 0;
    if ((rc = excl_n(&excl))) return rc;
    d.last_excl_n = excl;
    if ((rc = launch_k1(c, tb, (uint32_t)n_rec, (uint32_t)n_cig, excl, d.last_mate))) return rc;
  }
  CU_TRY(c, cudaEventRecord(d.ev[5], c->stream));
  return CMB_OK;
}

// K1's excl_n for the call's records: those that start before excl_end_block are this rank's exclusive share of the stream
// (cmb_kept_tid_range) -- none when the block lies before the range, all when it lies after it
int BgzfCall::excl_n(uint32_t* n) {
  *n = 0xffffffffu;
  if (in->ranged && in->excl_end_block < walk_end) {
    if (in->excl_end_block <= first_block) *n = 0;
    else {
      uint64_t base = 0;
      CU_TRY(c, cudaMemcpyAsync(&base, d.d_rec_base + in->excl_end_block, 8, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaStreamSynchronize(c->stream));
      *n = (uint32_t)base;
    }
  }
  return CMB_OK;
}

int BgzfCall::stage_times() {
  CU_TRY(c, cudaEventSynchronize(d.ev[4]));
  cudaEventElapsedTime(&out->ms_copy_inflate, d.ev[0], d.ev[2]);
  cudaEventElapsedTime(&out->ms_chain, d.ev[2], d.ev[3]);
  cudaEventElapsedTime(&out->ms_extract, d.ev[3], d.ev[4]);
  cudaEventElapsedTime(&out->ms_total, d.ev[0], d.ev[4]);
  return CMB_OK;
}

// ------------------------------------------------------------------------------------------------ mate matching
int cmb::match_mates(cmb_ctx* c, const uint8_t* infl_base, uint32_t n_rec, bool filter_out, const char* who, uint32_t carry,
                     uint32_t* largest) {
  auto& d = c->dec;
  int rc;
  d.last_mate = nullptr;
  d.filter_planned = false;
  if (d.d_pair_key.cap < n_rec) {  // growing: give the filter's buffers back first (cmb_filter_plan sizes them again)
    d.d_filter_anchor.release();
    d.d_filter_role.release();
    d.d_filter_out.release();
  }
  const size_t want = with_slack(n_rec);
  const uint32_t n_chunks = (n_rec + PAIR_ORDER_CHUNK - 1) / PAIR_ORDER_CHUNK;
  if ((rc = d.d_pair_key.ensure(c, n_rec, want)) || (rc = d.d_pair_mate.ensure(c, n_rec, want)) || (rc = d.d_pair_next.ensure(c, n_rec, want)) ||
      (rc = d.d_pair_order.ensure(c, n_chunks, with_slack(n_chunks))))
    return rc;
  size_t table = 1u << 16;
  while (table < 2 * (size_t)n_rec) table <<= 1;
  if ((rc = d.d_pair_tag.ensure(c, table)) || (rc = d.d_pair_head.ensure(c, table))) return rc;
  CU_TRY(c, cudaMemsetAsync(d.d_pair_tag, 0, 8 * table, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_pair_head, 0xff, 4 * table, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.d_cnt + 1, 0, 4, c->stream));
  PairArgs pa{};
  pa.data = infl_base; pa.rec_off = d.d_rec_off; pa.n_records = n_rec; pa.key = d.d_pair_key; pa.mate = d.d_pair_mate;
  pa.next = d.d_pair_next; pa.slot_tag = d.d_pair_tag; pa.slot_head = d.d_pair_head; pa.table_mask = (uint32_t)(table - 1);
  pa.flags = d.d_cnt + 1; pa.order = d.d_pair_order; pa.filter_out = filter_out ? 1 : 0;
  const uint32_t gr = (n_rec + 255) / 256;
  kd_pair_keys<<<gr, 256, 0, c->stream>>>(pa);
  kd_pair_order<<<(n_chunks + 255) / 256, 256, 0, c->stream>>>(pa);
  kd_pair_order_fold<<<1, 1024, 0, c->stream>>>(d.d_pair_order, n_chunks, pa.flags, carry, largest);
  kd_pair_insert<<<gr, 256, 0, c->stream>>>(pa);
  kd_pair_resolve<<<(uint32_t)((table + 255) / 256), 256, 0, c->stream>>>(pa);
  CU_TRY(c, cudaGetLastError());
  uint32_t flags = 0;
  CU_TRY(c, cudaMemcpyAsync(&flags, d.d_cnt + 1, 4, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (flags)
    return fail(c, CMB_E_DECLINED, "%s: mate matching gave up (flags %u: %s)", who, flags,
                (flags & DEC_ERR_PAIR_ORDER) ? "the proper-pair records' reference ids are not sorted" : "too many records of one name");
  d.last_mate = d.d_pair_mate;
  d.last_mate_inverse = !filter_out;
  return CMB_OK;
}

void cmb::launch_scan(cmb_ctx* c, unsigned long long* v, uint32_t n) { kf_scan<<<1, 1024, 0, c->stream>>>(v, n); }

// ------------------------------------------------------------------------------------------------ entry points
namespace {

int submit_bgzf_impl(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out, bool decode_only) {
  NvtxRange nvtx_fn("cmb_submit_bgzf");
  if (!c || !in || !out || !in->data || !in->block_coffset || !in->block_clen || !in->block_isize)
    return fail(c, CMB_E_ARG, "cmb_submit_bgzf: null argument");
  if (!decode_only && !c->in_sample) return fail(c, CMB_E_ARG, "cmb_submit_bgzf: no sample in progress");
  if (decode_only && (c->in_sample || !c->have_params)) return fail(c, CMB_E_ARG, "cmb_decode_bgzf: set the parameters first; not inside a sample");
  if (c->n_acquired) return fail(c, CMB_E_ARG, "cmb_submit_bgzf: a staging batch is still acquired");
  *out = cmb_bgzf_result{};
  if (in->n_blocks == 0) return CMB_OK;
  CU_TRY(c, cudaSetDevice(c->device));
  BgzfCall j{c, c->dec, in, out, decode_only, in->n_blocks};
  const int rc = j.run();
  if (rc || j.nothing_to_decode) return rc;
  return j.stage_times();
}

// A whole-stream call that ran out of device memory did so before anything was accumulated (K1) or handed over (the filter's
// sink): its buffers go back, so that the rest has room, and slices() takes the stream instead.
template <class Slices>
int whole_or_slices(cmb_ctx* c, int rc, Slices slices) {
  if (rc != CMB_E_NOMEM) return rc;
  release_decode(c);
  return slices();
}

// Device bytes of the mate-matching buffers
uint64_t pair_bytes(const cmb_ctx* c) {
  const auto& d = c->dec;
  return d.d_pair_key.bytes() + d.d_pair_mate.bytes() + d.d_pair_next.bytes() + d.d_pair_tag.bytes() + d.d_pair_head.bytes();
}

// Pair mode: the mates of the slice j decoded, matched after the slices before it (`carry`: their largest eligible tid), and
// unless it is the stream's `last` slice, the trailing run of its last eligible tid held back for the next one (cmb_slices.hpp).
// *largest: the slice's largest eligible tid; *cut: the records it keeps, and when that is fewer than it decoded, *next: record
// `cut`'s offset, where the next slice starts.  A run that is the whole slice declines, the message naming the entry point
// (`who`) and where the stream goes instead (`host_route`).  SLICE_HALVE when mate matching runs out of memory.
int pair_cut(BgzfCall& j, bool filter_out, uint32_t carry, bool last, const char* who, const char* host_route, uint32_t* largest,
             uint32_t* cut, uint64_t* next) {
  cmb_ctx* c = j.c;
  auto& d = j.d;
  const uint32_t n = (uint32_t)j.n_rec;
  // words 12..14 of d_cnt: the slice's largest eligible tid, then the cut's `after` and n - cut (zeroed by copy_inflate)
  uint32_t* w = d.d_cnt + 12;
  const int rc = match_mates(c, d.last_infl_base, n, filter_out, who, carry, w);
  if (rc == CMB_E_NOMEM) return SLICE_HALVE;
  if (rc) return rc;
  j.out->n_launches += 5;
  if (!last) {
    cmb_read_batch tb;
    carve_batch(d.d_tuple_slab, n, (uint32_t)j.n_cig, &tb);
    const uint32_t g = (n + 255) / 256;
    kd_pair_cut_after<<<g, 256, 0, c->stream>>>(d.d_pair_key, tb.tid, n, w, w + 1);
    kd_pair_cut_at<<<g, 256, 0, c->stream>>>(d.d_pair_key, tb.tid, n, w, w + 1, w + 2);
    CU_TRY(c, cudaGetLastError());
    j.out->n_launches += 2;
  }
  uint32_t h[3] = {0, 0, 0};
  CU_TRY(c, cudaMemcpyAsync(h, w, 12, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  *largest = h[0];
  *cut = n - h[2];
  if (*cut == 0)
    return fail(c, CMB_E_DECLINED, "%s: the proper-pair records of reference %d do not fit in one decode slice; %s", who, (int32_t)h[0],
                host_route);
  if (*cut < n) {
    CU_TRY(c, cudaMemcpyAsync(next, d.d_rec_off + *cut, 8, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
  }
  return CMB_OK;
}

// An ordinary stream (the whole stream, or a rank's block range in a group) in block slices (decode_in_slices), for the
// sliced decode (decode_sliced) and the sliced filter (FilterCall::sliced): in `pair` mode each slice is cut (pair_cut), then
// work(j, r, cut) takes its records [0, cut).
//   held()  device bytes the caller holds that count as room, since they are reused or freed to grow
//   events  K1 appends to the sample's event list: the budget keeps room for its growth
//   other() bytes the last slice needed beside its compressed and inflated bytes (the budget's `side`, per byte of those)
// CMB_PIPELINE_STATS prints #<stats>_slices.  Every exit releases the decode buffers: what comes next needs the room, and a
// sliced decode has no resident stream to keep.
template <class Held, class Other, class Work>
int stream_in_slices(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out, SliceStats& ss, const char* who, const char* host_route,
                     const char* stats, bool pair, bool filter_out, bool events, Held held, Other other, Work work) {
  auto room = [&] { return device_room(held()); };
  if (room() < SLICE_MIN_BYTES) {
    const int rc = fail(c, CMB_E_DECLINED, "%s: not enough device memory for device-side decode", who);
    release_decode(c);
    return rc;
  }
  const uint32_t walk_end = in->ranged ? std::min(in->walk_end_block, in->n_blocks) : in->n_blocks;
  uint64_t stream_end = 0;  // end of the inflated bytes whose records are walked
  for (uint32_t b = 0; b < walk_end; ++b) stream_end += in->block_isize[b];
  const uint64_t iv0 = c->n_intervals;
  double side = 0;     // the last slice's other buffers per compressed + inflated byte
  uint32_t carry = 0;  // pair mode: the largest eligible tid of the slices so far
  auto budget = [&](uint64_t at) -> uint64_t {
    const uint64_t done = at > in->records_at ? at - in->records_at : 0;
    const uint64_t total = stream_end > in->records_at ? stream_end - in->records_at : 0;
    return decode_slice_budget(room(), events, c->d_events.bytes(), done, total, c->n_intervals - iv0, side);
  };
  auto step = [&](BgzfCall& j, cmb_bgzf_result& r, uint64_t* next) -> int {
    const uint32_t n = (uint32_t)j.n_rec;
    uint32_t cut = n, largest = carry;
    int rc;
    if (pair) {
      const auto t0 = std::chrono::steady_clock::now();
      if ((rc = pair_cut(j, filter_out, carry, j.walk_end >= walk_end, who, host_route, &largest, &cut, next))) return rc;
      ss.ms_mates += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    if ((rc = work(j, r, cut))) return rc;
    carry = largest;
    ss.pair_cut_records += n - cut;
    side = (double)other() / (double)std::max<uint64_t>(1, (j.byte_hi - j.byte_lo) + (j.total - j.u_lo));
    return CMB_OK;
  };
  auto nomem = [&](const SliceBlocks&, uint32_t, uint32_t, uint64_t) {
    return fail(c, CMB_E_DECLINED, "%s: not enough device memory for device-side decode", who);
  };
  const int rc = decode_in_slices(c, in, out, ss, budget, step, nomem);
  release_decode(c);
  if (rc) return rc;
  if (getenv("CMB_PIPELINE_STATS"))
    fprintf(stderr, "#%s_slices\tslices=%u\tmax_slice_bytes=%llu\thalvings=%u\tpair_cut_records=%llu\n", stats, ss.n_slices,
            (unsigned long long)ss.max_slice, ss.halvings, (unsigned long long)ss.pair_cut_records);
  return CMB_OK;
}

// cmb_submit_bgzf when the whole-stream buffers do not fit: each slice submitted to K1 as one batch at the sample's running
// interval base, in pair mode only up to its cut.  A decline leaves the sample as cmb_begin_sample left it, for the host decoder.
int decode_sliced(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out) {
  auto& d = c->dec;
  *out = cmb_bgzf_result{};
  const bool pair = c->mode.filter_pairs;
  auto work = [&](BgzfCall& j, cmb_bgzf_result& r, uint32_t cut) -> int {
    const uint32_t n = (uint32_t)j.n_rec;
    uint32_t iv_sub = (uint32_t)j.n_cig;
    cmb_read_batch tb;
    carve_batch(d.d_tuple_slab, n, (uint32_t)j.n_cig, &tb);
    if (cut < n) {  // records [cut, n) start the next slice: they leave this slice's counters
      CU_TRY(c, cudaMemcpyAsync(&iv_sub, tb.iv_begin + cut, 4, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaMemsetAsync(d.d_cnt + 16, 0, 16, c->stream));
      kd_count_held<<<(n - cut + 255) / 256, 256, 0, c->stream>>>(tb.tid, tb.flag, cut, n, j.in->own_tid_begin, j.in->own_tid_end, j.in->own_unplaced,
                                                                 (unsigned long long*)(d.d_cnt + 16), (unsigned long long*)(d.d_cnt + 18));
      CU_TRY(c, cudaGetLastError());
      uint64_t held[2] = {0, 0};
      CU_TRY(c, cudaMemcpyAsync(held, d.d_cnt + 16, 16, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaStreamSynchronize(c->stream));
      r.n_primary -= held[0];
      r.n_records -= held[1];
      r.n_intervals = iv_sub;
      r.n_launches += 1;
    }
    if (!k1_active(c)) return CMB_OK;
    uint32_t excl = 0;
    if (int rc = j.excl_n(&excl)) return rc;
    const int rc = launch_k1(c, tb, cut, iv_sub, excl, pair ? d.d_pair_mate.p : nullptr);
    return rc == CMB_E_NOMEM ? SLICE_HALVE : rc;  // the event list did not grow: nothing of the slice was accumulated
  };
  SliceStats ss;
  const int rc = stream_in_slices(
      c, in, out, ss, "cmb_submit_bgzf", "mates are matched on the host", "decode", pair, true, !c->gene_mode, [&] { return decode_bytes(c); },
      [&] { return d.d_tuple_slab.bytes() + d.d_rec_off.bytes() + (pair ? pair_bytes(c) : 0); }, work);
  if (rc == CMB_E_DECLINED)
    if (int e = reset_sample(c)) return e;
  if (rc) return rc;
  out->ms_copy_inflate = ss.ms_inflate;
  out->ms_chain = ss.ms_chain;
  out->ms_extract = ss.ms_extract;
  return CMB_OK;
}

int bgzf_entry(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out, bool decode_only) {
  if (c) {
    c->dec.last_valid = false;
    c->dec.filter_planned = false;
  }
  const auto t_call0 = std::chrono::steady_clock::now();
  const int rc = whole_or_slices(c, submit_bgzf_impl(c, in, out, decode_only), [&] {
    return decode_only ? fail(c, CMB_E_DECLINED, "cmb_submit_bgzf: not enough device memory for device-side decode") : decode_sliced(c, in, out);
  });
  if (out) out->ms_host_wall = (float)std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_call0).count();
  return rc;
}

// The filter kernels over records [0, n) of the resident decode, its mates matched on the pair path (filter.rs:117-233; else
// the singles path, filter.rs:88-116): kf_decide, kf_scan, and kf_gather of the *total bytes of the *n_emit returned records
// into d_filter_out.
int filter_kernels(cmb_ctx* c, bool pair_path, int inverse, uint32_t n, uint64_t* total, uint64_t* n_emit) {
  auto& d = c->dec;
  int rc;
  if ((rc = d.d_filter_anchor.ensure(c, (size_t)n + 1, with_slack(n))) || (rc = d.d_filter_role.ensure(c, (size_t)n + 1, with_slack(n))))
    return rc;
  cmb_read_batch tb;
  carve_batch(d.d_tuple_slab, d.last_n_rec, d.last_n_cig, &tb);
  FilterArgs a{};
  a.data = d.last_infl_base; a.rec_off = d.d_rec_off; a.n = n; a.flag = tb.flag; a.mapq = tb.mapq; a.nm_state = tb.nm_state; a.nm = tb.nm;
  a.l_seq = tb.l_seq; a.aligned = tb.aligned; a.del = tb.del; a.mate = pair_path ? d.last_mate : nullptr; a.p = c->params;
  a.filter_single = c->mode.filter_single_reads; a.pair_path = pair_path; a.filter_out = inverse ? 0 : 1;
  a.anchor_bytes = d.d_filter_anchor; a.role = d.d_filter_role; a.error_flags = d.d_cnt + 12; a.n_emit = (unsigned long long*)(d.d_cnt + 14);
  CU_TRY(c, cudaMemsetAsync(d.d_cnt + 12, 0, 16, c->stream));
  kf_decide<<<(n + 255) / 256, 256, 0, c->stream>>>(a);
  kf_scan<<<1, 1024, 0, c->stream>>>(d.d_filter_anchor, n);
  CU_TRY(c, cudaGetLastError());
  uint32_t h[4];
  CU_TRY(c, cudaMemcpyAsync(h, d.d_cnt + 12, 16, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(total, d.d_filter_anchor + n, 8, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (h[0] & ERR_NM) return fail(c, CMB_E_NM, "%s", NM_PANIC);
  memcpy(n_emit, h + 2, 8);
  if (!*total) return CMB_OK;
  if ((rc = d.d_filter_out.ensure(c, *total, (size_t)*total + (size_t)*total / 8 + 4096))) return rc;
  a.out = d.d_filter_out;
  kf_gather<<<(n + 7) / 8, 256, 0, c->stream>>>(a);
  CU_TRY(c, cudaGetLastError());
  return CMB_OK;
}
}  // namespace

// Device memory for the whole-stream decode buffers (compressed file + inflated stream + tuples) is requested before anything
// is accumulated; when it runs out, the stream is decoded in block slices (decode_sliced), and a sample that declines there is
// reset to its empty state first, so that the host decoder can take it over with only the staging batches.
extern "C" int cmb_last_bgzf_batch(cmb_ctx* c, cmb_read_batch* dev_batch, uint32_t* n_records, uint32_t* n_intervals) {
  if (!c || !dev_batch || !n_records || !n_intervals) return fail(c, CMB_E_ARG, "cmb_last_bgzf_batch: null argument");
  if (!c->dec.last_valid || !c->dec.d_tuple_slab) return fail(c, CMB_E_ARG, "cmb_last_bgzf_batch: no device-decoded sample is resident");
  carve_batch(c->dec.d_tuple_slab, c->dec.last_n_rec, c->dec.last_n_cig, dev_batch);
  *n_records = c->dec.last_n_rec;
  *n_intervals = c->dec.last_n_cig;
  return CMB_OK;
}

extern "C" int cmb_submit_bgzf(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out) { return bgzf_entry(c, in, out, false); }
extern "C" int cmb_decode_bgzf(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out) { return bgzf_entry(c, in, out, true); }

extern "C" int cmb_filter_plan(cmb_ctx* c, int inverse, uint64_t* n_records, uint64_t* n_bytes) {
  if (!c || !n_records || !n_bytes) return fail(c, CMB_E_ARG, "cmb_filter_plan: null argument");
  auto& d = c->dec;
  if (!d.last_valid || !d.d_tuple_slab || !c->have_params) return fail(c, CMB_E_ARG, "cmb_filter_plan: no device-decoded sample is resident (cmb_decode_bgzf first)");
  CU_TRY(c, cudaSetDevice(c->device));
  *n_records = 0;
  *n_bytes = 0;
  d.filter_planned = false;
  const uint32_t n = d.last_n_rec;
  if (n == 0) {
    d.filter_bytes = 0;
    d.filter_planned = true;
    return CMB_OK;
  }
  const bool pair_path = !(c->mode.filter_single_reads && !c->mode.filter_pairs);
  int rc;
  if (pair_path && (rc = match_mates(c, d.last_infl_base, n, !inverse, "cmb_filter_plan"))) return rc;
  uint64_t total = 0, n_emit = 0;
  if ((rc = filter_kernels(c, pair_path, inverse, n, &total, &n_emit))) return rc;
  d.filter_bytes = total;
  d.filter_planned = true;
  *n_records = n_emit;
  *n_bytes = total;
  return CMB_OK;
}

extern "C" int cmb_filter_fetch(cmb_ctx* c, uint8_t* records, uint64_t n_bytes) {
  if (!c || (!records && n_bytes)) return fail(c, CMB_E_ARG, "cmb_filter_fetch: null argument");
  auto& d = c->dec;
  if (!d.filter_planned || n_bytes != d.filter_bytes) return fail(c, CMB_E_ARG, "cmb_filter_fetch: call cmb_filter_plan first and pass the size it reported");
  CU_TRY(c, cudaSetDevice(c->device));
  if (n_bytes) CU_TRY(c, cudaMemcpyAsync(records, d.d_filter_out, n_bytes, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}

// ------------------------------------------------------------------------------------------------ coverm filter, streamed
namespace {

using Clock = std::chrono::steady_clock;
constexpr uint64_t FILTER_PIECE_BYTES = 64u << 20;  // most bytes per sink call, and the size of each pinned staging buffer
double ms_since(Clock::time_point t0) { return std::chrono::duration<double, std::milli>(Clock::now() - t0).count(); }

// One cmb_filter_bgzf call: the filter over the records of the resident decode (the whole stream, or one slice), and the
// hand-over of what it returns to the sink.
struct FilterCall {
  cmb_ctx* c;
  int inverse;
  cmb_filter_sink sink;
  void* user;
  cmb_filter_result* out;
  bool pair_path;  // filter.rs:117-233 (mates matched), else the singles path (filter.rs:88-116)
  bool deflate;    // the returned records to the deflate stream (cmb_filter_bgzf_deflate), not to the staging buffers

  // filter_kernels over records [0, n) of the last decode (its mates matched on the pair path), then the returned records to
  // the sink in pieces of at most FILTER_PIECE_BYTES, each through the next staging buffer.  Every allocation comes before the
  // first sink call: CMB_E_NOMEM means nothing was handed over.
  int filter(uint32_t n) {
    auto& d = c->dec;
    const auto t0 = Clock::now();
    uint64_t total = 0, n_emit = 0;
    int rc;
    if ((rc = filter_kernels(c, pair_path, inverse, n, &total, &n_emit))) return rc;
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    out->ms_filter += (float)ms_since(t0);
    if (!total) return CMB_OK;
    if (deflate) {  // cmb_filter_bgzf_deflate: the records go to the context's deflate stream from device memory
      if ((rc = deflate_feed_device(c, d.d_filter_out, total, sink, user, &out->n_sink_calls))) return rc;
      out->n_bytes += total;
      out->n_records += n_emit;
      return CMB_OK;
    }
    // Both staging buffers have their fixed size once allocated, so that none is freed while the caller still reads it
    for (auto& stage : d.filter_stage)
      if ((rc = stage.ensure(c, FILTER_PIECE_BYTES))) return rc;
    for (uint64_t o = 0; o < total; o += FILTER_PIECE_BYTES) {
      // sink call k - 1's bytes are in the other buffer, which its caller may still be reading
      const auto t1 = Clock::now();
      const uint64_t len = std::min<uint64_t>(FILTER_PIECE_BYTES, total - o);
      uint8_t* stage = d.filter_stage[out->n_sink_calls & 1];
      CU_TRY(c, cudaMemcpyAsync(stage, d.d_filter_out + o, len, cudaMemcpyDeviceToHost, c->stream));
      CU_TRY(c, cudaStreamSynchronize(c->stream));
      out->ms_d2h += (float)ms_since(t1);
      if (const int s = sink(user, stage, len)) return fail(c, CMB_E_ARG, "cmb_filter_bgzf: the sink returned %d", s);
      out->n_sink_calls += 1;
      out->n_bytes += len;
    }
    out->n_records += n_emit;
    return CMB_OK;
  }

  // Device bytes the filter holds beside the decode buffers: they count as room, since they are reused or freed to grow
  uint64_t held() const {
    const auto& d = c->dec;
    return decode_bytes(c) + d.d_filter_anchor.bytes() + d.d_filter_role.bytes() + d.d_filter_out.bytes() + (pair_path ? pair_bytes(c) : 0);
  }
  void release_filter() {
    auto& d = c->dec;
    d.d_filter_anchor.release();
    d.d_filter_role.release();
    d.d_filter_out.release();
  }

  // The whole stream when its buffers fit; else slices
  int whole(const cmb_bgzf_input* in) {
    auto& d = c->dec;
    d.last_valid = false;
    d.filter_planned = false;
    cmb_bgzf_result br{};
    int rc = submit_bgzf_impl(c, in, &br, true);
    if (!rc && d.last_valid) {
      out->ms_decode = br.ms_total;
      const uint32_t n = d.last_n_rec;
      const auto t0 = Clock::now();
      if (pair_path && n) rc = match_mates(c, d.last_infl_base, n, !inverse, "cmb_filter_bgzf");
      out->ms_filter += (float)ms_since(t0);
      if (!rc && n) rc = filter(n);
    }
    return whole_or_slices(c, rc, [&] {
      release_filter();
      return sliced(in);
    });
  }

  // The stream in block slices, each filtered up to its cut and handed to the sink
  int sliced(const cmb_bgzf_input* in) {
    auto& d = c->dec;
    auto work = [&](BgzfCall&, cmb_bgzf_result&, uint32_t cut) {
      const int rc = filter(cut);
      if (rc != CMB_E_NOMEM) return rc;
      release_filter();
      return SLICE_HALVE;
    };
    SliceStats ss;
    cmb_bgzf_result r{};
    const int rc = stream_in_slices(
        c, in, &r, ss, "cmb_filter_bgzf", "the filter runs on the host", "filter", pair_path, !inverse, false, [&] { return held(); },
        [&] { return held() - d.d_comp.bytes() - d.d_inflated.bytes(); }, work);
    out->n_slices = ss.n_slices;  // on a decline: the slices handed over before it
    out->halvings = ss.halvings;
    out->pair_cut_records = ss.pair_cut_records;
    out->ms_filter += ss.ms_mates;
    if (rc) return rc;
    out->ms_decode = ss.ms_inflate + ss.ms_chain + ss.ms_extract;
    return CMB_OK;
  }
};

}  // namespace

namespace {
int filter_entry(cmb_ctx* c, const cmb_bgzf_input* in, int inverse, cmb_filter_sink sink, void* user, cmb_filter_result* out, bool deflate) {
  if (!c || !in || !sink || !out) return fail(c, CMB_E_ARG, "cmb_filter_bgzf: null argument");
  *out = cmb_filter_result{};
  if (!c->have_params || c->in_sample) return fail(c, CMB_E_ARG, "cmb_filter_bgzf: set the parameters first; not inside a sample");
  if (c->n_acquired) return fail(c, CMB_E_ARG, "cmb_filter_bgzf: a staging batch is still acquired");
  if (deflate && !c->dfl.active) return fail(c, CMB_E_ARG, "cmb_filter_bgzf_deflate: no stream begun (cmb_deflate_begin first)");
  CU_TRY(c, cudaSetDevice(c->device));
  FilterCall f{c, inverse, sink, user, out, !(c->mode.filter_single_reads && !c->mode.filter_pairs), deflate};
  return f.whole(in);
}
}  // namespace

extern "C" int cmb_filter_bgzf(cmb_ctx* c, const cmb_bgzf_input* in, int inverse, cmb_filter_sink sink, void* user, cmb_filter_result* out) {
  NvtxRange nvtx("cmb_filter_bgzf");
  return filter_entry(c, in, inverse, sink, user, out, false);
}

extern "C" int cmb_filter_bgzf_deflate(cmb_ctx* c, const cmb_bgzf_input* in, int inverse, cmb_filter_sink sink, void* user,
                                       cmb_filter_result* out) {
  NvtxRange nvtx("cmb_filter_bgzf_deflate");
  return filter_entry(c, in, inverse, sink, user, out, true);
}
