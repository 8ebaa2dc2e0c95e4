// TEST INFRASTRUCTURE ONLY — never linked into libcoverm_b200.so or the `coverm` product binary.
//
// The filter emulator (filter_emulator.cpp, whose scripted cmb_filter_bgzf outcomes CMB_EMU_FILTER picks) with the deflate
// stream of the device ABI on top of the encoder core's host build (coverm_b200/csrc/cmb_deflate.cuh): `coverm filter
// --device-deflate` then runs without a GPU and writes, block for block, the bytes kz_deflate writes.
// cmb_filter_bgzf_deflate follows the same script, feeding its filler pieces to the stream instead of to the sink.
#include "filter_emulator.cpp"

#include <memory>

#include "../../coverm_b200/csrc/cmb_deflate.cuh"

namespace {
struct EmuDeflate {
  std::unique_ptr<cmb_dfl::DflSmem> smem{new cmb_dfl::DflSmem};
  std::vector<uint8_t> carry, stage[2];
  cmb_deflate_stats stats{};
  bool active = false;

  int hand(cmb_ctx* c, std::vector<uint8_t>& out, cmb_filter_sink sink, void* user) {
    if (out.empty()) return CMB_OK;
    stage[stats.sink_calls & 1].swap(out);
    const std::vector<uint8_t>& s = stage[stats.sink_calls & 1];
    if (const int r = sink(user, s.data(), s.size())) {
      active = false;
      return fail(c, CMB_E_ARG, "cmb_deflate: the sink returned " + std::to_string(r));
    }
    stats.sink_calls += 1;
    stats.bgzf_bytes += s.size();
    out.clear();
    return CMB_OK;
  }
  void block(const uint8_t* p, size_t n, std::vector<uint8_t>& out) {
    std::vector<uint8_t> b(cmb_dfl::DFL_MAX_OUT);
    cmb_dfl::dfl_encode_block(*smem, p, (uint32_t)n, b.data());
    out.insert(out.end(), b.begin(), b.begin() + smem->size);
    stats.blocks += 1;
    stats.stored_blocks += smem->stored ? 1 : 0;
    stats.raw_bytes += n;
  }
  int feed(cmb_ctx* c, const uint8_t* p, uint64_t n, cmb_filter_sink sink, void* user) {
    if (!active) return fail(c, CMB_E_ARG, "cmb_deflate: no stream begun (cmb_deflate_begin first)");
    carry.insert(carry.end(), p, p + n);
    std::vector<uint8_t> out;
    size_t o = 0;
    for (; carry.size() - o >= cmb_dfl::DFL_BLOCK; o += cmb_dfl::DFL_BLOCK) block(carry.data() + o, cmb_dfl::DFL_BLOCK, out);
    carry.erase(carry.begin(), carry.begin() + (ptrdiff_t)o);
    return hand(c, out, sink, user);
  }
} emu_dfl;
}  // namespace

extern "C" int cmb_deflate_begin(cmb_ctx* c) {
  if (!c) return fail(c, CMB_E_ARG, "cmb_deflate_begin: null argument");
  emu_dfl.carry.clear();
  emu_dfl.stats = cmb_deflate_stats{};
  emu_dfl.active = true;
  return CMB_OK;
}

extern "C" int cmb_deflate_feed(cmb_ctx* c, const uint8_t* bytes, uint64_t n_bytes, cmb_filter_sink sink, void* user) {
  if (!c || !sink || (!bytes && n_bytes)) return fail(c, CMB_E_ARG, "cmb_deflate_feed: null argument");
  return emu_dfl.feed(c, bytes, n_bytes, sink, user);
}

extern "C" int cmb_deflate_finish(cmb_ctx* c, cmb_filter_sink sink, void* user, cmb_deflate_stats* stats) {
  if (!c || !sink || !stats) return fail(c, CMB_E_ARG, "cmb_deflate_finish: null argument");
  if (!emu_dfl.active) return fail(c, CMB_E_ARG, "cmb_deflate_finish: no stream begun (cmb_deflate_begin first)");
  std::vector<uint8_t> out;
  if (!emu_dfl.carry.empty()) emu_dfl.block(emu_dfl.carry.data(), emu_dfl.carry.size(), out);
  static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  out.insert(out.end(), eof, eof + sizeof eof);
  if (int rc = emu_dfl.hand(c, out, sink, user)) return rc;
  emu_dfl.carry.clear();
  emu_dfl.active = false;
  *stats = emu_dfl.stats;
  return CMB_OK;
}

extern "C" int cmb_filter_bgzf_deflate(cmb_ctx* c, const cmb_bgzf_input* in, int, cmb_filter_sink sink, void* user, cmb_filter_result* out) {
  if (!c || !in || !sink || !out) return fail(c, CMB_E_ARG, "cmb_filter_bgzf: null argument");
  *out = cmb_filter_result{};
  if (!emu_dfl.active) return fail(c, CMB_E_ARG, "cmb_filter_bgzf_deflate: no stream begun (cmb_deflate_begin first)");
  const char* e = getenv("CMB_EMU_FILTER");
  const std::string mode = e ? e : "";
  auto hand = [&](size_t n, char fill) {
    const std::vector<uint8_t> filler(n, (uint8_t)fill);
    const uint32_t before = emu_dfl.stats.sink_calls;
    const int r = emu_dfl.feed(c, filler.data(), n, sink, user);
    out->n_sink_calls += emu_dfl.stats.sink_calls - before;
    return r;
  };
  if (mode == "decline_late") {
    for (int k = 0; k < 3; ++k)
      if (int r = hand(300000, (char)('a' + k))) return r;
    out->n_slices = 3;
    return fail(c, CMB_E_DECLINED, "emulator: declined after three slices");
  }
  if (mode == "nm")
    return fail(c, CMB_E_NM, "Mapping record encountered that does not have an 'NM' auxiliary tag in the SAM/BAM format. This is "
                             "required to work out some coverage statistics");
  if (mode == "sink_error") {
    hand(100000, 'a');
    return fail(c, CMB_E_ARG, "emulator: stopped after one piece");
  }
  return fail(c, CMB_E_DECLINED, "emulator: no device-side filter");
}
