// TEST INFRASTRUCTURE ONLY — never linked into libcoverm_b200.so or the `coverm` product binary.
//
// The CPU emulator of the device ABI (oracle/device_emulator.cpp) with a cmb_filter_bgzf on top whose outcome the test picks
// with CMB_EMU_FILTER, so that `coverm filter`'s handling of it (coverm_b200/csrc/host/filter_command.hpp) runs without a GPU
// (tests/test_filter_slices.py builds this file with the product's host code into a `coverm` binary):
//   decline_late  hands three pieces of filler bytes to the sink, then declines: the host must drop them and write the file
//                 its own loop writes;
//   nm            raises the reference's NM panic before any sink call: the host must leave no output file, and must not
//                 unwind past the header bytes it is still compressing;
//   sink_error    hands one piece, then declines with CMB_E_ARG as if the sink had failed.
// Unset, it declines at once, like the plain emulator's cmb_decode_bgzf.
#include "../../oracle/device_emulator.cpp"

extern "C" int cmb_filter_bgzf(cmb_ctx* c, const cmb_bgzf_input* in, int, cmb_filter_sink sink, void* user, cmb_filter_result* out) {
  if (!c || !in || !sink || !out) return fail(c, CMB_E_ARG, "cmb_filter_bgzf: null argument");
  *out = cmb_filter_result{};
  const char* e = getenv("CMB_EMU_FILTER");
  const std::string mode = e ? e : "";
  static std::vector<uint8_t> stage[2];  // the pieces stay valid until the next call, as the library's staging buffers do
  auto hand = [&](size_t n) {
    auto& s = stage[out->n_sink_calls & 1];
    s.assign(n, (uint8_t)('a' + out->n_sink_calls));
    const int r = sink(user, s.data(), n);
    out->n_sink_calls += 1;
    return r;
  };
  if (mode == "decline_late") {
    for (int k = 0; k < 3; ++k)
      if (int r = hand(300000)) return fail(c, CMB_E_ARG, "cmb_filter_bgzf: the sink returned " + std::to_string(r));
    out->n_slices = 3;
    return fail(c, CMB_E_DECLINED, "emulator: declined after three slices");
  }
  if (mode == "nm")
    return fail(c, CMB_E_NM, "Mapping record encountered that does not have an 'NM' auxiliary tag in the SAM/BAM format. This is "
                             "required to work out some coverage statistics");
  if (mode == "sink_error") {
    hand(1000);
    return fail(c, CMB_E_ARG, "emulator: stopped after one piece");
  }
  return fail(c, CMB_E_DECLINED, "emulator: no device-side filter");
}
