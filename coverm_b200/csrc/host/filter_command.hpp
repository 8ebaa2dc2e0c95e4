// `coverm filter` (src/bin/coverm.rs:408-472): ReferenceSortedBamFilter (src/filter.rs:36-234) used as a record sink --
// every record the filter returns is written, in the order it returns them, into a new BAM file with the input's header.
//
// Fast path: the sample is decoded on the GPU (cmb_filter_bgzf: whole, or in block slices when it does not fit), the device
// decides and orders the returned records (cmb_filter.cuh) and hands their bytes back piece by piece; this file compresses and
// writes each piece while the device works on the next (BgzfWriter).  With --device-deflate the records are compressed on the
// device instead (cmb_filter_bgzf_deflate) and only BGZF bytes come back; the host loop's output goes through the same encoder.  Fallback (SAM / uncompressed input, a stream the device
// declines): filter_on_host below runs the reference's loop on the host.
// `filter-names` prints the returned records' names instead of writing a BAM: the form in which the reference's unit tests
// (filter.rs:342-844) state their expectations.
#pragma once
#include <cstdio>
#include <exception>
#include <fstream>
#include <utility>

#include "bgzf_writer.hpp"
#include "sample_processor.hpp"

// Referenced weakly: the host code also links against stand-ins of the device library without it (the CPU emulator of the ABI),
// where every input takes the host loop.  libcoverm_b200 always defines it.
extern "C" int cmb_filter_bgzf(cmb_ctx* ctx, const cmb_bgzf_input* in, int inverse, cmb_filter_sink sink, void* user,
                               cmb_filter_result* out) __attribute__((weak));
extern "C" int cmb_filter_bgzf_deflate(cmb_ctx* ctx, const cmb_bgzf_input* in, int inverse, cmb_filter_sink sink, void* user,
                                       cmb_filter_result* out) __attribute__((weak));
extern "C" int cmb_deflate_begin(cmb_ctx* ctx) __attribute__((weak));
extern "C" int cmb_deflate_feed(cmb_ctx* ctx, const uint8_t* bytes, uint64_t n_bytes, cmb_filter_sink sink, void* user) __attribute__((weak));
extern "C" int cmb_deflate_finish(cmb_ctx* ctx, cmb_filter_sink sink, void* user, cmb_deflate_stats* stats) __attribute__((weak));

namespace cmbh {

// The filter's predicates on the host, over the tuple of a record (filter.rs:243-336): the same f32 expressions as the kernels.
struct HostFilterParams {
  cmb_params p{};
  bool filter_single = false, filter_pairs = false, filter_out = true;
};
inline bool host_single_read_passes(const Tuple& t, const cmb_params& p) {
  if (p.min_mapq != 255 && (t.mapq < p.min_mapq || t.mapq == 255)) return false;
  if (t.nm_state != 1)
    throw Panic("Mapping record encountered that does not have an 'NM' auxiliary tag in the SAM/BAM format. This is required to work out some coverage statistics");
  const float aligned = (float)t.aligned;
  return t.aligned >= p.min_aligned_length_single && aligned / (float)t.l_seq >= p.min_aligned_percent_single &&
         1.0f - (float)t.nm / aligned >= p.min_percent_identity_single;
}
inline bool host_read_pair_passes(const Tuple& a, const Tuple& b, const cmb_params& p) {
  if (p.min_mapq != 255 && (a.mapq < p.min_mapq || b.mapq < p.min_mapq || a.mapq == 255 || b.mapq == 255)) return false;
  if (a.nm_state != 1 || b.nm_state != 1)
    throw Panic("Mapping record encountered that does not have an 'NM' auxiliary tag in the SAM/BAM format. This is required to work out some coverage statistics");
  const uint32_t aligned = (a.aligned - a.del) + (b.aligned - b.del);
  const float aligned_f = (float)aligned;
  return aligned >= p.min_aligned_length_pair && aligned_f / (float)((uint64_t)a.l_seq + b.l_seq) >= p.min_aligned_percent_pair &&
         1.0f - ((float)((uint64_t)a.nm + b.nm) / aligned_f) >= p.min_percent_identity_pair;
}

// ReferenceSortedBamFilter::read over an uncompressed BAM record stream: appends the returned records to `out`.
inline void filter_on_host(const uint8_t* recs, size_t n_bytes, const HostFilterParams& f, std::vector<uint8_t>& out, uint64_t& n_out) {
  struct Stored {
    Tuple t;
    size_t off, size;
  };
  HostMates<Stored> mates;
  std::vector<int32_t> ivs, ivl;
  auto emit = [&](size_t off, size_t size) {
    out.insert(out.end(), recs + off, recs + off + size);
    ++n_out;
  };
  const bool singles = f.filter_single && !f.filter_pairs;
  walk_records(recs, 0, n_bytes, true, [&](size_t o) {
    const size_t size = 4 + (size_t)rd_u32(recs + o);
    Tuple t;
    ivs.clear();
    ivl.clear();
    decode_bam_record(recs + o, t, ivs, ivl);
    const bool unmapped = t.flag & 0x4, secondary = t.flag & 0x100, supplementary = t.flag & 0x800, proper = t.flag & 0x2;
    if (singles) {  // filter.rs:88-116
      if (unmapped && !f.filter_out) emit(o, size);
      else {
        const bool passes_filter1 = !unmapped && (f.p.include_supplementary || !supplementary) && (f.p.include_secondary || !secondary);
        if (passes_filter1 && host_single_read_passes(t, f.p) == f.filter_out) emit(o, size);
      }
    } else {  // filter.rs:117-233
      if (unmapped && !f.filter_out) emit(o, size);
      else if (secondary || supplementary) {
      } else if (!proper) {
        if (!f.filter_out) emit(o, size);
      } else if (const std::optional<Stored> s = mates.match(t, bam_qname(recs + o), [&] { return Stored{t, o, size}; })) {
        const bool passes = (!f.filter_single || (host_single_read_passes(s->t, f.p) && host_single_read_passes(t, f.p))) &&
                            host_read_pair_passes(t, s->t, f.p);
        if (passes == f.filter_out) {
          emit(s->off, s->size);
          emit(o, size);
        }
      }
    }
    return true;
  });
}

// Where `coverm filter` sends one input's output: the header bytes, then the returned records in the reference's order, in
// as many pieces as they arrive.  A piece's bytes stay valid until the next call into the sink returns; after the last piece
// the caller calls finish() or restart() before they go.
struct FilterSink {
  virtual ~FilterSink() = default;
  virtual void header(const uint8_t* p, size_t n) = 0;
  virtual void records(const uint8_t* p, size_t n) = 0;
  // Forget everything received (the input is filtered again from its start, or it ended in an error); nothing received is
  // read after this returns.  Does not throw.
  virtual void restart() noexcept = 0;
  virtual void finish() = 0;  // the input is done: nothing of it is still being written after this returns
  // true: the sink's BGZF stream is the device's (cmb_deflate_*), and the device path hands it compressed bytes through
  // compressed() instead of records through records()
  virtual bool device_deflate() const { return false; }
  virtual void compressed(const uint8_t*, size_t) {}
};

// `coverm filter`'s output BAM, compressed and written while the device works.  The file is created by the first piece and
// removed again unless finish() is reached: an input that ends in an error leaves no output file.
class BamFileSink : public FilterSink {
 public:
  BamFileSink(std::string path, ThreadPool& pool) : path_(std::move(path)), pool_(pool) {}
  ~BamFileSink() override {
    if (done_ || !created_) return;
    writer_.reset();
    if (file_.is_open()) file_.close();
    std::remove(path_.c_str());
  }
  void header(const uint8_t* p, size_t n) override { open().feed(p, n); }
  void records(const uint8_t* p, size_t n) override { open().feed(p, n); }
  void restart() noexcept override {
    writer_.reset();  // waits for the blocks being deflated, and drops their error
    if (file_.is_open()) file_.close();  // the next piece truncates it
  }
  void finish() override {
    open().finish();
    file_.flush();
    if (!file_) throw Panic("Failed to write BAM record");
    done_ = true;
  }

 private:
  BgzfWriter& open() {
    if (!writer_) {
      file_.open(path_, std::ios::binary | std::ios::trunc);
      if (!file_) throw Panic("Failed to write BAM file " + path_);
      created_ = true;
      writer_ = std::make_unique<BgzfWriter>(file_, pool_);
    }
    return *writer_;
  }
  std::string path_;
  ThreadPool& pool_;
  std::ofstream file_;
  std::unique_ptr<BgzfWriter> writer_;
  bool created_ = false, done_ = false;
};

// `coverm filter --device-deflate`'s output BAM: the header and the host loop's records are fed to the context's deflate
// stream, the device path's records reach it on the device, and the stream's BGZF bytes are written as they arrive.  Restarting
// truncates the file and begins the stream again.  Like BamFileSink, it leaves no file unless finish() is reached.
class DeviceDeflateBamSink : public FilterSink {
 public:
  DeviceDeflateBamSink(std::string path, cmb_ctx* ctx) : path_(std::move(path)), ctx_(ctx) {
    if (!cmb_deflate_begin || !cmb_deflate_feed || !cmb_deflate_finish || !cmb_filter_bgzf_deflate)
      throw ExitError(1, "--device-deflate: this build of the device library has no deflate encoder");
  }
  ~DeviceDeflateBamSink() override {
    if (done_ || !created_) return;
    if (file_.is_open()) file_.close();
    std::remove(path_.c_str());
  }
  void header(const uint8_t* p, size_t n) override { feed(p, n); }
  void records(const uint8_t* p, size_t n) override { feed(p, n); }
  void compressed(const uint8_t* p, size_t n) override {
    open();
    file_.write((const char*)p, (std::streamsize)n);
    if (!file_) throw Panic("Failed to write BAM record");
  }
  void restart() noexcept override {
    if (file_.is_open()) file_.close();  // the next piece truncates it and begins the stream again
  }
  void finish() override {
    open();
    const int rc = cmb_deflate_finish(ctx_, &piece, this, &stats_);
    settle(rc);
    file_.flush();
    if (!file_) throw Panic("Failed to write BAM record");
    done_ = true;
  }
  bool device_deflate() const override { return true; }
  const cmb_deflate_stats& stats() const { return stats_; }

 private:
  void open() {
    if (file_.is_open()) return;
    file_.open(path_, std::ios::binary | std::ios::trunc);
    if (!file_) throw Panic("Failed to write BAM file " + path_);
    created_ = true;
    if (const int rc = cmb_deflate_begin(ctx_)) throw_device_error(ctx_, rc);
  }
  void feed(const uint8_t* p, size_t n) {
    open();
    settle(cmb_deflate_feed(ctx_, p, n, &piece, this));
  }
  void settle(int rc) {  // the sink's own error first, then the library's
    if (error_) std::rethrow_exception(std::exchange(error_, nullptr));
    if (rc) throw_device_error(ctx_, rc);
  }
  static int piece(void* user, const uint8_t* p, uint64_t n) {
    auto* s = static_cast<DeviceDeflateBamSink*>(user);
    try {
      s->compressed(p, n);
      return 0;
    } catch (...) {
      s->error_ = std::current_exception();
      return 1;
    }
  }
  std::string path_;
  cmb_ctx* ctx_;
  std::ofstream file_;
  std::exception_ptr error_;
  cmb_deflate_stats stats_{};
  bool created_ = false, done_ = false;
};

// `filter-names`: the returned records, kept until the input is done
struct RecordsSink : FilterSink {
  std::vector<uint8_t> bytes;
  void header(const uint8_t*, size_t) override {}
  void records(const uint8_t* p, size_t n) override { bytes.insert(bytes.end(), p, p + n); }
  void restart() noexcept override { bytes.clear(); }
  void finish() override {}
};

struct FilterRun {
  uint64_t n_records = 0;
  bool on_device = false;
};

// cmb_filter_bgzf's sink: the pieces to a FilterSink, whose first error is kept for the caller to rethrow
struct DeviceSinkCall {
  FilterSink* sink = nullptr;
  std::exception_ptr error;
  static int piece(void* user, const uint8_t* p, uint64_t n) {
    auto* s = static_cast<DeviceSinkCall*>(user);
    try {
      if (s->sink->device_deflate()) s->sink->compressed(p, n);
      else s->sink->records(p, n);
      return 0;
    } catch (...) {
      s->error = std::current_exception();
      return 1;
    }
  }
};

// Restarts the sink on every exit but a finished one: the pieces it was fed from buffers that go with the caller's frame are not
// read after they are gone.
class SinkSettle {
 public:
  explicit SinkSettle(FilterSink& sink) : sink_(sink) {}
  ~SinkSettle() {
    if (!finished_) sink_.restart();
  }
  SinkSettle(const SinkSettle&) = delete;
  SinkSettle& operator=(const SinkSettle&) = delete;
  void finish() {
    sink_.finish();
    finished_ = true;
  }

 private:
  FilterSink& sink_;
  bool finished_ = false;
};

// One input through the filter into `sink`.  `params`: thresholds + flag includes with filtering = 1; inverse = --inverse.
inline FilterRun filter_one_input(DeviceSession& session, const InputSpec& in, const cmb_params& params, bool inverse, FilterSink& sink) {
  FilterRun run;
  const BamInput input(in);
  cmb_ctx* ctx = session.ctx();
  cmb_filter_mode mode{};
  int rc = cmb_set_params(ctx, &params, &mode);
  if (rc) throw_device_error(ctx, rc);
  InflateStream stream(input.data(), input.size(), session.pool(), 1u << 20);
  std::vector<uint8_t> buf;
  const BamHeader h = read_bam_header(stream, buf, in.path);
  const std::vector<uint8_t> header(buf.begin(), buf.begin() + (ptrdiff_t)h.records_at);  // magic .. last reference entry
  std::vector<uint8_t> records;  // the host loop's output
  SinkSettle settle(sink);       // after `header` and `records`: gone before them
  const BlockIndex& bx = stream.index();
  if (bx.bgzf && cmb_filter_bgzf && !getenv("CMB_HOST_DECODE")) {
    sink.header(header.data(), header.size());  // written on the pool while the device decodes, which does not use it (or
                                                // fed to the device's deflate stream)
    const BgzfInput bi(bx, (uint32_t)h.header->names.size(), h.records_at, session.pool().size());
    DeviceSinkCall sc;
    sc.sink = &sink;
    cmb_filter_result fr{};
    rc = (sink.device_deflate() ? cmb_filter_bgzf_deflate : cmb_filter_bgzf)(ctx, &bi.in, inverse ? 1 : 0, &DeviceSinkCall::piece, &sc, &fr);
    if (sc.error) std::rethrow_exception(sc.error);
    if (rc == CMB_OK) {
      settle.finish();
      run.n_records = fr.n_records;
      run.on_device = true;
      return run;
    }
    // the device declines a stream whose mates it cannot match in file order (cmb_pairs.cuh), among others: the host loop
    // takes it from the start, whatever was handed over already
    if (rc != CMB_E_DECLINED) throw_device_error(ctx, rc);
    if (getenv("CMB_PIPELINE_STATS")) {
      fprintf(stderr, "#device_decode\tdeclined: %s\n", cmb_last_error(ctx));
      fprintf(stderr, "#filter_declined\tslices_before=%u\tsink_calls=%u\n", fr.n_slices, fr.n_sink_calls);
    }
    sink.restart();  // the writer is idle after this: the host decoder below needs the pool
  }
  // host fallback: the whole record stream in memory, then the reference's loop
  while (stream.fill(buf)) {
  }
  HostFilterParams f;
  f.p = params;
  f.filter_single = mode.filter_single_reads;
  f.filter_pairs = mode.filter_pairs;
  f.filter_out = !inverse;
  filter_on_host(buf.data() + h.records_at, buf.size() - h.records_at, f, records, run.n_records);
  sink.header(header.data(), header.size());
  sink.records(records.data(), records.size());
  settle.finish();
  return run;
}

}  // namespace cmbh
