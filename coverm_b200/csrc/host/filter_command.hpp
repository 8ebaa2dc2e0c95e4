// `coverm filter` (src/bin/coverm.rs:408-472): ReferenceSortedBamFilter (src/filter.rs:36-234) used as a record sink --
// every record the filter returns is written, in the order it returns them, into a new BAM file with the input's header.
//
// Fast path: the sample is decoded on the GPU (cmb_decode_bgzf), the device decides and orders the returned records
// (cmb_filter_plan, cmb_filter.cuh) and hands their bytes back; this file then only compresses and writes.  Fallback (SAM /
// uncompressed input, a stream the device declines): FilterOnHost below runs the reference's loop on the host.
// `filter-names` prints the returned records' names instead of writing a BAM: the form in which the reference's unit tests
// (filter.rs:342-844) state their expectations.
#pragma once
#include <fstream>

#include "sample_processor.hpp"

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

// BGZF writer: `data` cut into blocks of at most 0xff00 bytes, deflated on all threads, followed by the EOF marker.
inline void write_bgzf(std::ostream& os, const std::vector<const uint8_t*>& parts, const std::vector<size_t>& sizes, ThreadPool& pool) {
  // flatten the parts into block jobs (a block may span parts: assemble per job)
  size_t total = 0;
  for (size_t s : sizes) total += s;
  const size_t BLOCK = 0xff00;
  const size_t n_blocks = (total + BLOCK - 1) / BLOCK;
  std::vector<size_t> part_start(parts.size() + 1, 0);
  for (size_t i = 0; i < parts.size(); ++i) part_start[i + 1] = part_start[i] + sizes[i];
  auto copy_range = [&](size_t from, size_t len, uint8_t* dst) {
    size_t i = (size_t)(std::upper_bound(part_start.begin(), part_start.end(), from) - part_start.begin()) - 1;
    while (len) {
      const size_t in_part = from - part_start[i];
      const size_t take = std::min(len, sizes[i] - in_part);
      memcpy(dst, parts[i] + in_part, take);
      dst += take;
      from += take;
      len -= take;
      ++i;
    }
  };
  const size_t GROUP = 64;  // blocks per task, written in order group by group
  std::vector<std::vector<uint8_t>> done((n_blocks + GROUP - 1) / GROUP);
  pool.parallel_for(done.size(), [&](size_t g, int) {
    std::vector<uint8_t> raw(BLOCK), comp(BLOCK + 1024);
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (deflateInit2(&zs, Z_DEFAULT_COMPRESSION, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) throw ExitError(1, "zlib init failed");
    std::vector<uint8_t>& outb = done[g];
    for (size_t b = g * GROUP; b < std::min(n_blocks, (g + 1) * GROUP); ++b) {
      const size_t from = b * BLOCK, len = std::min(BLOCK, total - from);
      copy_range(from, len, raw.data());
      deflateReset(&zs);
      zs.next_in = raw.data();
      zs.avail_in = (uInt)len;
      zs.next_out = comp.data();
      zs.avail_out = (uInt)comp.size();
      if (deflate(&zs, Z_FINISH) != Z_STREAM_END) throw ExitError(1, "deflate failed");
      const size_t clen = zs.total_out;
      const uint32_t bsize = (uint32_t)(12 + 6 + clen + 8 - 1);
      const uint8_t head[18] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, (uint8_t)(bsize & 0xff), (uint8_t)(bsize >> 8)};
      outb.insert(outb.end(), head, head + 18);
      outb.insert(outb.end(), comp.data(), comp.data() + clen);
      const uint32_t crc = (uint32_t)crc32(0, raw.data(), (uInt)len), isz = (uint32_t)len;
      uint8_t tail[8];
      memcpy(tail, &crc, 4);
      memcpy(tail + 4, &isz, 4);
      outb.insert(outb.end(), tail, tail + 8);
    }
    deflateEnd(&zs);
  });
  for (auto& b : done) os.write((const char*)b.data(), (std::streamsize)b.size());
  static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  os.write((const char*)eof, sizeof eof);
}

struct FilterRun {
  std::vector<uint8_t> header_bytes;  // the uncompressed BAM header block: magic .. last reference entry
  std::vector<uint8_t> records;       // returned records, back to back
  uint64_t n_records = 0;
  bool on_device = false;
};

// One input through the filter.  `params`: thresholds + flag includes with filtering = 1; inverse = --inverse.
inline FilterRun filter_one_input(DeviceSession& session, const InputSpec& in, const cmb_params& params, bool inverse) {
  FilterRun run;
  const BamInput input(in);
  cmb_ctx* ctx = session.ctx();
  cmb_filter_mode mode{};
  int rc = cmb_set_params(ctx, &params, &mode);
  if (rc) throw_device_error(ctx, rc);
  InflateStream stream(input.data(), input.size(), session.pool(), 1u << 20);
  std::vector<uint8_t> buf;
  const BamHeader h = read_bam_header(stream, buf, in.path);
  run.header_bytes.assign(buf.begin(), buf.begin() + (ptrdiff_t)h.records_at);
  const BlockIndex& bx = stream.index();
  if (bx.bgzf && !getenv("CMB_HOST_DECODE")) {
    const BgzfInput bi(bx, (uint32_t)h.header->names.size(), h.records_at, session.pool().size());
    cmb_bgzf_result br{};
    rc = cmb_decode_bgzf(ctx, &bi.in, &br);
    uint64_t n_rec = 0, n_bytes = 0;
    // the plan declines a stream whose mates the device cannot match in file order (cmb_pairs.cuh): the host loop takes it
    if (rc == CMB_OK) rc = cmb_filter_plan(ctx, inverse ? 1 : 0, &n_rec, &n_bytes);
    if (rc == CMB_OK) {
      run.records.resize(n_bytes);
      rc = cmb_filter_fetch(ctx, run.records.data(), n_bytes);
      if (rc) throw_device_error(ctx, rc);
      run.n_records = n_rec;
      run.on_device = true;
      return run;
    }
    if (rc != CMB_E_DECLINED) throw_device_error(ctx, rc);
    if (getenv("CMB_PIPELINE_STATS")) fprintf(stderr, "#device_decode\tdeclined: %s\n", cmb_last_error(ctx));
  }
  // host fallback: the whole record stream in memory, then the reference's loop
  while (stream.fill(buf)) {
  }
  HostFilterParams f;
  f.p = params;
  f.filter_single = mode.filter_single_reads;
  f.filter_pairs = mode.filter_pairs;
  f.filter_out = !inverse;
  filter_on_host(buf.data() + h.records_at, buf.size() - h.records_at, f, run.records, run.n_records);
  return run;
}

}  // namespace cmbh
