// Host record source of libcoverm_b200: BGZF / BAM / SAM -> per-read tuples written straight into the pinned SoA
// staging batch of the device library (include/coverm_b200.h, cmb_read_batch).
//
// Replaces, for the coverage path, what the reference gets from rust-htslib 0.46.0 (Cargo.lock:1643-1646):
// bam::Reader::from_path + read (bam_generator.rs:103-134), record.tid/pos/flags/mapq/cigar/seq().len()
// (contig.rs:124,166-168; filter.rs:251-277) and the NM aux lookup (lib.rs:138-158).  Written from the SAM/BAM
// specification (SAMv1 §4.1 BGZF, §4.2 BAM, §1.4 SAM); BGZF blocks are inflated with zlib on a thread pool
// (the reference's set_threads, bam_generator.rs:125-129) and tuples are extracted in parallel.
//
// Every BAM-format rule of the host lives here, once: opening an input (SAM converted to BAM), the BGZF block index,
// the header, the record decoder, the walk of an in-memory record stream and the host's mate matching.
#pragma once
#include <functional>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include "fast_inflate.hpp"

#include <climits>
#include <cstring>
#include <map>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../../include/coverm_b200.h"
#include "thread_pool.hpp"

namespace cmbh {

struct Panic : std::runtime_error {  // the reference would panic!() here (exit status 101)
  using std::runtime_error::runtime_error;
};

// One BGZF block -> its uncompressed bytes: the fast decoder first, checked against the block footer's CRC32; zlib's
// inflate() when the fast decoder declines or the checksum disagrees (htslib verifies the same CRC in bgzf.c).
class BgzfInflater {
 public:
  BgzfInflater() : fast_(new FastInflate) {
    memset(&zs_, 0, sizeof zs_);
    if (inflateInit2(&zs_, -15) != Z_OK) throw Panic("zlib init failed");
  }
  ~BgzfInflater() { inflateEnd(&zs_); }
  BgzfInflater(const BgzfInflater&) = delete;
  BgzfInflater& operator=(const BgzfInflater&) = delete;
  // cdata[clen .. clen+8) is the footer (CRC32, ISIZE).  Returns false on a corrupt block.
  bool block(const uint8_t* cdata, size_t clen, uint8_t* out, uint32_t isize) {
    if (isize == 0) return true;
    uint32_t want;
    memcpy(&want, cdata + clen, 4);
    if (fast_->run(cdata, clen, out, isize) && (uint32_t)crc32(0, out, isize) == want) return true;
    ++slow_blocks;
    inflateReset(&zs_);
    zs_.next_in = const_cast<Bytef*>(cdata);
    zs_.avail_in = (uInt)clen;
    zs_.next_out = out;
    zs_.avail_out = isize;
    if (inflate(&zs_, Z_FINISH) != Z_STREAM_END || zs_.avail_out != 0) return false;
    return (uint32_t)crc32(0, out, isize) == want;
  }
  uint64_t slow_blocks = 0;

 private:
  std::unique_ptr<FastInflate> fast_;
  z_stream zs_;
};
struct ExitError : std::runtime_error {  // error!(..); process::exit(code)
  int code;
  ExitError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

struct Header {
  std::vector<std::string> names;
  std::vector<uint64_t> lens;
};

// A BAM/SAM input: a file path or a caller-owned memory buffer holding the file's bytes.
struct InputSpec {
  std::string path;              // used for the sample name (file stem) and, when data == nullptr, opened
  const uint8_t* data = nullptr;
  size_t size = 0;
  // --sharded: one sample made of these read-name-sorted shards (the same read set mapped to each reference shard), and which
  // of the concatenated reference's contigs belong to excluded genomes (0 no, 1 yes, 2 its genome cannot be told)
  std::vector<InputSpec> shards;
  std::function<uint8_t(const std::string&)> excluded;
  std::string unknown_genome_panic;  // the reference's panic when a candidate's first mate lies on a contig marked 2
};

// One decoded record, fixed part (everything the device tuple needs) + qname location for mate matching.
struct Tuple {
  int32_t tid, pos;
  uint32_t nm, l_seq, aligned, del, ins;
  uint16_t flag;
  uint8_t mapq, nm_state;
  int32_t mtid;
  uint32_t n_iv;
};

inline uint32_t rd_u32(const uint8_t* p) {
  uint32_t v;
  memcpy(&v, p, 4);
  return v;
}
inline uint16_t rd_u16(const uint8_t* p) {
  uint16_t v;
  memcpy(&v, p, 2);
  return v;
}

class ByteSource {  // whole input mapped (file) or borrowed (memory)
 public:
  explicit ByteSource(const InputSpec& in) {
    if (in.data) {
      p_ = in.data;
      n_ = in.size;
      return;
    }
    fd_ = open(in.path.c_str(), O_RDONLY);
    if (fd_ < 0) throw Panic("Unable to find BAM file " + in.path);
    struct stat st;
    if (fstat(fd_, &st) != 0) throw Panic("Unable to stat BAM file " + in.path);
    n_ = (size_t)st.st_size;
    if (n_) {
      void* m = mmap(nullptr, n_, PROT_READ, MAP_PRIVATE, fd_, 0);
      if (m == MAP_FAILED) throw Panic("Unable to map BAM file " + in.path);
      madvise(m, n_, MADV_SEQUENTIAL);
      p_ = (const uint8_t*)m;
      mapped_ = true;
    }
  }
  ~ByteSource() {
    if (mapped_) munmap((void*)p_, n_);
    if (fd_ >= 0) close(fd_);
  }
  ByteSource(const ByteSource&) = delete;
  const uint8_t* data() const { return p_; }
  size_t size() const { return n_; }

 private:
  const uint8_t* p_ = nullptr;
  size_t n_ = 0;
  int fd_ = -1;
  bool mapped_ = false;
};

// Converts SAM text to BAM record bytes so that one decoder serves both (htslib reads SAM through the same
// bam::Reader; tests/data/mapq_test.sam).  Integer aux tags get htslib's smallest-fitting type.
class SamToBam {
 public:
  static bool looks_like_sam(const uint8_t* p, size_t n) { return n == 0 || p[0] == '@' || (n > 4 && memcmp(p, "BAM\1", 4) != 0); }
  static void convert(const uint8_t* p, size_t n, Header& header, std::vector<uint8_t>& out) {
    std::unordered_map<std::string, int32_t> name_to_tid;
    size_t o = 0;
    auto next_line = [&](std::string& line) {
      if (o >= n) return false;
      size_t e = o;
      while (e < n && p[e] != '\n') ++e;
      line.assign((const char*)p + o, e - o);
      o = e < n ? e + 1 : e;
      if (!line.empty() && line.back() == '\r') line.pop_back();
      return true;
    };
    auto split = [](const std::string& s) {
      std::vector<std::string> v;
      size_t a = 0;
      for (;;) {
        size_t b = s.find('\t', a);
        if (b == std::string::npos) { v.push_back(s.substr(a)); break; }
        v.push_back(s.substr(a, b - a));
        a = b + 1;
      }
      return v;
    };
    out.assign({'B', 'A', 'M', 1});
    std::string line;
    std::vector<uint8_t> body;
    auto put32 = [](std::vector<uint8_t>& v, uint32_t x) { for (int k = 0; k < 4; ++k) v.push_back((x >> (8 * k)) & 0xff); };
    auto put16 = [](std::vector<uint8_t>& v, uint32_t x) { v.push_back(x & 0xff); v.push_back((x >> 8) & 0xff); };
    bool header_done = false;
    std::vector<uint8_t> recs;
    while (next_line(line)) {
      if (line.empty()) continue;
      if (line[0] == '@' && !header_done) {
        if (line.compare(0, 3, "@SQ") == 0) {
          std::string sn;
          uint64_t ln = 0;
          for (auto& f : split(line)) {
            if (f.compare(0, 3, "SN:") == 0) sn = f.substr(3);
            if (f.compare(0, 3, "LN:") == 0) ln = strtoull(f.c_str() + 3, nullptr, 10);
          }
          name_to_tid[sn] = (int32_t)header.names.size();
          header.names.push_back(sn);
          header.lens.push_back(ln);
        }
        continue;
      }
      header_done = true;
      auto f = split(line);
      if (f.size() < 11) throw Panic("Error reading BAM record: malformed SAM line");
      auto tid_of = [&](const std::string& s) -> int32_t {
        if (s == "*") return -1;
        auto it = name_to_tid.find(s);
        if (it == name_to_tid.end()) throw Panic("Error reading BAM record: unknown reference " + s);
        return it->second;
      };
      const int32_t tid = tid_of(f[2]);
      std::vector<uint32_t> cigar;
      if (f[5] != "*") {
        const char* c = f[5].c_str();
        while (*c) {
          char* e;
          const uint32_t len = (uint32_t)strtoul(c, &e, 10);
          static const char* ops = "MIDNSHP=X";
          const char* w = *e ? strchr(ops, *e) : nullptr;
          if (!w) throw Panic("Error reading BAM record: bad CIGAR");
          cigar.push_back((len << 4) | (uint32_t)(w - ops));
          c = e + 1;
        }
      }
      const uint32_t l_seq = f[9] == "*" ? 0 : (uint32_t)f[9].size();
      body.clear();
      put32(body, (uint32_t)tid);
      put32(body, (uint32_t)((int32_t)strtol(f[3].c_str(), nullptr, 10) - 1));
      body.push_back((uint8_t)std::min<size_t>(255, f[0].size() + 1));
      body.push_back((uint8_t)strtoul(f[4].c_str(), nullptr, 10));
      put16(body, 0);
      put16(body, (uint32_t)cigar.size());
      put16(body, (uint32_t)strtoul(f[1].c_str(), nullptr, 10));
      put32(body, l_seq);
      put32(body, (uint32_t)(f[6] == "=" ? tid : tid_of(f[6])));
      put32(body, (uint32_t)((int32_t)strtol(f[7].c_str(), nullptr, 10) - 1));
      put32(body, (uint32_t)strtol(f[8].c_str(), nullptr, 10));
      body.insert(body.end(), f[0].begin(), f[0].begin() + std::min<size_t>(254, f[0].size()));
      body.push_back(0);
      for (uint32_t cg : cigar) put32(body, cg);
      body.insert(body.end(), (l_seq + 1) / 2 + l_seq, 0);
      for (size_t i = 11; i < f.size(); ++i) {
        if (f[i].size() < 5 || f[i][2] != ':' || f[i][4] != ':') continue;
        if (f[i][0] != 'N' || f[i][1] != 'M') continue;  // only NM matters on this path
        body.push_back('N');
        body.push_back('M');
        if (f[i][3] == 'i') {
          const long long v = strtoll(f[i].c_str() + 5, nullptr, 10);
          if (v < 0) { body.push_back('i'); put32(body, (uint32_t)(int32_t)v); }
          else if (v <= 0xff) { body.push_back('C'); body.push_back((uint8_t)v); }
          else if (v <= 0xffff) { body.push_back('S'); put16(body, (uint32_t)v); }
          else { body.push_back('I'); put32(body, (uint32_t)v); }
        } else {
          body.push_back('A');
          body.push_back('?');
        }
      }
      put32(recs, (uint32_t)body.size());
      recs.insert(recs.end(), body.begin(), body.end());
    }
    put32(out, 0);  // l_text
    put32(out, (uint32_t)header.names.size());
    for (size_t i = 0; i < header.names.size(); ++i) {
      put32(out, (uint32_t)header.names[i].size() + 1);
      out.insert(out.end(), header.names[i].begin(), header.names[i].end());
      out.push_back(0);
      put32(out, (uint32_t)header.lens[i]);
    }
    out.insert(out.end(), recs.begin(), recs.end());
    header = Header{};  // re-parsed from the BAM bytes by the caller
  }
};

// The BAM bytes of an input: the file mapped (or the caller's buffer), or its SAM text converted to BAM.
class BamInput {
 public:
  explicit BamInput(const InputSpec& in) : src_(in), p_(src_.data()), n_(src_.size()) {
    if (!(n_ >= 2 && p_[0] == 0x1f && p_[1] == 0x8b) && SamToBam::looks_like_sam(p_, n_)) {
      Header sam_header;
      SamToBam::convert(p_, n_, sam_header, sam_as_bam_);
      p_ = sam_as_bam_.data();
      n_ = sam_as_bam_.size();
    }
  }
  const uint8_t* data() const { return p_; }
  size_t size() const { return n_; }

 private:
  ByteSource src_;
  const uint8_t* p_;
  size_t n_;
  std::vector<uint8_t> sam_as_bam_;
};

struct BlockRef {
  size_t cdata, clen;  // compressed payload (BGZF) or raw slice [cdata, cdata+clen)
  uint32_t isize;      // uncompressed size
};

// The blocks of an input with their uncompressed offsets: its BGZF blocks (SAMv1 §4.1) when it starts with one, otherwise
// 64 KB slices of the bytes as they are.  The only BGZF block-header parser of the host: InflateStream grows the table
// block by block as it reads, the decoders take it whole (finish()).
class BlockIndex {
 public:
  std::vector<BlockRef> blocks;
  std::vector<uint64_t> ustart{0};  // blocks.size()+1 cumulative uncompressed offsets
  bool bgzf = false;
  const uint8_t* p = nullptr;
  size_t n = 0;

  void build(const uint8_t* data, size_t size) {
    start(data, size);
    finish();
  }
  // An empty table over a BGZF input, or every slice of any other (or of one that must not be taken for BGZF).
  void start(const uint8_t* data, size_t size, bool may_be_bgzf = true) {
    p = data;
    n = size;
    next_header_ = 0;
    blocks.clear();
    ustart.assign(1, 0);
    BlockRef b;
    size_t end;
    bgzf = may_be_bgzf && !parse(0, b, end);
    if (!bgzf)
      for (size_t o = 0; o < size; o += 65536) add({o, std::min<size_t>(65536, size - o), (uint32_t)std::min<size_t>(65536, size - o)});
  }
  // BGZF: appends the block whose header comes next.  false at the end of the input.
  bool next() {
    if (!bgzf || next_header_ >= n) return false;
    BlockRef b;
    if (const char* bad = parse(next_header_, b, next_header_)) throw Panic(std::string("Error reading BAM record: ") + bad);
    add(b);
    return true;
  }
  const BlockIndex& finish() {
    while (next()) {
    }
    return *this;
  }

  // Inflate blocks [b0, b1) into dst (which has room for ustart[b1]-ustart[b0] bytes).
  void inflate(size_t b0, size_t b1, uint8_t* dst, BgzfInflater& inf) const {
    for (size_t b = b0; b < b1; ++b) {
      const BlockRef& r = blocks[b];
      uint8_t* out = dst + (ustart[b] - ustart[b0]);
      if (!bgzf) {
        memcpy(out, p + r.cdata, r.clen);
        continue;
      }
      if (!inf.block(p + r.cdata, r.clen, out, r.isize)) throw Panic("Error reading BAM record: BGZF inflate failed");
    }
  }

 private:
  size_t next_header_ = 0;  // BGZF: file offset of the first block header not in the table yet

  void add(const BlockRef& b) {
    blocks.push_back(b);
    ustart.push_back(ustart.back() + b.isize);
  }
  // The block whose header is at `o`, and the offset after it; nullptr, or what is wrong with the header.
  const char* parse(size_t o, BlockRef& b, size_t& end) const {
    if (o + 18 > n || p[o] != 0x1f || p[o + 1] != 0x8b || p[o + 2] != 8 || !(p[o + 3] & 4)) return "corrupt BGZF block header";
    const size_t xlen = p[o + 10] | (p[o + 11] << 8);
    size_t x = o + 12;
    const size_t xend = x + xlen;
    if (xend > n) return "truncated BGZF block";
    int bsize = -1;
    while (x + 4 <= xend) {
      const size_t slen = p[x + 2] | (p[x + 3] << 8);
      if (p[x] == 'B' && p[x + 1] == 'C' && slen == 2) bsize = p[x + 4] | (p[x + 5] << 8);
      x += 4 + slen;
    }
    if (bsize < 0) return "gzip member without a BGZF block size";
    const size_t e = o + (size_t)bsize + 1;
    if (e > n || e < xend + 8) return "truncated BGZF block";
    b.cdata = xend;
    b.clen = e - 8 - xend;
    b.isize = rd_u32(p + e - 4);
    end = e;
    return nullptr;
  }
};

// Streams the uncompressed bytes of a BGZF (or plain gzip, or uncompressed) input in windows, building its block index on
// the way.
class InflateStream {
 public:
  InflateStream(const uint8_t* p, size_t n, ThreadPool& pool, size_t window_bytes) : pool_(pool), window_(window_bytes) {
    index_.start(p, n);
    if (!index_.bgzf && n >= 2 && p[0] == 0x1f && p[1] == 0x8b) {  // plain gzip, not block-indexable: inflate it whole
      inflate_whole(p, n);                                           // (small inputs only)
      index_.start(whole_.data(), whole_.size(), false);
    }
  }
  // Appends up to ~window bytes of uncompressed data to buf (after buf.size()). Returns false at EOF (nothing appended).
  bool fill(std::vector<uint8_t>& buf) {
    const size_t b0 = next_;
    while (index_.ustart[next_] - index_.ustart[b0] < window_ && (next_ < index_.blocks.size() || index_.next())) ++next_;
    if (next_ == b0) return false;
    const size_t o = buf.size();
    buf.resize(o + (index_.ustart[next_] - index_.ustart[b0]));
    uint8_t* out = buf.data() + o;
    const size_t per = 4;  // blocks per task: ~256 KB of output
    pool_.parallel_for((next_ - b0 + per - 1) / per, [&](size_t task, int) {
      BgzfInflater inf;
      const size_t t0 = b0 + task * per;
      index_.inflate(t0, std::min(next_, t0 + per), out + (index_.ustart[t0] - index_.ustart[b0]), inf);
    });
    return true;
  }
  void set_window(size_t window_bytes) { window_ = window_bytes; }
  bool is_bgzf() const { return index_.bgzf; }
  // The whole block table (of the inflated bytes for plain gzip); a Panic at the first bad block header.
  const BlockIndex& index() { return index_.finish(); }

 private:
  ThreadPool& pool_;
  size_t window_;
  BlockIndex index_;
  size_t next_ = 0;  // first block fill() has not returned yet
  std::vector<uint8_t> whole_;

  void inflate_whole(const uint8_t* p, size_t n) {
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, 15 + 32) != Z_OK) throw Panic("zlib init failed");
    zs.next_in = const_cast<Bytef*>(p);
    zs.avail_in = (uInt)n;
    std::vector<uint8_t> chunk(1 << 20);
    for (;;) {
      zs.next_out = chunk.data();
      zs.avail_out = (uInt)chunk.size();
      int rc = inflate(&zs, Z_NO_FLUSH);
      whole_.insert(whole_.end(), chunk.data(), chunk.data() + (chunk.size() - zs.avail_out));
      if (rc == Z_STREAM_END) {
        if (zs.avail_in == 0) break;
        inflateReset(&zs);
      } else if (rc != Z_OK) {
        inflateEnd(&zs);
        throw Panic("Error reading BAM record: gzip inflate failed");
      }
    }
    inflateEnd(&zs);
  }
};

// The BAM header (SAMv1 §4.2) read from the start of a stream.
struct BamHeader {
  std::shared_ptr<Header> header;  // nullptr: the reference list is byte for byte the caller's `known_refs`
  size_t refs_at = 0;              // offset of n_ref; the @-text in front of it (e.g. @PG) may differ between samples
  uint64_t records_at = 0;         // offset of the first record: [refs_at, records_at) is the raw reference list
};
// Reads the header into the empty `buf`, which then holds at least the header's bytes.
inline BamHeader read_bam_header(InflateStream& stream, std::vector<uint8_t>& buf, const std::string& path,
                                 const std::vector<uint8_t>& known_refs = {}) {
  auto need = [&](size_t bytes) {  // buf[0, bytes) available; false at EOF
    while (buf.size() < bytes)
      if (!stream.fill(buf)) return false;
    return true;
  };
  BamHeader h;
  if (!need(12) || memcmp(buf.data(), "BAM\1", 4) != 0) throw Panic("Error reading BAM header: not a BAM/SAM file: " + path);
  const uint32_t l_text = rd_u32(buf.data() + 4);
  if (!need(12 + (size_t)l_text)) throw Panic("Error reading BAM header: truncated");
  h.refs_at = 8 + (size_t)l_text;
  if (known_refs.size() >= 4 && need(h.refs_at + known_refs.size()) &&
      memcmp(buf.data() + h.refs_at, known_refs.data(), known_refs.size()) == 0) {
    h.records_at = h.refs_at + known_refs.size();
    return h;
  }
  h.header = std::make_shared<Header>();
  const uint32_t n_ref = rd_u32(buf.data() + h.refs_at);
  size_t o = h.refs_at + 4;
  h.header->names.reserve(n_ref);
  h.header->lens.reserve(n_ref);
  for (uint32_t i = 0; i < n_ref; ++i) {
    if (!need(o + 4)) throw Panic("Error reading BAM header: truncated");
    const uint32_t l_name = rd_u32(buf.data() + o);
    if (!need(o + 8 + l_name)) throw Panic("Error reading BAM header: truncated");
    h.header->names.emplace_back((const char*)buf.data() + o + 4, l_name ? l_name - 1 : 0);
    h.header->lens.push_back(rd_u32(buf.data() + o + 4 + l_name));
    o += 8 + l_name;
  }
  h.records_at = o;
  return h;
}

// cmb_bgzf_input over the blocks of a BGZF index (the device inflates and decodes them itself), with the per-block arrays it
// points at.
class BgzfInput {
 public:
  cmb_bgzf_input in{};
  BgzfInput(const BlockIndex& bx, uint32_t n_ref, uint64_t records_at, int threads)
      : coff_(bx.blocks.size()), clen_(bx.blocks.size()), isz_(bx.blocks.size()) {
    for (size_t b = 0; b < bx.blocks.size(); ++b) {
      coff_[b] = bx.blocks[b].cdata;
      clen_[b] = (uint32_t)bx.blocks[b].clen;
      isz_[b] = bx.blocks[b].isize;
    }
    in.data = bx.p;
    in.size = bx.n;
    in.n_blocks = (uint32_t)bx.blocks.size();
    in.n_ref = n_ref;
    in.block_coffset = coff_.data();
    in.block_clen = clen_.data();
    in.block_isize = isz_.data();
    in.records_at = records_at;
    in.copy_threads = (uint32_t)std::min(threads, 8);
  }
  BgzfInput(const BgzfInput&) = delete;

 private:
  std::vector<uint64_t> coff_;
  std::vector<uint32_t> clen_, isz_;
};

// A BAM record header that could be real: sane block_size, reference ids, name length and NUL, field sizes.  Shared by
// the speculative record alignment of the host decoder (decode_runner.hpp) and the block-range probe (shard_range.hpp).
inline bool record_plausible(const uint8_t* buf, size_t s, size_t usize, uint32_t n_ref) {
  if (s + 36 > usize) return false;
  const uint32_t bs = rd_u32(buf + s);
  if (bs < 32 || bs > (64u << 20)) return false;
  const int32_t tid = (int32_t)rd_u32(buf + s + 4), pos = (int32_t)rd_u32(buf + s + 8), mtid = (int32_t)rd_u32(buf + s + 24);
  if (tid < -1 || tid >= (int32_t)n_ref || mtid < -1 || mtid >= (int32_t)n_ref || pos < -1) return false;
  const uint32_t l_name = buf[s + 12], n_cig = rd_u16(buf + s + 16), l_seq = rd_u32(buf + s + 20);
  if (l_name == 0 || l_seq > (1u << 28)) return false;
  const uint64_t fixed = 32ull + l_name + 4ull * n_cig + (l_seq + 1) / 2 + l_seq;
  if (fixed > bs) return false;
  if (s + 36 + l_name <= usize && buf[s + 36 + l_name - 1] != 0) return false;
  return true;
}

// Walks the block_size chain of the records in buf[from, size): f(offset) for every complete record, until f returns false.
// Returns where the walk stopped.  `at_eof`: the stream ends at `size`, and bytes left over there are a record cut short --
// htslib's bam_read1 fails on it and the reference panics on the Err (contig.rs:113-115).
template <class F>
inline size_t walk_records(const uint8_t* buf, size_t from, size_t size, bool at_eof, F f) {
  size_t q = from;
  while (q + 4 <= size) {
    const uint32_t bs = rd_u32(buf + q);
    if (bs < 32) throw Panic("Error reading BAM record: corrupt block_size");
    if (q + 4 + (size_t)bs > size) break;
    const size_t rec = q;
    q += 4 + (size_t)bs;
    if (!f(rec)) break;
  }
  if (at_eof && q != size) throw Panic("Error reading BAM record: truncated");
  return q;
}

// Walks the aux fields in [a, end) (SAMv1 §4.2.4): f(tag0, tag1, type, value, size) for each, until f returns true.  A 'B'
// array cut short by `end` comes with the bytes that are left (size < 5).  Returns false at an unknown type.
template <class F>
inline bool walk_aux(const uint8_t* a, const uint8_t* end, F f) {
  while (a + 3 <= end) {
    const uint8_t t0 = a[0], t1 = a[1], ty = a[2];
    a += 3;
    size_t sz;
    switch (ty) {
      case 'A': case 'c': case 'C': sz = 1; break;
      case 's': case 'S': sz = 2; break;
      case 'i': case 'I': case 'f': sz = 4; break;
      case 'Z': case 'H': {
        const uint8_t* e = (const uint8_t*)memchr(a, 0, (size_t)(end - a));
        sz = e ? (size_t)(e - a) + 1 : (size_t)(end - a);
        break;
      }
      case 'B': {
        if (a + 5 > end) { sz = (size_t)(end - a); break; }
        const uint8_t sub = a[0];
        const size_t es = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4;
        sz = 5 + es * (size_t)rd_u32(a + 1);
        break;
      }
      default: return false;
    }
    if (f(t0, t1, ty, a, sz)) return true;
    a += sz;
  }
  return true;
}

// ---- record layout checks shared by every host decoder -------------------------------------------------------------
// htslib's bam_read1 rejects a record whose fixed-size fields do not fit its block_size (the reference then panics with
// "Error reading BAM record", contig.rs:113-115); the CIGAR / aux walks below rely on that having been checked.
// It also restores CIGARs of more than 65535 operations from the CG:B,I tag (bam_tag2cigar: the in-record CIGAR is then the
// placeholder `<l_seq>S<reflen>N`).  `rec` points at block_size and the whole record is in memory.
struct CigarView {
  const uint8_t* ops = nullptr;  // n little-endian u32 operations (len << 4 | op)
  uint32_t n = 0;
  bool valid = false;            // false: the fixed fields overrun block_size
};
inline CigarView effective_cigar(const uint8_t* rec) {
  CigarView v;
  const uint32_t block_size = rd_u32(rec);
  const uint8_t* o = rec + 4;
  const uint32_t l_read_name = o[8], n_cigar = rd_u16(o + 12), l_seq = rd_u32(o + 16);
  const uint64_t fixed = 32ull + l_read_name + 4ull * n_cigar + ((uint64_t)l_seq + 1) / 2 + l_seq;
  if (block_size < 32 || fixed > block_size) return v;
  v.valid = true;
  v.ops = o + 32 + l_read_name;
  v.n = n_cigar;
  if (n_cigar == 0) return v;
  const uint32_t op0 = rd_u32(v.ops);
  if ((op0 & 0xf) != 4 || (op0 >> 4) != l_seq) return v;  // not the placeholder: the common case ends here
  if ((int32_t)rd_u32(o) < 0 || (int32_t)rd_u32(o + 4) < 0) return v;
  const uint8_t* end = o + block_size;
  // bam_aux_get(b, "CG"); an unknown aux type ends the search (the NM walk raises the error)
  walk_aux(o + fixed, end, [&](uint8_t t0, uint8_t t1, uint8_t ty, const uint8_t* a, size_t sz) {
    if (ty != 'B') return false;
    if (sz < 5) return true;
    if (t0 != 'C' || t1 != 'G') return false;
    const uint8_t sub = a[0];
    const uint32_t cnt = rd_u32(a + 1);
    if ((sub == 'I' || sub == 'i') && cnt >= n_cigar && cnt < (1u << 29) && sz <= (size_t)(end - a)) {
      v.ops = a + 5;
      v.n = cnt;
    }
    return true;
  });
  return v;
}
[[noreturn]] inline void throw_bad_record_layout() {
  throw Panic("Error reading BAM record: the record's name, CIGAR and sequence fields do not fit its block_size");
}
// Upper bound of the intervals a record can produce (the operation count of its effective CIGAR); -1: invalid layout.
inline int64_t record_cigar_ops(const uint8_t* rec) {
  const CigarView v = effective_cigar(rec);
  return v.valid ? (int64_t)v.n : -1;
}

// Decode the fixed fields, CIGAR summary and NM aux of one BAM record (`rec` points at block_size); M/=/X blocks
// (contig.rs:171-186) are written to ivs/ivl (room for record_cigar_ops entries).  A block starting before the contig is
// clamped to -1 as on the device (cmb_decode.cuh), which K1 rejects as out of bounds.  Returns the number of intervals.
inline uint32_t decode_bam_record(const uint8_t* rec, Tuple& t, int32_t* ivs, int32_t* ivl) {
  const uint32_t block_size = rd_u32(rec);
  const uint8_t* o = rec + 4;
  t.tid = (int32_t)rd_u32(o);
  t.pos = (int32_t)rd_u32(o + 4);
  const uint32_t l_read_name = o[8];
  t.mapq = o[9];
  const uint32_t n_cigar = rd_u16(o + 12);
  t.flag = rd_u16(o + 14);
  t.l_seq = rd_u32(o + 16);
  t.mtid = (int32_t)rd_u32(o + 20);
  const CigarView cv = effective_cigar(rec);
  if (!cv.valid) throw_bad_record_layout();
  uint32_t aligned = 0, del = 0, ins = 0, n_iv = 0;
  int64_t cursor = t.pos;
  for (uint32_t i = 0; i < cv.n; ++i) {
    const uint32_t v = rd_u32(cv.ops + 4 * (size_t)i);
    const uint32_t op = v & 0xf, len = v >> 4;
    switch (op) {
      case 0: case 7: case 8:  // M = X
        ivs[n_iv] = cursor < 0 ? -1 : (int32_t)std::min<int64_t>(cursor, INT32_MAX);
        ivl[n_iv] = (int32_t)len;
        ++n_iv;
        cursor += len;
        aligned += len;
        break;
      case 2: cursor += len; del += len; aligned += len; break;  // D
      case 3: cursor += len; break;                              // N
      case 1: ins += len; aligned += len; break;                 // I
      default: break;                                            // S H P
    }
  }
  t.aligned = aligned;
  t.del = del;
  t.ins = ins;
  t.n_iv = n_iv;
  // aux: NM (lib.rs:139-156: U8/U16/U32 accepted, anything else is a type panic, absent is a panic)
  t.nm_state = 0;
  t.nm = 0;
  const uint8_t* aux = o + 32 + l_read_name + 4 * (size_t)n_cigar + (t.l_seq + 1) / 2 + t.l_seq;
  const bool known = walk_aux(aux, o + block_size, [&](uint8_t t0, uint8_t t1, uint8_t ty, const uint8_t* a, size_t) {
    if (t0 == 'N' && t1 == 'M' && t.nm_state == 0) {
      if (ty == 'C') { t.nm_state = 1; t.nm = a[0]; }
      else if (ty == 'S') { t.nm_state = 1; t.nm = rd_u16(a); }
      else if (ty == 'I') { t.nm_state = 1; t.nm = rd_u32(a); }
      else t.nm_state = 2;
    }
    return false;  // the whole list is walked: an unknown type further on is still an error
  });
  if (!known) throw Panic("Error reading BAM record: unknown aux type");
  return n_iv;
}
// The same, appending the intervals to ivs/ivl.
inline void decode_bam_record(const uint8_t* rec, Tuple& t, std::vector<int32_t>& ivs, std::vector<int32_t>& ivl) {
  const int64_t ops = record_cigar_ops(rec);
  if (ops < 0) throw_bad_record_layout();
  const size_t at = ivs.size();
  ivs.resize(at + (size_t)ops);
  ivl.resize(at + (size_t)ops);
  const uint32_t n_iv = decode_bam_record(rec, t, ivs.data() + at, ivl.data() + at);
  ivs.resize(at + n_iv);
  ivl.resize(at + n_iv);
}

// Row r of a tuple table in SoA form (a cmb_read_batch, or cmbh_tuples) whose intervals start at `iv`; ivs/ivl are copied
// there, or are there already when nullptr.
template <class Soa>
inline void put_tuple(const Soa& b, size_t r, uint32_t iv, const Tuple& t, const int32_t* ivs, const int32_t* ivl) {
  b.tid[r] = t.tid; b.pos[r] = t.pos; b.flag[r] = t.flag; b.mapq[r] = t.mapq; b.nm_state[r] = t.nm_state;
  b.nm[r] = t.nm; b.l_seq[r] = t.l_seq; b.aligned[r] = t.aligned; b.del[r] = t.del; b.ins[r] = t.ins;
  b.iv_begin[r] = iv;
  if (ivs)
    for (uint32_t k = 0; k < t.n_iv; ++k) {
      b.iv_start[iv + k] = ivs[k];
      b.iv_len[iv + k] = ivl[k];
    }
}

inline std::string bam_qname(const uint8_t* rec) {
  const uint32_t l = rec[4 + 8];
  return std::string((const char*)rec + 4 + 32, l ? l - 1 : 0);
}

// The host's mate matching, ReferenceSortedBamFilter's (filter.rs:149-224), over the proper-pair records of a stream in
// stream order: the names kept are forgotten when the reference changes, a first mate is kept only when its mate maps to
// the current reference, and the second record of a name hands the kept first mate back.  Which records take part is the
// caller's business.
template <class Stored>
class HostMates {
 public:
  // The kept first mate of `t`, if any; otherwise make()'s copy of `t` is kept when its mate maps to the current reference.
  template <class Make>
  std::optional<Stored> match(const Tuple& t, std::string qname, Make make) {
    if (t.tid != current_reference_) {
      current_reference_ = t.tid;
      first_set_.clear();
    }
    auto it = first_set_.find(qname);
    if (it == first_set_.end()) {
      if (t.mtid == current_reference_) first_set_.emplace(std::move(qname), make());
      return std::nullopt;
    }
    std::optional<Stored> first(std::move(it->second));
    first_set_.erase(it);
    return first;
  }

 private:
  std::map<std::string, Stored> first_set_;  // filter.rs:16-18
  int32_t current_reference_ = -1;
};

}  // namespace cmbh
