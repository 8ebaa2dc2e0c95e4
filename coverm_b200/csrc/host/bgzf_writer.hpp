// BGZF output of `coverm filter`, written as the records arrive.  The concatenation of everything fed is cut into blocks of
// 0xff00 bytes (the last one shorter), each deflated alone (zlib level 6, raw deflate) with its BGZF header and CRC32/ISIZE
// footer, then the 28-byte EOF block.  Each block depends only on its own bytes, so the file is the same however the stream
// was cut into feeds: a filter run decoded in slices writes the file a whole-stream run writes.
#pragma once
#include <zlib.h>

#include <cstring>
#include <future>
#include <ostream>
#include <vector>

#include "bam_source.hpp"

namespace cmbh {

class BgzfWriter {
 public:
  static constexpr size_t BLOCK = 0xff00;  // uncompressed bytes per block
  static constexpr size_t GROUP = 16;      // blocks per pool task

  BgzfWriter(std::ostream& os, ThreadPool& pool) : os_(os), pool_(pool) {}
  ~BgzfWriter() {
    if (job_.valid()) job_.wait();
  }
  BgzfWriter(const BgzfWriter&) = delete;
  BgzfWriter& operator=(const BgzfWriter&) = delete;

  // Appends p[0, n).  The full blocks it completes are deflated on the pool and written in the background: p must stay valid
  // until the next call into the writer returns.  Rethrows an error of the previous feed's background work.
  void feed(const uint8_t* p, size_t n) {
    wait();
    if (!n) return;
    job_ = std::async(std::launch::async, [this, p, n] { write_blocks(p, n); });
  }
  // Waits for the background work, writes the partial last block and the EOF block
  void finish() {
    wait();
    if (!carry_.empty()) write_blocks(nullptr, 0, true);
    static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    os_.write((const char*)eof, sizeof eof);
  }
  // Forgets everything fed that is not written yet (the caller empties the stream itself); an error of the background work is
  // dropped with it
  void reset() {
    if (job_.valid()) job_.wait();
    job_ = {};
    carry_.clear();
  }

 private:
  void wait() {
    if (job_.valid()) job_.get();
  }
  // carry_ + p[0, n) in blocks: every full block (and with `last` the partial one) deflated and written; the rest kept in carry_
  void write_blocks(const uint8_t* p, size_t n, bool last = false) {
    const size_t total = carry_.size() + n;
    const size_t n_blocks = last ? (total + BLOCK - 1) / BLOCK : total / BLOCK;
    if (n_blocks) {
      // block 0 may start in carry_: assemble it; the others lie in p
      const size_t head = std::min(total, BLOCK) - carry_.size();
      carry_.insert(carry_.end(), p, p + head);
      auto block = [&](size_t b, size_t* len) -> const uint8_t* {
        *len = std::min(BLOCK, total - b * BLOCK);
        return b == 0 ? carry_.data() : p + (b * BLOCK - (carry_.size() - head));
      };
      std::vector<std::vector<uint8_t>> done((n_blocks + GROUP - 1) / GROUP);
      pool_.parallel_for(done.size(), [&](size_t g, int) {
        std::vector<uint8_t> comp(BLOCK + 1024);
        z_stream zs;
        memset(&zs, 0, sizeof zs);
        if (deflateInit2(&zs, Z_DEFAULT_COMPRESSION, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) throw ExitError(1, "zlib init failed");
        std::vector<uint8_t>& outb = done[g];
        for (size_t b = g * GROUP; b < std::min(n_blocks, (g + 1) * GROUP); ++b) {
          size_t len;
          const uint8_t* raw = block(b, &len);
          deflateReset(&zs);
          zs.next_in = const_cast<Bytef*>(raw);
          zs.avail_in = (uInt)len;
          zs.next_out = comp.data();
          zs.avail_out = (uInt)comp.size();
          if (deflate(&zs, Z_FINISH) != Z_STREAM_END) {
            deflateEnd(&zs);
            throw ExitError(1, "deflate failed");
          }
          const size_t clen = zs.total_out;
          const uint32_t bsize = (uint32_t)(12 + 6 + clen + 8 - 1);
          const uint8_t hdr[18] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, (uint8_t)(bsize & 0xff), (uint8_t)(bsize >> 8)};
          outb.insert(outb.end(), hdr, hdr + 18);
          outb.insert(outb.end(), comp.data(), comp.data() + clen);
          const uint32_t crc = (uint32_t)crc32(0, raw, (uInt)len), isz = (uint32_t)len;
          uint8_t tail[8];
          memcpy(tail, &crc, 4);
          memcpy(tail + 4, &isz, 4);
          outb.insert(outb.end(), tail, tail + 8);
        }
        deflateEnd(&zs);
      });
      for (auto& b : done) os_.write((const char*)b.data(), (std::streamsize)b.size());
      if (!os_) throw Panic("Failed to write BAM record");
      const size_t used = std::min(total, n_blocks * BLOCK);
      carry_.clear();
      const size_t from = used - (total - n);  // first byte of p not yet written
      carry_.assign(p + from, p + n);
    } else {
      carry_.insert(carry_.end(), p, p + n);
    }
  }

  std::ostream& os_;
  ThreadPool& pool_;
  std::vector<uint8_t> carry_;  // bytes fed past the last full block
  std::future<void> job_;
};

}  // namespace cmbh
