// BgzfWriter (coverm_b200/csrc/host/bgzf_writer.hpp) fed a byte stream in arbitrary pieces writes exactly the file a one-shot
// BGZF writer writes for the concatenation, and that file inflates back to the stream.  Pieces: random lengths, empty pieces,
// pieces ending on multiples of the 0xff00-byte block, single bytes, one piece for everything, and nothing at all.
// Prints "ok <cases>" on success.
#include <cstdio>
#include <random>
#include <sstream>
#include <string>

#include "host/bgzf_writer.hpp"

using cmbh::BgzfWriter;

// The concatenation cut into 0xff00-byte blocks, each deflated alone at zlib's default level, then the EOF block
static std::string one_shot(const std::vector<uint8_t>& data) {
  std::string out;
  const size_t B = 0xff00;
  for (size_t from = 0; from < data.size(); from += B) {
    const size_t len = std::min(B, data.size() - from);
    z_stream zs{};
    deflateInit2(&zs, Z_DEFAULT_COMPRESSION, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY);
    std::vector<uint8_t> comp(B + 1024);
    zs.next_in = const_cast<Bytef*>(data.data() + from);
    zs.avail_in = (uInt)len;
    zs.next_out = comp.data();
    zs.avail_out = (uInt)comp.size();
    if (deflate(&zs, Z_FINISH) != Z_STREAM_END) abort();
    const size_t clen = zs.total_out;
    deflateEnd(&zs);
    const uint32_t bsize = (uint32_t)(18 + clen + 8 - 1);
    const uint8_t hdr[18] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, (uint8_t)(bsize & 0xff), (uint8_t)(bsize >> 8)};
    out.append((const char*)hdr, 18);
    out.append((const char*)comp.data(), clen);
    const uint32_t crc = (uint32_t)crc32(0, data.data() + from, (uInt)len), isz = (uint32_t)len;
    out.append((const char*)&crc, 4);
    out.append((const char*)&isz, 4);
  }
  static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  out.append((const char*)eof, 28);
  return out;
}

// zlib's inflate of every block of a BGZF file, checked against each footer
static bool inflate_all(const std::string& f, std::vector<uint8_t>& out) {
  size_t o = 0;
  while (o < f.size()) {
    if (o + 18 > f.size() || (uint8_t)f[o] != 0x1f || (uint8_t)f[o + 1] != 0x8b) return false;
    const size_t bsize = (size_t)(uint8_t)f[o + 16] + ((size_t)(uint8_t)f[o + 17] << 8) + 1;
    uint32_t crc, isz;
    memcpy(&crc, f.data() + o + bsize - 8, 4);
    memcpy(&isz, f.data() + o + bsize - 4, 4);
    std::vector<uint8_t> buf(isz + 1);
    z_stream zs{};
    inflateInit2(&zs, -15);
    zs.next_in = (Bytef*)f.data() + o + 18;
    zs.avail_in = (uInt)(bsize - 26);
    zs.next_out = buf.data();
    zs.avail_out = (uInt)buf.size();
    const int r = inflate(&zs, Z_FINISH);
    const size_t got = zs.total_out;
    inflateEnd(&zs);
    if (r != Z_STREAM_END || got != isz || (uint32_t)crc32(0, buf.data(), isz) != crc) return false;
    out.insert(out.end(), buf.begin(), buf.begin() + isz);
    o += bsize;
  }
  return o == f.size();
}

int main() {
  std::mt19937_64 rng(12345);
  cmbh::ThreadPool pool(4);
  const size_t B = BgzfWriter::BLOCK;
  int cases = 0;
  for (size_t total : {(size_t)0, (size_t)1, B - 1, B, B + 1, 3 * B, 64 * B + 17, (size_t)5'000'000}) {
    // compressible but not trivial: runs of random bytes from a small alphabet
    std::vector<uint8_t> data(total);
    for (size_t i = 0; i < total; ++i) data[i] = (uint8_t)((rng() % 7 == 0) ? rng() : 'A' + rng() % 4);
    const std::string want = one_shot(data);
    std::vector<uint8_t> back;
    if (!inflate_all(want, back) || back != data) {
      fprintf(stderr, "the one-shot writer does not round-trip (%zu bytes)\n", total);
      return 1;
    }
    for (int kind = 0; kind < 6; ++kind) {
      // the piece lengths
      std::vector<size_t> lens;
      size_t left = total;
      while (left) {
        size_t n = 0;
        switch (kind) {
          case 0: n = left; break;                                   // one piece
          case 1: n = 1; break;                                      // single bytes
          case 2: n = 1 + rng() % (2 * B); break;                    // random
          case 3: n = (rng() % 3) * B; break;                        // block multiples, some empty
          case 4: n = rng() % 2 ? 0 : 1 + rng() % 1000; break;       // small, many empty
          default: n = lens.size() % 2 ? B - lens.size() % 5 : 1 + rng() % (8 * B); break;  // around the block edge
        }
        if (lens.size() >= 400) n = left;  // the rest in one piece: a feed costs a thread
        n = std::min(n, left);
        lens.push_back(n);
        left -= n;
      }
      if (kind == 4) lens.insert(lens.begin(), 0);
      std::ostringstream os;
      {
        BgzfWriter w(os, pool);
        // every piece in a buffer of its own that lives until the next call returns, as the writer requires
        std::vector<uint8_t> piece[2];
        size_t at = 0, k = 0;
        for (size_t n : lens) {
          auto& buf = piece[k++ & 1];
          buf.assign(data.begin() + at, data.begin() + at + n);
          w.feed(buf.data(), n);
          at += n;
        }
        w.finish();
      }
      const std::string got = os.str();
      if (got != want) {
        fprintf(stderr, "total %zu, pieces kind %d (%zu pieces): %zu bytes written, %zu expected\n", total, kind, lens.size(), got.size(), want.size());
        return 1;
      }
      ++cases;
    }
    // reset drops everything fed that is not written yet; the stream written after it is a file of its own
    if (total >= B) {
      std::ostringstream os;
      BgzfWriter w(os, pool);
      std::vector<uint8_t> junk(B / 2, 'x');
      w.feed(junk.data(), junk.size());
      w.reset();
      w.feed(data.data(), data.size());
      w.finish();
      if (os.str() != want) {
        fprintf(stderr, "total %zu: reset kept bytes fed before it\n", total);
        return 1;
      }
      ++cases;
    }
  }
  printf("ok %d\n", cases);
  return 0;
}
