// Host-side check of the BGZF deflate encoder (coverm_b200/csrc/cmb_deflate.cuh), compiled as plain C++: the same code the
// kz_deflate kernel runs, its CTA's threads run one after the other.  Every block it makes must inflate (zlib, raw) to its
// input, carry a correct header, BSIZE, CRC32 and ISIZE, fit in 64 KiB, use complete Huffman codes within their length
// limits, be stored when the input is incompressible, come out the same on a second run, and inflate through the project's
// own first-pass decoder (kd_inflate_t1, cmb_decode_t1.cuh, host build as in t1_inflate_check.cpp) to the same bytes.
//
//   deflate_check <bam>...               the checks over the BAMs' inflated streams and over synthetic buffers
//   deflate_check --recompress in out    writes in's inflated stream as the encoder's BGZF file (blocks of 0xff00 bytes + EOF)
#include <zlib.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <vector>

#define __device__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__
#define __align__(x)
#define T1_HOST_TEST 1
struct Dim3 { unsigned x = 0, y = 0, z = 0; };
static Dim3 threadIdx, blockIdx, gridDim;
static inline uint32_t __brev(uint32_t v) {
  v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
  v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
  v = ((v >> 4) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4);
  v = ((v >> 8) & 0x00ff00ffu) | ((v & 0x00ff00ffu) << 8);
  return (v >> 16) | (v << 16);
}
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline uint32_t atomicAdd(uint32_t* p, uint32_t v) { uint32_t o = *p; *p += v; return o; }
static inline void __threadfence_system() {}
static inline void __nanosleep(unsigned) {}
using std::min;
static const uint8_t c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
struct InflateArgs {
  const uint8_t* comp; const uint64_t* coff; const uint32_t* clen; const uint32_t* isize; const uint64_t* uoff;
  uint32_t b0, b1; uint8_t* out; uint32_t* status; uint32_t* ticket; uint32_t* fail_count;
  const uint32_t* block_window; const uint32_t* ready; uint32_t lane_limit;
  const uint32_t* block_list; uint8_t* scratch;
};
uint8_t t1_smem[4096];
#include "../../coverm_b200/csrc/cmb_decode_t1.cuh"
#undef __device__
#undef __forceinline__
#include "../../coverm_b200/csrc/cmb_deflate.cuh"

using namespace std;
using namespace cmb_dfl;

static int fails = 0;
#define CHECK(cond, ...)                                   \
  do {                                                     \
    if (!(cond)) {                                         \
      if (++fails < 20) {                                  \
        printf("FAIL %s:%d: ", __FILE__, __LINE__);        \
        printf(__VA_ARGS__);                               \
        printf("\n");                                      \
      }                                                    \
    }                                                      \
  } while (0)

static unique_ptr<DflSmem> S(new DflSmem);

static vector<uint8_t> encode(const uint8_t* p, size_t n) {
  vector<uint8_t> out(DFL_MAX_OUT);
  dfl_encode_block(*S, p, (uint32_t)n, out.data());
  out.resize(S->size);
  return out;
}

static vector<uint8_t> inflate_raw(const uint8_t* p, size_t n, size_t want, bool* ok) {
  vector<uint8_t> out(want + 16);
  z_stream zs{};
  inflateInit2(&zs, -15);
  zs.next_in = (Bytef*)p; zs.avail_in = (uInt)n; zs.next_out = out.data(); zs.avail_out = (uInt)out.size();
  const int r = inflate(&zs, Z_FINISH);
  *ok = r == Z_STREAM_END && zs.avail_in == 0;
  out.resize(zs.total_out);
  inflateEnd(&zs);
  return out;
}

static bool complete(const uint8_t* len, uint32_t n, uint32_t maxlen) {
  uint64_t kraft = 0;
  for (uint32_t s = 0; s < n; ++s) {
    if (len[s] > maxlen) return false;
    if (len[s]) kraft += 1ull << (maxlen - len[s]);
  }
  return kraft == (1ull << maxlen);
}

struct T1Batch {  // blocks for one run of the t1 decoder's host build
  vector<vector<uint8_t>> comp, want;
};
static uint64_t n_t1 = 0, t1_declined = 0;
static void run_t1(T1Batch& b) {
  vector<uint8_t> file(64, 0xEE);
  vector<uint64_t> coff, uoff;
  vector<uint32_t> clen, isize;
  uint64_t u = 7;
  for (size_t i = 0; i < b.comp.size(); ++i) {
    coff.push_back(file.size());
    clen.push_back((uint32_t)b.comp[i].size());
    file.insert(file.end(), b.comp[i].begin(), b.comp[i].end());
    file.insert(file.end(), 8, 0xAB);
    isize.push_back((uint32_t)b.want[i].size());
    uoff.push_back(u);
    u += b.want[i].size() + 3;
  }
  file.resize(file.size() + 1024, 0);
  vector<uint8_t> inflated(u + 1024, 0x5A);
  vector<uint32_t> status(b.comp.size(), 99);
  uint32_t ticket = 0, nf = 0;
  InflateArgs a{};
  a.comp = file.data(); a.coff = coff.data(); a.clen = clen.data(); a.isize = isize.data(); a.uoff = uoff.data();
  a.b0 = 0; a.b1 = (uint32_t)b.comp.size(); a.out = inflated.data(); a.status = status.data(); a.ticket = &ticket; a.fail_count = &nf;
  vector<uint8_t> scratch(b.comp.size() * 160 + 16, 0x77);
  a.scratch = scratch.data();
  kd_inflate_t1(a);
  for (size_t i = 0; i < b.comp.size(); ++i) {
    ++n_t1;
    if (status[i] != 0) {  // declined: the second pass (kd_inflate) takes such a block on the device
      ++t1_declined;
      continue;
    }
    CHECK(equal(b.want[i].begin(), b.want[i].end(), inflated.begin() + uoff[i]), "t1 decoder: block %zu inflates to other bytes", i);
  }
  b.comp.clear();
  b.want.clear();
}

static uint64_t n_blocks = 0, n_stored = 0, raw_total = 0, bgzf_total = 0, zlib6_total = 0;
static T1Batch t1;

// Encodes p[0, n), checks the block, and returns it
static vector<uint8_t> check_block(const uint8_t* p, size_t n, const char* what, int expect_stored = -1) {
  vector<uint8_t> blk = encode(p, n);
  const bool stored = S->stored;
  if (!stored) {
    CHECK(complete(S->t.llen, 286, 15), "%s n=%zu: literal/length code incomplete or too long", what, n);
    CHECK(complete(S->t.dlen, 30, 15), "%s n=%zu: distance code incomplete or too long", what, n);
    CHECK(complete(S->t.clen, 19, 7), "%s n=%zu: code-length code incomplete or too long", what, n);
  }
  if (expect_stored >= 0) CHECK(stored == (bool)expect_stored, "%s n=%zu: stored=%d", what, n, (int)stored);
  CHECK(blk.size() <= 65536 && blk.size() >= 26, "%s n=%zu: block of %zu bytes", what, n, blk.size());
  static const uint8_t hdr[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
  CHECK(memcmp(blk.data(), hdr, 16) == 0, "%s n=%zu: header", what, n);
  CHECK((size_t)(blk[16] | blk[17] << 8) == blk.size() - 1, "%s n=%zu: BSIZE", what, n);
  uint32_t crc, isz;
  memcpy(&crc, blk.data() + blk.size() - 8, 4);
  memcpy(&isz, blk.data() + blk.size() - 4, 4);
  CHECK(crc == (uint32_t)crc32(0, p, (uInt)n), "%s n=%zu: CRC32", what, n);
  CHECK(isz == n, "%s n=%zu: ISIZE", what, n);
  bool ok;
  const vector<uint8_t> back = inflate_raw(blk.data() + 18, blk.size() - 26, n, &ok);
  CHECK(ok && back.size() == n && equal(back.begin(), back.end(), p), "%s n=%zu: does not inflate to its input", what, n);
  CHECK(encode(p, n) == blk, "%s n=%zu: a second run gives other bytes", what, n);
  t1.comp.emplace_back(blk.begin() + 18, blk.end() - 8);
  t1.want.emplace_back(p, p + n);
  if (t1.comp.size() == 64) run_t1(t1);
  ++n_blocks;
  n_stored += stored;
  raw_total += n;
  bgzf_total += blk.size();
  return blk;
}

static vector<uint8_t> read_bgzf(const char* path) {
  gzFile f = gzopen(path, "rb");
  if (!f) return {};
  vector<uint8_t> out;
  uint8_t buf[1 << 16];
  int r;
  while ((r = gzread(f, buf, sizeof buf)) > 0) out.insert(out.end(), buf, buf + r);
  gzclose(f);
  return out;
}

static size_t zlib6_block(const uint8_t* p, size_t n) {
  z_stream zs{};
  deflateInit2(&zs, 6, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY);
  vector<uint8_t> out(deflateBound(&zs, n) + 64);
  zs.next_in = (Bytef*)p; zs.avail_in = (uInt)n; zs.next_out = out.data(); zs.avail_out = (uInt)out.size();
  deflate(&zs, Z_FINISH);
  const size_t r = zs.total_out + 26;
  deflateEnd(&zs);
  return r;
}

int main(int argc, char** argv) {
  if (argc == 4 && string(argv[1]) == "--recompress") {
    const vector<uint8_t> s = read_bgzf(argv[2]);
    FILE* f = fopen(argv[3], "wb");
    if (!f) return 2;
    for (size_t o = 0; o < s.size(); o += DFL_BLOCK) {
      const vector<uint8_t> b = encode(s.data() + o, min<size_t>(DFL_BLOCK, s.size() - o));
      fwrite(b.data(), 1, b.size(), f);
    }
    static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    fwrite(eof, 1, sizeof eof, f);
    return fclose(f) ? 2 : 0;
  }
  // the BAMs' record streams, in the blocks a BGZF writer cuts them into
  uint64_t bam_raw = 0, bam_bgzf = 0, bam_zlib6 = 0;
  for (int k = 1; k < argc; ++k) {
    const vector<uint8_t> s = read_bgzf(argv[k]);
    CHECK(!s.empty(), "%s: not read", argv[k]);
    for (size_t o = 0; o < s.size(); o += DFL_BLOCK) {
      const size_t n = min<size_t>(DFL_BLOCK, s.size() - o);
      bam_bgzf += check_block(s.data() + o, n, argv[k]).size();
      bam_zlib6 += zlib6_block(s.data() + o, n);
      bam_raw += n;
    }
  }
  mt19937_64 rng(7);
  vector<uint8_t> d(DFL_BLOCK);
  // sizes at the edges, over several shapes
  const size_t sizes[] = {0, 1, 2, 3, 4, 257, 258, 259, 1000, 32768, 32769, 0xfeff, 0xff00};
  for (size_t n : sizes)
    for (int kind = 0; kind < 5; ++kind) {
      for (size_t i = 0; i < n; ++i) {
        switch (kind) {
          case 0: d[i] = (uint8_t)rng(); break;                 // incompressible
          case 1: d[i] = 0; break;                               // all zero: 258-byte matches
          case 2: d[i] = (uint8_t)(i % 37); break;               // periodic
          case 3: { static const char* w = "the quick brown fox jumps over the lazy dog "; d[i] = (uint8_t)w[(i + (rng() % 50 == 0)) % 44]; } break;
          case 4: d[i] = "ACGT"[rng() & 3]; break;               // 2 bits per byte
        }
      }
      check_block(d.data(), n, "synthetic", kind == 0 && n >= 64 ? 1 : kind == 1 && n >= 64 ? 0 : -1);
    }
  // long runs and far matches: a random 32 KiB half repeated at distance 32768 (and one at 40000, out of reach)
  for (size_t i = 0; i < 32768; ++i) d[i] = "ACGTN"[rng() % 5];
  for (size_t i = 32768; i < DFL_BLOCK; ++i) d[i] = d[i - 32768];
  check_block(d.data(), DFL_BLOCK, "distance 32768");
  for (size_t i = 0; i < 40000; ++i) d[i] = (uint8_t)rng();
  for (size_t i = 40000; i < DFL_BLOCK; ++i) d[i] = d[i - 40000];
  check_block(d.data(), DFL_BLOCK, "distance 40000");
  for (size_t i = 0; i < DFL_BLOCK; ++i) d[i] = (i / 300) & 1 ? 'A' : (uint8_t)(i / 600);
  check_block(d.data(), DFL_BLOCK, "runs of 300");
  // random sizes and mixtures
  for (int it = 0; it < 300; ++it) {
    const size_t n = it < 20 ? (size_t)it : rng() % (DFL_BLOCK + 1);
    const int kind = it % 4;
    for (size_t i = 0; i < n; ++i) {
      switch (kind) {
        case 0: d[i] = rng() % 8 ? 'A' : (uint8_t)rng(); break;
        case 1: d[i] = i > 3 && rng() % 4 ? d[i - 1 - rng() % min<size_t>(i - 1, 5)] : (uint8_t)rng(); break;
        case 2: d[i] = (uint8_t)((i % 37) ^ (rng() % 100 == 0)); break;
        case 3: d[i] = i > 1000 && rng() % 16 ? d[i - 1 - rng() % 1000] : "ACGT"[rng() & 3]; break;
      }
    }
    check_block(d.data(), n, "mixed");
  }
  if (!t1.comp.empty()) run_t1(t1);
  printf("%s %llu blocks (%llu stored), raw %llu -> BGZF %llu; t1 decoder read %llu of %llu blocks, declined %llu",
         fails ? "FAILED" : "ok", (unsigned long long)n_blocks, (unsigned long long)n_stored, (unsigned long long)raw_total,
         (unsigned long long)bgzf_total, (unsigned long long)(n_t1 - t1_declined), (unsigned long long)n_t1,
         (unsigned long long)t1_declined);
  if (bam_raw) printf("; BAM streams: raw %llu, encoder %llu, zlib-6 %llu (ratio %.4f)", (unsigned long long)bam_raw,
                      (unsigned long long)bam_bgzf, (unsigned long long)bam_zlib6, (double)bam_bgzf / (double)bam_zlib6);
  printf("\n");
  return fails ? 1 : 0;
}
