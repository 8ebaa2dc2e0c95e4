// The pair path of `coverm filter` and of the pair thresholds compiled as plain C++: kd_pair_keys / kd_pair_order /
// kd_pair_insert / kd_pair_resolve (coverm_b200/csrc/cmb_pairs.cuh) and kf_decide / kf_gather (cmb_filter.cuh), each kernel
// run thread by thread (CUDA keywords, atomics and the rounding intrinsics shimmed below; build with -ffp-contract=off).
// kd_pair_insert runs over a random permutation of the records, because the device's atomic order is arbitrary.  The two
// kernels that need a CTA barrier are replaced by sequential code: kd_pair_order_fold by the same fold over the chunk ranges,
// kf_scan by an exclusive scan (the GPU tests cover both).
//
// The expected result is ReferenceSortedBamFilter::read's walk (filter.rs:117-233) restated below in file order with a
// std::map cleared on every tid change.  Every stream must either give exactly its mate pairs, its filter roles and its
// output bytes (each byte written: the output is gathered twice, over two different fill bytes), or be declined -- and then
// only because its eligible tids go down in file order, or because a table slot holds more than PAIR_MAX_GROUP records.
// Collision mode cuts every key to four bits between kd_pair_keys and kd_pair_insert, so that distinct names and tids share a
// key and a slot.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <random>
#include <string>
#include <vector>

#include "../../include/coverm_b200.h"

#define __device__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__ static
#define __syncthreads()
struct Dim3 { unsigned x = 0, y = 0, z = 0; };
static Dim3 threadIdx, blockIdx;
struct uint2 { uint32_t x, y; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
using std::max;
using std::min;
static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
  const unsigned long long o = *p;
  if (o == cmp) *p = v;
  return o;
}
static inline uint32_t atomicExch(uint32_t* p, uint32_t v) { const uint32_t o = *p; *p = v; return o; }
static inline uint32_t atomicOr(uint32_t* p, uint32_t v) { const uint32_t o = *p; *p |= v; return o; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; *p += v; return o; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __uint2float_rn(uint32_t v) { return (float)v; }
static inline float __ull2float_rn(unsigned long long v) { return (float)v; }
static inline uint32_t ldu32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
constexpr uint32_t ERR_NM = 2u;  // cmb_common.cuh

#include "cmb_pairs.cuh"
#include "cmb_filter.cuh"

using namespace std;

namespace {

struct Rec {
  int32_t tid, mtid;
  uint16_t flag;
  string name;
  uint8_t mapq, nm_state;
  uint32_t nm, l_seq, aligned, del;
};

struct Stream {
  vector<Rec> recs;
  vector<uint8_t> data;  // BAM records back to back
  vector<uint64_t> off;
};

void encode(Stream& s, mt19937& rng) {
  s.data.assign(3, 0xEE);  // odd offsets on purpose
  s.off.clear();
  for (const Rec& r : s.recs) {
    const uint32_t l_name = (uint32_t)r.name.size() + 1, payload = rng() % 24;
    const uint32_t block_size = 32 + l_name + payload;
    s.off.push_back(s.data.size());
    uint8_t h[36] = {};
    auto put = [&](int at, uint32_t v) { memcpy(h + at, &v, 4); };
    put(0, block_size);
    put(4, (uint32_t)r.tid);
    put(8, rng() % 100000);                                       // pos
    put(12, l_name | (uint32_t)r.mapq << 8 | 4680u << 16);        // l_read_name, mapq, bin
    put(16, (uint32_t)r.flag << 16);                              // n_cigar_op = 0, flag
    put(20, r.l_seq);
    put(24, (uint32_t)r.mtid);
    put(28, rng() % 100000);                                      // next_pos
    put(32, rng());                                               // tlen
    s.data.insert(s.data.end(), h, h + 36);
    s.data.insert(s.data.end(), r.name.begin(), r.name.end());
    s.data.push_back(0);
    for (uint32_t k = 0; k < payload; ++k) s.data.push_back((uint8_t)rng());
  }
}

RecView view(const Rec& r) { return RecView{r.flag, r.mapq, r.nm_state, r.nm, r.l_seq, r.aligned, r.del}; }

struct Expected {
  vector<int32_t> mate;
  vector<uint8_t> role;
  vector<uint32_t> emitted;  // record indices in the order the reference returns them
  bool nm_panic = false;
  bool order_declines = false;  // eligible tids go down somewhere (the only order-based reason to decline)
};

bool eligible(const Rec& r, bool filter_out) { return !(r.flag & 0x900) && (r.flag & 0x2) && (filter_out || !(r.flag & 0x4)); }

// filter.rs:117-233 in file order, over records `recs` (filter_single: the single-read thresholds also apply to both mates).
Expected walk(const vector<Rec>& recs, const cmb_params& p, bool filter_single, bool filter_out) {
  Expected e;
  const size_t n = recs.size();
  e.mate.assign(n, -1);
  e.role.assign(n, 0);
  map<string, uint32_t> first_set;
  int32_t current_reference = -1;
  bool seen = false;
  uint32_t last_tid = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const Rec& r = recs[i];
    if (eligible(r, filter_out)) {
      if (seen && (uint32_t)r.tid < last_tid) e.order_declines = true;
      seen = true;
      last_tid = (uint32_t)r.tid;
    }
    if ((r.flag & 0x4) && !filter_out) {  // filter.rs:133-135
      e.emitted.push_back(i);
      e.role[i] = 1;
      continue;
    }
    if (r.flag & 0x900) continue;
    if (!(r.flag & 0x2)) {
      if (!filter_out) {
        e.emitted.push_back(i);
        e.role[i] = 1;
      }
      continue;
    }
    if (r.tid != current_reference) {
      current_reference = r.tid;
      first_set.clear();
    }
    auto it = first_set.find(r.name);
    if (it == first_set.end()) {
      if (r.mtid == current_reference) first_set.emplace(r.name, i);
      continue;
    }
    const uint32_t j = it->second;
    first_set.erase(it);
    e.mate[i] = (int32_t)j;
    e.mate[j] = (int32_t)i;
    bool nm_err = false;
    bool passes = true;  // && short-circuits: nm() is reached only where the reference reaches it
    if (filter_single) passes = single_read_passes(view(recs[j]), p, &nm_err) && single_read_passes(view(r), p, &nm_err);
    if (passes) passes = read_pair_passes(view(r), view(recs[j]), p, &nm_err);
    if (nm_err) e.nm_panic = true;
    if (passes == filter_out) {
      e.emitted.push_back(j);
      e.emitted.push_back(i);
      e.role[j] = 2;
      e.role[i] = 1;
    }
  }
  return e;
}

const char* ALPHA = "ABCxyz:/_#0123456789";

string random_name(mt19937& rng) {
  const uint32_t pick = rng() % 8;
  const uint32_t len = pick == 0 ? 254 : pick == 1 ? 1 : 1 + rng() % (pick < 4 ? 3 : 40);
  string s;
  for (uint32_t k = 0; k < len; ++k) s.push_back(ALPHA[rng() % 20]);
  return s;
}

Stream random_stream(mt19937& rng, uint32_t max_records) {
  Stream s;
  vector<string> pool;
  const uint32_t n_names = 1 + rng() % 12;
  for (uint32_t k = 0; k < n_names; ++k) {
    string nm = random_name(rng);
    if (!pool.empty() && rng() % 3 == 0) nm = pool[rng() % pool.size()].substr(0, 1 + rng() % 4);  // a prefix of another name
    pool.push_back(nm);
  }
  const uint32_t n = 1 + rng() % max_records, n_tids = 1 + rng() % 4;
  const bool interleaved = rng() % 4 == 0;
  const uint32_t unplaced_from = rng() % 3 == 0 ? n - rng() % (n / 8 + 1) : n;
  int32_t tid = 0;
  for (uint32_t i = 0; i < n; ++i) {
    Rec r{};
    if (interleaved) tid = (int32_t)(rng() % n_tids);
    else if (rng() % 12 == 0) tid = min<int32_t>(tid + 1, (int32_t)n_tids - 1);
    r.tid = i >= unplaced_from || rng() % 500 == 0 ? -1 : tid;  // unplaced: mostly at the end, as in a sorted file
    r.mtid = rng() % 6 == 0 ? (int32_t)(rng() % n_tids) : r.tid;
    static const uint16_t FLAGS[] = {0x1 | 0x2 | 0x40, 0x1 | 0x2 | 0x80, 0x1 | 0x2 | 0x10 | 0x80, 0x1 | 0x2 | 0x20 | 0x40,
                                     0x1 | 0x40,       0x1 | 0x2 | 0x100, 0x1 | 0x2 | 0x800,        0x1 | 0x2 | 0x4 | 0x40,
                                     0x1 | 0x2 | 0x8 | 0x80, 0x0,       0x1 | 0x2 | 0x4 | 0x100,  0x1 | 0x2 | 0x80};
    r.flag = FLAGS[rng() % 12];
    r.name = pool[rng() % pool.size()];
    r.mapq = (uint8_t)(rng() % 5 == 0 ? 255 : rng() % 61);
    r.nm_state = rng() % 50 == 0 ? 0 : 1;
    r.l_seq = 1 + rng() % 300;
    r.aligned = rng() % 8 == 0 ? 0 : rng() % (r.l_seq + 20);
    r.del = r.aligned ? rng() % min<uint32_t>(r.aligned, 6) : 0;
    r.nm = rng() % 12;
    s.recs.push_back(r);
  }
  encode(s, rng);
  return s;
}

cmb_params random_params(mt19937& rng, bool& filter_single) {
  cmb_params p{};
  p.filtering = 1;
  p.min_mapq = rng() % 3 == 0 ? (uint8_t)(rng() % 40) : 255;
  p.min_aligned_length_pair = rng() % 2 ? rng() % 400 : 0;
  p.min_percent_identity_pair = rng() % 2 ? (float)(rng() % 100) / 100.0f : 0.0f;
  p.min_aligned_percent_pair = rng() % 3 == 0 ? (float)(rng() % 100) / 100.0f : 0.0f;
  if (!p.min_aligned_length_pair && p.min_percent_identity_pair == 0.0f && p.min_aligned_percent_pair == 0.0f) p.min_aligned_length_pair = 1;
  filter_single = rng() % 3 == 0;
  if (filter_single) p.min_aligned_length_single = 1 + rng() % 100;
  return p;
}

struct Outcome {
  bool ok;
  string why;
};

// The kernels over one stream, checked against walk().
Outcome check(const Stream& s, const cmb_params& p, bool filter_single, bool filter_out, bool collide, mt19937& rng) {
  const uint32_t n = (uint32_t)s.recs.size();
  const Expected e = walk(s.recs, p, filter_single, filter_out);
  const uint32_t table = 64;
  vector<uint64_t> key(n);
  vector<int32_t> mate(n, 77);
  vector<uint32_t> next(n, 12345), slot_head(table, PAIR_NIL), flags(1, 0);
  vector<unsigned long long> slot_tag(table, 0);
  const uint32_t n_chunks = (n + PAIR_ORDER_CHUNK - 1) / PAIR_ORDER_CHUNK;
  vector<uint2> order(n_chunks, uint2{1, 1});
  PairArgs pa{};
  pa.data = s.data.data(); pa.rec_off = s.off.data(); pa.n_records = n; pa.key = key.data(); pa.mate = mate.data();
  pa.next = next.data(); pa.slot_tag = slot_tag.data(); pa.slot_head = slot_head.data(); pa.table_mask = table - 1;
  pa.flags = flags.data(); pa.order = order.data(); pa.filter_out = filter_out ? 1 : 0;
  auto at = [](uint32_t i) { blockIdx.x = i / 256; threadIdx.x = i % 256; };
  for (uint32_t i = 0; i < (n + 255) / 256 * 256; ++i) at(i), kd_pair_keys(pa);
  for (uint32_t c = 0; c < (n_chunks + 255) / 256 * 256; ++c) at(c), kd_pair_order(pa);
  uint32_t run_max = 0;  // kd_pair_order_fold
  for (uint32_t c = 0; c < n_chunks; ++c) {
    if (order[c].x < run_max) flags[0] |= DEC_ERR_PAIR_ORDER;
    run_max = max(run_max, order[c].y);
  }
  for (uint32_t i = 0; i < n; ++i)
    if ((key[i] != 0) != eligible(s.recs[i], filter_out)) return {false, "eligibility of record " + to_string(i)};
  if (collide)
    for (auto& k : key)
      if (k) k = (k & 0xf00000ull) | 1;
  vector<uint32_t> perm(n);
  for (uint32_t i = 0; i < n; ++i) perm[i] = i;
  shuffle(perm.begin(), perm.end(), rng);
  for (uint32_t i : perm) at(i), kd_pair_insert(pa);
  vector<uint32_t> slots(table);
  for (uint32_t t = 0; t < table; ++t) slots[t] = t;
  shuffle(slots.begin(), slots.end(), rng);
  for (uint32_t t : slots) at(t), kd_pair_resolve(pa);
  uint32_t biggest = 0;
  for (uint32_t t = 0; t < table; ++t) {
    uint32_t len = 0;
    for (uint32_t r = slot_head[t]; r != PAIR_NIL; r = next[r]) ++len;
    biggest = max(biggest, len);
  }
  const bool big = biggest > PAIR_MAX_GROUP;
  if (e.order_declines != (bool)(flags[0] & DEC_ERR_PAIR_ORDER)) return {false, e.order_declines ? "eligible tids go down, not declined" : "declined for order, but the tids do not go down"};
  if (big != (bool)(flags[0] & DEC_ERR_PAIRS)) return {false, big ? "a slot over PAIR_MAX_GROUP, not declined" : "declined for group size without a big group"};
  if (flags[0] & ~(DEC_ERR_PAIR_ORDER | DEC_ERR_PAIRS)) return {false, "unknown flag"};
  if (flags[0]) return {true, "declined"};
  for (uint32_t i = 0; i < n; ++i)
    if (mate[i] != e.mate[i]) return {false, "mate[" + to_string(i) + "] = " + to_string(mate[i]) + ", reference " + to_string(e.mate[i])};

  // kf_decide, the scan, kf_gather
  vector<uint16_t> flag(n);
  vector<uint8_t> mapq(n), nm_state(n), role(n, 9);
  vector<uint32_t> nm(n), l_seq(n), aligned(n), del(n), err(1, 0);
  for (uint32_t i = 0; i < n; ++i) {
    const Rec& r = s.recs[i];
    flag[i] = r.flag; mapq[i] = r.mapq; nm_state[i] = r.nm_state; nm[i] = r.nm; l_seq[i] = r.l_seq; aligned[i] = r.aligned; del[i] = r.del;
  }
  vector<unsigned long long> anchor(n + 1, 999), n_emit(1, 0);
  FilterArgs fa{};
  fa.data = s.data.data(); fa.rec_off = s.off.data(); fa.n = n; fa.flag = flag.data(); fa.mapq = mapq.data(); fa.nm_state = nm_state.data();
  fa.nm = nm.data(); fa.l_seq = l_seq.data(); fa.aligned = aligned.data(); fa.del = del.data(); fa.mate = mate.data(); fa.p = p;
  fa.filter_single = filter_single; fa.pair_path = 1; fa.filter_out = filter_out;
  fa.anchor_bytes = anchor.data(); fa.role = role.data(); fa.error_flags = err.data(); fa.n_emit = n_emit.data();
  for (uint32_t i = 0; i < (n + 255) / 256 * 256; ++i) at(i), kf_decide(fa);
  if (e.nm_panic != (bool)(err[0] & ERR_NM)) return {false, e.nm_panic ? "nm() panic missed" : "nm() panic the reference does not reach"};
  if (e.nm_panic) return {true, "nm"};
  for (uint32_t i = 0; i < n; ++i)
    if (role[i] != e.role[i]) return {false, "role[" + to_string(i) + "] = " + to_string(role[i]) + ", reference " + to_string(e.role[i])};
  if (n_emit[0] != e.emitted.size()) return {false, "n_emit"};
  unsigned long long run = 0;  // kf_scan
  for (uint32_t i = 0; i < n; ++i) {
    const unsigned long long x = anchor[i];
    anchor[i] = run;
    run += x;
  }
  anchor[n] = run;
  vector<uint8_t> want;
  for (uint32_t i : e.emitted) {
    const uint64_t o = s.off[i];
    want.insert(want.end(), s.data.begin() + (ptrdiff_t)o, s.data.begin() + (ptrdiff_t)(o + 4 + ldu32(s.data.data() + o)));
  }
  if (run != want.size()) return {false, "output size " + to_string(run) + ", reference " + to_string(want.size())};
  for (uint8_t fill : {0x00, 0xff}) {
    vector<uint8_t> out(run + 64, fill);
    fa.out = out.data();
    for (uint32_t i = 0; i < (n + 7) / 8 * 256; ++i) at(i), kf_gather(fa);
    if (!equal(want.begin(), want.end(), out.begin())) return {false, "output bytes"};
    for (size_t k = run; k < out.size(); ++k)
      if (out[k] != fill) return {false, "bytes written past the output"};
  }
  return {true, "ok"};
}

Rec rec(int32_t tid, uint16_t flag, const char* name, int32_t mtid) {
  Rec r{};
  r.tid = tid; r.mtid = mtid; r.flag = flag; r.name = name; r.mapq = 60; r.nm_state = 1; r.nm = 1; r.l_seq = 100; r.aligned = 100;
  return r;
}

}  // namespace

int main() {
  mt19937 rng(20261016);
  uint32_t tests = 0, fails = 0, declined = 0, nm = 0, order = 0;
  auto run = [&](const char* what, Stream& s, const cmb_params& p, bool fs, bool filter_out, bool collide) {
    const Outcome o = check(s, p, fs, filter_out, collide, rng);
    ++tests;
    if (o.why == "declined") ++declined;
    if (o.why == "declined" && walk(s.recs, p, fs, filter_out).order_declines) ++order;
    if (o.why == "nm") ++nm;
    if (!o.ok) {
      if (++fails <= 10) printf("FAIL %s (%zu records, filter_out %d, collide %d): %s\n", what, s.recs.size(), filter_out, collide, o.why.c_str());
    }
  };
  // the two streams of the pair path's known pitfalls
  cmb_params p1{};
  p1.filtering = 1;
  p1.min_mapq = 255;
  p1.min_aligned_length_pair = 1;
  {  // X on c0, Y on c1, X on c0: Y clears the set, the X records never meet
    Stream s;
    s.recs = {rec(0, 0x3, "X", 0), rec(1, 0x3, "Y", 1), rec(0, 0x3, "X", 0)};
    encode(s, rng);
    run("case 1", s, p1, false, true, false);
    const Expected e = walk(s.recs, p1, false, true);
    if (!e.order_declines || e.mate[0] != -1) ++fails, printf("FAIL case 1 reference\n");
  }
  {  // --inverse: an unmapped proper record is returned at once and never stored
    Stream s;
    s.recs = {rec(0, 0x1 | 0x2 | 0x4 | 0x40, "Z", 0), rec(0, 0x1 | 0x2 | 0x8 | 0x80, "Z", 0), rec(0, 0x1 | 0x2 | 0x80, "Z", 0)};
    p1.min_aligned_length_pair = 500;
    encode(s, rng);
    run("case 2", s, p1, false, false, false);
    const Expected e = walk(s.recs, p1, false, false);
    if (e.emitted != vector<uint32_t>{0, 1, 2}) ++fails, printf("FAIL case 2 reference\n");
  }
  for (uint32_t k = 0; k < 4000; ++k) {
    const bool collide = k % 4 == 3;
    Stream s = random_stream(rng, collide ? 40 : (k % 10 == 0 ? 400 : 80));
    bool fs = false;
    const cmb_params p = random_params(rng, fs);
    run("random", s, p, fs, true, collide);
    run("random", s, p, fs, false, collide);
  }
  {  // 25 eligible records of one (tid, name): more than one slot holds
    Stream s;
    for (int k = 0; k < 25; ++k) s.recs.push_back(rec(0, 0x3, "G", 0));
    encode(s, rng);
    const Outcome o = check(s, p1, false, true, false, rng);
    ++tests;
    if (!o.ok || o.why != "declined") ++fails, printf("FAIL 25 records of one name: %s\n", o.why.c_str());
  }
  printf("%u tests, %u fails (%u declined, %u of them for order; %u nm panics)\n", tests, fails, declined, order, nm);
  return fails ? 1 : 0;
}
