// C ABI of the host drivers (include/coverm_b200_host.h).
#include <memory>

#include "../../../include/coverm_b200_host.h"
#include "cli.hpp"

using namespace cmbh;

struct cmbh_session {
  std::unique_ptr<DeviceSession> dev;
};

namespace {
std::string g_err;
// An ostream buffer that grows a malloc'd array and hands it over (the table text reaches the caller without a copy).
class MallocBuf : public std::streambuf, public BulkSink {
 public:
  char* append_uninitialized(size_t n) override {
    reserve(n_ + n + 1);
    char* at = p_ + n_;
    n_ += n;
    return at;
  }
  ~MallocBuf() override { free(p_); }
  char* release(size_t* len) {
    if (!p_) reserve(1);
    p_[n_] = 0;
    *len = n_;
    char* r = p_;
    p_ = nullptr;
    n_ = cap_ = 0;
    return r;
  }

 protected:
  std::streamsize xsputn(const char* s, std::streamsize n) override {
    reserve(n_ + (size_t)n + 1);
    memcpy(p_ + n_, s, (size_t)n);
    n_ += (size_t)n;
    return n;
  }
  int_type overflow(int_type ch) override {
    if (ch != traits_type::eof()) {
      reserve(n_ + 2);
      p_[n_++] = (char)ch;
    }
    return ch;
  }

 private:
  void reserve(size_t need) {
    if (need <= cap_) return;
    size_t ncap = cap_ ? cap_ : (1u << 16);
    while (ncap < need) ncap *= 2;
    char* np = (char*)realloc(p_, ncap);
    if (!np) throw std::bad_alloc();
    p_ = np;
    cap_ = ncap;
  }
  char* p_ = nullptr;
  size_t n_ = 0, cap_ = 0;
};
char* dup_text(const std::string& s) {
  char* p = (char*)malloc(s.size() + 1);
  if (p) {
    memcpy(p, s.data(), s.size());
    p[s.size()] = 0;
  }
  return p;
}
}  // namespace

extern "C" {

const char* cmbh_last_error(void) { return g_err.c_str(); }

int cmbh_session_create(int device, int threads, cmbh_session** out) {
  if (!out) return -2;
  *out = nullptr;
  try {
    auto s = std::make_unique<cmbh_session>();
    s->dev = std::make_unique<DeviceSession>(device, threads);
    *out = s.release();
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

void cmbh_session_destroy(cmbh_session* s) { delete s; }

int cmbh_session_set_shard(cmbh_session* s, uint32_t tid_begin, uint32_t tid_end) {
  if (!s) return -2;
  s->dev->set_shard(tid_begin, tid_end);
  return 0;
}

int cmbh_session_set_group(cmbh_session* s, int rank, int n_ranks, const uint8_t* nccl_id, cmbh_allgather_fn allgather, void* user) {
  if (!s) return -2;
  try {
    s->dev->set_group(rank, n_ranks, nccl_id, allgather, user);
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

int cmbh_session_set_group_output(cmbh_session* s, int every_rank_prints) {
  if (!s) return -2;
  s->dev->set_every_rank_prints(every_rank_prints != 0);
  return 0;
}

void* cmbh_session_ctx(cmbh_session* s) { return s ? (void*)s->dev->ctx() : nullptr; }

int cmbh_run(cmbh_session* s, int argc, const char* const* argv, const cmbh_mem_input* mem, int n_mem, cmbh_result* res) {
  if (!res || (argc > 0 && !argv)) return -2;
  memset(res, 0, sizeof *res);
  std::vector<std::string> args(argv, argv + argc);
  std::vector<InputSpec> inputs;
  for (int i = 0; i < n_mem; ++i) {
    InputSpec in;
    in.path = mem[i].path;
    in.data = mem[i].data;
    in.size = mem[i].size;
    inputs.push_back(in);
  }
  MallocBuf out_buf;
  std::ostream out(&out_buf);
  std::ostringstream err;
  const CliResult r = run_cli(args, inputs, out, err, s ? s->dev.get() : nullptr);
  out.flush();
  res->status = r.status;
  const std::string se = err.str();
  res->out = out_buf.release(&res->out_len);
  res->err = dup_text(se);
  res->err_len = se.size();
  res->n_samples = (uint32_t)std::min<size_t>(CMBH_MAX_SAMPLES, r.timings.size());
  for (uint32_t i = 0; i < res->n_samples; ++i) {
    cmbh_sample_info& si = res->samples[i];
    if (i < r.reads_mapped.size()) {
      si.num_mapped_reads = r.reads_mapped[i].num_mapped_reads;
      si.num_reads = r.reads_mapped[i].num_reads;
    }
    si.n_records = r.record_counts[i];
    const SampleTiming& t = r.timings[i];
    si.total_s = t.total_s;
    si.decode_s = t.decode_s;
    si.submit_wait_s = t.submit_wait_s;
    si.end_sample_s = t.end_sample_s;
    si.k0_ms = t.device.ms_zero;
    si.k1_ms = t.device.ms_accumulate;
    si.k2_ms = t.device.ms_scan;
    si.k3_ms = t.device.ms_finalize;
    si.device_total_ms = t.device.ms_total;
    si.k1_launches = t.device.k1_launches;
    si.k2_launches = t.device.k2_launches;
    si.k3_launches = t.device.k3_launches;
    si.arena_elems = t.device.arena_elems;
    si.n_intervals = t.device.n_intervals;
    si.h2d_bytes = t.h2d_bytes;
    si.device_decode = t.device_decode ? 1u : 0u;
    si.decode_host_blocks = t.bgzf.n_blocks_host;
    si.decode_copy_inflate_ms = t.bgzf.ms_copy_inflate;
    si.decode_chain_ms = t.bgzf.ms_chain;
    si.decode_extract_ms = t.bgzf.ms_extract;
    si.decode_launches = t.decode_launches;
    si.group_ranks = t.group_ranks;
    si.shard_blocks = t.shard_blocks;
    si.total_blocks = t.total_blocks;
    si.range_probes = t.range_probes;
    si.tid_begin = t.tid_begin;
    si.tid_end = t.tid_end;
    si.decode_second_pass_blocks = t.bgzf.n_blocks_second_pass;
    si.gather_s = t.gather_s;
    si.decode_copy_enqueue_wall_ms = t.bgzf.ms_copy_enqueue_wall;
    si.decode_host_wall_ms = t.bgzf.ms_host_wall;
  }
  return 0;
}

int cmbh_plan_params(int argc, const char* const* argv, void* params) {
  if (!params || (argc > 0 && !argv)) return -2;
  try {
    const CliOptions o = parse_cli(std::vector<std::string>(argv, argv + argc));
    const Plan plan = make_plan(o);
    memcpy(params, &plan.params, sizeof(cmb_params));
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

void cmbh_free_result(cmbh_result* res) {
  if (!res) return;
  free(res->out);
  free(res->err);
  res->out = res->err = nullptr;
}

int cmbh_main(int argc, char** argv) {
  std::ios::sync_with_stdio(false);
  std::vector<std::string> args(argv + (argc > 0 ? 1 : 0), argv + argc);
  const CliResult r = run_cli(args, {}, std::cout, std::cerr);
  std::cout.flush();
  return r.status;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Whole-file tuple extraction (no GPU involved): the SoA columns the device ABI consumes, for callers that want to
// stage tuples in HBM themselves (bench.py's device-resident timing, cmb_submit_device_batch).
extern "C" {

int cmbh_extract_tuples(const char* path, const uint8_t* data, size_t size, int threads, cmbh_tuples* out) {
  if (!path || !out) return -2;
  memset(out, 0, sizeof *out);
  try {
    InputSpec in;
    in.path = path;
    in.data = data;
    in.size = size;
    ThreadPool pool(threads);
    const BamInput input(in);
    InflateStream stream(input.data(), input.size(), pool, 256u << 20);
    std::vector<uint8_t> buf;
    const BamHeader h = read_bam_header(stream, buf, in.path);
    while (stream.fill(buf)) {
    }
    std::vector<size_t> rec_off;
    walk_records(buf.data(), h.records_at, buf.size(), true, [&](size_t o) {
      rec_off.push_back(o);
      return true;
    });
    const std::vector<uint64_t>& lens = h.header->lens;
    const uint32_t n_ref = (uint32_t)lens.size();
    const size_t nrec = rec_off.size();
    constexpr size_t ITEM = 8192;
    const size_t n_items = (nrec + ITEM - 1) / ITEM;
    struct Item { std::vector<int32_t> s, l; };
    std::vector<Item> items(n_items);
    auto alloc = [](size_t bytes) { return malloc(bytes ? bytes : 1); };
    out->n_contigs = n_ref;
    out->contig_len = (uint64_t*)alloc(8 * (size_t)n_ref);
    memcpy(out->contig_len, lens.data(), 8 * (size_t)n_ref);
    out->n_records = nrec;
    out->tid = (int32_t*)alloc(4 * nrec); out->pos = (int32_t*)alloc(4 * nrec); out->flag = (uint16_t*)alloc(2 * nrec);
    out->mapq = (uint8_t*)alloc(nrec); out->nm_state = (uint8_t*)alloc(nrec); out->nm = (uint32_t*)alloc(4 * nrec);
    out->l_seq = (uint32_t*)alloc(4 * nrec); out->aligned = (uint32_t*)alloc(4 * nrec); out->del = (uint32_t*)alloc(4 * nrec);
    out->ins = (uint32_t*)alloc(4 * nrec); out->iv_begin = (uint32_t*)alloc(4 * (nrec + 1));
    pool.parallel_for(n_items, [&](size_t it, int) {
      Tuple t;
      for (size_t r = it * ITEM; r < std::min(nrec, (it + 1) * ITEM); ++r) {
        const uint32_t before = (uint32_t)items[it].s.size();  // made global below, once every item's count is known
        decode_bam_record(buf.data() + rec_off[r], t, items[it].s, items[it].l);
        put_tuple(*out, r, before, t, nullptr, nullptr);
      }
    });
    std::vector<uint64_t> base(n_items + 1, 0);
    for (size_t it = 0; it < n_items; ++it) base[it + 1] = base[it] + items[it].s.size();
    const uint64_t n_iv = base[n_items];
    if (n_iv > 0xffffffffull) throw Panic("too many intervals for 32-bit offsets");
    out->n_intervals = n_iv;
    out->iv_start = (int32_t*)alloc(4 * n_iv);
    out->iv_len = (int32_t*)alloc(4 * n_iv);
    pool.parallel_for(n_items, [&](size_t it, int) {
      for (size_t r = it * ITEM; r < std::min(nrec, (it + 1) * ITEM); ++r) out->iv_begin[r] += (uint32_t)base[it];
      if (!items[it].s.empty()) {
        memcpy(out->iv_start + base[it], items[it].s.data(), 4 * items[it].s.size());
        memcpy(out->iv_len + base[it], items[it].l.data(), 4 * items[it].l.size());
      }
    });
    out->iv_begin[nrec] = (uint32_t)n_iv;
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    cmbh_free_tuples(out);
    return -1;
  }
}

void cmbh_free_tuples(cmbh_tuples* t) {
  if (!t) return;
  free(t->contig_len); free(t->tid); free(t->pos); free(t->flag); free(t->mapq); free(t->nm_state); free(t->nm);
  free(t->l_seq); free(t->aligned); free(t->del); free(t->ins); free(t->iv_begin); free(t->iv_start); free(t->iv_len);
  memset(t, 0, sizeof *t);
}

}  // extern "C"
