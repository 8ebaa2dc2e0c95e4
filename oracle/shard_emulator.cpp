// TEST INFRASTRUCTURE ONLY — never linked into libcoverm_b200.so or the `coverm` product binary.
//
// The CPU device emulator (device_emulator.cpp, included whole) plus the sharded-input entry points cmb_shard_begin /
// cmb_shard_add / cmb_shard_finish, so that the product's host code for `--sharded` (sample_processor.hpp process_sharded, the
// CLI) runs without a GPU: `oracle/coverm_shardcheck` (oracle/sharded.mk), tests/test_sharded.py.
#include "device_emulator.cpp"

// Sharded input (cmb_shard_*): the shards are inflated with zlib and walked record by record; the choice of every pair, the
// reference's errors (shard_bam_reader.rs:55-296) and the tie rule follow the library (cmb_shards.cuh), met in the reference's
// serial order; the winners are stably sorted by tid and accumulated like any batch.
struct EmuShardRec {
  int32_t tid, pos;
  uint16_t flag;
  uint8_t mapq, nm_state, info;  // info: NM type (0 absent, 1 C, 2 other) | 4 when n_cigar > 0
  uint32_t nm, l_seq, aligned, del, ins;
  char as_type;
  int64_t as_value;
  std::string qname;
  std::vector<int32_t> ivs, ivl;
};
struct EmuShards {
  std::vector<uint32_t> offsets;
  std::vector<uint8_t> excluded;
  std::vector<std::vector<EmuShardRec>> prim;  // the primaries of every shard added so far
  std::vector<uint64_t> unpaired_at;           // per shard: primary set at which its first unpaired record was read, or -1
  bool active = false;
};
static std::map<const cmb_ctx*, EmuShards> g_shards;

static uint64_t emu_mix(uint64_t x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

int cmb_shard_begin(cmb_ctx* c, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded) {
  if (!c || !tid_offsets || !n_shards) return fail(c, CMB_E_ARG, "cmb_shard_begin: null argument or no shards");
  if (!c->in_sample) return fail(c, CMB_E_ARG, "cmb_shard_begin: no sample in progress");
  EmuShards& s = g_shards[c];
  s = EmuShards{};
  s.offsets.assign(tid_offsets, tid_offsets + n_shards);
  const size_t n_ref = c->gene_mode ? c->contig_lens.size() : c->lens.size();
  if (excluded) s.excluded.assign(excluded, excluded + n_ref);
  s.active = true;
  return CMB_OK;
}

int cmb_shard_add(cmb_ctx* c, const cmb_bgzf_input* in, cmb_bgzf_result* out) {
  if (!c || !in || !out) return fail(c, CMB_E_ARG, "cmb_shard_add: null argument");
  EmuShards& s = g_shards[c];
  if (!s.active || s.prim.size() >= s.offsets.size()) return fail(c, CMB_E_ARG, "cmb_shard_add: call cmb_shard_begin first, once per shard");
  *out = cmb_bgzf_result{};
  const uint32_t k = (uint32_t)s.prim.size();
  std::vector<uint8_t> stream;
  for (uint32_t b = 0; b < in->n_blocks; ++b) {
    const size_t at = stream.size();
    stream.resize(at + in->block_isize[b]);
    if (!in->block_isize[b]) continue;
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, -15) != Z_OK) return fail(c, CMB_E_NOMEM, "zlib");
    zs.next_in = const_cast<Bytef*>(in->data + in->block_coffset[b]);
    zs.avail_in = in->block_clen[b];
    zs.next_out = stream.data() + at;
    zs.avail_out = in->block_isize[b];
    const int zr = inflate(&zs, Z_FINISH);
    inflateEnd(&zs);
    if (zr != Z_STREAM_END || zs.avail_out) return fail(c, CMB_E_DECLINED, "shard " + std::to_string(k) + ": a BGZF block does not inflate");
  }
  auto u32 = [&](size_t o) { uint32_t v; memcpy(&v, stream.data() + o, 4); return v; };
  auto u16 = [&](size_t o) { uint16_t v; memcpy(&v, stream.data() + o, 2); return (uint32_t)v; };
  std::vector<EmuShardRec> prim;
  uint64_t unpaired_at = ~0ull;
  for (size_t o = in->records_at; o < stream.size();) {
    if (o + 36 > stream.size()) return fail(c, CMB_E_DECLINED, "shard " + std::to_string(k) + ": record cut short");
    const size_t r = o + 4, end = r + u32(o);
    if (end > stream.size()) return fail(c, CMB_E_DECLINED, "shard " + std::to_string(k) + ": record cut short");
    out->n_records += 1;
    EmuShardRec x{};
    const uint32_t l_name = stream[r + 8], n_cig = u16(r + 12);
    x.tid = (int32_t)u32(r) + (int32_t)s.offsets[k];
    x.pos = (int32_t)u32(r + 4);
    x.mapq = stream[r + 9];
    x.flag = (uint16_t)u16(r + 14);
    x.l_seq = u32(r + 16);
    x.qname.assign((const char*)stream.data() + r + 32, l_name ? l_name - 1 : 0);
    if (!(x.flag & 1) && unpaired_at == ~0ull) unpaired_at = prim.size();
    o = end;
    if (x.flag & 0x900) continue;
    const size_t cg = r + 32 + l_name;
    size_t aux = cg + 4ull * n_cig + (x.l_seq + 1) / 2 + x.l_seq;
    int64_t cur = x.pos;
    for (uint32_t q = 0; q < n_cig; ++q) {
      const uint32_t v = u32(cg + 4 * q), op = v & 15, len = v >> 4;
      if (op == 0 || op == 7 || op == 8) {
        x.ivs.push_back(cur < 0 ? -1 : (int32_t)std::min<int64_t>(cur, INT32_MAX));
        x.ivl.push_back((int32_t)len);
        cur += len;
        x.aligned += len;
      } else if (op == 2) { cur += len; x.del += len; x.aligned += len; }
      else if (op == 3) cur += len;
      else if (op == 1) { x.ins += len; x.aligned += len; }
    }
    uint32_t nm_type = 0;
    while (aux + 3 <= end) {
      const uint8_t t0 = stream[aux], t1 = stream[aux + 1], ty = stream[aux + 2];
      aux += 3;
      size_t sz;
      if (ty == 'A' || ty == 'c' || ty == 'C') sz = 1;
      else if (ty == 's' || ty == 'S') sz = 2;
      else if (ty == 'i' || ty == 'I' || ty == 'f') sz = 4;
      else if (ty == 'Z' || ty == 'H') { size_t e = aux; while (e < end && stream[e]) ++e; sz = e - aux + 1; }
      else if (ty == 'B') { const uint8_t sub = stream[aux]; sz = 5 + (size_t)u32(aux + 1) * ((sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4); }
      else return fail(c, CMB_E_DECLINED, "shard " + std::to_string(k) + ": unknown aux type");
      if (t0 == 'N' && t1 == 'M' && !nm_type) {
        nm_type = ty == 'C' ? 1 : 2;
        x.nm_state = (ty == 'C' || ty == 'S' || ty == 'I') ? 1 : 2;
        x.nm = ty == 'C' ? stream[aux] : ty == 'S' ? u16(aux) : ty == 'I' ? u32(aux) : 0;
      }
      if (t0 == 'A' && t1 == 'S' && !x.as_type) {
        x.as_type = (char)ty;
        x.as_value = ty == 'C' ? stream[aux] : ty == 'S' ? u16(aux) : 0;
      }
      aux += sz;
    }
    x.info = (uint8_t)(nm_type | (n_cig ? 4 : 0));
    prim.push_back(std::move(x));
  }
  out->n_primary = prim.size();
  s.prim.push_back(std::move(prim));
  s.unpaired_at.push_back(unpaired_at);
  return CMB_OK;
}

int cmb_shard_finish(cmb_ctx* c, cmb_shard_result* out) {
  if (!c || !out) return fail(c, CMB_E_ARG, "cmb_shard_finish: null argument");
  EmuShards& s = g_shards[c];
  if (!s.active || s.prim.size() != s.offsets.size()) return fail(c, CMB_E_ARG, "cmb_shard_finish: every shard must be added first");
  s.active = false;
  *out = cmb_shard_result{};
  const size_t K = s.prim.size();
  std::vector<std::pair<uint32_t, const EmuShardRec*>> winners;
  for (uint64_t set = 0;; set += 2) {  // the reference's loop, two primary sets at a time
    for (uint64_t q = set; q < set + 2; ++q) {
      bool some_unfinished = false, some_finished = false;
      for (size_t k = 0; k < K; ++k) {
        if (s.unpaired_at[k] == q) return fail(c, CMB_E_SHARD_EXIT, "This code can only handle paired-end input (at the moment), sorry. Found an unpaired record before primary " + std::to_string(q));
        if (q >= s.prim[k].size()) { some_finished = true; continue; }
        some_unfinished = true;
        if (k && q < s.prim[0].size() && s.prim[k][q].qname != s.prim[0][q].qname)
          return fail(c, CMB_E_SHARD_EXIT, "BAM files do not appear to be properly sorted by read name. The read names of primary alignment " + std::to_string(q) + " differ between the shards");
      }
      if (some_unfinished && some_finished) return fail(c, CMB_E_SHARD_EXIT, "Unexpectedly one BAM file input finished while another had further reads");
      if (!some_unfinished) {
        if (q == set + 1) return fail(c, CMB_E_SHARD_PANIC, "Unexpectedly was able to read a first read set, but not a second. Hmm.");
        goto done;
      }
    }
    {
      const uint64_t pair = set / 2;
      bool have = false;
      int64_t best = 0;
      uint32_t winner = 0, ties = 0;
      for (uint32_t k = 0; k < K; ++k) {
        const EmuShardRec& m1 = s.prim[k][set];
        const EmuShardRec& m2 = s.prim[k][set + 1];
        const int32_t local = m1.tid - (int32_t)s.offsets[k];
        const uint8_t ex = (local >= 0 && !s.excluded.empty()) ? s.excluded[(size_t)m1.tid] : 0;
        if (ex == 2) return fail(c, CMB_E_SHARD_PANIC, "Contig name does not contain split symbol, so cannot determine which genome it belongs to");
        if (ex) continue;
        int64_t score = 0;
        for (const EmuShardRec* m : {&m1, &m2}) {
          if (m->flag & 4) continue;
          if (m->as_type == 'C' || m->as_type == 'S') score += m->as_value;
          else if (m->as_type) return fail(c, CMB_E_SHARD_PANIC, std::string("Unexpected data type of AS aux tag, found ") + m->as_type);
          else return fail(c, CMB_E_SHARD_PANIC, "Mapping record encountered that does not have an 'AS' auxiliary tag in the SAM/BAM format. This is required for ranking pairs of alignments.");
        }
        if (!have || score > best) { have = true; best = score; winner = k; ties = 1; }
        else if (score == best) {
          ties += 1;
          const uint64_t r = emu_mix(emu_mix(pair) ^ ((uint64_t)k << 32 | ties));
          if ((uint32_t)(((r >> 32) * (uint64_t)ties) >> 32) == 0) winner = k;
        }
      }
      if (!have) return fail(c, CMB_E_SHARD_EXIT, "CoverM cannot currently deal with reads that only map to excluded genomes");
      for (uint64_t m = set; m < set + 2; ++m) {
        const EmuShardRec& w = s.prim[winner][m];
        if ((w.info & 3) == 2) return fail(c, CMB_E_NM, "Unexpected data type of NM aux tag");
        if ((w.info & 3) == 0 && w.tid - (int32_t)s.offsets[winner] >= 0 && (w.info & 4))
          return fail(c, CMB_E_NM, "record with name at primary alignment " + std::to_string(set + 1) + " had no NM tag");
        out->n_records += 1;
        if (!(w.flag & 4) && w.tid >= 0) winners.push_back({(uint32_t)w.tid, &w});
      }
      out->n_pairs += 1;
    }
  }
done:
  std::stable_sort(winners.begin(), winners.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  std::vector<int32_t> tid, pos, ivs, ivl;
  std::vector<uint16_t> flag;
  std::vector<uint8_t> mapq, nm_state;
  std::vector<uint32_t> nm, l_seq, aligned, del, ins, iv_begin;
  for (const auto& w : winners) {
    const EmuShardRec& x = *w.second;
    tid.push_back(x.tid); pos.push_back(x.pos); flag.push_back(x.flag); mapq.push_back(x.mapq); nm_state.push_back(x.nm_state);
    nm.push_back(x.nm); l_seq.push_back(x.l_seq); aligned.push_back(x.aligned); del.push_back(x.del); ins.push_back(x.ins);
    iv_begin.push_back((uint32_t)ivs.size());
    ivs.insert(ivs.end(), x.ivs.begin(), x.ivs.end());
    ivl.insert(ivl.end(), x.ivl.begin(), x.ivl.end());
  }
  iv_begin.push_back((uint32_t)ivs.size());
  out->n_emitted = tid.size();
  out->n_intervals = ivs.size();
  if (tid.empty()) return CMB_OK;
  if (ivs.empty()) { ivs.push_back(0); ivl.push_back(0); }
  cmb_read_batch b{};
  b.tid = tid.data(); b.pos = pos.data(); b.flag = flag.data(); b.mapq = mapq.data(); b.nm_state = nm_state.data(); b.nm = nm.data();
  b.l_seq = l_seq.data(); b.aligned = aligned.data(); b.del = del.data(); b.ins = ins.data(); b.iv_begin = iv_begin.data();
  b.iv_start = ivs.data(); b.iv_len = ivl.data();
  return submit(c, b, (uint32_t)tid.size(), (uint32_t)out->n_intervals);
}

