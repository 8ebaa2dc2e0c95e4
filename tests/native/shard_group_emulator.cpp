// TEST INFRASTRUCTURE ONLY — never linked into libcoverm_b200.so or the `coverm` product binary.
//
// The CPU device emulator with the sharded-input entry points (oracle/shard_emulator.cpp, included whole) plus those of sharded
// input over a group of ranks (cmb_shard_begin_range, cmb_shard_score, cmb_shard_export / cmb_shard_import, cmb_shard_choose,
// cmb_shard_finish_group) and cmb_set_genes_range, so that the host's group protocol for `--sharded` runs without a GPU
// (tests/test_sharded_group.py builds this file with coverm_b200/csrc/host/host_api.cpp into a shared library).
//
// Like the library, each rank scores the pairs of its own shards into a table of int32 columns, the ranks exchange the columns
// and shard 0's name hashes, and every rank walks the whole table with the tie rule of cmb_shards.cuh.  Errors are folded into
// the library's 64-bit keys (set index | phase | kind | detail), so that the smallest key over the ranks is the error the
// one-process run reports.
//
// cmb_set_genes_range here holds every gene: a group rank of a sharded sample submits only the winners of its own shards, which
// lie on its own contigs, so the rows, pairs, contig_seen and kept_primary of the other ranks' contigs stay empty.  (It is not a
// stand-in for ranged gene mode in general: tests/native/gene_range_emulator.cpp is.)
#include "../../oracle/shard_emulator.cpp"

namespace {
enum : uint32_t { K_UNPAIRED = 1, K_NAME = 2, K_AS_MISSING = 5, K_AS_TYPE = 6, K_EXCLUDED = 7, K_NM_TYPE = 8, K_NM_MISSING = 9, K_NO_SEPARATOR = 10 };
constexpr uint32_t P_SCORE = 0x100, P_CHOOSE = 0x200, P_CLONE = 0x300;
constexpr int32_t SCORE_NONE = -1, SCORE_ERR = -2;

uint64_t key_of(uint64_t set, uint32_t phase, uint32_t kind, uint32_t detail) {
  return (set << 24) | ((uint64_t)(phase & 0xfff) << 12) | ((kind & 0xf) << 8) | (detail & 0xff);
}

uint64_t name_hash(const std::string& s) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (unsigned char ch : s) h = (h ^ ch) * 0x100000001b3ull;
  return emu_mix(h ^ s.size());
}

struct EmuGroup {
  uint32_t first = 0, last = 0;
  std::vector<uint64_t> n_prim;
  uint64_t n_pairs = 0;
  std::vector<int32_t> score;    // [n_shards][n_pairs]
  std::vector<uint64_t> hash0;   // shard 0's name hashes
  std::vector<uint32_t> winner;  // per pair, UINT32_MAX: none
  uint64_t key = ~0ull;
  int stage = 0;
};
std::map<const cmb_ctx*, EmuGroup> g_group;
}  // namespace

extern "C" {

int cmb_set_genes_range(cmb_ctx* c, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes, uint32_t tid_begin,
                        uint32_t tid_end) {
  if (tid_begin > tid_end || tid_end > n_contigs) return fail(c, CMB_E_ARG, "cmb_set_genes_range: bad contig range");
  return cmb_set_genes(c, n_contigs, contig_len, n_genes, genes);
}

int cmb_shard_begin_range(cmb_ctx* c, uint32_t n_shards, const uint32_t* tid_offsets, const uint8_t* excluded, uint32_t shard_begin, uint32_t shard_end) {
  if (shard_begin > shard_end || shard_end > n_shards) return fail(c, CMB_E_ARG, "cmb_shard_begin_range: bad shard range");
  if (int rc = cmb_shard_begin(c, n_shards, tid_offsets, excluded)) return rc;
  EmuShards& s = g_shards[c];
  s.prim.resize(shard_begin);  // cmb_shard_add numbers the next shard by the stores so far
  s.unpaired_at.assign(shard_begin, ~0ull);
  EmuGroup& g = g_group[c];
  g = EmuGroup{};
  g.first = shard_begin;
  g.last = shard_end;
  return CMB_OK;
}

int cmb_shard_score(cmb_ctx* c, const uint64_t* n_primary) {
  EmuShards& s = g_shards[c];
  EmuGroup& g = g_group[c];
  if (!s.active || s.prim.size() != g.last || g.stage != 0) return fail(c, CMB_E_ARG, "cmb_shard_score: add this context's shards first");
  const uint32_t K = (uint32_t)s.offsets.size();
  for (uint32_t k = g.first; k < g.last; ++k)
    if (n_primary[k] != s.prim[k].size()) return fail(c, CMB_E_ARG, "cmb_shard_score: wrong primary count");
  g.n_prim.assign(n_primary, n_primary + K);
  const uint64_t n0 = g.n_prim[0];
  uint64_t n_min = n0;
  bool equal = true;
  for (uint64_t n : g.n_prim) {
    n_min = std::min(n_min, n);
    equal = equal && n == n0;
  }
  g.n_pairs = n_min / 2;
  if (!equal) g.key = (n_min << 24) | (0xfffull << 12) | (3ull << 8);  // the reader's own checks (cmb_shard_finish)
  else if (n0 % 2) g.key = (n0 << 24) | (0xfffull << 12) | (4ull << 8);
  g.score.assign((size_t)K * g.n_pairs, SCORE_NONE);
  g.hash0.assign(n0, 0);
  for (uint32_t k = g.first; k < g.last; ++k) {
    const auto& P = s.prim[k];
    if (s.unpaired_at[k] != ~0ull) g.key = std::min(g.key, key_of(s.unpaired_at[k], k, K_UNPAIRED, 0));
    if (k == 0)
      for (uint64_t j = 0; j < n0; ++j) g.hash0[j] = name_hash(P[j].qname);
    for (uint64_t j = 0; j < std::min<uint64_t>(P.size(), n0) / 2; ++j) {
      const EmuShardRec& m1 = P[2 * j];
      const int32_t local = m1.tid - (int32_t)s.offsets[k];
      const uint8_t ex = (local >= 0 && !s.excluded.empty()) ? s.excluded[(size_t)m1.tid] : 0;
      int32_t v = 0;
      if (ex == 2) {
        g.key = std::min(g.key, key_of(2 * j + 1, P_SCORE + k, K_NO_SEPARATOR, 0));
        v = SCORE_ERR;
      } else if (ex) {
        v = SCORE_NONE;
      } else {
        for (const EmuShardRec* m : {&m1, &P[2 * j + 1]}) {
          if (m->flag & 4) continue;
          if (m->as_type == 'C' || m->as_type == 'S') {
            v += (int32_t)m->as_value;
            continue;
          }
          g.key = std::min(g.key, key_of(2 * j + 1, P_SCORE + k, m->as_type ? K_AS_TYPE : K_AS_MISSING, (uint8_t)m->as_type));
          v = SCORE_ERR;
          break;
        }
      }
      if (j < g.n_pairs) g.score[(size_t)k * g.n_pairs + j] = v;
    }
  }
  g.stage = 1;
  return CMB_OK;
}

int cmb_shard_export(cmb_ctx* c, uint32_t shard, int32_t* scores, uint64_t* names) {
  EmuGroup& g = g_group[c];
  if (g.stage != 1 || shard >= g.n_prim.size() || !scores) return fail(c, CMB_E_ARG, "cmb_shard_export: no scored shard");
  std::copy_n(g.score.begin() + (ptrdiff_t)((size_t)shard * g.n_pairs), g.n_pairs, scores);
  if (shard == 0 && names) std::copy(g.hash0.begin(), g.hash0.end(), names);
  return CMB_OK;
}

int cmb_shard_import(cmb_ctx* c, uint32_t shard, const int32_t* scores, const uint64_t* names) {
  EmuGroup& g = g_group[c];
  if (g.stage != 1 || shard >= g.n_prim.size() || !scores) return fail(c, CMB_E_ARG, "cmb_shard_import: no scored shard");
  std::copy_n(scores, g.n_pairs, g.score.begin() + (ptrdiff_t)((size_t)shard * g.n_pairs));
  if (shard == 0 && names) std::copy_n(names, g.hash0.size(), g.hash0.begin());
  return CMB_OK;
}

int cmb_shard_choose(cmb_ctx* c, uint64_t* err_key) {
  EmuShards& s = g_shards[c];
  EmuGroup& g = g_group[c];
  if (g.stage != 1 || !err_key) return fail(c, CMB_E_ARG, "cmb_shard_choose: call cmb_shard_score first");
  const uint32_t K = (uint32_t)s.offsets.size();
  const uint64_t n0 = g.n_prim[0];
  for (uint32_t k = std::max<uint32_t>(1, g.first); k < g.last; ++k)
    for (uint64_t j = 0; j < std::min<uint64_t>(s.prim[k].size(), n0); ++j)
      if (name_hash(s.prim[k][j].qname) != g.hash0[j]) g.key = std::min(g.key, key_of(j, k, K_NAME, 0));
  g.winner.assign(g.n_pairs, UINT32_MAX);
  for (uint64_t j = 0; j < g.n_pairs; ++j) {
    int64_t best = 0;
    uint32_t w = UINT32_MAX, ties = 0;
    for (uint32_t k = 0; k < K; ++k) {
      const int32_t v = g.score[(size_t)k * g.n_pairs + j];
      if (v < 0) continue;
      if (w == UINT32_MAX || v > best) { best = v; w = k; ties = 1; }
      else if (v == best) {
        ties += 1;
        const uint64_t r = emu_mix(emu_mix(j) ^ ((uint64_t)k << 32 | ties));
        if ((uint32_t)(((r >> 32) * (uint64_t)ties) >> 32) == 0) w = k;
      }
    }
    g.winner[j] = w;
    if (w == UINT32_MAX) {
      g.key = std::min(g.key, key_of(2 * j + 1, P_CHOOSE, K_EXCLUDED, 0));
      continue;
    }
    if (w < g.first || w >= g.last) continue;
    for (uint64_t m = 2 * j; m < 2 * j + 2; ++m) {  // clone_record_into's NM checks, on the winner's owner
      const EmuShardRec& x = s.prim[w][m];
      if ((x.info & 3) == 2) g.key = std::min(g.key, key_of(2 * j + 1, P_CLONE + (uint32_t)(m & 1), K_NM_TYPE, 0));
      else if ((x.info & 3) == 0 && x.tid - (int32_t)s.offsets[w] >= 0 && (x.info & 4))
        g.key = std::min(g.key, key_of(2 * j + 1, P_CLONE + (uint32_t)(m & 1), K_NM_MISSING, 0));
    }
  }
  *err_key = g.key;
  g.stage = 2;
  return CMB_OK;
}

int cmb_shard_finish_group(cmb_ctx* c, uint64_t key, cmb_shard_result* out) {
  EmuShards& s = g_shards[c];
  EmuGroup& g = g_group[c];
  if (g.stage != 2 || !out) return fail(c, CMB_E_ARG, "cmb_shard_finish_group: call cmb_shard_choose first");
  s.active = false;
  g.stage = 0;
  *out = cmb_shard_result{};
  if (key != ~0ull) {
    const uint32_t kind = (uint32_t)(key >> 8) & 0xf, detail = (uint32_t)key & 0xff;
    const std::string set = std::to_string(key >> 24);
    switch (kind) {
      case 3: return fail(c, CMB_E_SHARD_EXIT, "Unexpectedly one BAM file input finished while another had further reads");
      case 4: return fail(c, CMB_E_SHARD_PANIC, "Unexpectedly was able to read a first read set, but not a second. Hmm.");
      case K_UNPAIRED: return fail(c, CMB_E_SHARD_EXIT, "This code can only handle paired-end input (at the moment), sorry. Found an unpaired record before primary " + set);
      case K_NAME: return fail(c, CMB_E_SHARD_EXIT, "BAM files do not appear to be properly sorted by read name. The read names of primary alignment " + set + " differ between the shards");
      case K_AS_MISSING: return fail(c, CMB_E_SHARD_PANIC, "Mapping record encountered that does not have an 'AS' auxiliary tag in the SAM/BAM format. This is required for ranking pairs of alignments.");
      case K_AS_TYPE: return fail(c, CMB_E_SHARD_PANIC, std::string("Unexpected data type of AS aux tag, found ") + (char)detail);
      case K_NO_SEPARATOR: return fail(c, CMB_E_SHARD_PANIC, "Contig name does not contain split symbol, so cannot determine which genome it belongs to");
      case K_EXCLUDED: return fail(c, CMB_E_SHARD_EXIT, "CoverM cannot currently deal with reads that only map to excluded genomes");
      case K_NM_TYPE: return fail(c, CMB_E_NM, "Unexpected data type of NM aux tag");
      case K_NM_MISSING: return fail(c, CMB_E_NM, "record with name at primary alignment " + set + " had no NM tag");
    }
    return fail(c, CMB_E_ARG, "cmb_shard_finish_group: unknown error key");
  }
  std::vector<std::pair<uint32_t, const EmuShardRec*>> winners;
  for (uint64_t j = 0; j < g.n_pairs; ++j) {
    const uint32_t w = g.winner[j];
    if (w < g.first || w >= g.last) continue;
    for (uint64_t m = 2 * j; m < 2 * j + 2; ++m) {
      const EmuShardRec& x = s.prim[w][m];
      if (!(x.flag & 4) && x.tid >= 0) winners.push_back({(uint32_t)x.tid, &x});
    }
  }
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
  out->n_pairs = g.n_pairs;
  out->n_records = 2 * g.n_pairs;
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

}  // extern "C"
