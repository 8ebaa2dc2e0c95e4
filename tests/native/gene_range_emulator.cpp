// TEST INFRASTRUCTURE ONLY — never linked into libcoverm_b200.so or the `coverm` product binary.
//
// The CPU emulator of the device ABI (oracle/device_emulator.cpp) with cmb_set_genes_range on top, so that the host's group
// protocol for per-gene coverage (--gff over several ranks) and the shard semantics of the ABI run without a GPU
// (tests/test_gene_shards.py builds this file with coverm_b200/csrc/host/host_api.cpp into a shared library).
//
// The emulator counts every kept record in gene mode.  A range context therefore hands it every gene of the header plus one
// whole-contig gene in front of each contig's genes, and after the sample keeps what a rank owns, as the CUDA library does:
//   * rows: the genes of the contigs [tid_begin, tid_end), at their global numbers, every other row zero (a gene's row only
//     ever receives its own contig's records, so the owned rows are already the shard's);
//   * histogram pairs: only those rows', offsets local to the shard;
//   * contig_seen: the owned contigs only;
//   * kept_primary: the primaries of the owned contigs' whole-contig genes (every kept record starts inside its contig).
// One difference remains: the emulator raises CMB_E_BOUNDS for blocks of other ranks' records too, the library only for its own.
#define cmb_set_reference emu_set_reference
#define cmb_set_genes emu_set_genes
#define cmb_end_sample_device emu_end_sample_device
#define cmb_end_sample emu_end_sample
#include "../../oracle/device_emulator.cpp"
#undef cmb_set_reference
#undef cmb_set_genes
#undef cmb_end_sample_device
#undef cmb_end_sample

namespace {
struct GeneRange {
  uint32_t tid_begin = 0, tid_end = 0, g_begin = 0, g_end = 0, n_seg = 1;
  std::vector<uint32_t> inner;  // emulator row of each global gene in [g_begin, g_end) (UINT32_MAX: the placeholder)
  std::vector<uint32_t> whole;  // emulator row of each owned contig's whole-contig gene
};
std::map<const cmb_ctx*, GeneRange> g_ranges;  // contexts set up by cmb_set_genes_range
}  // namespace

extern "C" {

int cmb_set_reference(cmb_ctx* c, uint32_t n, const uint64_t* len, uint32_t b, uint32_t e) {
  g_ranges.erase(c);
  return emu_set_reference(c, n, len, b, e);
}

int cmb_set_genes(cmb_ctx* c, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes) {
  g_ranges.erase(c);
  return emu_set_genes(c, n_contigs, contig_len, n_genes, genes);
}

int cmb_set_genes_range(cmb_ctx* c, uint32_t n_contigs, const uint64_t* contig_len, uint32_t n_genes, const cmb_gene* genes,
                        uint32_t tid_begin, uint32_t tid_end) {
  if (tid_begin > tid_end || tid_end > n_contigs) return fail(c, CMB_E_ARG, "cmb_set_genes_range: bad contig range");
  std::vector<uint32_t> first((size_t)n_contigs + 1, 0);
  for (uint32_t g = 0; g < n_genes; ++g) first[genes[g].tid + 1] += 1;
  for (uint32_t t = 0; t < n_contigs; ++t) first[t + 1] += first[t];
  GeneRange r;
  r.tid_begin = tid_begin;
  r.tid_end = tid_end;
  r.n_seg = std::max<uint32_t>(1, n_genes);
  auto seg_cut = [&](uint32_t t) { return t == n_contigs ? r.n_seg : first[t]; };  // the library's rule
  r.g_begin = tid_begin == 0 ? 0 : seg_cut(tid_begin);
  r.g_end = seg_cut(tid_end);
  r.inner.assign(r.g_end - r.g_begin, UINT32_MAX);
  std::vector<cmb_gene> in;
  uint32_t g = 0;
  for (uint32_t t = 0; t < n_contigs; ++t) {
    if (t >= tid_begin && t < tid_end) r.whole.push_back((uint32_t)in.size());
    in.push_back(cmb_gene{t, 0, (uint32_t)contig_len[t]});
    for (; g < n_genes && genes[g].tid == t; ++g) {
      if (g >= r.g_begin && g < r.g_end) r.inner[g - r.g_begin] = (uint32_t)in.size();
      in.push_back(genes[g]);
    }
  }
  const int rc = emu_set_genes(c, n_contigs, contig_len, (uint32_t)in.size(), in.data());
  if (rc) return rc;
  g_ranges[c] = std::move(r);
  return CMB_OK;
}

int cmb_end_sample_device(cmb_ctx* c, const cmb_contig_stats** out) {
  const int rc = emu_end_sample_device(c, nullptr);
  auto it = g_ranges.find(c);
  if (it != g_ranges.end()) {
    const GeneRange& r = it->second;
    const bool csr = c->p.want & CMB_WANT_HIST_CSR;
    std::vector<cmb_contig_stats> rows(r.n_seg);
    std::vector<cmb_hist_pair> pairs;
    for (uint32_t i = 0; i < r.inner.size(); ++i) {
      if (r.inner[i] == UINT32_MAX) continue;
      cmb_contig_stats row = c->rows[r.inner[i]];
      if (csr && row.hist_count) {
        pairs.insert(pairs.end(), c->pairs.begin() + (ptrdiff_t)row.hist_offset, c->pairs.begin() + (ptrdiff_t)(row.hist_offset + row.hist_count));
        row.hist_offset = pairs.size() - row.hist_count;
      }
      rows[r.g_begin + i] = row;
    }
    uint64_t kept = 0;
    for (uint32_t w : r.whole) kept += c->rows[w].n_primary;
    for (size_t t = 0; t < c->contig_seen.size(); ++t)
      if (t < r.tid_begin || t >= r.tid_end) c->contig_seen[t] = 0;
    c->rows.swap(rows);
    c->pairs.swap(pairs);
    c->kept_primary = kept;
  }
  if (rc) return rc;
  if (out) *out = c->rows.data();
  return CMB_OK;
}

int cmb_end_sample(cmb_ctx* c, cmb_contig_stats* stats, cmb_hist_pair* pairs, uint64_t cap, uint64_t* n_pairs) {
  const int rc = cmb_end_sample_device(c, nullptr);
  if (rc) return rc;
  if (stats) memcpy(stats, c->rows.data(), sizeof(cmb_contig_stats) * c->rows.size());
  if (pairs && cap >= c->pairs.size()) memcpy(pairs, c->pairs.data(), sizeof(cmb_hist_pair) * c->pairs.size());
  if (n_pairs) *n_pairs = c->pairs.size();
  return CMB_OK;
}

}  // extern "C"
