// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_bam.hpp header).
//
// `--sharded` input as the reference runs it: ReadSortedShardedBamReader + ShardedBamReaderGenerator
// (src/shard_bam_reader.rs:37-478) with the genome exclusion filters (src/genome_exclusion.rs), restated literally.  Like the
// reference, which writes the winners into `samtools sort` and reads the sorted stream back as an ordinary BAM, this program writes
// the winners -- cloned as clone_record_into does, tids shifted into the concatenated header -- as one uncompressed BAM, which
// oracle/coverm_oracle then reads like any sample.  Name it after the shards' stems joined with '|' to get the reference's sample
// name.  Two differences, both intended:
//   * ties between equally scored shards are broken by a deterministic uniform choice instead of thread_rng (:254): the t-th tied
//     candidate replaces the winner with probability 1/t, drawn from a hash of the pair index and the shard (the rule of the
//     device, cmb_shards.cuh sh_take_tie);
//   * where the reference runs `samtools sort`, the winners are stably sorted by (tid, pos), unplaced records last -- for the
//     coverage loop, which needs records grouped by tid in ascending order, the same stream.
//
//   shard_oracle --out OUT.bam [-s C | --genome-definition FILE | --single-genome] [--exclude-genomes-from-deshard FILE] SHARD...
#include <zlib.h>

#include <algorithm>
#include <fstream>
#include <iostream>

#include "oracle_core.hpp"

using namespace oracle;

namespace {

std::vector<uint8_t> slurp_inflated(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) throw Panic("Unable to open bam file " + path);
  std::vector<uint8_t> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  if (raw.size() < 2 || raw[0] != 0x1f || raw[1] != 0x8b) return raw;
  std::vector<uint8_t> out;
  size_t at = 0;
  std::vector<uint8_t> chunk(1 << 16);
  while (at < raw.size()) {  // one gzip member (BGZF block) after another
    z_stream zs{};
    if (inflateInit2(&zs, 15 + 16) != Z_OK) throw Panic("zlib");
    zs.next_in = raw.data() + at;
    zs.avail_in = (uInt)(raw.size() - at);
    int zr;
    do {
      zs.next_out = chunk.data();
      zs.avail_out = (uInt)chunk.size();
      zr = inflate(&zs, Z_NO_FLUSH);
      if (zr != Z_OK && zr != Z_STREAM_END) throw Panic("EFailure to read from a shard BAM file: " + path);
      out.insert(out.end(), chunk.data(), chunk.data() + (chunk.size() - zs.avail_out));
    } while (zr != Z_STREAM_END);
    at = raw.size() - zs.avail_in;
    inflateEnd(&zs);
  }
  return out;
}

uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
uint16_t rd16(const uint8_t* p) { uint16_t v; memcpy(&v, p, 2); return v; }

struct Rec {                // one alignment record: its bytes (block_size excluded) and what the reader looks at
  std::vector<uint8_t> b;
  int32_t tid, pos;
  uint16_t flag;
  std::string qname;
  uint32_t n_cigar;
  size_t aux_at;            // offset of the aux fields in b
  char as_type = 0, nm_type = 0;
  int64_t as_value = 0;
  uint8_t nm_c = 0;
  bool is_unmapped() const { return flag & 0x4; }
};

struct ShardFile {
  Header header;
  std::vector<uint8_t> data;
  size_t off = 0;
  explicit ShardFile(const std::string& path) : data(slurp_inflated(path)) {
    if (data.size() < 12 || memcmp(data.data(), "BAM\1", 4)) throw Panic("Unable to open bam file " + path);
    size_t o = 8 + rd32(data.data() + 4);
    const uint32_t n_ref = rd32(data.data() + o);
    o += 4;
    for (uint32_t i = 0; i < n_ref; ++i) {
      const uint32_t l = rd32(data.data() + o);
      header.names.emplace_back((const char*)data.data() + o + 4, l ? l - 1 : 0);
      header.lens.push_back(rd32(data.data() + o + 4 + l));
      o += 8 + l;
    }
    off = o;
  }
  bool read(Rec& r) {
    if (off + 4 > data.size()) return false;
    const uint32_t bs = rd32(data.data() + off);
    const uint8_t* p = data.data() + off + 4;
    if (bs < 32 || off + 4 + bs > data.size()) throw Panic("EFailure to read from a shard BAM file: truncated record");
    r = Rec{};
    r.b.assign(p, p + bs);
    r.tid = (int32_t)rd32(p);
    r.pos = (int32_t)rd32(p + 4);
    const uint32_t l_name = p[8], l_seq = rd32(p + 16);
    r.n_cigar = rd16(p + 12);
    r.flag = rd16(p + 14);
    r.qname.assign((const char*)p + 32, l_name ? l_name - 1 : 0);
    size_t o = 32 + l_name + 4ull * r.n_cigar + (l_seq + 1) / 2 + l_seq;
    r.aux_at = o;
    while (o + 3 <= bs) {  // record.aux(): the first tag of a name
      const char t0 = (char)p[o], t1 = (char)p[o + 1], ty = (char)p[o + 2];
      o += 3;
      size_t sz;
      if (ty == 'A' || ty == 'c' || ty == 'C') sz = 1;
      else if (ty == 's' || ty == 'S') sz = 2;
      else if (ty == 'i' || ty == 'I' || ty == 'f') sz = 4;
      else if (ty == 'Z' || ty == 'H') { size_t e = o; while (e < bs && p[e]) ++e; sz = e - o + 1; }
      else if (ty == 'B') { const char sub = (char)p[o]; sz = 5 + (size_t)rd32(p + o + 1) * ((sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4); }
      else throw Panic("EFailure to read from a shard BAM file: bad aux type");
      if (t0 == 'A' && t1 == 'S' && !r.as_type) {
        r.as_type = ty;
        r.as_value = ty == 'C' ? p[o] : ty == 'S' ? rd16(p + o) : 0;
      }
      if (t0 == 'N' && t1 == 'M' && !r.nm_type) {
        r.nm_type = ty;
        r.nm_c = p[o];
      }
      o += sz;
    }
    off += 4 + bs;
    return true;
  }
};

uint64_t shard_mix(uint64_t x) {  // splitmix64 finaliser
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
bool shard_take_tie(uint64_t pair, uint32_t shard, uint32_t t) {  // the t-th tied candidate wins with probability 1/t
  const uint64_t r = shard_mix(shard_mix(pair) ^ ((uint64_t)shard << 32 | t));
  return (uint32_t)(((r >> 32) * (uint64_t)t) >> 32) == 0;
}

int64_t aux_as(const Rec& r) {  // lib.rs:160-178
  if (r.as_type == 'C' || r.as_type == 'S') return r.as_value;
  if (r.as_type) throw Panic(std::string("Unexpected data type of AS aux tag, found ") + r.as_type);
  throw Panic("Mapping record encountered that does not have an 'AS' auxiliary tag in the SAM/BAM format. This is required for ranking pairs of alignments.");
}

// clone_record_into (:151-183): the record with only an NM tag of type C carried over, its tid shifted
Rec clone(const Rec& from, int32_t offset) {
  if (from.nm_type && from.nm_type != 'C') throw Panic("Unexpected data type of NM aux tag");
  if (!from.nm_type && from.tid >= 0 && from.n_cigar != 0) throw Panic("record with name " + from.qname + " had no NM tag");
  Rec to = from;
  to.b.resize(from.aux_at);
  if (from.nm_type == 'C') to.b.insert(to.b.end(), {'N', 'M', 'C', from.nm_c});
  to.tid = from.tid + offset;
  memcpy(to.b.data(), &to.tid, 4);
  return to;
}

using GenomeExclusion = std::function<bool(const std::string&)>;  // genome_exclusion.rs:16-18

int run(int argc, char** argv) {
  std::string out_path;
  std::optional<std::string> separator, definition, exclude;
  bool single_genome = false;
  std::vector<std::string> shards;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    auto val = [&]() -> std::string {
      if (i + 1 >= argc) throw ExitError(2, "error: missing value for " + a);
      return argv[++i];
    };
    if (a == "--out") out_path = val();
    else if (a == "-s" || a == "--separator") separator = val();
    else if (a == "--genome-definition") definition = val();
    else if (a == "--single-genome") single_genome = true;
    else if (a == "--exclude-genomes-from-deshard") exclude = val();
    else shards.push_back(a);
  }
  if (out_path.empty() || shards.empty()) throw ExitError(2, "error: --out and at least one shard are required");
  // the genome exclusion (coverm.rs:96-155): listed genomes, one per line, empty lines skipped; --single-genome excludes nothing
  GenomeExclusion excluded = [](const std::string&) { return false; };
  if (exclude) {
    std::ifstream f(*exclude, std::ios::binary);
    if (!f) throw Panic("Failed to open file '" + *exclude + "' containing list of excluded genomes");
    auto names = std::make_shared<std::set<std::string>>();
    std::string line;
    while (std::getline(f, line))
      if (!line.empty()) names->insert(line);
    if (!names->empty() && !single_genome) {
      if (separator) {  // SeparatorGenomeExclusionFilter (genome_exclusion.rs:45-64)
        const char split_char = (*separator)[0];
        excluded = [names, split_char](const std::string& contig) {
          const size_t offset = contig.find(split_char);
          if (offset == std::string::npos)
            throw Panic("Contig name " + std::to_string((unsigned)(uint8_t)split_char) + " does not contain split symbol, so cannot determine which genome it belongs to");
          return names->count(contig.substr(0, offset)) > 0;
        };
      } else if (definition) {  // GenomesAndContigsExclusionFilter (genome_exclusion.rs:25-43)
        auto gc = std::make_shared<GenomesAndContigs>(read_genome_definition_file(*definition));
        excluded = [names, gc](const std::string& contig) {
          auto it = gc->contig_to_genome.find(contig);
          return it != gc->contig_to_genome.end() && names->count(gc->genomes[it->second]) > 0;
        };
      }
    }
  }
  std::vector<std::unique_ptr<ShardFile>> readers;
  std::vector<int32_t> tid_offsets;
  Header hdr;
  for (const std::string& p : shards) {  // start (:315-336)
    readers.push_back(std::make_unique<ShardFile>(p));
    tid_offsets.push_back((int32_t)hdr.names.size());
    const Header& h = readers.back()->header;
    hdr.names.insert(hdr.names.end(), h.names.begin(), h.names.end());
    hdr.lens.insert(hdr.lens.end(), h.lens.begin(), h.lens.end());
  }
  // read_a_record_set (:55-129)
  auto read_a_record_set = [&](std::vector<Rec>& current) {
    current.clear();
    std::optional<std::string> current_qname;
    bool some_unfinished = false, some_finished = false;
    for (auto& reader : readers) {
      for (;;) {
        Rec record;
        if (!reader->read(record)) {
          some_finished = true;
          break;
        }
        if (!(record.flag & 0x1)) throw ExitError(1, "This code can only handle paired-end input (at the moment), sorry. Found record " + record.qname);
        if (!(record.flag & 0x900)) {
          some_unfinished = true;
          if (!current_qname) current_qname = record.qname;
          else if (*current_qname != record.qname)
            throw ExitError(1, "BAM files do not appear to be properly sorted by read name. Expected read name \"" + *current_qname +
                                   "\" from a previous reader but found \"" + record.qname + "\" in the current.");
          current.push_back(std::move(record));
          break;
        }
      }
    }
    if (some_unfinished && some_finished) throw ExitError(1, "Unexpectedly one BAM file input finished while another had further reads");
    return some_unfinished;
  };
  std::vector<Rec> previous, second, winners;
  for (uint64_t pair = 0; read_a_record_set(previous); ++pair) {  // read (:187-296)
    if (!read_a_record_set(second)) throw Panic("Unexpectedly was able to read a first read set, but not a second. Hmm.");
    std::optional<int64_t> max_score;
    uint32_t winner = 0, ties = 0;
    for (uint32_t i = 0; i < previous.size(); ++i) {
      const Rec& aln1 = previous[i];
      if (aln1.tid < 0 || !excluded(readers[i]->header.names.at((size_t)aln1.tid))) {
        int64_t score = 0;
        if (!aln1.is_unmapped()) score += aux_as(aln1);
        if (!second[i].is_unmapped()) score += aux_as(second[i]);
        if (max_score && score < *max_score) continue;
        if (max_score && score == *max_score) {
          ties += 1;
          if (shard_take_tie(pair, i, ties)) winner = i;
        } else {
          max_score = score;
          winner = i;
          ties = 1;
        }
      }
    }
    if (!max_score) throw ExitError(1, "CoverM cannot currently deal with reads that only map to excluded genomes");
    winners.push_back(clone(previous[winner], tid_offsets[winner]));
    winners.push_back(clone(second[winner], tid_offsets[winner]));
  }
  std::stable_sort(winners.begin(), winners.end(), [](const Rec& a, const Rec& b) {  // samtools sort
    return std::make_pair((uint32_t)a.tid, a.pos) < std::make_pair((uint32_t)b.tid, b.pos);
  });
  std::ofstream out(out_path, std::ios::binary);
  auto put32 = [&](uint32_t v) { out.write((const char*)&v, 4); };
  out.write("BAM\1", 4);
  put32(0);  // no header text
  put32((uint32_t)hdr.names.size());
  for (size_t t = 0; t < hdr.names.size(); ++t) {
    put32((uint32_t)hdr.names[t].size() + 1);
    out.write(hdr.names[t].c_str(), (std::streamsize)hdr.names[t].size() + 1);
    put32((uint32_t)hdr.lens[t]);
  }
  for (const Rec& r : winners) {
    put32((uint32_t)r.b.size());
    out.write((const char*)r.b.data(), (std::streamsize)r.b.size());
  }
  if (!out) throw Panic("Failed to write " + out_path);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  try {
    return run(argc, argv);
  } catch (const Panic& p) {
    std::cerr << "thread 'main' panicked: " << p.what() << "\n";
    return 101;
  } catch (const ExitError& e) {
    std::cerr << "[ERROR] " << e.what() << "\n";
    return e.code;
  }
}
