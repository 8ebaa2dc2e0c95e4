"""`--sharded` input (ReadSortedShardedBamReader, src/shard_bam_reader.rs): each read pair's best shard chosen, the winners
accumulated as one sample.

CPU: the oracle reproduces the reference's sharded goldens string for string, and the product's host code on the device
emulator matches the oracle on them and on seeded synthetic shard sets.  GPU (-m gpu): the `coverm` CLI against the oracle on
the goldens, on synthetic sets of 2-4 shards in every mode, on a large set spanning many decode windows, on every error the
reference raises, on the filter fall-back, and on the tie rule's determinism and balance."""
import os
import subprocess

import pytest

import shard_sets
from case_runner import DATA, ROOT
from sharded_oracle import run_oracle

HOSTCHECK_BIN = os.path.join(ROOT, "oracle", "coverm_shardcheck")  # the host code on the CPU emulator with cmb_shard_*
S1, S2 = os.path.join(DATA, "shard1.bam"), os.path.join(DATA, "shard2.bam")
DEFINITION = os.path.join(DATA, "shards_7seqs.definition")  # the FASTA headers of genomes_dir_7seqs/genome{1..6}.fasta

CONTIG_GOLDEN = """Contig	shard1|shard2 Mean
genome3~random_sequence_length_11001	0.110588886
genome4~random_sequence_length_11002	0.11057869
genome5~seq2	0
genome6~random_sequence_length_11003	0.11056851
genome1~random_sequence_length_11000	0.109861754
genome1~random_sequence_length_11010	0.110497236
genome2~seq1	0
"""
# tests/test_cmdline.rs test_sharding_*; `-p bwa-mem` only names the mapper, so that case is the contig case again
GOLDENS = {
    "test_sharding_no_exclusion_contig": (["contig", "--sharded", "-b", S1, S2], CONTIG_GOLDEN),
    "test_sharding_no_exclusion_bwa_contig": (["contig", "--sharded", "-b", S1, S2], CONTIG_GOLDEN),
    "test_sharding_no_exclusion_genome_separator": (["genome", "--sharded", "-b", S1, S2, "-s", "~"], """Genome	shard1|shard2 Relative Abundance (%)
unmapped	0
genome3	25.024881
genome4	25.022575
genome5	0
genome6	25.020271
genome1	24.932274
genome2	0
"""),
    "test_sharding_exclusion_genome_separator": (["genome", "--sharded", "-b", S1, S2, "-s", "~", "--exclude-genomes-from-deshard", "{EX}"],
                                                 """Genome	shard1|shard2 Relative Abundance (%)
unmapped	19.999998
genome3	0
genome4	26.699606
genome5	0
genome6	26.697144
genome1	26.60325
genome2	0
"""),
    "test_sharding_exclusion_genomes_fasta_files_definition": (
        ["genome", "--sharded", "-b", S1, S2, "--genome-definition", DEFINITION, "--exclude-genomes-from-deshard", "{EX}"],
        """Genome	shard1|shard2 Relative Abundance (%)
unmapped	19.999998
genome1	26.60325
genome2	0
genome3	0
genome4	26.699606
genome5	0
genome6	26.697144
"""),
}


@pytest.fixture(scope="module")
def genome3_list(tmp_path_factory):
    p = tmp_path_factory.mktemp("excl") / "genome3.txt"
    p.write_text("genome3\n")
    return str(p)


def _run(binary, argv, env=None, timeout=600):
    return subprocess.run([binary] + argv, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **(env or {})))


def _argv(name, ex):
    return [a.replace("{EX}", ex) for a in GOLDENS[name][0]]


@pytest.mark.parametrize("name", list(GOLDENS))
def test_oracle_reproduces_the_sharded_goldens(name, genome3_list):
    p = run_oracle(_argv(name, genome3_list))
    assert p.returncode == 0, p.stderr
    assert p.stdout == GOLDENS[name][1]


@pytest.mark.parametrize("name", list(GOLDENS))
def test_emulated_product_matches_the_goldens(name, genome3_list):
    p = _run(HOSTCHECK_BIN, _argv(name, genome3_list))
    assert p.returncode == 0, p.stderr
    assert p.stdout == GOLDENS[name][1]


# ---------------------------------------------------------------------------------------------- synthetic sets
@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    out = {}
    for K, n, seed in ((2, 1500, 11), (3, 1200, 12), (4, 900, 13)):
        d = tmp_path_factory.mktemp(f"k{K}")
        out[K] = shard_sets.rich_set(str(d), K, n, seed)
    return out


def modes(s):
    b = ["--sharded", "-b"] + s["shards"]
    return {
        "contig_mean": ["contig", "-m", "mean", "count", "covered_bases"] + b,
        "contig_hist": ["contig", "-m", "coverage_histogram"] + b,
        "contig_trim_var": ["contig", "-m", "trimmed_mean", "variance", "covered_fraction"] + b,
        "contig_anir": ["contig", "-m", "anir", "reads_per_base"] + b,
        "contig_gff": ["contig", "-m", "mean", "count", "--gff", s["gff"]] + b,
        "genome_sep": ["genome", "-s", "~", "-m", "relative_abundance", "mean", "count", "--min-covered-fraction", "0"] + b,
        "genome_sep_excl": ["genome", "-s", "~", "-m", "relative_abundance", "trimmed_mean", "--min-covered-fraction", "0",
                            "--exclude-genomes-from-deshard", s["excluded"]] + b,
        "genome_def_excl": ["genome", "--genome-definition", s["definition"], "-m", "relative_abundance", "variance",
                            "--exclude-genomes-from-deshard", s["excluded"]] + b,
    }


MODES = ["contig_mean", "contig_hist", "contig_trim_var", "contig_anir", "contig_gff", "genome_sep", "genome_sep_excl", "genome_def_excl"]


def _same_table(got, want, mode):
    if mode != "contig_anir":
        assert got == want
        return
    g, w = got.splitlines(), want.splitlines()  # ANIr sums identities in floating point, in an order that may differ
    assert len(g) == len(w) and g[0] == w[0]
    for a, b in zip(g[1:], w[1:]):
        fa, fb = a.split("\t"), b.split("\t")
        assert fa[0] == fb[0]
        for x, y in zip(fa[1:], fb[1:]):
            assert abs(float(x) - float(y)) <= 1e-6 * max(1.0, abs(float(y))), (a, b)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("K", [2, 3, 4])
def test_emulated_product_matches_oracle(sets, K, mode):
    argv = modes(sets[K])[mode] + ["--print-reads-mapped"]
    o, g = run_oracle(argv), _run(HOSTCHECK_BIN, argv)
    assert o.returncode == 0, o.stderr
    assert g.returncode == 0, g.stderr
    _same_table(g.stdout, o.stdout, mode)
    rm = lambda p: [l.split("\t")[2:] for l in p.stderr.splitlines() if l.startswith("#reads_mapped")]
    assert rm(g) == rm(o)


def test_sets_hold_what_they_claim(sets):
    """ties, unmapped records, secondaries / supplementaries and AS:S are all present in the synthetic shards"""
    import struct
    import zlib
    s = sets[3]
    raw = open(s["shards"][0], "rb").read()
    data, o = b"", 0
    while o < len(raw):
        bsize = struct.unpack_from("<H", raw, o + 16)[0] + 1
        data += zlib.decompress(raw[o + 18:o + bsize - 8], -15)
        o += bsize
    assert b"ASS" in data and b"ASC" in data
    text_len = struct.unpack_from("<I", data, 4)[0]
    n_ref = struct.unpack_from("<I", data, 8 + text_len)[0]
    o = 12 + text_len
    for _ in range(n_ref):
        o += 8 + struct.unpack_from("<I", data, o)[0]
    flags = []
    while o < len(data):
        bs = struct.unpack_from("<I", data, o)[0]
        flags.append(struct.unpack_from("<H", data, o + 18)[0])
        o += 4 + bs
    assert any(f & 0x4 for f in flags) and any(f & 0x100 for f in flags) and any(f & 0x800 for f in flags)


def _fallback_shards(d):
    """two shards that are name-sorted and, having one contig each, also reference-sorted: readable as ordinary samples (with
    one header, as the cached printers want)"""
    return _write_shards(d, [_pair("r0") + _pair("r1", as1=("AS", "C", 90)), _pair("r0") + _pair("r1")], prefix=False)


FALLBACK = [["contig", "--sharded", "--min-read-percent-identity", "90", "-b"], ["contig", "--sharded", "-m", "metabat", "-b"]]


@pytest.mark.parametrize("flags", range(len(FALLBACK)))
def test_filter_thresholds_make_sharded_fall_back(tmp_path, flags):
    """with a read filter the reference ignores --sharded: every BAM is its own sample (coverm.rs:168-187)"""
    argv = FALLBACK[flags] + _fallback_shards(str(tmp_path))
    o = run_oracle(argv)
    assert o.returncode == 0, o.stderr
    header = o.stdout.splitlines()[0]
    assert "e0" in header and "e1" in header and "|" not in header
    assert _run(HOSTCHECK_BIN, argv).stdout == o.stdout


def test_exclusion_file_needs_sharded():
    """clap's `requires("sharded")` (cli.rs:1698-1701): a usage error, exit status 2"""
    g = _run(HOSTCHECK_BIN, ["genome", "-s", "~", "--exclude-genomes-from-deshard", "x", "-b", S1])
    assert g.returncode == 2 and "--sharded" in g.stderr, g.stderr


# ---------------------------------------------------------------------------------------------- GPU
def _product(argv, env=None, timeout=900):
    import coverm_b200
    return _run(coverm_b200.COVERM_BIN, argv, env, timeout)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GOLDENS))
def test_goldens_on_the_device(name, genome3_list):
    p = _product(_argv(name, genome3_list))
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stdout == GOLDENS[name][1]


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 3, 4])
def test_synthetic_sets_on_the_device(sets, K):
    for mode, argv in modes(sets[K]).items():
        argv = argv + ["--print-reads-mapped", "-t", "4"]
        o, g = run_oracle(argv), _product(argv, {"CMB_PIPELINE_STATS": "1"})
        assert o.returncode == 0, o.stderr
        assert g.returncode == 0, (mode, g.stderr[-2000:])
        _same_table(g.stdout, o.stdout, mode)
        rm = lambda p: [l.split("\t")[2:] for l in p.stderr.splitlines() if l.startswith("#reads_mapped")]
        assert rm(g) == rm(o), mode
        assert any(l.startswith("#sharded\tpairs=") for l in g.stderr.splitlines()), mode


@pytest.mark.gpu
def test_large_set_over_many_decode_windows(tmp_path):
    shards = shard_sets.big_set(str(tmp_path), 3, 2_000_000, seed=5)
    argv = ["contig", "-m", "mean", "count", "variance", "--sharded", "-b"] + shards + ["-t", "8", "--print-reads-mapped"]
    o = run_oracle(argv)
    assert o.returncode == 0, o.stderr
    g = _product(argv, {"CMB_DECODE_WINDOW_KB": "4096", "CMB_PIPELINE_STATS": "1"})
    assert g.returncode == 0, g.stderr[-2000:]
    assert g.stdout == o.stdout
    assert [l for l in g.stderr.splitlines() if l.startswith("#reads_mapped")] == \
           [l for l in o.stderr.splitlines() if l.startswith("#reads_mapped")]


def _write_shards(d, per_shard, contigs=(("a~c0", 5000),), prefix=True):
    import bam_writer as bw
    paths = []
    for k, recs in enumerate(per_shard):
        p = os.path.join(d, f"e{k}.bam")
        cs = [((f"k{k}" if prefix else "") + n, l) for n, l in contigs]
        with open(p, "wb") as f:
            f.write(bw.bgzf(bw.bam_stream(cs, recs, text="@HD\tVN:1.6\tSO:queryname\n")))
        paths.append(p)
    return paths


def _pair(name, as1=("AS", "C", 50), as2=("AS", "C", 50), nm=("NM", "C", 1), flag1=0x43, flag2=0x83, tid=0):
    import bam_writer as bw
    t1 = [t for t in (nm, as1) if t]
    t2 = [t for t in (nm, as2) if t]
    return [bw.record(tid, 100, [("M", 50)], flag=flag1, qname=name, tags=t1), bw.record(tid, 300, [("M", 50)], flag=flag2, qname=name, tags=t2)]


def error_cases():
    ok = lambda i: _pair("r%d" % i)
    return {
        "names_differ": ([ok(0) + ok(1), ok(0) + _pair("x1")], 1, "BAM files do not appear to be properly sorted by read name"),
        "unequal_lengths": ([ok(0) + ok(1), ok(0)], 1, "Unexpectedly one BAM file input finished while another had further reads"),
        "odd_primaries": ([ok(0) + ok(1)[:1], ok(0) + ok(1)[:1]], 101, "Unexpectedly was able to read a first read set, but not a second"),
        "unpaired": ([ok(0) + _pair("r1", flag1=0x40), ok(0) + ok(1)], 1, "This code can only handle paired-end input"),
        "missing_as": ([ok(0) + _pair("r1", as2=None), ok(0) + ok(1)], 101, "does not have an 'AS' auxiliary tag"),
        "as_type_i": ([ok(0) + _pair("r1", as1=("AS", "i", 7)), ok(0) + ok(1)], 101, "Unexpected data type of AS aux tag"),
        "nm_type_s": ([ok(0) + _pair("r1", nm=("NM", "S", 1), as1=("AS", "C", 90)), ok(0) + ok(1)], 101, "Unexpected data type of NM aux tag"),
    }


EXCLUDED_ONLY = "CoverM cannot currently deal with reads that only map to excluded genomes"


def _error_bams(tmp_path, case):
    per_shard, status, msg = error_cases()[case]
    return _write_shards(str(tmp_path), per_shard), status, msg


@pytest.mark.parametrize("case", list(error_cases()))
def test_errors_oracle_and_emulator(tmp_path, case):
    shards, status, msg = _error_bams(tmp_path, case)
    for binary in (None, HOSTCHECK_BIN):
        argv = ["contig", "--sharded", "-b"] + shards
        p = run_oracle(argv) if binary is None else _run(binary, argv)
        assert p.returncode == status, (binary, p.stderr)
        assert msg in p.stderr, (binary, p.stderr)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(error_cases()))
def test_errors_on_the_device(tmp_path, case):
    shards, status, msg = _error_bams(tmp_path, case)
    p = _product(["contig", "--sharded", "-b"] + shards)
    assert p.returncode == status, p.stderr
    assert msg in p.stderr, p.stderr


def _excluded_only(tmp_path):
    shards = _write_shards(str(tmp_path), [_pair("r0") + _pair("r1"), _pair("r0") + _pair("r1")], contigs=(("a~c0", 5000),))
    ex = tmp_path / "ex.txt"
    ex.write_text("k0a\nk1a\n")
    return ["genome", "-s", "~", "--sharded", "--exclude-genomes-from-deshard", str(ex), "-b"] + shards


def test_excluded_only_oracle_and_emulator(tmp_path):
    argv = _excluded_only(tmp_path)
    for binary in (None, HOSTCHECK_BIN):
        p = run_oracle(argv) if binary is None else _run(binary, argv)
        assert p.returncode == 1 and EXCLUDED_ONLY in p.stderr, (binary, p.stderr)


@pytest.mark.gpu
def test_excluded_only_on_the_device(tmp_path):
    p = _product(_excluded_only(tmp_path))
    assert p.returncode == 1 and EXCLUDED_ONLY in p.stderr, p.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("flags", range(len(FALLBACK)))
def test_filter_fall_back_on_the_device(tmp_path, flags):
    argv = FALLBACK[flags] + _fallback_shards(str(tmp_path))
    o, g = run_oracle(argv), _product(argv)
    assert o.returncode == 0 and g.returncode == 0, g.stderr[-1500:]
    assert g.stdout == o.stdout


@pytest.mark.gpu
def test_sharded_with_two_gpus_exits_1():
    p = _product(["contig", "--sharded", "--gpus", "2", "-b", S1, S2])
    assert p.returncode == 1, p.stderr


@pytest.mark.gpu
def test_ties_are_deterministic_and_uniform(tmp_path):
    """200 000 pairs with the same score in both shards: two runs print the same bytes, each shard wins half of them"""
    import numpy as np
    n = 200_000
    shards = []
    for k in range(2):
        names = np.repeat(np.arange(n, dtype=np.int64), 2)
        pos = np.tile(np.array([100, 300], np.int32), n)
        flag = np.tile(np.array([0x43, 0x83], np.uint16), n)
        body = shard_sets.big_records(np.zeros(2 * n, np.int32), pos, flag, names, np.full(2 * n, 50, np.uint8), np.ones(2 * n, np.uint8), 100)
        import bam_writer as bw
        p = str(tmp_path / f"tie{k}.bam")
        with open(p, "wb") as f:
            f.write(bw.bgzf(bw.bam_stream([(f"k{k}~c", 100000)], [], text="@HD\tVN:1.6\n") + body, level=1))
        shards.append(p)
    argv = ["contig", "--sharded", "-m", "count", "-b"] + shards
    a, b = _product(argv), _product(argv)
    assert a.returncode == 0, a.stderr
    assert a.stdout == b.stdout
    counts = [int(l.split("\t")[1]) for l in a.stdout.splitlines()[1:]]
    assert sum(counts) == 2 * n
    for c in counts:
        assert abs(c / (2 * n) - 0.5) <= 0.01, counts
    o = run_oracle(argv)
    assert o.stdout == a.stdout
