"""Golden vectors transcribed from the reference's own tests (wwood/CoverM v0.8.0).

Every case cites the reference test it restates (file:line in wwood/CoverM v0.8.0).
The expected strings are the literal strings asserted there.  Inputs are the
reference's fixtures, stored as data files in tests/golden/data/ (they are test
inputs, not source code).

A case is a dict:
  ref      reference file:line
  sub      'contig' | 'genome' | 'filter-names'
  argv     arguments after the sub-command; '{D}' expands to the fixture dir,
           '{DEF}' to a temp file holding `definition`
  stdout   exact expected stdout                        (or)
  contains substring(s) expected in stdout              (or)
  table    expected table compared after sorting rows (assert_equal_table)
  reads_mapped  optional [[mapped,total],...] per sample (ReadsMapped)
  status   expected exit status (default 0); 101 = Rust panic, 1 = process::exit(1)

Library-level switches (--lib-*) reproduce the in-module unit-test harnesses
(contig.rs:290-322, genome.rs:940-1086): a streaming taker without header line,
explicit estimator constructor arguments and an explicit FlagFilter.
"""

S7 = "7seqs.reads_for_seq1_and_seq2"
S7A = "7seqs.reads_for_seq1"

# flag-filter triplets {include_improper_pairs, include_supplementary, include_secondary}
CONTIG_FLAGS = "1,0,0"          # contig.rs:300-304 (proper_pairs_only=false)
CONTIG_FLAGS_PP = "0,0,0"       # proper_pairs_only=true
GENOME_SEP_FLAGS = "1,1,1"      # genome.rs:958-962
GENOME_NAMES_FLAGS = "1,0,0"    # genome.rs:1035-1039, 994-998


def _contig(ref, bam, ests, expected, zeros, flags=CONTIG_FLAGS, reads_mapped=None):
    argv = ["-b", "{D}/" + bam, "--lib-streaming", "--lib-estimators", ests, "--lib-flags", flags,
            "--print-reads-mapped"]
    if not zeros:
        argv.append("--no-zeros")
    c = dict(ref=ref, sub="contig", argv=argv, stdout=expected)
    if reads_mapped is not None:
        c["reads_mapped"] = reads_mapped
    return c


def _genome_sep(ref, bams, sep, ests, expected, zeros, single=False, flags=GENOME_SEP_FLAGS, reads_mapped=None):
    argv = ["-b"] + ["{D}/" + b for b in bams] + ["--lib-streaming", "--lib-estimators", ests, "--lib-flags", flags,
                                                   "--print-reads-mapped"]
    if single:
        argv.append("--single-genome")
    else:
        argv += ["-s", sep]
    if not zeros:
        argv.append("--no-zeros")
    c = dict(ref=ref, sub="genome", argv=argv, stdout=expected)
    if reads_mapped is not None:
        c["reads_mapped"] = reads_mapped
    return c


def _genome_names(ref, bam, definition, ests, expected, zeros, reads_mapped=None):
    argv = ["-b", "{D}/" + bam, "--lib-streaming", "--lib-estimators", ests, "--lib-flags", GENOME_NAMES_FLAGS,
            "--print-reads-mapped", "--genome-definition", "{DEF}"]
    if not zeros:
        argv.append("--no-zeros")
    c = dict(ref=ref, sub="genome", argv=argv, stdout=expected, definition=definition)
    if reads_mapped is not None:
        c["reads_mapped"] = reads_mapped
    return c


DEF_SE = "se\tseq1\nse\tseq2\n"
DEF_S = "s\tseq1\ns\tseq2\n"
DEF_7 = ("genome1\tgenome1~random_sequence_length_11000\n"
         "genome1\tgenome1~random_sequence_length_11010\n"
         "genome2\tgenome2~seq1\n"
         "genome3\tgenome3~random_sequence_length_11001\n"
         "genome4\tgenome4~random_sequence_length_11002\n"
         "genome5\tgenome5~seq2\n"
         "genome6\tgenome6~random_sequence_length_11003\n")
DEF_23 = "genome2\tgenome2~seq1\ngenome3\tgenome3~random_sequence_length_11001\n"

CASES = [
    # ------------------------------------------------------------ src/contig.rs unit tests
    _contig("src/contig.rs:324-334", S7 + ".bam", "mean:0.0:0:0",
            f"{S7}\tgenome2~seq1\t1.2\n{S7}\tgenome5~seq2\t1.2\n", zeros=False),
    _contig("src/contig.rs:336-345", S7 + ".bam", "mean:0.0:0:0",
            f"{S7}\tgenome1~random_sequence_length_11000\t0\n{S7}\tgenome1~random_sequence_length_11010\t0\n"
            f"{S7}\tgenome2~seq1\t1.2\n{S7}\tgenome3~random_sequence_length_11001\t0\n"
            f"{S7}\tgenome4~random_sequence_length_11002\t0\n{S7}\tgenome5~seq2\t1.2\n"
            f"{S7}\tgenome6~random_sequence_length_11003\t0\n", zeros=True),
    _contig("src/contig.rs:367-376", "1.bam", "mean:0.0:0:0", "", zeros=False, flags=CONTIG_FLAGS_PP),
    _contig("src/contig.rs:378-388", "2seqs.reads_for_seq1.bam", "variance:0.0:0",
            "2seqs.reads_for_seq1\tseq1\t0.9489489\n2seqs.reads_for_seq1\tseq2\t0\n", zeros=True),
    _contig("src/contig.rs:417-430", "2seqs.reads_for_seq1.bam", "mean:0.0:0:0;variance:0.0:0",
            "2seqs.reads_for_seq1\tseq1\t1.2\t0.9489489\n2seqs.reads_for_seq1\tseq2\t0\t0\n", zeros=True),
    _contig("src/contig.rs:432-445", "2seqs.reads_for_seq1.with_unmapped.bam", "mean:0.0:0:1",
            "2seqs.reads_for_seq1.with_unmapped\tseq1\t1.497\n2seqs.reads_for_seq1.with_unmapped\tseq2\t1.5\n",
            zeros=True),
    _contig("src/contig.rs:447-458", "2seqs.reads_for_seq1.bam", "trimmed_mean:0.0:0.05:0.0:0",
            "2seqs.reads_for_seq1\tseq1\t0\n2seqs.reads_for_seq1\tseq2\t0\n", zeros=True),
    _contig("src/contig.rs:460-474", "2seqs.reads_for_seq1.bam", "mean:0.0:0:0;trimmed_mean:0.0:0.05:0.0:0",
            "2seqs.reads_for_seq1\tseq1\t1.2\t0\n", zeros=False),
    _contig("src/contig.rs:476-490", "2seqs.reads_for_seq1.bam", "trimmed_mean:0.0:0.05:0.0:0;mean:0.0:0:0",
            "2seqs.reads_for_seq1\tseq1\t0\t1.2\n", zeros=False),
    _contig("src/contig.rs:492-510", S7 + ".bam", "mean:0.0:75:0;variance:0.0:75",
            f"{S7}\tgenome2~seq1\t1.4117647\t1.3049262\n{S7}\tgenome5~seq2\t1.2435294\t0.6862065\n", zeros=False),
    _contig("src/contig.rs:512-522", "1read_of_pair_mapped.bam", "mean:0.0:75:1",
            "1read_of_pair_mapped\t73.20100900_E1D.16_contig_9606\t0.011293635\n", zeros=False),
    _contig("src/contig.rs:524-534", "k141_2005182.bam", "variance:0.0:75",
            "k141_2005182\tk141_2005182\t5.107387\n", zeros=False),
    _contig("src/contig.rs:536-556", "2seqs.reads_for_seq1_and_seq2.bam", "variance:0.0:75",
            "2seqs.reads_for_seq1_and_seq2\tseq1\t1.3049262\n2seqs.reads_for_seq1_and_seq2\tseq2\t0.6862065\n",
            zeros=False, reads_mapped=[[24, 24]]),
    _contig("src/contig.rs:558-577", "2seqs.reads_for_seq1_and_seq2.bam", "variance:0.99:75", "",
            zeros=False, reads_mapped=[[0, 24]]),

    # ------------------------------------------------------------ src/genome.rs unit tests
    _genome_sep("src/genome.rs:1088-1099", ["2seqs.reads_for_seq1.bam"], "q", "mean:0.0:0:0",
                "2seqs.reads_for_seq1\tse\t0.6\n", zeros=True),
    _genome_names("src/genome.rs:1101-1115", "2seqs.reads_for_seq1.bam", DEF_SE, "mean:0.0:0:0",
                  "2seqs.reads_for_seq1\tse\t0.6\n", zeros=True),
    _genome_sep("src/genome.rs:1117-1128", ["2seqs.reads_for_seq2.bam"], "q", "mean:0.0:0:0",
                "2seqs.reads_for_seq2\tse\t0.6\n", zeros=True),
    _genome_names("src/genome.rs:1130-1144", "2seqs.reads_for_seq2.bam", DEF_SE, "mean:0.0:0:0",
                  "2seqs.reads_for_seq2\tse\t0.6\n", zeros=True),
    _genome_sep("src/genome.rs:1146-1159", ["2seqs.reads_for_seq1_and_seq2.bam"], "e", "mean:0.0:0:0",
                "2seqs.reads_for_seq1_and_seq2\ts\t1.2\n", zeros=True),
    _genome_names("src/genome.rs:1161-1177", "2seqs.reads_for_seq1_and_seq2.bam", DEF_S, "mean:0.0:0:0",
                  "2seqs.reads_for_seq1_and_seq2\ts\t1.2\n", zeros=True),
    _genome_sep("src/genome.rs:1179-1192", ["2seqs.reads_for_seq1_and_seq2.bam"], "e", "mean:0.76:0:0",
                "2seqs.reads_for_seq1_and_seq2\ts\t0\n", zeros=True),
    _genome_names("src/genome.rs:1194-1210", "2seqs.reads_for_seq1_and_seq2.bam", DEF_S, "mean:0.76:0:0",
                  "", zeros=False),
    _genome_sep("src/genome.rs:1212-1225", ["2seqs.reads_for_seq1_and_seq2.bam"], "e", "mean:0.759:0:0",
                "2seqs.reads_for_seq1_and_seq2\ts\t1.2\n", zeros=True),
    _genome_names("src/genome.rs:1227-1243", "2seqs.reads_for_seq1_and_seq2.bam", DEF_S, "mean:0.759:0:0",
                  "2seqs.reads_for_seq1_and_seq2\ts\t1.2\n", zeros=True),
    _genome_sep("src/genome.rs:1245-1260", ["2seqs.reads_for_seq1_and_seq2.bam"], "e",
                "trimmed_mean:0.1:0.9:0.759:0", "2seqs.reads_for_seq1_and_seq2\ts\t1.08875\n", zeros=True),
    _genome_names("src/genome.rs:1262-1280", "2seqs.reads_for_seq1_and_seq2.bam", DEF_S,
                  "trimmed_mean:0.1:0.9:0.0:0", "2seqs.reads_for_seq1_and_seq2\ts\t1.08875\n", zeros=True),
    _genome_sep("src/genome.rs:1282-1292", ["2seqs.reads_for_seq1_and_seq2.bam"], "e", "coverage_histogram:0.0:0",
                "".join(f"2seqs.reads_for_seq1_and_seq2\ts\t{d}\t{n}\n" for d, n in
                        [(0, 482), (1, 922), (2, 371), (3, 164), (4, 61)]),
                zeros=True, flags="1,0,0"),
    _genome_names("src/genome.rs:1294-1307", "2seqs.reads_for_seq1_and_seq2.bam", DEF_S, "coverage_histogram:0.0:0",
                  "".join(f"2seqs.reads_for_seq1_and_seq2\ts\t{d}\t{n}\n" for d, n in
                          [(0, 482), (1, 922), (2, 371), (3, 164), (4, 61)]), zeros=True),
    _genome_sep("src/genome.rs:1309-1318", [S7 + ".bam"], "~", "mean:0.1:0:0",
                f"{S7}\tgenome1\t0\n{S7}\tgenome2\t1.2\n{S7}\tgenome3\t0\n{S7}\tgenome4\t0\n{S7}\tgenome5\t1.2\n"
                f"{S7}\tgenome6\t0\n", zeros=True),
    _genome_sep("src/genome.rs:1320-1328", [S7 + ".bam"], "~", "mean:0.1:0:0",
                f"{S7}\tgenome2\t1.2\n{S7}\tgenome5\t1.2\n", zeros=False),
    _genome_sep("src/genome.rs:1373-1383", [S7 + ".bam"], "~", "mean:0.759:0:0",
                f"{S7}\tgenome1\t0\n{S7}\tgenome2\t0\n{S7}\tgenome3\t0\n{S7}\tgenome4\t0\n{S7}\tgenome5\t1.2\n"
                f"{S7}\tgenome6\t0\n", zeros=True),
    _genome_sep("src/genome.rs:1385-1398", [S7 + ".bam"], "~", "mean:0.0:0:0",
                f"{S7}\tgenome1\t0.04209345\n", zeros=True, single=True),
    _genome_sep("src/genome.rs:1400-1417", [S7 + ".bam"], "~", "covered_bases:0.0",
                f"{S7}\tgenome2\t669\n{S7}\tgenome5\t849\n", zeros=False),
    _genome_names("src/genome.rs:1438-1479", S7 + ".bam", DEF_7, "mean:0.1:0:0",
                  f"{S7}\tgenome1\t0\n{S7}\tgenome2\t1.2\n{S7}\tgenome3\t0\n{S7}\tgenome4\t0\n{S7}\tgenome5\t1.2\n"
                  f"{S7}\tgenome6\t0\n", zeros=True),
    _genome_names("src/genome.rs:1481-1487", S7 + ".bam", DEF_7, "mean:0.1:0:0",
                  f"{S7}\tgenome2\t1.2\n{S7}\tgenome5\t1.2\n", zeros=False),
    _genome_names("src/genome.rs:1489-1531", S7 + ".bam", DEF_7, "mean:0.1:0:0;variance:0.1:0",
                  f"{S7}\tgenome1\t0\t0\n{S7}\tgenome2\t1.2\t1.3633634\n{S7}\tgenome3\t0\t0\n{S7}\tgenome4\t0\t0\n"
                  f"{S7}\tgenome5\t1.2\t0.6166166\n{S7}\tgenome6\t0\t0\n", zeros=True),
    _genome_names("src/genome.rs:1533-1548", S7 + ".bam", DEF_7, "mean:0.1:0:0;variance:0.1:0",
                  f"{S7}\tgenome2\t1.2\t1.3633634\n{S7}\tgenome5\t1.2\t0.6166166\n", zeros=False,
                  reads_mapped=[[24, 24]]),
    _genome_names("src/genome.rs:1550-1586", S7 + ".bam", DEF_23, "mean:0.1:0:0;variance:0.1:0",
                  f"{S7}\tgenome2\t1.2\t1.3633634\n{S7}\tgenome3\t0\t0\n", zeros=True, reads_mapped=[[12, 24]]),
    _genome_sep("src/genome.rs:1588-1609", ["2seqs.reads_for_seq1.with_unmapped.bam"], None, "mean:0.1:0:1",
                "2seqs.reads_for_seq1.with_unmapped\tgenome1\t1.4985\n", zeros=True, single=True,
                reads_mapped=[[20, 24]]),
    _genome_sep("src/genome.rs:1611-1627", ["2seqs.reads_for_seq1.bam"], None,
                "mean:0.0:0:0;trimmed_mean:0.0:0.05:0.0:0", "2seqs.reads_for_seq1\tgenome1\t0.6\t0\n",
                zeros=False, single=True),
    _genome_sep("src/genome.rs:1629-1645", ["2seqs.reads_for_seq1.bam"], None,
                "trimmed_mean:0.0:0.05:0.0:0;mean:0.0:0:0", "2seqs.reads_for_seq1\tgenome1\t0\t0.6\n",
                zeros=False, single=True),
    _genome_sep("src/genome.rs:1647-1661", [S7A + ".bam"], "~", "mean:0.0:0:0;trimmed_mean:0.0:0.05:0.0:0",
                f"{S7A}\tgenome1\t0\t0\n{S7A}\tgenome2\t1.2\t0\n{S7A}\tgenome3\t0\t0\n{S7A}\tgenome4\t0\t0\n"
                f"{S7A}\tgenome5\t0\t0\n{S7A}\tgenome6\t0\t0\n", zeros=True),
    _genome_sep("src/genome.rs:1663-1677", [S7A + ".bam"], "~", "trimmed_mean:0.0:0.05:0.0:0;mean:0.0:0:0",
                f"{S7A}\tgenome1\t0\t0\n{S7A}\tgenome2\t0\t1.2\n{S7A}\tgenome3\t0\t0\n{S7A}\tgenome4\t0\t0\n"
                f"{S7A}\tgenome5\t0\t0\n{S7A}\tgenome6\t0\t0\n", zeros=True),
    _genome_sep("src/genome.rs:1794-1836", [S7A + ".bam", S7 + ".bam"], "~", "count",
                "".join(f"{S7A}\tgenome{i}\t{12 if i == 2 else 0}\n" for i in range(1, 7)) +
                "".join(f"{S7}\tgenome{i}\t{12 if i in (2, 5) else 0}\n" for i in range(1, 7)),
                zeros=True, reads_mapped=[[12, 12], [24, 24]]),
    _genome_sep("src/genome.rs:1838-1885", [S7A + ".bam", S7 + ".bam"], "~", "count;covered_fraction:0.1",
                f"{S7A}\tgenome1\t0\t0\n{S7A}\tgenome2\t12\t0.727\n{S7A}\tgenome3\t0\t0\n{S7A}\tgenome4\t0\t0\n"
                f"{S7A}\tgenome5\t0\t0\n{S7A}\tgenome6\t0\t0\n"
                f"{S7}\tgenome1\t0\t0\n{S7}\tgenome2\t12\t0.669\n{S7}\tgenome3\t0\t0\n{S7}\tgenome4\t0\t0\n"
                f"{S7}\tgenome5\t12\t0.849\n{S7}\tgenome6\t0\t0\n",
                zeros=True, reads_mapped=[[12, 12], [24, 24]]),
    _genome_sep("src/genome.rs:1887-1927", [S7A + ".bam", S7 + ".bam"], "~", "covered_fraction:0.99",
                "".join(f"{S7A}\tgenome{i}\t0\n" for i in range(1, 7)) +
                "".join(f"{S7}\tgenome{i}\t0\n" for i in range(1, 7)),
                zeros=True, reads_mapped=[[0, 12], [0, 24]]),
    _genome_names("src/genome.rs:1929-1964", S7 + ".bam", DEF_7, "mean:0.1:0:0;variance:0.1:0",
                  f"{S7}\tgenome2\t1.2\t1.3633634\n{S7}\tgenome5\t1.2\t0.6166166\n", zeros=False,
                  reads_mapped=[[24, 24]]),
    _genome_names("src/genome.rs:1966-1986", S7 + ".bam", DEF_7, "mean:0.99:0:0;variance:0.99:0", "", zeros=False,
                  reads_mapped=[[0, 24]]),
]


def _filter(ref, bam, names, pair=(0, 0.0, 0.0), single=(0, 0.0, 0.0), mapq=0, flags="0,0,0", inverse=False,
            count=None, exact=False):
    argv = ["-b", "{D}/" + bam, "--lib-flags", flags, "--min-mapq", str(mapq)]
    if flags.startswith("0"):
        argv.append("--proper-pairs-only")
    if single[0]:
        argv += ["--min-read-aligned-length", str(single[0])]
    if single[1]:
        argv += ["--min-read-percent-identity", str(single[1])]
    if single[2]:
        argv += ["--min-read-aligned-percent", str(single[2])]
    if pair[0]:
        argv += ["--min-read-aligned-length-pair", str(pair[0])]
    if pair[1]:
        argv += ["--min-read-percent-identity-pair", str(pair[1])]
    if pair[2]:
        argv += ["--min-read-aligned-percent-pair", str(pair[2])]
    if inverse:
        argv.append("--inverse")
    c = dict(ref=ref, sub="filter-names", argv=argv)
    if count is not None:
        c["line_count"] = count
    elif exact:
        c["stdout"] = "".join(n + "\n" for n in names)
    else:  # the reference test reads exactly len(names) records and does not assert EOF
        c["stdout_prefix"] = "".join(n + "\n" for n in names)
    return c


_HW = ["9", "9", "12", "12", "7", "7", "11", "11", "10", "10", "8", "8", "4", "4", "6", "6", "1", "1", "2", "2",
       "3", "3", "5", "5"]

# ---------------------------------------------------------------- src/filter.rs unit tests
# (ReferenceSortedBamFilter::new(reader, flags, len_s, id_s, pct_s, mapq, len_p, id_p, pct_p, filter_out))
FILTER_CASES = [
    _filter("src/filter.rs:342-374", S7 + ".bam", _HW, pair=(90, 0.99, 0.0), exact=True),
    _filter("src/filter.rs:376-405", S7 + ".bam", [], pair=(90, 0.99, 0.0), inverse=True, exact=True),
    _filter("src/filter.rs:407-432", "2seqs.bad_read.1.bam", ["2", "2", "3", "3"], pair=(250, 0.99, 0.0)),
    _filter("src/filter.rs:434-456", "2seqs.bad_read.1.bam", ["2", "2", "3", "3"], pair=(300, 0.98, 0.0)),
    _filter("src/filter.rs:458-480", "2seqs.bad_read.1.with_extra.bam", ["2", "2", "3", "3"], pair=(0, 0.98, 0.94)),
    _filter("src/filter.rs:482-502", "2seqs.bad_read.1.bam", ["1", "1", "2", "2"], pair=(299, 0.98, 0.0)),
    _filter("src/filter.rs:504-530", "2seqs.bad_read.1.bam", ["1", "1"], pair=(250, 0.99, 0.0), inverse=True),
    _filter("src/filter.rs:532-553", "2seqs.bad_read.1.bam", ["1", "1"], pair=(300, 0.98, 0.0), inverse=True),
    _filter("src/filter.rs:555-576", "2seqs.bad_read.1.with_extra.bam", ["1", "1"], pair=(0, 0.98, 0.94),
            inverse=True),
    _filter("src/filter.rs:578-599", "2seqs.bad_read.1.bam", [], pair=(299, 0.98, 0.0), inverse=True),
    _filter("src/filter.rs:602-630", "2seqs.bad_read.1.bam", ["2", "3", "4", "1"], single=(0, 0.99, 0.0),
            flags="1,0,0"),
    _filter("src/filter.rs:632-660", "2seqs.bad_read.1.bam", ["1"], single=(0, 0.99, 0.0), flags="1,0,0",
            inverse=True),
    _filter("src/filter.rs:662-690", "2seqs.bad_read.1.bam", ["2", "2", "3", "3", "4", "4"], single=(0, 0.95, 0.0),
            pair=(300, 0.0, 0.0)),
    _filter("src/filter.rs:692-720", "2seqs.bad_read.1.bam", ["1", "1"], single=(0, 0.95, 0.0),
            pair=(300, 0.0, 0.0), inverse=True),
    _filter("src/filter.rs:722-750", "eg2.bam", None, pair=(1, 0.0, 0.0), count=11192),
    _filter("src/filter.rs:752-781", "mapq_test.sam", ["1", "1", "2", "2"], mapq=1, flags="1,0,0"),
    _filter("src/filter.rs:783-812", "mapq_test.sam", ["1", "2", "2"], mapq=51, flags="1,0,0"),
    _filter("src/filter.rs:814-844", "mapq_test.sam", ["2", "2"], mapq=51, pair=(1, 0.0, 0.0), flags="1,0,0"),
]


def _cli(ref, sub, argv, **kw):
    c = dict(ref=ref, sub=sub, argv=argv)
    c.update(kw)
    return c


V = "7seqs.fnaVbad_read"
_ZC = ["genome1~random_sequence_length_11000", "genome1~random_sequence_length_11010", "genome2~seq1",
       "genome3~random_sequence_length_11001", "genome4~random_sequence_length_11002", "genome5~seq2",
       "genome6~random_sequence_length_11003"]


def _contig_rows(prefix, vals):
    """rows for the 7seqs reference; vals maps contig -> tab-joined value string, others get zeros."""
    return prefix, vals


# ---------------------------------------------------------------- tests/test_cmdline.rs (only `-b` tests)
CLI_CASES = [
    _cli("tests/test_cmdline.rs:1145-1172", "genome",
         ["-m", "relative_abundance", "mean", "-b", "{D}/" + S7 + ".bam", "--output-format", "sparse", "-s", "~"],
         contains=["Sample\tGenome\tRelative Abundance (%)\tMean\n"
                   f"{S7}\tunmapped\t0\tNA\n{S7}\tgenome1\t0\t0\n{S7}\tgenome2\t53.16792\t1.4117647\n"
                   f"{S7}\tgenome3\t0\t0\n{S7}\tgenome4\t0\t0\n{S7}\tgenome5\t46.832077\t1.2435294\n"
                   f"{S7}\tgenome6\t0\t0"]),
    _cli("tests/test_cmdline.rs:1174-1197", "contig", ["-b", "{D}/" + S7 + ".bam", "--output-format", "dense"],
         contains=[f"Contig\t{S7} Mean\n"
                   "genome1~random_sequence_length_11000\t0\ngenome1~random_sequence_length_11010\t0\n"
                   "genome2~seq1\t1.4117647\ngenome3~random_sequence_length_11001\t0\n"
                   "genome4~random_sequence_length_11002\t0\ngenome5~seq2\t1.2435294\n"
                   "genome6~random_sequence_length_11003\t0"]),
    _cli("tests/test_cmdline.rs:1199-1226", "genome",
         ["-m", "relative_abundance", "-b", "{D}/" + S7 + ".bam", "-s", "~", "--output-format", "dense"],
         contains=[f"Genome\t{S7} Relative Abundance (%)\nunmapped\t0\ngenome1\t0\ngenome2\t53.167923\ngenome3\t0\n"
                   "genome4\t0\ngenome5\t46.832077\ngenome6\t0"]),
    _cli("tests/test_cmdline.rs:1561-1578", "contig", ["-m", "metabat", "-b", "{D}/k141_7.reheadered.bam"],
         contains=["contigName\tcontigLen\ttotalAvgDepth\tk141_7.reheadered.bam\tk141_7.reheadered.bam-var\n"
                   "k141_7\t350\t0.69\t0.69\t2.0843"]),
    _cli("tests/test_cmdline.rs:1580-1598", "contig", ["-m", "metabat", "-b", "{D}/k141_2005182.head11.bam"],
         contains=["contigName\tcontigLen\ttotalAvgDepth\tk141_2005182.head11.bam\tk141_2005182.head11.bam-var\n"
                   "k141_2005182\t225\t1.9333\t1.9333\t0.0631"]),
    _cli("tests/test_cmdline.rs:1600-1612", "contig", ["-m", "metabat", "-b", "{D}/k141_109815.stray_read.bam"],
         contains=["contigName\tcontigLen\ttotalAvgDepth\tk141_109815.stray_read.bam\tk141_109815.stray_read.bam-var\n"
                   "k141_109815\t362\t0.6274\t0.6274\t0.2349"]),
    _cli("tests/test_cmdline.rs:2262-2279", "genome",
         ["--genome-definition", "{D}/7seqs.definition", "-b", "{D}/" + S7 + ".bam"],
         contains=[f"Genome\t{S7} Relative Abundance (%)\n", "genome2\t53.167923\n", "genome5\t46.832077\n"]),
    _cli("tests/test_cmdline.rs:2465-2491", "contig",
         ["-m", "rpkm", "reads_per_base", "length", "count", "-b", "{D}/" + V + ".bam", "--output-format", "sparse"],
         stdout="Sample\tContig\tRPKM\tReads per base\tLength\tRead Count\n"
                f"{V}\tgenome1~random_sequence_length_11000\t0\t0\t11000\t0\n"
                f"{V}\tgenome1~random_sequence_length_11010\t0\t0\t11010\t0\n"
                f"{V}\tgenome2~seq1\t500000\t0.01\t1000\t10\n"
                f"{V}\tgenome3~random_sequence_length_11001\t0\t0\t11001\t0\n"
                f"{V}\tgenome4~random_sequence_length_11002\t0\t0\t11002\t0\n"
                f"{V}\tgenome5~seq2\t500000\t0.01\t1000\t10\n"
                f"{V}\tgenome6~random_sequence_length_11003\t0\t0\t11003\t0\n"),
    _cli("tests/test_cmdline.rs:2493-2517", "contig",
         ["-m", "rpkm", "reads_per_base", "length", "count", "-b", "{D}/" + V + ".bam"],
         stdout=f"Contig\t{V} RPKM\t{V} Reads per base\t{V} Length\t{V} Read Count\n"
                "genome1~random_sequence_length_11000\t0\t0\t11000\t0\n"
                "genome1~random_sequence_length_11010\t0\t0\t11010\t0\n"
                "genome2~seq1\t500000\t0.01\t1000\t10\n"
                "genome3~random_sequence_length_11001\t0\t0\t11001\t0\n"
                "genome4~random_sequence_length_11002\t0\t0\t11002\t0\n"
                "genome5~seq2\t500000\t0.01\t1000\t10\n"
                "genome6~random_sequence_length_11003\t0\t0\t11003\t0\n"),
    _cli("tests/test_cmdline.rs:2519-2540", "genome",
         ["--single-genome", "-m", "rpkm", "reads_per_base", "length", "count", "--min-covered-fraction", "0",
          "-b", "{D}/" + V + ".bam"],
         stdout=f"Genome\t{V} RPKM\t{V} Reads per base\t{V} Length\t{V} Read Count\n"
                "genome1\t17538.936\t0.00035077872\t57016\t20\n"),
    _cli("tests/test_cmdline.rs:2542-2557", "genome", ["--single-genome", "-m", "rpkm", "-b", "{D}/" + V + ".bam"],
         stdout=f"Genome\t{V} RPKM\ngenome1\t0\n"),
    # --genome-fasta-directory tests/data/genomes_dir_7seqs restated as the equivalent definition file
    # (FASTA parsing is out of scope); rows compared after sorting as the reference does.
    _cli("tests/test_cmdline.rs:2784-2814", "genome",
         ["--output-format", "sparse", "-b", "{D}/" + V + ".bam", "--genome-definition", "{D}/7seqs.definition",
          "-t", "5", "--methods", "covered_bases", "covered_fraction", "mean", "variance", "trimmed_mean", "rpkm",
          "relative_abundance", "length", "--min-covered-fraction", "0"],
         table="Sample\tGenome\tCovered Bases\tCovered Fraction\tMean\tVariance\tTrimmed Mean\tRPKM\t"
               "Relative Abundance (%)\tLength\n"
               f"{V}\tunmapped\tNA\tNA\tNA\tNA\tNA\tNA\t0\tNA\n"
               f"{V}\tgenome2\t899\t0.899\t1.6764706\t0.51357985\t1.6788511\t500000\t50\t1000\n"
               f"{V}\tgenome6\t0\t0\t0\t0\t0\t0\t0\t11003\n"
               f"{V}\tgenome4\t0\t0\t0\t0\t0\t0\t0\t11002\n"
               f"{V}\tgenome3\t0\t0\t0\t0\t0\t0\t0\t11001\n"
               f"{V}\tgenome5\t900\t0.9\t1.6764706\t0.51357985\t1.6788511\t500000\t50\t1000\n"
               f"{V}\tgenome1\t0\t0\t0\t0\t0\t0\t0\t22010\n"),
    _cli("tests/test_cmdline.rs:3072-3080", "contig", ["-b", "{D}/2seqs.bad_read.1.unsorted.bam"],
         status=101, stderr_contains="BAM file appears to be unsorted"),
    _cli("tests/test_cmdline.rs:3082-3096", "genome", ["-s", "e", "-b", "{D}/2seqs.bad_read.1.unsorted.bam"],
         status=101, stderr_contains="BAM file appears to be unsorted"),
    # names mode (the reference test uses --genome-fasta-directory genomes_dir = seq1.fna, seq2.fna)
    _cli("tests/test_cmdline.rs:3098-3113", "genome",
         ["--genome-definition", "{D}/2seqs.genome-definition", "-b", "{D}/2seqs.bad_read.1.unsorted.bam"],
         status=101, stderr_contains="BAM file appears to be unsorted"),
    _cli("tests/test_cmdline.rs:3456-3480", "contig",
         ["--output-format", "sparse", "-m", "mean", "tpm", "-b", "{D}/tpm_test.bam"],
         stdout="Sample\tContig\tMean\tTPM\n"
                "tpm_test\tgenome1~random_sequence_length_11000\t0\t0\n"
                "tpm_test\tgenome1~random_sequence_length_11010\t0\t0\n"
                "tpm_test\tgenome2~seq1\t1.5882353\t900000.0357627869\n"
                "tpm_test\tgenome3~random_sequence_length_11001\t0\t0\n"
                "tpm_test\tgenome4~random_sequence_length_11002\t0\t0\n"
                "tpm_test\tgenome5~seq2\t0.14467005\t99999.99403953552\n"
                "tpm_test\tgenome6~random_sequence_length_11003\t0\t0\n"),
    _cli("tests/test_cmdline.rs:3482-3504", "contig", ["-m", "mean", "tpm", "-b", "{D}/tpm_test.bam"],
         stdout="Contig\ttpm_test Mean\ttpm_test TPM\n"
                "genome1~random_sequence_length_11000\t0\t0\n"
                "genome1~random_sequence_length_11010\t0\t0\n"
                "genome2~seq1\t1.5882353\t900000.06\n"
                "genome3~random_sequence_length_11001\t0\t0\n"
                "genome4~random_sequence_length_11002\t0\t0\n"
                "genome5~seq2\t0.14467005\t99999.99\n"
                "genome6~random_sequence_length_11003\t0\t0\n"),
    _cli("tests/test_cmdline.rs:3506-3533", "genome",
         ["--output-format", "sparse", "-m", "mean", "tpm", "-b", "{D}/tpm_test.bam", "-s", "~",
          "--min-covered-fraction", "0"],
         stdout="Sample\tGenome\tMean\tTPM\n"
                "tpm_test\tgenome1\t0\t0\n"
                "tpm_test\tgenome2\t1.5882353\t900000.0357627869\n"
                "tpm_test\tgenome3\t0\t0\n"
                "tpm_test\tgenome4\t0\t0\n"
                "tpm_test\tgenome5\t0.14467005\t99999.99403953552\n"
                "tpm_test\tgenome6\t0\t0\n"),
    _cli("tests/test_cmdline.rs:3535-3560", "genome",
         ["-m", "mean", "tpm", "-b", "{D}/tpm_test.bam", "-s", "~", "--min-covered-fraction", "0"],
         stdout="Genome\ttpm_test Mean\ttpm_test TPM\n"
                "genome1\t0\t0\ngenome2\t1.5882353\t900000.06\ngenome3\t0\t0\ngenome4\t0\t0\n"
                "genome5\t0.14467005\t99999.99\ngenome6\t0\t0\n"),
    _cli("tests/test_cmdline.rs:3585-3604", "genome",
         ["-m", "count", "-b", "{D}/2seqs.bad_read.1.with_supplementary.bam", "--single-genome",
          "--min-covered-fraction", "0"],
         stdout="Genome\t2seqs.bad_read.1.with_supplementary Read Count\ngenome1\t20\n"),
    _cli("tests/test_cmdline.rs:4069-4090", "genome",
         ["-m", "mean", "covered_fraction", "-b", "{D}/mapq_test.sam", "--single-genome",
          "--min-covered-fraction", "0"],
         stdout="Genome\tmapq_test Mean\tmapq_test Covered Fraction\ngenome1\t0.009380695\t0.00875193\n"),
    _cli("tests/test_cmdline.rs:4092-4111", "genome",
         ["-m", "mean", "covered_fraction", "-b", "{D}/mapq_test.sam", "--single-genome",
          "--min-covered-fraction", "0", "--min-mapq", "100"],
         stdout="Genome\tmapq_test Mean\tmapq_test Covered Fraction\ngenome1\t0\t0\n"),
    _cli("tests/test_cmdline.rs:4114-4137", "contig", ["-m", "mean", "covered_fraction", "-b", "{D}/mapq_test.sam"],
         stdout="Contig\tmapq_test Mean\tmapq_test Covered Fraction\n"
                "genome1~random_sequence_length_11000\t0\t0\ngenome1~random_sequence_length_11010\t0\t0\n"
                "genome2~seq1\t0.61764705\t0.499\ngenome3~random_sequence_length_11001\t0\t0\n"
                "genome4~random_sequence_length_11002\t0\t0\ngenome5~seq2\t0\t0\n"
                "genome6~random_sequence_length_11003\t0\t0\n"),
    _cli("tests/test_cmdline.rs:4139-4160", "contig",
         ["-m", "mean", "covered_fraction", "-b", "{D}/mapq_test.sam", "--min-mapq", "51"],
         stdout="Contig\tmapq_test Mean\tmapq_test Covered Fraction\n"
                "genome1~random_sequence_length_11000\t0\t0\ngenome1~random_sequence_length_11010\t0\t0\n"
                "genome2~seq1\t0.5294118\t0.4\ngenome3~random_sequence_length_11001\t0\t0\n"
                "genome4~random_sequence_length_11002\t0\t0\ngenome5~seq2\t0\t0\n"
                "genome6~random_sequence_length_11003\t0\t0\n"),
    _cli("tests/test_cmdline.rs:4163-4188", "contig",
         ["-m", "mean", "covered_fraction", "-b", "{D}/mapq_test.sam", "--min-mapq", "51", "--proper-pairs-only"],
         stdout="Contig\tmapq_test Mean\tmapq_test Covered Fraction\n"
                "genome1~random_sequence_length_11000\t0\t0\ngenome1~random_sequence_length_11010\t0\t0\n"
                "genome2~seq1\t0.3529412\t0.3\ngenome3~random_sequence_length_11001\t0\t0\n"
                "genome4~random_sequence_length_11002\t0\t0\ngenome5~seq2\t0\t0\n"
                "genome6~random_sequence_length_11003\t0\t0\n"),
    _cli("tests/test_cmdline.rs:4190-4208", "genome",
         ["-m", "anir", "-b", "{D}/2seqs.bad_read.1.with_supplementary.bam", "--single-genome",
          "--min-covered-fraction", "0"],
         stdout="Genome\t2seqs.bad_read.1.with_supplementary ANIr\ngenome1\t0.999\n"),
]

# ---------------------------------------------------------------- per-gene coverage (src/genes.rs, --gff)
# genes.rs unit tests build GeneDefinitions in code (whole-contig genes on seq1 / seq2 of the 2seqs reference);
# 2seqs_whole_contig_genes.gff (written for these cases, not a reference file) states the same two genes as GFF lines.
# Harness of genes.rs:577-618: streaming taker, mean(0.0, 0, false) / read-count estimator, FlagFilter {improper: true,
# secondary: false, supplementary: false}.
_G2 = "2seqs.reads_for_seq1"
_WHOLE = "{D}/2seqs_whole_contig_genes.gff"
GENE_CASES = [
    _cli("src/genes.rs:646-679", "contig",
         ["-b", "{D}/" + _G2 + ".bam", "--gff", _WHOLE, "--lib-streaming", "--lib-estimators", "mean:0.0:0:0", "--lib-flags", "1,0,0"],
         stdout=f"{_G2}\tgene_seq1\tseq1\t1.2\n{_G2}\tgene_seq2\tseq2\t0\n"),
    _cli("src/genes.rs:681-718", "genome",
         ["-b", "{D}/" + _G2 + ".bam", "--gff", _WHOLE, "--genome-definition", "{DEF}", "--lib-streaming", "--lib-estimators", "mean:0.0:0:0",
          "--lib-flags", "1,0,0"],
         definition="genomeA\tseq1\n", stdout=f"{_G2}\tgene_seq1\tseq1\tgenomeA\t1.2\n"),
    _cli("src/genes.rs:720-745", "contig",
         ["-b", "{D}/" + _G2 + ".bam", "--gff", _WHOLE, "--lib-streaming", "--lib-estimators", "mean:0.0:0:0", "--lib-flags", "1,0,0", "--no-zeros"],
         stdout=f"{_G2}\tgene_seq1\tseq1\t1.2\n"),
    _cli("src/genes.rs:747-765", "contig",
         ["-b", "{D}/" + _G2 + ".bam", "--gff", "{D}/2seqs_gene_seq1_only.gff", "--lib-streaming", "--lib-estimators", "count", "--lib-flags", "1,0,0",
          "--no-zeros"],
         stdout=f"{_G2}\tgene_seq1\tseq1\t12\n"),
    _cli("tests/test_cmdline.rs:134-158", "contig",
         ["--bam-files", "{D}/" + _G2 + ".bam", "--gff", "{D}/2seqs.gff", "--methods", "mean", "--contig-end-exclusion", "0", "--output-format", "sparse"],
         contains=["Sample\tGene\tContig\tMean", f"{_G2}\tgene1\tseq1\t1.2", f"{_G2}\tgene3\tseq2\t0"]),
    _cli("tests/test_cmdline.rs:160-179", "contig",
         ["--bam-files", "{D}/" + _G2 + ".bam", "--gff", "{D}/2seqs.gff", "--methods", "count", "--output-format", "sparse", "--no-zeros"],
         contains=[f"{_G2}\tgene1\tseq1\t12"]),
    _cli("tests/test_cmdline.rs:181-209", "genome",
         ["--bam-files", "{D}/" + _G2 + ".bam", "--gff", "{D}/2seqs.gff", "--genome-definition", "{D}/2seqs.genome-definition", "--methods", "mean",
          "--contig-end-exclusion", "0", "--min-covered-fraction", "0", "--output-format", "sparse"],
         contains=["Sample\tGene\tContig\tGenome\tMean", f"{_G2}\tgene1\tseq1\tgenomeA\t1.2", f"{_G2}\tgene3\tseq2\tgenomeB\t0"]),
]
OWN_GFF_FIXTURES = {  # GFF statements of the gene sets genes.rs's unit tests construct in code
    "2seqs_whole_contig_genes.gff": "seq1\ttest\tgene\t1\t1000\t.\t+\t.\tID=gene_seq1\nseq2\ttest\tgene\t1\t1000\t.\t+\t.\tID=gene_seq2\n",
    "2seqs_gene_seq1_only.gff": "seq1\ttest\tgene\t1\t1000\t.\t+\t.\tID=gene_seq1\n",
}
CLI_CASES = CLI_CASES + GENE_CASES

ALL_CASES = CASES + FILTER_CASES + CLI_CASES
