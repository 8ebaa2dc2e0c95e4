"""The pair path of ReferenceSortedBamFilter (filter.rs:117-233): `--proper-pairs-only` with a pair threshold in `coverm contig`
and `coverm genome`, and `coverm filter` with and without `--inverse`.

tests/pair_reference.py restates the reference's walk over decoded records.  On the CPU it is checked against the oracle on
every BAM below (filter-names in both modes, read counts of `contig`), and tests/native/pairs_check.cpp runs the device's
mate matching and filter kernels, compiled as plain C++, over thousands of random record streams against the same walk.
Marked gpu: the `coverm` CLI on every BAM below against the oracle and the reference -- filter output records byte for byte
and in order, contig tables and read counts -- with the device path asserted where the stream should stay on it, and the
host's HostMates path (CMB_HOST_DECODE=1) as a check on the fallback.

Each BAM pins one way a table keyed by (tid, qname) could differ from the reference's BTreeMap, cleared on every tid change."""
import os
import random
import re
import subprocess

import pytest

import bam_writer as bw
import pair_reference as pr
from case_runner import ORACLE_BIN, ROOT
from device_reference import default_params

P = 0x1 | 0x2  # paired, proper
R1, R2, UNMAPPED, MATE_UNMAPPED, SECONDARY, SUPPLEMENTARY = 0x40, 0x80, 0x4, 0x8, 0x100, 0x800
CONTIGS = [("gA~c0", 5000), ("gA~c1", 5000), ("gB~c2", 5000), ("gB~c3", 5000)]  # genomes gA, gB for `genome -s ~`


def rec(tid, pos, name, flag=P | R1, mtid=None, nm=1, length=100, mapq=60, tags=None):
    return bw.record(tid, pos, [("M", length)], flag=flag, mapq=mapq, qname=name, mtid=tid if mtid is None else mtid, mpos=pos,
                     tags=(("NM", "C", nm),) if tags is None else tags)


def split_by_other_contig():
    """X on c0, Y on c1, X on c0 (then Z on c2, W on c3, Z on c2): the record of another tid clears the stored first mates, so the
    two X records (and the Z records) never meet.  The eligible tids go down: the device declines to the host."""
    return [rec(0, 100, "X"), rec(1, 100, "Y"), rec(0, 300, "X", P | R2), rec(2, 50, "Z"), rec(3, 60, "W"), rec(2, 70, "Z", P | R2),
            rec(3, 80, "V"), rec(3, 90, "V", P | R2)]


def unmapped_proper_first():
    """Z unmapped (proper flag set), Z mapped with its mate unmapped, Z mapped: with --inverse the unmapped record is returned at
    once and never stored, so the two mapped records are the pair; without it the unmapped record pairs with the second."""
    return [rec(0, 100, "Z", P | UNMAPPED | R1), rec(0, 100, "Z", P | MATE_UNMAPPED | R2), rec(0, 120, "Z", P | R2),
            rec(0, 200, "Q"), rec(0, 240, "Q", P | R2, length=30)]


def three_and_four_of_a_name():
    """Three records of A (the third is stored again, alone) and four of B (two pairs)."""
    return [rec(0, 10, "A"), rec(0, 20, "A", P | R2), rec(0, 30, "A"), rec(0, 40, "B"), rec(0, 50, "B", P | R2, length=20),
            rec(0, 60, "B"), rec(0, 70, "B", P | R2)]


def mtid_elsewhere():
    """A first record whose mtid is another contig is not stored (so the next record of its name is stored instead); a stored
    record is completed by a second one whose own mtid is another contig."""
    return [rec(0, 10, "M", mtid=1), rec(0, 20, "M", P | R2), rec(0, 30, "M"), rec(0, 40, "N"), rec(0, 50, "N", P | R2, mtid=2)]


def one_name_two_contigs():
    """One name paired on c0 and again on c1, and a name stored on c0 whose mate is the first of its name on c1."""
    return [rec(0, 10, "D"), rec(0, 20, "D", P | R2), rec(0, 30, "E"), rec(1, 10, "D"), rec(1, 15, "E", P | R2),
            rec(1, 20, "D", P | R2), rec(1, 30, "E")]


def name_lengths():
    """Names that are prefixes of each other, a 1-byte name and two 254-byte names that differ in their last byte."""
    long_a, long_b = "L" * 253 + "a", "L" * 253 + "b"
    return [rec(0, 10, "ab"), rec(0, 11, "a"), rec(0, 12, "abc"), rec(0, 13, long_a), rec(0, 14, "a", P | R2),
            rec(0, 15, long_b), rec(0, 16, "abc", P | R2), rec(0, 17, long_b, P | R2), rec(0, 18, "ab", P | R2), rec(0, 19, long_a, P | R2)]


def secondary_between():
    """Secondary and supplementary records of the name between its mates (and an improper pair of it)."""
    return [rec(0, 10, "S"), rec(0, 20, "S", P | SECONDARY), rec(0, 25, "S", P | SUPPLEMENTARY | R2), rec(0, 28, "S", 0x1 | R2),
            rec(0, 30, "S", P | R2), rec(0, 40, "S", P | SECONDARY | R2)]


def unmapped_mate_on_contig():
    """An unmapped proper mate placed on its contig next to its mapped mate, in both orders."""
    return [rec(0, 10, "U"), rec(0, 10, "U", P | UNMAPPED | R2), rec(0, 50, "V", P | UNMAPPED | R1), rec(0, 50, "V", P | R2),
            rec(1, 70, "W"), rec(1, 90, "W", P | R2)]


def missing_nm():
    """A proper pair whose second mate has no NM tag: nm() panics when the pair predicates are reached."""
    return [rec(0, 10, "K"), rec(0, 30, "K", P | R2, tags=())]


def big_group():
    """25 proper records of one (tid, name): more than the device's 24 per table slot, so it declines to the host."""
    return [rec(0, 10 + k, "G", P | (R1 if k % 2 == 0 else R2)) for k in range(25)] + [rec(0, 100, "H"), rec(0, 110, "H", P | R2)]


def many_blocks():
    """A sorted file of 3000 pairs over all four contigs, cut into small BGZF blocks, so that mates and names lie in different
    blocks and (with 64 KB decode windows) different windows."""
    rng = random.Random(5)
    out = []
    for t in range(4):
        pending = []
        for k in range(750):
            pending.append((rng.randrange(4000), f"p{t}_{k}", P | R1))
            pending.append((rng.randrange(4000), f"p{t}_{k}", P | R2))
        pending.sort()
        for pos, name, flag in pending:
            out.append(rec(t, pos, name, flag, nm=rng.randrange(6), length=rng.randint(30, 150), mapq=rng.choice([0, 20, 60])))
    return out


CASES = {f.__name__: f for f in (split_by_other_contig, unmapped_proper_first, three_and_four_of_a_name, mtid_elsewhere,
                                 one_name_two_contigs, name_lengths, secondary_between, unmapped_mate_on_contig, missing_nm,
                                 big_group, many_blocks)}
DECLINED = {"split_by_other_contig", "big_group"}  # the device hands these to the host's mate matching

# pair thresholds and MAPQ; identity 0.99 is 1 - 2/200 in f32, the identity of two 100-base mates with NM 1, at the threshold
SETTINGS = {
    "len1": (["--min-read-aligned-length-pair", "1"], dict(min_aligned_length_pair=1)),
    "len150_mapq20": (["--min-read-aligned-length-pair", "150", "--min-mapq", "20"], dict(min_aligned_length_pair=150, min_mapq=20)),
    "ident_pct": (["--min-read-percent-identity-pair", "0.99", "--min-read-aligned-percent-pair", "0.5"],
                  dict(min_percent_identity_pair=0.99, min_aligned_percent_pair=0.5)),
    "len500": (["--min-read-aligned-length-pair", "500"], dict(min_aligned_length_pair=500)),
}


def params(setting):
    return default_params(filtering=1, include_improper_pairs=0, **SETTINGS[setting][1])


@pytest.fixture(scope="module")
def bams(tmp_path_factory):
    d = tmp_path_factory.mktemp("pairs")
    out = {}
    for name, f in CASES.items():
        stream = bw.bam_stream(CONTIGS, f())
        path = str(d / f"{name}.bam")
        with open(path, "wb") as fh:
            fh.write(bw.bgzf(stream, block_sizes=(300, 2000), seed=3) if name == "many_blocks" else bw.bgzf(stream))
        out[name] = path
    return out


def _oracle(argv):
    return subprocess.run([ORACLE_BIN] + argv, capture_output=True, text=True, timeout=300)


def _counts(stdout):
    return [int(line.split("\t")[1]) for line in stdout.splitlines()[1:]]


# ---------------------------------------------------------------------------------------------- CPU
def test_pairs_kernels_model(tmp_path):
    """kd_pair_* and kf_decide / kf_gather compiled with g++ (ASan/UBSan) over random streams, against filter.rs's walk."""
    src = os.path.join(ROOT, "tests", "native", "pairs_check.cpp")
    exe = str(tmp_path / "pairs_check")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined", "-I",
                    os.path.join(ROOT, "coverm_b200", "csrc"), src, "-o", exe], check=True)
    p = subprocess.run([exe], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    m = re.search(r"\b(\d+) tests, 0 fails \((\d+) declined, (\d+) of them for order; (\d+) nm panics\)", p.stdout)
    assert m, p.stdout
    tests, declined, order, nm = map(int, m.groups())
    assert tests > 8000 and declined - order < tests // 10 and tests - declined - nm > tests // 3, p.stdout  # most streams are checked whole


@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("case", list(CASES))
def test_reference_matches_oracle(bams, case, setting):
    """pair_reference.py against the oracle: filter-names in both modes, the read counts of `contig`, and the nm() panic."""
    _, recs = pr.read_bam(bams[case])
    flags, p = SETTINGS[setting][0], params(setting)
    for inverse in (False, True):
        o = _oracle(["filter-names", "-b", bams[case], "--proper-pairs-only"] + flags + (["--inverse"] if inverse else []))
        emitted, panicked = pr.run(recs, p, not inverse)
        assert (o.returncode != 0) == panicked, o.stderr[-500:]
        if panicked:
            assert pr.NM_PANIC in o.stderr
        else:
            assert o.stdout.split("\n")[:-1] == [recs[i].name for i in emitted]
    o = _oracle(["contig", "-m", "count", "-b", bams[case], "--proper-pairs-only"] + flags)
    want = pr.contig_read_counts(recs, p, len(CONTIGS))
    assert (o.returncode != 0) == (want is None), o.stderr[-500:]
    if want is not None:
        assert _counts(o.stdout) == want


def test_cases_pin_what_they_claim(bams):
    p = params("len1")
    _, recs = pr.read_bam(bams["split_by_other_contig"])
    assert pr.run(recs, p, True)[0] == [6, 7]  # only V pairs
    _, recs = pr.read_bam(bams["unmapped_proper_first"])
    assert pr.run(recs, params("len500"), False)[0] == [0, 1, 2, 3, 4]  # flags 71, 139, 131 in file order, then Q
    assert pr.run(recs, p, True)[0] == [0, 1, 3, 4]
    _, recs = pr.read_bam(bams["three_and_four_of_a_name"])
    assert pr.run(recs, p, True)[0] == [0, 1, 3, 4, 5, 6]
    _, recs = pr.read_bam(bams["missing_nm"])
    assert pr.run(recs, p, True)[1]


# ---------------------------------------------------------------------------------------------- GPU
def _product(argv, env=None):
    import coverm_b200
    return subprocess.run([coverm_b200.COVERM_BIN] + argv, capture_output=True, text=True, timeout=300,
                          env=dict(os.environ, **(env or {})))


COVERAGE = [["contig", "-m", "count", "mean", "covered_bases"], ["genome", "-s", "~", "-m", "count", "mean", "--min-covered-fraction", "0"]]


@pytest.mark.gpu
@pytest.mark.parametrize("setting", ["len1", "len150_mapq20", "ident_pct"])
@pytest.mark.parametrize("case", list(CASES))
def test_coverage_on_the_device(bams, case, setting):
    """`contig` and `genome` with pair thresholds: table text and #reads_mapped as the oracle, contig read counts as the
    reference; the device decoder keeps the sample unless the case declines, and the host decode path agrees."""
    _, recs = pr.read_bam(bams[case])
    flags = ["--proper-pairs-only"] + SETTINGS[setting][0] + ["-b", bams[case], "-t", "4", "--print-reads-mapped"]
    rm = lambda p: [l for l in p.stderr.splitlines() if l.startswith("#reads_mapped")]
    for cmd in COVERAGE:
        o = _oracle(cmd + flags)
        for env in ({"CMB_PIPELINE_STATS": "1"}, {"CMB_HOST_DECODE": "1"}):
            g = _product(cmd + flags, env)
            assert g.returncode == o.returncode, f"{env}: exit {g.returncode} vs oracle {o.returncode}\n{g.stderr[-1500:]}"
            if o.returncode:
                assert pr.NM_PANIC in o.stderr and pr.NM_PANIC in g.stderr, g.stderr[-800:]
                continue
            assert g.stdout == o.stdout, env
            assert rm(g) == rm(o), env
            if "CMB_PIPELINE_STATS" in env:
                lines = g.stderr.splitlines()
                if case in DECLINED:
                    assert any(l.startswith("#device_decode\tdeclined") and "mate matching gave up" in l for l in lines), lines[-8:]
                else:
                    assert any(l.startswith("#device_decode\tblocks=") for l in lines), lines[-8:]
        if cmd[0] == "contig" and not o.returncode:
            assert _counts(o.stdout) == pr.contig_read_counts(recs, params(setting), len(CONTIGS))


@pytest.mark.gpu
@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("case", list(CASES))
def test_filter_on_the_device(bams, tmp_path, case, setting):
    """`coverm filter` with and without --inverse: the records written are the reference's, byte for byte and in its order,
    and their names are the oracle's; on the device unless the case declines, and the host loop writes the same."""
    header, recs = pr.read_bam(bams[case])
    for inverse in (False, True):
        flt = ["--proper-pairs-only"] + SETTINGS[setting][0] + (["--inverse"] if inverse else [])
        emitted, panicked = pr.run(recs, params(setting), not inverse)
        o = _oracle(["filter-names", "-b", bams[case]] + flt)
        assert (o.returncode != 0) == panicked
        envs = [{"CMB_PIPELINE_STATS": "1"}, {"CMB_HOST_DECODE": "1"}]
        if case == "many_blocks":
            envs.append({"CMB_DECODE_WINDOW_KB": "64"})
        for env in envs:
            out = str(tmp_path / f"out{inverse:d}.bam")
            g = _product(["filter", "-b", bams[case], "-o", out, "-t", "4", "--timing"] + flt, env)
            if panicked:
                assert g.returncode != 0 and pr.NM_PANIC in g.stderr, g.stderr[-800:]
                continue
            assert g.returncode == 0, g.stderr[-800:]
            on_device = "device=1" in g.stderr
            assert on_device == ("CMB_HOST_DECODE" not in env and case not in DECLINED), g.stderr[-800:]
            got_header, got = pr.read_bam(out)
            assert got_header == header
            assert [r.raw for r in got] == [recs[i].raw for i in emitted], (env, inverse)
            assert [r.name for r in got] == o.stdout.split("\n")[:-1]
