"""The host's BAM input (coverm_b200/csrc/host/bam_source.hpp) on the paths the device decode never takes, through the
test-only CPU emulator (oracle/coverm_hostcheck, oracle/libcoverm_hostcheck.so; the emulator declines device decode):
the host mate matching of `--proper-pairs-only` and of `coverm filter`, cut-short headers and records, a first mate left of
its contig, and one sample as BGZF, plain gzip, uncompressed BAM and SAM.  Everything is checked against the oracle."""
import ctypes as C
import gzip
import os
import subprocess

import numpy as np
import pytest

import bam_writer as bw
from case_runner import ORACLE_BIN, ROOT
from test_decode_edge_cases import METHODS, NAMES, _files

HOSTCHECK = os.path.join(ROOT, "oracle", "coverm_hostcheck")
EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")
CONTIGS = [("ctgA", 5000), ("ctgB", 30000), ("ctgC", 800)]


@pytest.fixture(scope="module", autouse=True)
def _hostcheck_built():
    if not (os.path.exists(HOSTCHECK) and os.path.exists(EMU_LIB)):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])


@pytest.fixture(scope="module")
def edge_files(tmp_path_factory):
    return _files(tmp_path_factory)


def _run(binary, argv, threads="3"):
    return subprocess.run([binary] + argv + ["-t", threads], capture_output=True, text=True, timeout=600)


def _same(a, o):
    """Status, then the table (or the returned names) and #reads_mapped lines."""
    assert a.returncode == o.returncode, (a.returncode, o.returncode, a.stderr[-400:], o.stderr[-300:])
    if o.returncode == 0:
        assert a.stdout == o.stdout
        rm = lambda p: [l for l in p.stderr.splitlines() if l.startswith("#reads_mapped")]
        assert rm(a) == rm(o)


PAIR_FILTER = ["--proper-pairs-only", "--min-read-aligned-length-pair", "30"]  # a pair threshold: the filter's mate-matching path


def _contig_pairs(path):
    return ["contig", "-m"] + METHODS + ["--min-covered-fraction", "0", "-b", path, "--print-reads-mapped"] + PAIR_FILTER


FILTERS = {"pairs": ["--proper-pairs-only", "--min-read-aligned-length-pair", "60"],
           "pairs_inverse": ["--proper-pairs-only", "--min-read-aligned-length-pair", "60", "--inverse"],
           "singles": ["--min-read-percent-identity", "97"],
           "singles_inverse": ["--min-read-percent-identity", "97", "--inverse"]}


@pytest.mark.parametrize("name", NAMES)
def test_edge_cases_through_the_host_pair_fallback(edge_files, name):
    _same(_run(HOSTCHECK, _contig_pairs(edge_files[name])), _run(ORACLE_BIN, _contig_pairs(edge_files[name])))


@pytest.mark.parametrize("mode", list(FILTERS))
@pytest.mark.parametrize("name", NAMES)
def test_edge_cases_through_the_host_filter_loop(edge_files, name, mode):
    argv = ["filter-names", "-b", edge_files[name]] + FILTERS[mode]
    _same(_run(HOSTCHECK, argv), _run(ORACLE_BIN, argv))


# ---- a small sample with real mate pairs, written in every input format the host reads
def _pairs(n, seed):
    """(qname, tid, pos, cigar, flag, mtid, mpos, nm) of n proper pairs and a few unpaired reads, sorted by position."""
    rng = np.random.default_rng(seed)
    recs = []
    for i in range(n):
        tid = int(rng.integers(len(CONTIGS)))
        L = CONTIGS[tid][1]
        a, b = sorted(int(x) for x in rng.integers(0, L - 200, 2))
        la, lb = int(rng.integers(40, 150)), int(rng.integers(40, 150))
        cig_b = [("M", lb)] if i % 3 else [("M", lb // 2), ("D", 2), ("M", lb - lb // 2)]
        recs.append(("p%05d" % i, tid, a, [("S", 3), ("M", la)], 99, tid, b, int(rng.integers(0, 4))))
        recs.append(("p%05d" % i, tid, b, cig_b, 147, tid, a, int(rng.integers(0, 4))))
        if i % 7 == 0:
            recs.append(("u%05d" % i, tid, a, [("M", 80)], 0, -1, -1, 1))
    recs.sort(key=lambda r: (r[1], r[2]))
    return recs


def _bam_records(recs):
    return [bw.record(t, p, cig, flag=f, qname=q, mtid=mt, mpos=mp, tags=[("NM", "C", nm)]) for q, t, p, cig, f, mt, mp, nm in recs]


def _sam(recs):
    lines = ["@HD\tVN:1.6\tSO:coordinate"] + [f"@SQ\tSN:{n}\tLN:{l}" for n, l in CONTIGS]
    for q, t, p, cig, f, mt, mp, nm in recs:
        l_seq = sum(n for c, n in cig if c in "MIS=X")
        mate = "*" if mt < 0 else ("=" if mt == t else CONTIGS[mt][0])
        lines.append("\t".join([q, str(f), CONTIGS[t][0], str(p + 1), "60", "".join(f"{n}{c}" for c, n in cig), mate, str(mp + 1), "0",
                                "A" * l_seq, "I" * l_seq, f"NM:i:{nm}"]))
    return ("\n".join(lines) + "\n").encode()


@pytest.fixture(scope="module")
def formats(tmp_path_factory):
    d = tmp_path_factory.mktemp("formats")
    recs = _pairs(1500, seed=3)
    stream = bw.bam_stream(CONTIGS, _bam_records(recs))
    out = {}
    for kind, data, ext in (("bgzf", bw.bgzf(stream, level=6, block_sizes=(300, 9000), seed=1), "bam"), ("gzip", gzip.compress(stream), "bam"),
                            ("raw", stream, "bam"), ("sam", _sam(recs), "sam")):
        os.mkdir(d / kind)
        out[kind] = str(d / kind / f"sample.{ext}")  # one file stem: the tables' column names agree
        with open(out[kind], "wb") as f:
            f.write(data)
    return out


def _extract(path):
    """cmbh_extract_tuples on the emulator build: the columns as numpy arrays, or None when it fails."""
    import coverm_b200
    lib = coverm_b200.load_library(EMU_LIB)
    t = coverm_b200.Tuples()
    if lib.cmbh_extract_tuples(path.encode(), None, 0, 3, C.byref(t)) != 0:
        return None
    n, ni = t.n_records, t.n_intervals
    cols = {"contig_len": np.ctypeslib.as_array(t.contig_len, (t.n_contigs,)).copy()}
    for name, cnt in (("tid", n), ("pos", n), ("flag", n), ("mapq", n), ("nm_state", n), ("nm", n), ("l_seq", n), ("aligned", n),
                      ("del_", n), ("ins", n), ("iv_begin", n + 1), ("iv_start", ni), ("iv_len", ni)):
        cols[name] = np.ctypeslib.as_array(getattr(t, name), (cnt,)).copy() if cnt else np.zeros(0)
    lib.cmbh_free_tuples(C.byref(t))
    return cols


@pytest.mark.parametrize("extra", [[], PAIR_FILTER], ids=["all", "pairs"])
def test_every_input_format_gives_the_same_table(formats, extra):
    argv = lambda p: ["contig", "-m", "mean", "covered_bases", "variance", "count", "-b", p, "--print-reads-mapped"] + extra
    want = _run(ORACLE_BIN, argv(formats["bgzf"]))
    assert want.returncode == 0 and want.stdout.count("\n") == len(CONTIGS) + 1
    for kind, path in formats.items():
        _same(_run(HOSTCHECK, argv(path)), want)


def test_every_input_format_gives_the_same_tuples(formats):
    want = _extract(formats["bgzf"])
    assert want is not None and want["tid"].size > 3000
    for kind in ("gzip", "raw", "sam"):
        got = _extract(formats[kind])
        assert got is not None, kind
        for col, a in want.items():
            np.testing.assert_array_equal(got[col], a, err_msg=f"{kind}: {col}")


def test_every_input_format_gives_the_same_filtered_names(formats):
    for mode in ("pairs", "singles_inverse"):
        want = _run(ORACLE_BIN, ["filter-names", "-b", formats["bgzf"]] + FILTERS[mode])
        assert want.returncode == 0 and want.stdout
        for path in formats.values():
            _same(_run(HOSTCHECK, ["filter-names", "-b", path] + FILTERS[mode]), want)


# ---- cut-short headers and records
@pytest.fixture(scope="module")
def cut_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("cut")
    header = bw.bam_stream(CONTIGS, [])
    recs = _bam_records(_pairs(40, seed=5))
    l_text = int.from_bytes(header[4:8], "little")
    cuts = {"in_l_text": header[:8 + l_text // 2],               # inside the @-text
            "in_reference_list": header[:len(header) - 6],     # inside the last reference entry
            "last_record": bw.bam_stream(CONTIGS, recs)[:-7]}  # header intact, the last record cut short
    out = {}
    for name, stream in cuts.items():
        out[name] = str(d / f"{name}.bam")
        with open(out[name], "wb") as f:
            f.write(bw.bgzf(stream, level=6))
    return out


@pytest.mark.parametrize("where", ["in_l_text", "in_reference_list"])
def test_cut_short_header_is_a_header_error(cut_files, tmp_path, where):
    path = cut_files[where]
    for argv in (["contig", "-m", "mean", "-b", path], ["filter", "-b", path, "-o", str(tmp_path / "out.bam")]):
        p = _run(HOSTCHECK, argv)
        assert p.returncode == 101 and "Error reading BAM header" in p.stderr, (argv, p.returncode, p.stderr[-300:])
    assert _extract(path) is None


def test_cut_short_last_record_fails_tuple_extraction(cut_files):
    assert _extract(cut_files["last_record"]) is None
    for argv in (["contig", "-m", "mean", "-b", cut_files["last_record"]], _contig_pairs(cut_files["last_record"])):
        _same(_run(HOSTCHECK, argv), _run(ORACLE_BIN, argv))
        assert _run(HOSTCHECK, argv).returncode == 101


def test_first_mate_left_of_its_contig_is_a_bounds_error_on_the_pair_fallback(tmp_path):
    """The host decoder clamps a block starting left of the contig to -1 as the device does, so K1 raises its bounds error
    instead of taking INT32_MIN for an unused interval slot."""
    recs = [bw.record(0, -2 ** 31, [("M", 50)], flag=99, qname="left", mtid=0, mpos=100),
            bw.record(0, 100, [("M", 50)], flag=147, qname="left", mtid=0, mpos=-2 ** 31)]
    path = str(tmp_path / "left.bam")
    with open(path, "wb") as f:
        f.write(bw.bgzf(bw.bam_stream(CONTIGS, recs), level=6))
    argv = _contig_pairs(path)
    o, a = _run(ORACLE_BIN, argv), _run(HOSTCHECK, argv)
    assert o.returncode == 101
    _same(a, o)


def test_unknown_aux_type_on_the_parallel_host_paths(tmp_path):
    """A decode error raised on a worker thread (the host pair fallback's and cmbh_extract_tuples' parallel decode) reaches
    the caller as the reference's panic instead of ending the process on the worker; the filter's serial loop agrees."""
    recs = _bam_records(_pairs(6000, seed=9))
    bad = bytearray(recs[9000]) + b"XXQ\0"  # 'Q' is no SAM aux type
    bad[0:4] = (len(bad) - 4).to_bytes(4, "little")
    recs[9000] = bytes(bad)
    path = str(tmp_path / "aux.bam")
    with open(path, "wb") as f:
        f.write(bw.bgzf(bw.bam_stream(CONTIGS, recs), level=6))
    for argv in (_contig_pairs(path), ["filter-names", "-b", path] + FILTERS["pairs"]):
        a, o = _run(HOSTCHECK, argv), _run(ORACLE_BIN, argv)
        assert a.returncode == o.returncode == 101 and "Error reading BAM record" in a.stderr, (argv, a.returncode, o.returncode, a.stderr[-300:])
    assert _extract(path) is None
