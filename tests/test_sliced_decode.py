"""The ordinary device decode in block slices (cmb_submit_bgzf when the whole-stream buffers do not fit;
coverm_b200/csrc/cmb_slices.hpp).

CPU: the pair-mode cut and the slice budget against a brute-force walk (tests/native/decode_slices_check.cpp).  GPU (-m gpu):
with CMB_DECODE_MEM_LIMIT_MB low enough for four or more slices, `coverm` prints what the unlimited run and the oracle print,
decodes every sample on the device (a `#decode_slices` line, no host `#pipeline` line), and a sample that declines in a late
slice -- a corrupted block, a malformed record, unsorted proper pairs, one reference's proper pairs larger than a slice --
ends as the host route ends it."""
import json
import os
import re
import struct
import subprocess
import sys
import zlib

import pytest

import bam_writer as bw
import coverm_b200
from case_runner import ORACLE_BIN, ROOT
from test_genes import bam_header, write_gff
from test_multirank_gloo import GROUP_WORKER, _free_port
from test_gpu_multi import _n_gpus

SRC = os.path.join(ROOT, "tests", "native", "decode_slices_check.cpp")


def test_pair_cut_and_budget_rules(tmp_path):
    exe = str(tmp_path / "decode_slices_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "coverm_b200", "csrc"), SRC, "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("ok "), r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------- GPU
ALL_METHODS = ["mean", "trimmed_mean", "covered_fraction", "covered_bases", "variance", "length", "count",
               "reads_per_base", "rpkm", "tpm", "anir"]
MB = 1 << 20


def _inflate(path):
    raw, out, o = open(path, "rb").read(), bytearray(), 0
    while o < len(raw):
        bsize = struct.unpack_from("<H", raw, o + 16)[0] + 1
        out += zlib.decompress(raw[o + 18:o + bsize - 8], -15)
        o += bsize
    return bytes(out)


def _records_start(stream):
    """offset of the first alignment record of an inflated BAM stream"""
    l_text = struct.unpack_from("<i", stream, 4)[0]
    o = 8 + l_text
    n_ref = struct.unpack_from("<i", stream, o)[0]
    o += 4
    for _ in range(n_ref):
        l_name = struct.unpack_from("<i", stream, o)[0]
        o += 4 + l_name + 4
    return o


def _record_offsets(stream):
    offs, o = [], _records_start(stream)
    while o < len(stream):
        offs.append(o)
        o += 4 + struct.unpack_from("<i", stream, o)[0]
    return offs


def limit_for(path, slices=4):
    """CMB_DECODE_MEM_LIMIT_MB that gives at least `slices` slices: the first slice takes half the room, the others less than
    all of it"""
    whole = os.path.getsize(path) + len(_inflate(path))
    mb = max(64, whole // (slices * MB))
    assert whole > 2.5 * mb * MB, "the file is too small to be sliced with a limit of at least 64 MB"
    return str(mb)


def _run(argv, env=None, binary=None):
    return subprocess.run([binary or coverm_b200.COVERM_BIN] + argv + ["-t", "8", "--print-reads-mapped"], capture_output=True,
                          text=True, timeout=1800, env=dict(os.environ, CMB_PIPELINE_STATS="1", **(env or {})))


def _oracle(argv):
    return subprocess.run([ORACLE_BIN] + argv + ["-t", "8", "--print-reads-mapped"], capture_output=True, text=True, timeout=1800)


def _reads_mapped(p):
    return [l for l in p.stderr.splitlines() if l.startswith("#reads_mapped")]


def _same_table(got, want, anir):
    """identical text, or (anir) identical but for the ANI columns, which agree to 1e-6"""
    if got == want:
        return
    assert anir, (got[:2000], want[:2000])
    gl, wl = got.splitlines(), want.splitlines()
    assert len(gl) == len(wl)
    for a, b in zip(gl, wl):
        for x, y in zip(a.split("\t"), b.split("\t")):
            if x == y:
                continue
            assert abs(float(x) - float(y)) <= 1e-6 * max(1.0, abs(float(y))), (a, b)


def decode_slices(p):
    m = re.search(r"^#decode_slices\tslices=(\d+)\tmax_slice_bytes=(\d+)\thalvings=(\d+)\tpair_cut_records=(\d+)$", p.stderr, re.M)
    return tuple(int(g) for g in m.groups()) if m else None


def _gen(d, name, *args):
    p = os.path.join(d, f"{name}.bam")
    subprocess.check_call([coverm_b200.BAMGEN_BIN, "--out", p, "--threads", "16"] + [str(a) for a in args], stdout=subprocess.DEVNULL)
    return p


def _reblock(src, dst, block_sizes):
    with open(dst, "wb") as f:
        f.write(bw.bgzf(_inflate(src), level=1, block_sizes=block_sizes, seed=7))
    return dst


def long_reads(path, n=2000):
    """100 kb reads (records of 150 kB, more than a slice's first tail), proper pairs over four contigs, in small blocks"""
    import random
    rng = random.Random(41)
    contigs = [(f"lc{k}", 2_000_000) for k in range(4)]
    recs = []
    per = n // 4
    for k in range(4):
        starts = sorted(rng.randrange(0, 1_800_000) for _ in range(per))
        for i, pos in enumerate(starts):
            recs.append(bw.record(k, pos, [("M", 100_000)], flag=0x1 | 0x2 | (0x40 if i % 2 == 0 else 0x80), qname="L%d_%d" % (k, i // 2),
                                  mtid=k, mpos=pos, tags=[("NM", "C", rng.randint(0, 50))]))
    with open(path, "wb") as f:
        f.write(bw.bgzf(bw.bam_stream(contigs, recs, text="@HD\tVN:1.6\tSO:coordinate\n"), level=1, block_sizes=(8000, 40000), seed=5))
    return path


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("sliced"))
    out = {
        "small": _gen(d, "small", "--contigs", 3000, "--reads", 1_200_000, "--seed", 61, "--median-len", 2500, "--min-len", 200, "--max-len", 60000),
        "long": _gen(d, "long", "--contigs", 12, "--reads", 1_000_000, "--seed", 62, "--median-len", 900000, "--sigma", 0.6, "--min-len", 50000,
                     "--max-len", 5000000),
        "mags": _gen(d, "mags", "--contigs", 2500, "--genomes", 60, "--reads", 1_000_000, "--seed", 63, "--median-len", 8000,
                     "--definition-out", os.path.join(d, "mags.tsv")),
        "one_ref": _gen(d, "one_ref", "--contigs", 1, "--reads", 1_000_000, "--seed", 64, "--median-len", 3000000, "--min-len", 3000000,
                        "--max-len", 3000000),
    }
    out["mags_def"] = os.path.join(d, "mags.tsv")
    out["reblocked"] = _reblock(out["small"], os.path.join(d, "small_reblocked.bam"), (600, 5000))
    out["long_reads"] = long_reads(os.path.join(d, "long_reads.bam"))
    gff = os.path.join(d, "small.gff")
    write_gff(gff, bam_header(out["small"]), 4000, seed=3)
    out["gff"] = gff
    return out


RUNS = [
    ("small", ["contig", "-m"] + ALL_METHODS),
    ("small", ["contig", "-m", "trimmed_mean", "mean"]),
    ("small", ["contig", "-m", "coverage_histogram"]),
    ("small", ["contig", "-m", "metabat"]),
    ("small", ["contig", "-m", "mean", "count", "--gff", "{gff}"]),
    ("small", ["contig", "-m", "mean", "trimmed_mean", "covered_fraction", "--min-read-percent-identity", "97", "--min-mapq", "20"]),
    ("small", ["contig", "-m", "mean", "variance", "--proper-pairs-only", "--min-read-aligned-length-pair", "250",
               "--min-read-percent-identity-pair", "95"]),
    ("long", ["contig", "-m"] + ALL_METHODS),
    ("mags", ["genome", "-s", "~", "-m", "relative_abundance", "mean", "trimmed_mean", "variance", "covered_fraction", "--min-covered-fraction", "0"]),
    ("mags", ["genome", "--genome-definition", "{mags_def}", "-m", "relative_abundance", "mean", "trimmed_mean", "--min-covered-fraction", "5"]),
    ("reblocked", ["contig", "-m", "mean", "count", "covered_bases"]),
    ("reblocked", ["contig", "-m", "mean", "count", "--proper-pairs-only", "--min-read-percent-identity-pair", "95"]),
    ("long_reads", ["contig", "-m", "mean", "count", "variance"]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("which,argv", RUNS, ids=[f"{w}:{' '.join(a[:5])}#{i}" for i, (w, a) in enumerate(RUNS)])
def test_sliced_equals_whole_and_oracle(inputs, which, argv):
    argv = [a.format(**inputs) for a in argv] + ["-b", inputs[which]]
    anir = "anir" in argv
    whole = _run(argv)
    sliced = _run(argv, {"CMB_DECODE_MEM_LIMIT_MB": limit_for(inputs[which])})
    o = _oracle(argv)
    assert o.returncode == 0, o.stderr[-2000:]
    for g in (whole, sliced):
        assert g.returncode == 0, g.stderr[-2000:]
        _same_table(g.stdout, o.stdout, anir)
        assert _reads_mapped(g) == _reads_mapped(o)
        assert not any(l.startswith("#pipeline") for l in g.stderr.splitlines()), g.stderr[-2000:]
    assert sliced.stdout == whole.stdout
    assert decode_slices(whole) is None
    s = decode_slices(sliced)
    assert s and s[0] >= 4, sliced.stderr[-2000:]
    if any(a.endswith("-pair") for a in argv):  # mates matched on the device: slices end before their last reference's run
        assert s[3] > 0, sliced.stderr[-2000:]


@pytest.mark.gpu
def test_one_reference_larger_than_a_slice_declines(inputs):
    argv = ["contig", "-m", "mean", "count", "--proper-pairs-only", "--min-read-aligned-length-pair", "100", "-b", inputs["one_ref"]]
    p = _run(argv, {"CMB_DECODE_MEM_LIMIT_MB": limit_for(inputs["one_ref"])})
    o = _oracle(argv)
    assert p.returncode == 0 == o.returncode, p.stderr[-2000:]
    assert p.stdout == o.stdout
    assert re.search(r"^#device_decode\tdeclined: .*proper-pair records of reference 0 do not fit in one decode slice", p.stderr, re.M), p.stderr[-2000:]
    assert decode_slices(p) is None


def _late_bad(inputs, d, kind):
    """the small file with a fault at 85 % of its records"""
    src = inputs["small"]
    if kind == "corrupt_block":
        raw = bytearray(open(src, "rb").read())
        o, blocks = 0, []
        while o < len(raw):
            bsize = struct.unpack_from("<H", raw, o + 16)[0] + 1
            blocks.append((o, bsize))
            o += bsize
        bo, bs = blocks[int(len(blocks) * 0.85)]
        for k in range(bo + 40, bo + bs - 20, 97):
            raw[k] ^= 0x5a
        p = os.path.join(d, "corrupt.bam")
        open(p, "wb").write(bytes(raw))
        return p
    stream = bytearray(_inflate(src))
    offs = _record_offsets(stream)
    if kind == "malformed_record":
        o = offs[int(len(offs) * 0.85)]
        struct.pack_into("<H", stream, o + 4 + 12, 0xffff)  # n_cigar_op: the CIGAR runs past the record's end
    else:  # unsorted: the last 40 % of the records before the rest
        start, cut = offs[0], offs[int(len(offs) * 0.6)]
        stream = stream[:start] + stream[cut:] + stream[start:cut]
    p = os.path.join(d, kind + ".bam")
    with open(p, "wb") as f:
        f.write(bw.bgzf(bytes(stream), level=1))
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("kind,pairs", [("corrupt_block", False), ("malformed_record", False), ("unsorted", True), ("unsorted", False)])
def test_late_slice_faults_end_like_the_host_route(inputs, tmp_path, kind, pairs):
    bam = _late_bad(inputs, str(tmp_path), kind)
    argv = ["contig", "-m", "mean", "count", "-b", bam] + (["--proper-pairs-only", "--min-read-percent-identity-pair", "95"] if pairs else [])
    p = _run(argv, {"CMB_DECODE_MEM_LIMIT_MB": limit_for(inputs["small"])})
    host = _run(argv, {"CMB_HOST_DECODE": "1"})
    o = _oracle(argv)
    assert p.returncode == o.returncode == host.returncode, (p.stderr[-2000:], o.stderr[-2000:])
    assert p.stdout == host.stdout
    last = lambda g: [l for l in g.stderr.splitlines() if l.strip() and not l.startswith("#")][-1:]
    assert last(p) == last(host), (last(p), last(host))
    if not o.returncode:
        assert p.stdout == o.stdout
    if kind != "unsorted" or pairs:  # declined in a late slice: the host decoded the sample again from its start
        assert any(l.startswith("#device_decode\tdeclined") for l in p.stderr.splitlines()), p.stderr[-2000:]


@pytest.mark.gpu
def test_group_of_two_processes_in_slices(inputs, tmp_path):
    """2 processes on one GPU in a cmbh_session_set_group group, each slicing its block range: the one-process whole run"""
    runs = [["contig", "-m", "mean", "trimmed_mean", "count", "-b", inputs["small"]],
            ["contig", "-m", "mean", "count", "--proper-pairs-only", "--min-read-percent-identity-pair", "95", "-b", inputs["small"]]]
    script = tmp_path / "group_worker.py"
    script.write_text(GROUP_WORKER)
    port = str(_free_port())
    env = dict(os.environ, CMB_PIPELINE_STATS="1", CMB_DECODE_MEM_LIMIT_MB=limit_for(inputs["small"], 8))
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, str(r), "2", port, coverm_b200.LIB_PATH, json.dumps(runs)],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env) for r in range(2)]
    outs = [p.communicate(timeout=1800) for p in procs]
    for p, (o, er) in zip(procs, outs):
        assert p.returncode == 0, er[-3000:]
        assert re.search(r"^#decode_slices\tslices=([4-9]|\d\d+)\t", er, re.M), er[-3000:]
    results = [json.loads(o.strip().splitlines()[-1]) for o, _ in outs]
    for i, argv in enumerate(runs):
        whole = _run(argv)
        assert whole.returncode == 0
        for r in results:
            assert r[i]["status"] == 0 and r[i]["device_decode"], r[i]
            assert r[i]["out"] == whole.stdout
            assert r[i]["rm"] == _reads_mapped(whole)


@pytest.mark.gpu
@pytest.mark.skipif(_n_gpus() < 2, reason="needs at least 2 GPUs")
def test_two_gpus_in_slices(inputs):
    argv = ["contig", "-m", "mean", "trimmed_mean", "count", "-b", inputs["small"]]
    whole = _run(argv)
    p = _run(argv + ["--gpus", "2"], {"CMB_DECODE_MEM_LIMIT_MB": limit_for(inputs["small"], 8)})
    assert p.returncode == 0 == whole.returncode, p.stderr[-2000:]
    assert p.stdout == whole.stdout
    assert decode_slices(p), p.stderr[-2000:]
