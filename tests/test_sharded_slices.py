"""`--sharded` input decoded in block slices (cmb_shard_add, coverm_b200/csrc/cmb_slices.hpp).

CPU: the slice planner's invariants on random block tables (tests/native/shard_slices_check.cpp).  GPU (-m gpu): with
CMB_DECODE_MEM_LIMIT_MB low enough that the shards after the first are decoded in many slices (the first, like a whole-shard
decode, takes all the room the limit leaves), `coverm` prints what the unsliced run and the
oracle print -- on the reference's goldens and on synthetic sets cut into small BGZF blocks, so that slice edges split pairs,
fall between a primary and its secondary or supplementary records and cut through records that straddle blocks -- raises every
sharded error from a late slice of a later shard as the oracle does, and fails clearly when the stores alone do not fit."""
import os
import re
import struct
import subprocess
import zlib

import pytest

import bam_writer as bw
import shard_sets
from case_runner import DATA, ROOT
from sharded_oracle import run_oracle
from test_sharded import EXCLUDED_ONLY, GOLDENS, _argv, _same_table, _write_shards, modes

SRC = os.path.join(ROOT, "tests", "native", "shard_slices_check.cpp")


def test_slice_plan_invariants(tmp_path):
    exe = str(tmp_path / "shard_slices_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "coverm_b200", "csrc"), SRC, "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("ok "), r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------- GPU
def _inflate(path):
    raw, out, o = open(path, "rb").read(), bytearray(), 0
    while o < len(raw):
        bsize = struct.unpack_from("<H", raw, o + 16)[0] + 1
        out += zlib.decompress(raw[o + 18:o + bsize - 8], -15)
        o += bsize
    return bytes(out)


def reblock(src, dst, block_sizes=(150, 900)):
    """the same BAM stream in small BGZF blocks of random size: many blocks, most records straddling one"""
    with open(dst, "wb") as f:
        f.write(bw.bgzf(_inflate(src), level=1, block_sizes=block_sizes, seed=len(dst)))
    return dst


def _product(argv, env=None, timeout=900):
    import coverm_b200
    return subprocess.run([coverm_b200.COVERM_BIN] + argv, capture_output=True, text=True, timeout=timeout,
                          env=dict(os.environ, CMB_PIPELINE_STATS="1", **(env or {})))


def slices(p):
    """slices per shard from the #shard_slices lines"""
    return [int(m.group(1)) for m in re.finditer(r"^#shard_slices\tshard=\d+\tslices=(\d+)\tmax_slice_bytes=\d+\t", p.stderr, re.M)]


def sliced_limit(whole, shards, parts=4):
    """CMB_DECODE_MEM_LIMIT_MB for room for what the unsliced run's stores held and a `parts`-th of the largest shard's decode
    (its compressed and inflated bytes)"""
    m = re.search(r"^#reference_bytes\tshards=\d+\tshard_store=(\d+)$", whole.stderr, re.M)
    assert m, whole.stderr[-2000:]
    decode = max(os.path.getsize(p) + len(_inflate(p)) for p in shards)
    return "%.6f" % ((int(m.group(1)) + decode / parts) / 1048576)


def _reads_mapped(p):
    return [l.split("\t")[2:] for l in p.stderr.splitlines() if l.startswith("#reads_mapped")]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GOLDENS))
def test_goldens_in_slices(name, tmp_path):
    ex = tmp_path / "genome3.txt"
    ex.write_text("genome3\n")
    d = tmp_path / "small"
    d.mkdir()
    argv = _argv(name, str(ex))
    for src in (os.path.join(DATA, "shard1.bam"), os.path.join(DATA, "shard2.bam")):
        argv[argv.index(src)] = reblock(src, str(d / os.path.basename(src)), 200)
    whole = _product(argv)
    assert whole.returncode == 0, whole.stderr[-2000:]
    p = _product(argv, {"CMB_DECODE_MEM_LIMIT_MB": sliced_limit(whole, argv[argv.index("-b") + 1:argv.index("-b") + 3])})
    assert p.returncode == 0, p.stderr[-2000:]
    assert p.stdout == GOLDENS[name][1]
    assert len(slices(p)) == 2 and slices(p)[1] > 1, p.stderr[-2000:]


@pytest.fixture(scope="module")
def small_sets(tmp_path_factory):
    out = {}
    for K, n, seed in ((2, 1500, 21), (3, 1000, 22), (4, 700, 23)):
        d = tmp_path_factory.mktemp(f"slices{K}")
        s = shard_sets.rich_set(str(d), K, n, seed)
        s["shards"] = [reblock(p, p[:-4] + ".small.bam") for p in s["shards"]]
        out[K] = s
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 3, 4])
def test_synthetic_sets_in_slices(small_sets, K):
    for mode, argv in modes(small_sets[K]).items():
        argv = argv + ["--print-reads-mapped", "-t", "4"]
        o = run_oracle(argv)
        whole = _product(argv)
        sliced = _product(argv, {"CMB_DECODE_MEM_LIMIT_MB": sliced_limit(whole, small_sets[K]["shards"])})
        assert o.returncode == 0, o.stderr
        for g in (whole, sliced):
            assert g.returncode == 0, (mode, g.stderr[-2000:])
            _same_table(g.stdout, o.stdout, mode)
            assert _reads_mapped(g) == _reads_mapped(o), mode
        assert sliced.stdout == whole.stdout or mode == "contig_anir", mode
        assert slices(whole) == [1] * K, whole.stderr[-2000:]
        assert len(slices(sliced)) == K and min(slices(sliced)[1:]) > 1, sliced.stderr[-2000:]


def long_read_set(d, K=2, n_pairs=600, seed=31):
    """pairs of 3 kb mates, a few of 100 kb (longer than a slice's first tail), in small blocks: stores far smaller than the decode"""
    import random
    rng = random.Random(seed)
    recs = [[] for _ in range(K)]
    for i in range(n_pairs):
        for k in range(K):
            for m in range(2):
                rl = 100_000 if i % 97 == 13 and m == 1 else 3000
                flag = 0x1 | 0x2 | (0x40 if m == 0 else 0x80)
                recs[k].append(bw.record(0, rng.randrange(0, 150_000), [("M", rl)], flag=flag, qname="L%06d" % i,
                                         tags=[("NM", "C", rng.randint(0, 9)), ("AS", "S", rng.randint(100, 400))]))
    paths = []
    for k in range(K):
        p = os.path.join(d, f"long{k}.bam")
        with open(p, "wb") as f:
            f.write(bw.bgzf(bw.bam_stream([(f"s{k}g0~c0", 300_000)], recs[k], text="@HD\tVN:1.6\tSO:queryname\n"), level=1,
                            block_sizes=(4000, 20000), seed=seed + k))
        paths.append(p)
    return paths


@pytest.mark.gpu
def test_many_slices_and_long_records(tmp_path):
    shards = long_read_set(str(tmp_path))
    argv = ["contig", "-m", "mean", "count", "variance", "--sharded", "-b"] + shards + ["--print-reads-mapped"]
    o = run_oracle(argv)
    assert o.returncode == 0, o.stderr
    whole = _product(argv)
    sliced = _product(argv, {"CMB_DECODE_MEM_LIMIT_MB": sliced_limit(whole, shards, 20)})
    for g in (whole, sliced):
        assert g.returncode == 0, g.stderr[-2000:]
        assert g.stdout == o.stdout
        assert _reads_mapped(g) == _reads_mapped(o)
    assert max(slices(sliced)) >= 10, sliced.stderr[-2000:]


@pytest.mark.gpu
def test_ties_in_slices(tmp_path):
    """the tie set of test_ties_are_deterministic_and_uniform: the same bytes sliced and whole"""
    import numpy as np
    n = 200_000
    shards = []
    for k in range(2):
        names = np.repeat(np.arange(n, dtype=np.int64), 2)
        pos = np.tile(np.array([100, 300], np.int32), n)
        flag = np.tile(np.array([0x43, 0x83], np.uint16), n)
        body = shard_sets.big_records(np.zeros(2 * n, np.int32), pos, flag, names, np.full(2 * n, 50, np.uint8), np.ones(2 * n, np.uint8), 100)
        p = str(tmp_path / f"tie{k}.bam")
        with open(p, "wb") as f:
            f.write(bw.bgzf(bw.bam_stream([(f"k{k}~c", 100000)], [], text="@HD\tVN:1.6\n") + body, level=1))
        shards.append(p)
    argv = ["contig", "--sharded", "-m", "count", "-b"] + shards
    whole = _product(argv)
    # the stores' need by the library's accounting (2 x 45 B per primary, 5 B of AS scratch, 16 B of name hash and pair state,
    # 60 B per sorted winner with its one interval slot) and an eighth of a shard's decode: stores' slack would give one slice
    need = 2 * n * (2 * 45 + 5 + 16 + 60)
    decode = os.path.getsize(shards[0]) + len(_inflate(shards[0]))
    sliced = _product(argv, {"CMB_DECODE_MEM_LIMIT_MB": "%.6f" % ((need + decode / 8) / 1048576)})
    assert whole.returncode == 0 and sliced.returncode == 0, sliced.stderr[-2000:]
    assert sliced.stdout == whole.stdout
    assert slices(sliced)[1] > 1, sliced.stderr[-2000:]


def _long_pair(name, as1=("AS", "C", 50), as2=("AS", "C", 50), nm=("NM", "C", 1), flag1=0x43, flag2=0x83):
    """_pair with 1 kb mates"""
    t1 = [t for t in (nm, as1) if t]
    t2 = [t for t in (nm, as2) if t]
    return [bw.record(0, 100, [("M", 1000)], flag=flag1, qname=name, tags=t1), bw.record(0, 300, [("M", 1000)], flag=flag2, qname=name, tags=t2)]


def late_error_cases():
    """each error in pair 950 of 1000 of the last shard (EXCLUDED_ONLY: every pair)"""
    _pair = _long_pair
    ok = lambda i: _pair("r%d" % i)
    head = [r for i in range(950) for r in ok(i)]
    tail = [r for i in range(951, 1000) for r in ok(i)]
    good = head + ok(950) + tail
    return {
        "names_differ": ([good, head + _pair("x950") + tail], 1, "BAM files do not appear to be properly sorted by read name"),
        "unequal_lengths": ([good, head], 1, "Unexpectedly one BAM file input finished while another had further reads"),
        "odd_primaries": ([good + ok(1000)[:1], good + ok(1000)[:1]], 101, "Unexpectedly was able to read a first read set, but not a second"),
        "unpaired": ([good, head + _pair("r950", flag1=0x40) + tail], 1, "This code can only handle paired-end input"),
        "missing_as": ([good, head + _pair("r950", as2=None) + tail], 101, "does not have an 'AS' auxiliary tag"),
        "as_type_i": ([good, head + _pair("r950", as1=("AS", "i", 7)) + tail], 101, "Unexpected data type of AS aux tag"),
        "nm_type_s": ([good, head + _pair("r950", nm=("NM", "S", 1), as1=("AS", "C", 90)) + tail], 101, "Unexpected data type of NM aux tag"),
        "excluded_only": ([good, good], 1, EXCLUDED_ONLY),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(late_error_cases()))
def test_errors_from_a_late_slice(tmp_path, case):
    per_shard, status, msg = late_error_cases()[case]
    shards = [reblock(p, p[:-4] + ".small.bam", (2000, 8000)) for p in _write_shards(str(tmp_path), per_shard)]
    argv = ["contig", "--sharded", "-b"] + shards
    if case == "excluded_only":
        ex = tmp_path / "ex.txt"
        ex.write_text("k0a\nk1a\n")
        argv = ["genome", "-s", "~", "--sharded", "--exclude-genomes-from-deshard", str(ex), "-b"] + shards
    o = run_oracle(argv)
    assert o.returncode == status and msg in o.stderr, o.stderr
    p = _product(argv, {"CMB_DECODE_MEM_LIMIT_MB": "1"})
    assert p.returncode == status, p.stderr[-2000:]
    assert msg in p.stderr, p.stderr[-2000:]
    if len(slices(p)) == 2:  # errors found by the kernels are raised once every shard is in
        assert slices(p)[1] > 1, p.stderr[-2000:]


@pytest.mark.gpu
def test_limit_below_the_stores_fails_clearly(small_sets):
    argv = ["contig", "--sharded", "-b"] + small_sets[2]["shards"]
    p = _product(argv, {"CMB_DECODE_MEM_LIMIT_MB": "0.05"})
    assert p.returncode == 1, p.stderr[-2000:]
    m = re.search(r"sharded input needs (\d+) bytes of device memory for its shard stores, pair state, name hashes, AS scratch and "
                  r"sorted winners; the device has (\d+) bytes free for them", p.stderr)
    assert m and int(m.group(1)) > int(m.group(2)) == int(0.05 * 1048576), p.stderr[-2000:]
