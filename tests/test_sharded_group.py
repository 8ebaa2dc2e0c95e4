"""`--sharded` input over a group of ranks: rank r decodes a contiguous run of whole shards and owns their contigs, the ranks
exchange every pair's scores (and shard 0's read-name hashes), and every rank reaches the winners and the errors the one-GPU
run reaches (cmb_shard_begin_range .. cmb_shard_finish_group).

CPU: the shard-run cut planner (tests/native/shard_run_cuts_check.cpp); gloo groups of 2, 3 and 5 ranks (5 > K: ranks without
shards) on the CPU emulator with the group entry points (tests/native/shard_group_emulator.cpp, built here), against the oracle
in every mode of tests/test_sharded.py and on the sharded goldens; every sharded error in a group of 2, including an earlier
error on rank 1's shard beside a later one on rank 0's; and a device library without the group entry points.
GPU (-m gpu): the same groups as processes on device 0 with the CUDA library (the host all-gather path) against the
one-process `coverm --sharded`, on errors, on the tie set, in block slices, and the stores' split over the ranks;
`coverm --sharded --gpus N` (NCCL) where N GPUs are present."""
import itertools
import json
import os
import re
import struct
import subprocess
import sys
import zlib

import pytest

import shard_sets
from case_runner import DATA, ROOT
from sharded_oracle import run_oracle
from test_gene_shards import GROUP_WORKER, _free_port, _n_gpus
from test_sharded import EXCLUDED_ONLY, GOLDENS, MODES, _argv, _excluded_only, _pair, _same_table, _write_shards, error_cases, modes

EMU_SRC = os.path.join(ROOT, "tests", "native", "shard_group_emulator.cpp")
CUTS_SRC = os.path.join(ROOT, "tests", "native", "shard_run_cuts_check.cpp")
EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")  # the plain emulator: no group entry points


@pytest.fixture(scope="module")
def group_emu_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("shard_group_emu") / "libshard_group_emulator.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-Wl,--exclude-libs,ALL",
                    "-o", so, EMU_SRC, os.path.join(ROOT, "coverm_b200", "csrc", "host", "host_api.cpp"), "-lz", "-lpthread"], check=True)
    return so


# ------------------------------------------------------------------------------------------------------------ cut planner
def _best_max(sizes, n):
    """the smallest possible largest run over every contiguous cut of `sizes` into n runs (brute force)"""
    K = len(sizes)
    best = None
    for inner in itertools.combinations_with_replacement(range(K + 1), n - 1):
        cuts = [0] + list(inner) + [K]
        m = max(sum(sizes[cuts[r]:cuts[r + 1]]) for r in range(n))
        best = m if best is None else min(best, m)
    return best


def test_shard_run_cuts(tmp_path):
    exe = str(tmp_path / "shard_run_cuts_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "coverm_b200", "csrc", "host"), "-I", os.path.join(ROOT, "include"),
                    CUTS_SRC, "-o", exe], check=True)
    import random
    rng = random.Random(7)
    cases = [([5], 1), ([5], 3), ([10, 1, 1], 2), ([10, 1, 1], 3), ([1, 1, 1, 1], 2), ([3, 3, 3], 5), ([7, 2, 9, 4, 4], 3)]
    cases += [([rng.randint(1, 1000) for _ in range(rng.randint(1, 7))], rng.randint(1, 6)) for _ in range(150)]
    for sizes, n in cases:
        r = subprocess.run([exe, str(n)] + [str(x) for x in sizes], capture_output=True, text=True, check=True)
        cuts = [int(x) for x in r.stdout.split()]
        K = len(sizes)
        assert len(cuts) == n + 1 and cuts[0] == 0 and cuts[-1] == K, (sizes, n, cuts)
        assert all(a <= b for a, b in zip(cuts, cuts[1:])), (sizes, n, cuts)
        runs = [sum(sizes[cuts[r]:cuts[r + 1]]) for r in range(n)]
        assert max(runs) == _best_max(sizes, n), (sizes, n, cuts)
        used = [cuts[r + 1] > cuts[r] for r in range(n)]
        assert used == sorted(used, reverse=True), (sizes, n, cuts)  # ranks without shards come last
        if n >= K:
            assert sum(used) <= K


# ------------------------------------------------------------------------------------------------------------ groups
def _run_group(tmp_path, world, runs, lib_path, env=None):
    """`world` gloo processes running `runs` as one group; per rank the worker's results, and each process's stderr"""
    script = tmp_path / "shard_group_worker.py"
    script.write_text(GROUP_WORKER)
    port = str(_free_port())
    e = dict(os.environ, **(env or {}))
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, str(r), str(world), port, lib_path, json.dumps(runs)],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=e) for r in range(world)]
    outs = [p.communicate(timeout=1800) for p in procs]
    for p, (o, er) in zip(procs, outs):
        assert p.returncode == 0, er[-3000:]
    return [json.loads(o.strip().splitlines()[-1]) for o, _ in outs], [er for _, er in outs]


def _inflate(path):
    raw, out, o = open(path, "rb").read(), bytearray(), 0
    while o < len(raw):
        bsize = struct.unpack_from("<H", raw, o + 16)[0] + 1
        out += zlib.decompress(raw[o + 18:o + bsize - 8], -15)
        o += bsize
    return bytes(out)


def _n_targets(path):
    data = _inflate(path)
    return struct.unpack_from("<I", data, 8 + struct.unpack_from("<I", data, 4)[0])[0]


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    out = {}
    for K, n, seed in ((2, 1500, 11), (3, 1200, 12), (4, 900, 13)):
        out[K] = shard_sets.rich_set(str(tmp_path_factory.mktemp(f"group{K}")), K, n, seed)
    return out


@pytest.fixture(scope="module")
def genome3_list(tmp_path_factory):
    p = tmp_path_factory.mktemp("excl") / "genome3.txt"
    p.write_text("genome3\n")
    return str(p)


def _runs(sets, genome3_list):
    """(mode, argv, shard paths): every mode on every synthetic set, and the goldens"""
    runs = [(mode, modes(sets[K])[mode], sets[K]["shards"]) for K in (2, 3, 4) for mode in MODES]
    for name in GOLDENS:
        argv = _argv(name, genome3_list)
        runs.append((name, argv, [a for a in argv if a.endswith(".bam")]))
    return runs


def _reads_mapped(err):
    return [l.split("\t")[2:] for l in err.splitlines() if l.startswith("#reads_mapped")]


def _check_group(res, runs, world, want):
    """every rank's table and #reads_mapped against want[i] = (status, stdout, reads_mapped); the ranks' contig ranges cut the
    concatenated header exactly at shard boundaries"""
    for i, (mode, argv, shards) in enumerate(runs):
        status, out, rm = want[i]
        bounds = list(itertools.accumulate([0] + [_n_targets(p) for p in shards]))
        for r in range(world):
            got = res[r][i]
            assert got["status"] == status == 0, (mode, r, got["err"])
            _same_table(got["out"], out, mode if mode in MODES else "")
            assert [l.split("\t")[2:] for l in got["rm"]] == rm, (mode, r)
            assert got["ranks"] == world
        ranges = [(res[r][i]["tid_begin"], res[r][i]["tid_end"]) for r in range(world)]
        assert ranges[0][0] == 0 and ranges[-1][1] == bounds[-1], (mode, ranges)
        assert all(ranges[r][1] == ranges[r + 1][0] for r in range(world - 1)), (mode, ranges)
        assert all(b in bounds and e in bounds for b, e in ranges), (mode, ranges, bounds)


def _oracle_wants(runs):
    wants = []
    for _, argv, _ in runs:
        o = run_oracle(argv + ["--print-reads-mapped"])
        wants.append((o.returncode, o.stdout, _reads_mapped(o.stderr)))
    return wants


@pytest.mark.parametrize("world", [2, 3, 5])
def test_group_matches_the_oracle_emulator(tmp_path, sets, genome3_list, group_emu_lib, world):
    runs = _runs(sets, genome3_list)
    res, _ = _run_group(tmp_path, world, [a for _, a, _ in runs], group_emu_lib)
    _check_group(res, runs, world, _oracle_wants(runs))


def _error_inputs(tmp_path):
    """every sharded error case: (name, argv, status, message); `earlier_on_rank1`: shard 1 (rank 1's) fails at pair 1, shard 0
    (rank 0's) only at pair 2 -- the reference meets shard 1's error first"""
    out = []
    for case, (per_shard, status, msg) in error_cases().items():
        d = tmp_path / case
        d.mkdir()
        out.append((case, ["contig", "--sharded", "-b"] + _write_shards(str(d), per_shard), status, msg))
    d = tmp_path / "excluded_only"
    d.mkdir()
    out.append(("excluded_only", _excluded_only(d), 1, EXCLUDED_ONLY))
    d = tmp_path / "earlier_on_rank1"
    d.mkdir()
    ok = lambda i: _pair("r%d" % i)
    shards = _write_shards(str(d), [ok(0) + ok(1) + _pair("r2", as2=None), ok(0) + _pair("r1", as1=("AS", "i", 7)) + ok(2)])
    out.append(("earlier_on_rank1", ["contig", "--sharded", "-b"] + shards, 101, "Unexpected data type of AS aux tag"))
    return out


def _check_errors(res, cases, world, one):
    for i, (case, argv, status, msg) in enumerate(cases):
        assert one[i].returncode == status and msg in one[i].stderr, (case, one[i].stderr)
        for r in range(world):
            got = res[r][i]
            assert got["status"] == status, (case, r, got["err"])
            assert msg in got["err"], (case, r, got["err"])


def test_errors_in_a_group_emulator(tmp_path, group_emu_lib):
    cases = _error_inputs(tmp_path)
    res, _ = _run_group(tmp_path, 2, [a for _, a, _, _ in cases], group_emu_lib)
    _check_errors(res, cases, 2, [run_oracle(a) for _, a, _, _ in cases])


def test_group_needs_the_entry_points(tmp_path, sets):
    """the plain emulator lacks the group entry points: a group --sharded run stops on every rank; the same group still runs
    without --sharded"""
    if not os.path.exists(EMU_LIB):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    runs = [["contig", "-m", "mean", "--sharded", "-b"] + sets[2]["shards"], ["contig", "-m", "mean", "-b", DATA + "/7seqs.reads_for_seq1_and_seq2.bam"]]
    res, _ = _run_group(tmp_path, 2, runs, EMU_LIB)
    o = run_oracle(runs[1] + ["--print-reads-mapped"])
    for r in range(2):
        assert res[r][0]["status"] == 1 and "cmb_shard_begin_range" in res[r][0]["err"], res[r][0]
        assert res[r][1]["status"] == o.returncode == 0 and res[r][1]["out"] == o.stdout


# ------------------------------------------------------------------------------------------------------------ GPU
def _product(argv, env=None, timeout=900):
    import coverm_b200
    return subprocess.run([coverm_b200.COVERM_BIN] + argv, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **(env or {})))


def _product_wants(runs, env=None):
    wants = []
    for _, argv, _ in runs:
        p = _product(argv + ["--print-reads-mapped"], env)
        wants.append((p.returncode, p.stdout, _reads_mapped(p.stderr)))
    return wants


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_group_matches_one_process_gpu(tmp_path, sets, genome3_list, world):
    """`world` processes on device 0 with the CUDA library (scores exchanged through the host all-gather)"""
    import coverm_b200
    runs = _runs(sets, genome3_list)
    res, _ = _run_group(tmp_path, world, [a for _, a, _ in runs], coverm_b200.LIB_PATH)
    _check_group(res, runs, world, _product_wants(runs))
    cases = _error_inputs(tmp_path)
    res, _ = _run_group(tmp_path, world, [a for _, a, _, _ in cases], coverm_b200.LIB_PATH)
    _check_errors(res, cases, world, [_product(a) for _, a, _, _ in cases])


@pytest.mark.gpu
def test_group_ties_gpu(tmp_path):
    """200 000 pairs tied in both shards: ks_choose over the exchanged columns picks the winners ks_pairs picks on one GPU"""
    import numpy as np
    import bam_writer as bw
    import coverm_b200
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
    argv = ["contig", "--sharded", "-m", "count", "mean", "-b"] + shards
    one = _product(argv)
    assert one.returncode == 0, one.stderr
    res, _ = _run_group(tmp_path, 2, [argv], coverm_b200.LIB_PATH)
    for r in range(2):
        assert res[r][0]["status"] == 0 and res[r][0]["out"] == one.stdout, (r, res[r][0]["err"])


@pytest.mark.gpu
def test_group_in_slices_gpu(tmp_path):
    """test_sharded_slices.py's small-block sets, with room for a few slices of each rank's later shards"""
    import coverm_b200
    from test_sharded_slices import reblock, sliced_limit
    for K, n, seed in ((3, 1000, 22), (4, 700, 23)):
        d = tmp_path / f"slices{K}"
        d.mkdir()
        s = shard_sets.rich_set(str(d), K, n, seed)
        s["shards"] = [reblock(p, p[:-4] + ".small.bam") for p in s["shards"]]
        runs = [(mode, modes(s)[mode], s["shards"]) for mode in ("contig_mean", "genome_sep_excl")]
        whole = _product(runs[0][1], {"CMB_PIPELINE_STATS": "1"})
        assert whole.returncode == 0, whole.stderr[-2000:]
        env = {"CMB_DECODE_MEM_LIMIT_MB": sliced_limit(whole, s["shards"], parts=8), "CMB_PIPELINE_STATS": "1"}
        res, errs = _run_group(tmp_path, 2, [a for _, a, _ in runs], coverm_b200.LIB_PATH, env=env)
        _check_group(res, runs, 2, _product_wants(runs))
        sl = [int(x) for e in errs for x in re.findall(r"^#shard_slices\tshard=\d+\tslices=(\d+)", e, re.M)]
        assert sl and max(sl) > 1, (K, errs[0][-1500:], errs[1][-1500:])


@pytest.mark.gpu
def test_group_splits_the_stores_gpu(tmp_path):
    """K = 4 over 2 processes: each rank holds about half the stores of the one-process run"""
    import coverm_b200
    s = shard_sets.big_set(str(tmp_path), 4, 200_000, seed=9)
    argv = ["contig", "-m", "mean", "--sharded", "-b"] + s
    one = _product(argv, {"CMB_PIPELINE_STATS": "1"})
    assert one.returncode == 0, one.stderr[-2000:]
    store = lambda err: [int(x) for x in re.findall(r"^#reference_bytes\tshards=\d+\tshard_store=(\d+)$", err, re.M)]
    whole = store(one.stderr)[0]
    res, errs = _run_group(tmp_path, 2, [argv], coverm_b200.LIB_PATH, env={"CMB_PIPELINE_STATS": "1"})
    for r in range(2):
        assert res[r][0]["status"] == 0 and res[r][0]["out"] == one.stdout, (r, res[r][0]["err"])
        got = store(errs[r])
        assert len(got) == 1 and got[0] < 0.75 * whole, (r, got, whole)
        assert re.search(r"^#shard_exchange\tbytes=\d+\tms=", errs[r], re.M), errs[r][-2000:]


@pytest.mark.gpu
@pytest.mark.parametrize("gpus", [2, 4])
def test_coverm_sharded_gpus(sets, genome3_list, gpus):
    """`coverm --sharded --gpus N`: the scores exchanged over NCCL"""
    if _n_gpus() < gpus:
        pytest.skip(f"needs {gpus} GPUs, {_n_gpus()} present")
    for mode, argv, _ in _runs(sets, genome3_list):
        args = argv + ["-t", "8", "--print-reads-mapped"]
        one, many = _product(args), _product(args + ["--gpus", str(gpus)])
        assert one.returncode == many.returncode == 0, (mode, many.stderr[-1500:])
        _same_table(many.stdout, one.stdout, mode if mode in MODES else "")
        assert _reads_mapped(many.stderr) == _reads_mapped(one.stderr), mode
