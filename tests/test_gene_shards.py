"""Per-gene coverage (`--gff`) over contig shards: several ranks each own a contig range, count only its records and hold only
its genes (cmb_set_genes_range), and one gather of the gene rows, `contig_seen` and `kept_primary` completes the sample.

* Device ABI: the same records on a whole-range gene context and on the shard contexts of several cut sets.  Each shard's
  gene rows must equal the whole run's in every integer field and histogram pair (the f64 identity sums to 1e-12 relative),
  its other rows must stay zero, the shards' contig_seen must OR and their kept_primary add up to the whole run's.  Every
  shard is given every record, so records of other ranks' contigs (the one-block overlap of ranged decode) must add nothing.
  On the CPU emulator with cmb_set_genes_range on top (tests/native/gene_range_emulator.cpp, built here) and, marked gpu, on
  the CUDA library.
* Group mode: gloo workers run tests/test_genes.py's runs with `--gff` as one group (the host all-gather callback); every
  rank's table and `#reads_mapped` must equal the oracle's.  On that emulator at 2, 3 and 8 ranks with ranged device decode
  and with host decode; marked gpu, 2 and 3 processes on device 0 with the real library.  A device library without
  cmb_set_genes_range (the plain emulator) stops such a run on every rank with an error.
* `coverm --gpus N --gff` (NCCL gather) against the oracle when N GPUs are present."""
import json
import os
import random
import socket
import subprocess
import sys

import numpy as np
import pytest

import coverm_b200
import device_reference as ref
import device_scenarios as ds
from case_runner import DATA, ORACLE_BIN, ROOT
from test_genes import RUNS, bam_header, write_gff

EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")
RANGE_EMU_SRC = os.path.join(ROOT, "tests", "native", "gene_range_emulator.cpp")


@pytest.fixture(scope="module")
def range_emu_lib(tmp_path_factory):
    """Path of the emulator with cmb_set_genes_range, linked with the product's host code like oracle/libcoverm_hostcheck.so."""
    so = str(tmp_path_factory.mktemp("gene_range_emu") / "libgene_range_emulator.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-Wl,--exclude-libs,ALL",
                    "-o", so, RANGE_EMU_SRC, os.path.join(ROOT, "coverm_b200", "csrc", "host", "host_api.cpp"), "-lz", "-lpthread"],
                   check=True)
    return so


# ------------------------------------------------------------------------------------------------------------ device ABI
LENS = [4000, 2500, 9000, 300, 1200, 8200, 700]
# contig 0's and 1's last genes end at the contig end (a GFF gene running past it is clamped there); contigs 2 and 4 carry none
GENES = [(0, 0, 100), (0, 50, 4000), (0, 3999, 4000), (1, 10, 2000), (1, 1500, 2500), (3, 0, 300), (5, 100, 8200), (5, 4000, 4100),
         (5, 8190, 8200), (6, 0, 5)]
CUT_SETS = {
    "cut_at_tid0": [0, 0, 7],
    "between_gene_contigs": [0, 1, 7],          # right after contig 0, whose genes run to its end; contig 1 carries genes too
    "after_contig_end_genes": [0, 2, 7],        # right after contig 1 (genes to its end), before contig 2 (no genes)
    "ranks_without_genes": [0, 2, 3, 4, 5, 7],  # [2, 3) and [4, 5) own contigs but no gene
    "rank_without_contigs": [0, 3, 3, 7],
    "all_genes_on_one_rank": [0, 7, 7],
    "eight_ranks": [0, 0, 1, 1, 3, 5, 5, 6, 7],
}


def seg_cut(first, n_seg, t):
    """cmb_set_genes_range's row bound of contig cut t."""
    return n_seg if t == len(first) - 1 else first[t]


def _records(seed):
    rng = random.Random(seed)
    recs = ds.Records()
    for t, L in enumerate(LENS):
        ds._reads(rng, recs, t, L, 120, pads=True)
    recs.add(0, 3990, 10).add(1, 2490, 200).add(5, 8185, 30).add(2, 0, 9000)
    return recs.columns()


def _samples():
    cols = _records(61)
    filt = ref.default_params(filtering=1, min_mapq=20, min_percent_identity_single=0.9, include_secondary=1)
    return [(cols, ref.default_params()), (cols, ref.default_params(contig_end_exclusion=3, trim_min=0.1, trim_max=0.9)), (cols, filt)]


def _run(lib, genes, tid_range, cols, p):
    ctx = coverm_b200.DeviceContext(lib=lib, batch_records=700)  # several batches
    try:
        if tid_range is None:
            ctx.set_genes(LENS, genes)
        else:
            ctx.set_genes(LENS, genes, *tid_range)
        ctx.set_params(ds.to_params(p))
        ctx.begin_sample()
        ctx.submit_columns(cols)
        rows, pairs = ctx.end_sample(want_pairs=True)
        seen, kept = ctx.fetch_gene_extras()
        return rows, pairs, seen.copy(), kept
    finally:
        ctx.close()


def _hist(rows, pairs, g):
    o, n = int(rows["hist_offset"][g]), int(rows["hist_count"][g])
    return pairs[o:o + n]


def check_shards(lib, genes, cuts, want):
    n_seg = max(1, len(genes))
    first = [0] * (len(LENS) + 1)
    for t, _, _ in genes:
        first[t + 1] += 1
    first = list(np.cumsum(first))
    for i, (cols, p) in enumerate(_samples()):
        p = dict(p, want=want)
        w_rows, w_pairs, w_seen, w_kept = _run(lib, genes, None, cols, p)
        # the whole run is the single-GPU path already checked against the reference; anchor it anyway
        exp = ref.expected(LENS, p, cols, genes=genes)
        assert np.array_equal(w_seen, exp.contig_seen) and w_kept == exp.kept_primary
        seen_or, kept_sum = np.zeros_like(w_seen), 0
        for r in range(len(cuts) - 1):
            tb, te = cuts[r], cuts[r + 1]
            gb = 0 if tb == 0 else seg_cut(first, n_seg, tb)
            ge = seg_cut(first, n_seg, te)
            rows, pairs, seen, kept = _run(lib, genes, (tb, te), cols, p)
            where = f"sample {i} want={want} rank {r} contigs [{tb}, {te}) genes [{gb}, {ge})"
            for f in ref.INT_FIELDS:
                assert np.array_equal(rows[f][gb:ge], w_rows[f][gb:ge]), (where, f, rows[f][gb:ge], w_rows[f][gb:ge])
            for f in ref.FLOAT_FIELDS:
                assert np.allclose(rows[f][gb:ge], w_rows[f][gb:ge], rtol=1e-12, atol=0.0), (where, f)
            outside = np.ones(len(rows), dtype=bool)
            outside[gb:ge] = False
            for f in ref.INT_FIELDS + ref.FLOAT_FIELDS + ["hist_offset"]:
                assert not rows[f][outside].any(), (where, f, "row outside the shard touched")
            if want & ref.WANT_HIST_CSR:
                assert len(pairs) == int(rows["hist_count"][gb:ge].sum()), where
                for g in range(gb, ge):
                    a, b = _hist(rows, pairs, g), _hist(w_rows, w_pairs, g)
                    assert np.array_equal(a["depth"], b["depth"]) and np.array_equal(a["count"], b["count"]), (where, g)
            mask = np.zeros(len(LENS), dtype=bool)
            mask[tb:te] = True
            assert not seen[~mask].any(), (where, "contig_seen set outside the rank's contigs")
            seen_or |= seen
            kept_sum += kept
        assert np.array_equal(seen_or, w_seen) and kept_sum == w_kept, (i, want, seen_or, w_seen, kept_sum, w_kept)


@pytest.fixture(scope="module")
def emu(range_emu_lib):
    return coverm_b200.load_library(range_emu_lib)


@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("cuts", list(CUT_SETS.values()), ids=list(CUT_SETS))
def test_gene_shards_emulator(emu, cuts, want):
    check_shards(emu, GENES, cuts, want)


def test_gene_shards_without_genes_emulator(emu):
    """A GFF with no gene on these contigs: the placeholder row goes with the last contig range."""
    check_shards(emu, [], [0, 3, 7], ds.WANTS["hist_csr"])


def test_gene_range_bad_arguments_emulator(emu):
    ctx = coverm_b200.DeviceContext(lib=emu)
    try:
        with pytest.raises(coverm_b200.CmbError):
            ctx.set_genes(LENS, GENES, 5, 3)
        with pytest.raises(coverm_b200.CmbError):
            ctx.set_genes(LENS, GENES, 0, len(LENS) + 1)
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("cuts", list(CUT_SETS.values()), ids=list(CUT_SETS))
def test_gene_shards_gpu(cuts, want):
    check_shards(coverm_b200.load_library(), GENES, cuts, want)


@pytest.mark.gpu
def test_gene_shards_without_genes_gpu():
    check_shards(coverm_b200.load_library(), [], [0, 3, 7], ds.WANTS["hist_csr"])


@pytest.mark.gpu
def test_gene_range_bad_arguments_gpu():
    ctx = coverm_b200.DeviceContext()
    try:
        with pytest.raises(coverm_b200.CmbError):
            ctx.set_genes(LENS, GENES, 5, 3)
        with pytest.raises(coverm_b200.CmbError):
            ctx.set_genes(LENS, GENES, 0, len(LENS) + 1)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------------------ group mode
GROUP_WORKER = r'''
import os, sys, json
sys.path.insert(0, sys.argv[1])
import torch
import torch.distributed as dist
import coverm_b200
rank, world, port, lib_path = int(sys.argv[2]), int(sys.argv[3]), sys.argv[4], sys.argv[5]
runs = json.loads(sys.argv[6])
dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
lib = coverm_b200.load_library(lib_path)

def allgather(send):  # the caller-supplied host all-gather of cmbh_session_set_group (here: gloo)
    mine = torch.frombuffer(bytearray(send), dtype=torch.uint8)
    outs = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(outs, mine)
    return b"".join(bytes(o.numpy()) for o in outs)

sess = coverm_b200.Session(device=0, threads=2, lib=lib)
sess.set_group(rank, world, allgather=allgather)
sess.set_group_output(every_rank_prints=True)
results = []
for argv in runs:
    r = sess.run(argv + ["-t", "2", "--print-reads-mapped"])
    s = r.samples[0] if r.samples else {}
    results.append({"status": r.status, "out": r.out, "rm": [l for l in r.err.splitlines() if l.startswith("#reads_mapped")],
                    "err": r.err[-300:] if r.status else "", "device_decode": s.get("device_decode"), "ranks": s.get("group_ranks"),
                    "tid_begin": s.get("tid_begin"), "tid_end": s.get("tid_end")})
sess.close()
print(json.dumps(results))
dist.destroy_process_group()
'''


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run_group(tmp_path, world, runs, lib_path, env=None):
    script = tmp_path / "gene_group_worker.py"
    script.write_text(GROUP_WORKER)
    port = str(_free_port())
    e = dict(os.environ, **(env or {}))
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, str(r), str(world), port, lib_path, json.dumps(runs)],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=e) for r in range(world)]
    outs = [p.communicate(timeout=900) for p in procs]
    for p, (o, er) in zip(procs, outs):
        assert p.returncode == 0, er[-3000:]
    return [json.loads(o.strip().splitlines()[-1]) for o, _ in outs]


def _oracle(argv):
    p = subprocess.run([ORACLE_BIN] + argv + ["--print-reads-mapped"], capture_output=True, text=True, timeout=600)
    return p.returncode, p.stdout, [l for l in p.stderr.splitlines() if l.startswith("#reads_mapped")], p.stderr


@pytest.fixture(scope="module")
def gene_inputs(tmp_path_factory):
    """tests/test_genes.py's inputs: bamgen BAMs and random GFFs over their headers."""
    d = tmp_path_factory.mktemp("gene_shards")
    out = {}
    for name, args, n_genes in (("small", ["--contigs", "400", "--reads", "60000", "--seed", "51", "--median-len", "3000", "--min-len", "200", "--max-len", "40000"], 1500),
                                ("long", ["--contigs", "6", "--reads", "80000", "--seed", "52", "--median-len", "300000", "--sigma", "0.5", "--min-len", "50000", "--max-len", "900000"], 800),
                                ("mags", ["--contigs", "300", "--genomes", "12", "--reads", "50000", "--seed", "53", "--median-len", "6000"], 900)):
        bam = str(d / f"{name}.bam")
        subprocess.check_call([coverm_b200.BAMGEN_BIN, "--out", bam, "--threads", "4"] + args, stdout=subprocess.DEVNULL)
        gff = str(d / f"{name}.gff")
        write_gff(gff, bam_header(bam), n_genes, seed=len(name))
        out[name] = (bam, gff)
    return out


def _group_runs(gene_inputs):
    runs = [argv + ["-b", gene_inputs[w][0], "--gff", gene_inputs[w][1]] for w, argv in RUNS]
    runs.append(["contig", "-m", "mean", "-b", DATA + "/2seqs.bad_read.1.unsorted.bam", "--gff", DATA + "/2seqs.gff"])
    return runs


def _check_group(res, runs, world):
    for i, argv in enumerate(runs):
        rc, out, rm, err = _oracle(argv)
        for r in range(world):
            got = res[r][i]
            assert got["status"] == rc, (argv, r, got["err"])
            assert got["out"] == out, (argv, r)
            assert got["rm"] == rm, (argv, r, got["rm"], rm)
            if rc == 101:  # the unsorted input: the reference's panic, on every rank
                assert "BAM file appears to be unsorted" in got["err"] and "BAM file appears to be unsorted" in err, (r, got["err"])
            else:
                assert got["ranks"] == world


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("emu_bgzf", ["1", None], ids=["ranged-device-decode", "host-decode"])
def test_gene_group_matches_the_oracle_emulator(tmp_path, gene_inputs, range_emu_lib, world, emu_bgzf):
    runs = _group_runs(gene_inputs)
    res = _run_group(tmp_path, world, runs, range_emu_lib, env={"CMB_EMU_BGZF": emu_bgzf or ""})
    _check_group(res, runs, world)
    if emu_bgzf:  # the ranks' contig ranges partition the header, cut by gene bases
        first = [res[r][0] for r in range(world)]
        assert all(x["device_decode"] == 1 for x in first)
        assert first[0]["tid_begin"] == 0 and all(first[r]["tid_end"] == first[r + 1]["tid_begin"] for r in range(world - 1))


def test_gene_group_eight_ranks_emulator(tmp_path, gene_inputs, range_emu_lib):
    """More ranks than `long` has contigs: several ranks own no contig, others contigs without genes."""
    runs = _group_runs(gene_inputs)
    for emu_bgzf in ("1", ""):
        res = _run_group(tmp_path, 8, runs, range_emu_lib, env={"CMB_EMU_BGZF": emu_bgzf})
        _check_group(res, runs, 8)


def test_gene_group_needs_the_range_entry_point(tmp_path, gene_inputs):
    """The plain emulator has no cmb_set_genes_range: a group run with --gff stops on every rank with that error, while the
    same group still runs without --gff."""
    if not os.path.exists(EMU_LIB):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    bam, gff = gene_inputs["small"]
    runs = [["contig", "-m", "mean", "-b", bam, "--gff", gff], ["contig", "-m", "mean", "-b", bam]]
    res = _run_group(tmp_path, 2, runs, EMU_LIB)
    rc, out, rm, _ = _oracle(runs[1])
    for r in range(2):
        assert res[r][0]["status"] == 1 and "cmb_set_genes_range" in res[r][0]["err"], res[r][0]
        assert res[r][1]["status"] == rc == 0 and res[r][1]["out"] == out and res[r][1]["rm"] == rm


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_gene_group_matches_the_oracle_gpu(tmp_path, gene_inputs, world):
    """`world` processes on device 0 with the CUDA library: the real K1 gating, and the gather through the host callback."""
    runs = _group_runs(gene_inputs)
    res = _run_group(tmp_path, world, runs, coverm_b200.LIB_PATH)
    _check_group(res, runs, world)
    assert all(res[r][0]["device_decode"] == 1 for r in range(world))


@pytest.mark.gpu
def test_gene_group_host_decode_gpu(tmp_path, gene_inputs):
    """The same with CMB_HOST_DECODE: every rank decodes the whole file, K1 counts only its own contigs."""
    runs = _group_runs(gene_inputs)
    res = _run_group(tmp_path, 2, runs, coverm_b200.LIB_PATH, env={"CMB_HOST_DECODE": "1"})
    _check_group(res, runs, 2)


# ------------------------------------------------------------------------------------------------- coverm --gpus N --gff
def _n_gpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
        return sum(1 for l in out.splitlines() if l.startswith("GPU "))
    except Exception:
        return 0


@pytest.mark.gpu
@pytest.mark.skipif(_n_gpus() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("which,argv", RUNS, ids=[f"{w}:{' '.join(a[:6])}#{i}" for i, (w, a) in enumerate(RUNS)])
@pytest.mark.parametrize("gpus", [2, 4, 8])
def test_coverm_gpus_gff_matches_the_oracle(gene_inputs, which, argv, gpus):
    if _n_gpus() < gpus:
        pytest.skip(f"needs {gpus} GPUs")
    bam, gff = gene_inputs[which]
    args = argv + ["-b", bam, "--gff", gff, "-t", "8", "--print-reads-mapped"]
    g = subprocess.run([coverm_b200.COVERM_BIN] + args + ["--gpus", str(gpus)], capture_output=True, text=True, timeout=600)
    o = subprocess.run([ORACLE_BIN] + args, capture_output=True, text=True, timeout=600)
    assert g.returncode == o.returncode == 0, g.stderr[-1500:]
    assert g.stdout == o.stdout
    rm = lambda p: [l for l in p.stderr.splitlines() if l.startswith("#reads_mapped")]
    assert rm(g) == rm(o)
