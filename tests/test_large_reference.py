"""References larger than one GPU's memory at 4 B per base: contig mode keeps no per-base array on the device, so its memory
grows with the contigs and the records, not with the bases, up to CMB_MAX_SPANS 32-base spans (about 2^37 bases) per context.

CPU: the run-length restatement of the exact reference (tests/sparse_reference.py) against the dense one on the kernel
scenarios, and the host's advice to split a reference beyond one context's limit over more GPUs (CPU emulator of the ABI).
GPU: the whole CLI on a reference whose dense arena would not fit the device, the ABI at exactly the per-context limit
(64 contigs, 2^32 - 16 spans) against the sparse reference, contig / gene / contig references on one context, and `--gpus 2`
over a reference beyond one context's limit."""
import os
import random
import subprocess

import numpy as np
import pytest

import bam_writer as bw
import coverm_b200
import device_reference as ref
import device_scenarios as ds
import sparse_reference as sparse
from case_runner import ORACLE_BIN, ROOT

EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")
MAX_SPANS = 0xFFFFFFF0  # CMB_MAX_SPANS
BIG = (1 << 31) - 1     # the longest contig the device takes: 2^26 spans
CMB_E_ARG = -2


# ------------------------------------------------------------------------------------------------ sparse vs dense (CPU)
def _same_expectation(where, a, b):
    assert a.error == b.error, f"{where}: error {a.error} != {b.error}"
    if a.error:
        return
    for r, (x, y) in enumerate(zip(a.rows, b.rows)):
        assert x == y, f"{where}: row {r}: {x} != {y}"
    for r, (x, y) in enumerate(zip(a.pairs, b.pairs)):
        assert (x is None) == (y is None), f"{where}: row {r} histogram presence"
        if x is not None:
            assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]), f"{where}: row {r} histogram"


CONTIG_SCENARIOS = [n for n in ds.BUILDERS if n != "e_genes"]


@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", CONTIG_SCENARIOS)
def test_sparse_reference_matches_dense(name, want):
    sc = ds.build(name)
    for i, smp in enumerate(sc.samples):
        p = dict(smp.params, want=want)
        _same_expectation(f"{name} sample {i}", sparse.expected(sc.lens, p, smp.records, shard=sc.shard),
                          ref.expected(sc.lens, p, smp.records, shard=sc.shard))


@pytest.mark.parametrize("seed", ds.SWEEP_SEEDS)
def test_sparse_reference_matches_dense_seeded(seed):
    sc = ds.sweep(seed)  # random E, trims, want (CSR included), flags, filter, every fourth on a shard
    smp = sc.samples[0]
    _same_expectation(sc.name, sparse.expected(sc.lens, smp.params, smp.records, shard=sc.shard),
                      ref.expected(sc.lens, smp.params, smp.records, shard=sc.shard))


def test_depth_runs():
    s, e, d = sparse.depth_runs(100, [0, 10, 10, 50], [20, 30, 100, 60])
    assert s.tolist() == [0, 10, 20, 30, 50, 60] and e.tolist() == [10, 20, 30, 50, 60, 100]
    assert d.tolist() == [1, 3, 2, 1, 2, 1]
    s, e, d = sparse.depth_runs(7, [], [])
    assert (s.tolist(), e.tolist(), d.tolist()) == ([0], [7], [0])


# ------------------------------------------------------------------------------------------------ host limit (CPU emulator)
def _header_only_sam(path, lens):
    with open(path, "w") as f:
        f.write("@HD\tVN:1.6\tSO:coordinate\n" + "".join(f"@SQ\tSN:c{t:03d}\tLN:{L}\n" for t, L in enumerate(lens)))


@pytest.mark.parametrize("n_big,gpus", [(65, 2), (200, 4)])
def test_reference_beyond_one_context_names_gpus(tmp_path, n_big, gpus):
    """A header of n_big contigs of 2^31 - 1 bases (65: 2^32 + 2^26 spans) and no records: the run stops before any device
    call with the smallest --gpus whose contig cuts fit every rank."""
    if not os.path.exists(EMU_LIB):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    sam = str(tmp_path / "big.sam")
    _header_only_sam(sam, [BIG] * n_big + [5000])
    sess = coverm_b200.Session(device=0, threads=2, lib=coverm_b200.load_library(EMU_LIB))
    try:
        res = sess.run(["contig", "-m", "mean", "-b", sam])
    finally:
        sess.close()
    assert res.status != 0
    assert f"run with --gpus {gpus} or more" in res.err and "2^37" in res.err, res.err[-500:]
    assert not res.samples or res.samples[0]["k2_launches"] == 0


def test_reference_within_one_context_runs(tmp_path):
    """Just at the limit: the same header with 64 contigs taking exactly CMB_MAX_SPANS spans passes the host check."""
    if not os.path.exists(EMU_LIB):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    sam = str(tmp_path / "limit.sam")
    _header_only_sam(sam, LIMIT_LENS)
    sess = coverm_b200.Session(device=0, threads=2, lib=coverm_b200.load_library(EMU_LIB))
    try:
        res = sess.run(["contig", "-m", "mean", "-b", sam])
    finally:
        sess.close()
    assert res.status == 0, res.err[-500:]
    assert res.out.count("\n") == len(LIMIT_LENS) + 1


# 63 contigs of 2^31 - 1 bases (2^26 spans each) and one of 2^26 - 16 spans: exactly CMB_MAX_SPANS spans
LIMIT_LENS = [BIG] * 63 + [((1 << 26) - 16) * 32]
assert sum(-(-L // 32) for L in LIMIT_LENS) == MAX_SPANS


# ------------------------------------------------------------------------------------------------------------ GPU tests
def _reference_bytes(text):
    lines = [ln for ln in text.splitlines() if ln.startswith("#reference_bytes")]
    assert lines, "no #reference_bytes line"
    return [{k: int(v) for k, v in (f.split("=") for f in ln.split("\t")[1:])} for ln in lines]


def _limit_records(seed):
    """A few thousand records on LIMIT_LENS: at every contig's start and end (e == L), in the last span, across bitmap word
    (1024) and chunk (8192) boundaries near both ends of each contig, at the far end of the layout, and random ones."""
    rng = random.Random(seed)
    recs = ds.Records()
    for t, L in enumerate(LIMIT_LENS):
        recs.add(t, 0, 1).add(t, 0, 150).add(t, L - 1, 1).add(t, L - 150, 150).add(t, L - 40, 60)
        for b in (1024, 8192, 3 * 8192, L - L % 8192, L - L % 1024 - 1024):
            if 0 < b < L - 4:
                recs.add(t, b - 2, 4).add(t, b, 1).add(t, b - 1, blocks=[(b - 1, 1), (b + 7, 20)], dels=7)
        ds._reads(rng, recs, t, L, 20, max_len=2000)
    last, L = len(LIMIT_LENS) - 1, LIMIT_LENS[-1]
    for k in range(1, 33):  # the last span, one base each, and blocks ending there
        recs.add(last, L - k, k)
    recs.add(last, L - 5000, 5000).add(last, L - 8192 - 3, 8195)
    return recs.columns()


def _run_sparse(ctx, lens, cols, p, where):
    exp = sparse.expected(lens, p, cols)
    ctx.set_params(ds.to_params(p))
    ctx.begin_sample()
    ctx.submit_columns(cols)
    rows, pairs = ctx.end_sample(want_pairs=True)
    assert not exp.error, exp.error
    ds._compare(where, rows, pairs, exp, bool(p["want"] & ref.WANT_HIST_CSR))


@pytest.mark.gpu
def test_one_span_over_the_limit_is_refused():
    ctx = coverm_b200.DeviceContext()
    try:
        over = LIMIT_LENS[:-1] + [LIMIT_LENS[-1] + 32]
        with pytest.raises(coverm_b200.CmbError) as e:
            ctx.set_reference(over)
        assert e.value.code == CMB_E_ARG and "2^37" in str(e.value)
        with pytest.raises(coverm_b200.CmbError) as e:  # no reference was laid out
            ctx.begin_sample()
        assert e.value.code == CMB_E_ARG
    finally:
        ctx.close()


@pytest.mark.gpu
def test_abi_at_the_per_context_limit(monkeypatch, capfd):
    """2^32 - 16 spans (137 Gbp) on one context, records at its edges, every row field and histogram pair against the sparse
    reference; the layout holds no arena."""
    monkeypatch.setenv("CMB_PIPELINE_STATS", "1")
    cols = _limit_records(5)
    ctx = coverm_b200.DeviceContext(batch_records=1 << 12)
    try:
        ctx.set_reference(LIMIT_LENS)
        for i, p in enumerate([ref.default_params(want=ds.WANTS["hist_csr"]),
                               ref.default_params(want=ds.WANTS["hist_csr"], contig_end_exclusion=1000, trim_min=0.1, trim_max=0.9),
                               ref.default_params(want=0, contig_end_exclusion=75)]):
            capfd.readouterr()
            _run_sparse(ctx, LIMIT_LENS, cols, p, f"limit sample {i}")
            rb = _reference_bytes(capfd.readouterr().err)[-1]
            assert rb["arena"] == 0 and rb["layout_elems"] == -(-MAX_SPANS // 256) * 8192, rb
            assert rb["total"] < 2 << 30, rb  # 4 B per base would be 512 GiB
    finally:
        ctx.close()


@pytest.mark.gpu
def test_contig_gene_contig_on_one_context(monkeypatch, capfd):
    """Contig, gene, then contig references on one context give what fresh contexts give; only the gene reference holds an
    arena."""
    monkeypatch.setenv("CMB_PIPELINE_STATS", "1")
    steps = [ds.build("a_layout_edges"), ds.build("e_genes"), ds.build("c_carries")]
    want = ds.WANTS["hist_csr"]

    def run(ctx, sc):
        if sc.genes is not None:
            ctx.set_genes(sc.lens, sc.genes)
        else:
            ctx.set_reference(sc.lens)
        out = []
        for smp in sc.samples:
            p = dict(smp.params, want=want)
            exp = ref.expected(sc.lens, p, smp.records, genes=sc.genes)
            ctx.set_params(ds.to_params(p))
            ctx.begin_sample()
            ctx.submit_columns(smp.records)
            rows, pairs = ctx.end_sample(want_pairs=True)
            ds._compare(sc.name, rows, pairs, exp, True)
            out.append((rows, pairs))
        return out

    shared = coverm_b200.DeviceContext()
    try:
        for sc in steps:
            capfd.readouterr()
            got = run(shared, sc)
            arenas = {rb["arena"] for rb in _reference_bytes(capfd.readouterr().err)}
            assert all(a > 0 for a in arenas) if sc.genes is not None else arenas == {0}, (sc.name, arenas)
            fresh = coverm_b200.DeviceContext()
            try:
                want_out = run(fresh, sc)
            finally:
                fresh.close()
            for (r1, p1), (r2, p2) in zip(got, want_out):  # K3 places each row's pairs in whatever order its contigs finish
                for f in ref.INT_FIELDS:
                    assert np.array_equal(r1[f], r2[f]), (sc.name, f)
                for f in ref.FLOAT_FIELDS:  # f64 REDs in any order
                    assert np.allclose(r1[f], r2[f], rtol=1e-12, atol=0.0), (sc.name, f)
                for r in range(len(r1)):
                    o1, o2, n = int(r1["hist_offset"][r]), int(r2["hist_offset"][r]), int(r1["hist_count"][r])
                    assert np.array_equal(p1[o1:o1 + n], p2[o2:o2 + n]), (sc.name, r)
    finally:
        shared.close()


def _cli(argv, threads="16", gpus=None):
    extra = ["--gpus", str(gpus)] if gpus else []
    return subprocess.run([coverm_b200.COVERM_BIN] + argv + ["-t", threads] + extra, capture_output=True, text=True, timeout=1800,
                          env=dict(os.environ, CMB_PIPELINE_STATS="1"))


def _oracle(argv, threads="16"):
    return subprocess.Popen([ORACLE_BIN] + argv + ["-t", threads], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)


def _same_as_oracle(g, o):
    out, err = o.communicate(timeout=1800)
    assert g.returncode == o.returncode == 0, (g.stderr[-1500:], err[-500:])
    assert g.stdout == out


@pytest.mark.gpu
def test_cli_on_a_reference_beyond_device_memory(tmp_path):
    """231 contigs of about 100 Mbp and 2769 small ones (23.3 Gbp: 93 GB as a dense i32 arena), 3.2 M reads: `coverm contig`
    and `coverm genome` as text against the oracle, the sample decoded on the device, and no arena.  The oracle walks every
    base (minutes at this size), so its two runs go in parallel."""
    rng = random.Random(2026)
    table = str(tmp_path / "contigs.tsv")
    lens = []
    with open(table, "w") as f:
        for c in range(3000):
            L = rng.randint(95_000_000, 105_000_000) if c % 13 == 0 else rng.randint(500, 50_000)
            lens.append(L)
            f.write(f"g{c % 40:02d}~c{c:05d}\t{L}\n")
    total_mib = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=memory.total", "--format=csv,noheader,nounits"],
                               capture_output=True, text=True, check=True).stdout.split()[0]
    assert 4 * sum(lens) > int(total_mib) << 20  # the dense i32 arena of earlier versions would not fit
    bam = str(tmp_path / "big.bam")
    subprocess.run([coverm_b200.BAMGEN_BIN, "--out", bam, "--threads", "16", "--contig-table", table, "--reads", "3000000",
                    "--seed", "77"], check=True, capture_output=True)
    contig = ["contig", "-m", "mean", "trimmed_mean", "covered_fraction", "variance", "-b", bam]
    genome = ["genome", "-s", "~", "-m", "relative_abundance", "mean", "covered_fraction", "--min-covered-fraction", "0", "-b", bam]
    oracles = [_oracle(contig), _oracle(genome)]
    try:
        g = _cli(contig)
        assert any(ln.startswith("#device_decode\tblocks=") for ln in g.stderr.splitlines()), g.stderr[-800:]
        assert all(rb["arena"] == 0 for rb in _reference_bytes(g.stderr))
        _same_as_oracle(g, oracles[0])
        _same_as_oracle(_cli(genome), oracles[1])
    finally:
        for o in oracles:
            if o.poll() is None:
                o.kill()
                o.wait()
        os.remove(bam)


def _n_gpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
        return sum(1 for ln in out.splitlines() if ln.startswith("GPU "))
    except Exception:
        return 0


@pytest.mark.gpu
@pytest.mark.skipif(_n_gpus() < 2, reason="needs at least 2 GPUs")
def test_gpus_2_over_a_reference_beyond_one_context(tmp_path):
    """65 contigs of 2^31 - 1 bases (more than one context holds) over two GPUs, reads on the contigs on both sides of the
    cut and at the reference's ends, against the oracle."""
    lens = [BIG] * 65
    contigs = [(f"c{t:03d}", L) for t, L in enumerate(lens)]
    rng = random.Random(9)
    recs = []
    for t in (0, 31, 32, 33, 64):
        for k in range(400):
            pos = rng.randrange(BIG - 200) if k > 1 else (0 if k == 0 else BIG - 150)
            recs.append((t, pos, [("M", 150)], f"r{t}_{k}"))
    recs.sort(key=lambda r: (r[0], r[1]))
    stream = bw.bam_stream(contigs, [bw.record(t, p, cig, qname=q, tags=[("NM", "C", 1)]) for t, p, cig, q in recs])
    bam = str(tmp_path / "huge.bam")
    with open(bam, "wb") as f:
        f.write(bw.bgzf(stream))
    argv = ["contig", "-m", "mean", "covered_fraction", "variance", "-b", bam]
    o = _oracle(argv)
    _same_as_oracle(_cli(argv, gpus=2), o)
