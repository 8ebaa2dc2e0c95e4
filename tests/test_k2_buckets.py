"""Contig mode writes each interval's two delta events to an event list (K1), buckets them by span-bitmap word (K1e), and K2
builds each round's 32 rows in shared memory from the buckets of the words its slots lie in.  These scenarios put that path
at its edges: rounds that share a partial word with their neighbours, a dense chunk whose words hold more events than a
fetch stage, thousands of events on one position, blocks that end at the contig's end (no -1), events on word, chunk and
contig edges, a sample whose list grows over many staging batches, samples after a failed one (with and without cleaning as
K2 goes), contig shards of 2 and 3 ranks, and the pair filter through the `coverm` CLI.

test_bucket_rows_model builds tests/native/k2_buckets_check.cpp: the row building of cmb_k2_slots.cuh as plain C++ against
rows cut from a dense arena.  The scenarios run on the CPU emulator of the ABI and, marked gpu, on the CUDA library through
tests/device_scenarios.py's harness (every row field, the histogram pairs and K2's load counts exactly), where the
`#k2_events` line must also show every event read once or, in a word shared by two rounds, twice."""
import os
import random
import re
import subprocess

import pytest

import bam_writer as bw
import coverm_b200
import device_reference as ref
import device_scenarios as ds
from case_runner import ORACLE_BIN, ROOT

EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")
CHUNK, SPAN, WORD = ds.CHUNK, ref.SPAN, 1024
STAGE_CODES = 1024  # K2_STAGE_CODES: bucket entries a fetch stage holds


def _samples(recs, excl=(0, 21)):
    cols = recs.columns()
    return [ds.Sample(cols, ref.default_params(contig_end_exclusion=e)) for e in excl]


def straddle():
    """Chunks whose rounds share partial words: spans 0..19 and 32..51 of chunk 0, so that round 0 ends and round 1 starts
    inside word 1; 70 spans in chunk 1 spread over every word; 33 spans in chunk 2, the last one alone in the next word."""
    recs = ds.Records()
    for s in list(range(20)) + list(range(32, 52)):
        recs.add(0, SPAN * s + s % 27, 5)
    for i in range(70):
        recs.add(0, CHUNK + (i * 113) % CHUNK // SPAN * SPAN + i % 20, 3)
    for i in range(33):
        recs.add(0, 2 * CHUNK + 3 * WORD + i * SPAN, 1 + i % 31)
    return ds.Scenario("straddle", [3 * CHUNK], _samples(recs))


def dense_deep():
    """A dense chunk (every span occupied) with 1500 short reads inside word 0: that word's bucket holds far more entries than
    a fetch stage, so the round reads the rest straight from global memory.  Depth goes up to 1500."""
    recs = ds.Records()
    for p0 in range(0, CHUNK, SPAN):
        recs.add(0, p0 + 3, 20)
    rng = random.Random(5)
    for _ in range(1500):
        recs.add(0, rng.randrange(WORD - 4), rng.randint(1, 3))
    cols = recs.columns()
    return ds.Scenario("dense_deep", [CHUNK + 500], [ds.Sample(cols, ref.default_params()),
                                                     ds.Sample(cols, ref.default_params(contig_end_exclusion=300))])


def one_position():
    """2000 identical reads, 700 reads ending on one position, and reads starting where the others end."""
    recs = ds.Records()
    for _ in range(2000):
        recs.add(0, 777, 50)
    for i in range(700):
        recs.add(0, 900 + i % 100, 1000 - i % 100)
    for _ in range(300):
        recs.add(0, 827, 10)
    return ds.Scenario("one_position", [5000], _samples(recs))


def contig_end():
    """Blocks ending exactly at the contig's end (e == L: no -1 event) and one position before it, on contigs that end on,
    just before and just after a chunk boundary, and a read covering a whole contig."""
    recs = ds.Records()
    lens = [1000, CHUNK, CHUNK + 1, 3 * WORD - 1]
    for t, L in enumerate(lens):
        recs.add(t, 0, L).add(t, L - 40, 40).add(t, L - 1, 1).add(t, L - 41, 40).add(t, L // 2, L)
    return ds.Scenario("contig_end", lens, _samples(recs, excl=(0, 1, 40)))


def edges():
    """Events on the first and last element of words, chunks and contigs, with contigs that start inside words."""
    lens = [1000, 1025, 8190, 3 * CHUNK + 5, 33]
    recs = ds.Records()
    for t, L in enumerate(lens):
        for p in (0, 31, 32, WORD - 1, WORD, CHUNK - 1, CHUNK, CHUNK + 1, L - 1):
            if p < L:
                for n in (1, WORD - p % WORD, CHUNK - p % CHUNK, L - p):
                    recs.add(t, p, max(1, n))
    return ds.Scenario("edges", lens, _samples(recs))


def batches_grow():
    """4000 records in staging batches of 150: the event list grows between batches, keeping the earlier ones' entries."""
    lens = [30_000, 1, 8192, 50_000, 777]
    return ds.Scenario("batches_grow", lens, [ds.Sample(ds._mixed(61, lens, 4000), ref.default_params(contig_end_exclusion=20))],
                       batch_records=150)


def _after_failure_samples():
    lens = [2 * CHUNK, 3000, 5000]
    rng = random.Random(67)
    a = ds.Records()
    for _ in range(600):
        t = rng.choice([0, 0, 1, 2])
        a.add(t, rng.randrange(lens[t]), rng.randint(1, 400))
    bad = ds.Records()  # events on every contig before the block that starts at contig 1's end
    for t in range(3):
        for _ in range(50):
            bad.add(t, rng.randrange(lens[t] - 10), 5)
    bad.add(1, 3000, 1)
    b = ds.Records().add(2, 10, 20).add(0, CHUNK - 3, 6)
    pa = ref.default_params(contig_end_exclusion=3)
    A, B = ds.Sample(a.columns(), pa), ds.Sample(b.columns(), ref.default_params())
    return lens, [A, ds.Sample(bad.columns(), pa), B, A, ds.Sample(bad.columns(), pa), A]


def after_failure():
    """A, a sample rejected with CMB_E_BOUNDS after K1 had listed and counted events on every contig, B, A, the failure again,
    A: counts, bits or entries left by the failed sample would show in the next one."""
    lens, samples = _after_failure_samples()
    return ds.Scenario("after_failure", lens, samples)


def after_failure_no_clean():
    """The same with CMB_CLEAN_AS_YOU_GO=0: the bitmap and word counts are zeroed at the start of every sample instead."""
    lens, samples = _after_failure_samples()
    return ds.Scenario("after_failure_no_clean", lens, samples, env={"CMB_CLEAN_AS_YOU_GO": "0"})


SHARD_LENS = [9000, 300, 17_000, 1025, 8193, 40, 12_000, 500, CHUNK, 3]
SHARD_CUTS = {"2ranks": [0, 4, 10], "3ranks": [0, 3, 7, 10]}


def shard_rank(cuts, rank):
    """Rank `rank` of a contig shard cut at `cuts`: every rank gets every record and keeps its own contigs' events."""
    recs = ds._mixed(71, SHARD_LENS, 3000)
    return ds.Scenario(f"shard_{len(cuts) - 1}_{rank}", SHARD_LENS, [ds.Sample(recs, ref.default_params(contig_end_exclusion=5))],
                       shard=(cuts[rank], cuts[rank + 1]))


SCENARIOS = {f.__name__: f for f in (straddle, dense_deep, one_position, contig_end, edges, batches_grow, after_failure,
                                     after_failure_no_clean)}
SCENARIOS.update({f"shard_{k}_{r}": (lambda c=c, r=r: shard_rank(c, r)) for k, c in SHARD_CUTS.items() for r in range(len(c) - 1)})


def _word_events(sc):
    """The largest number of events in one bitmap word over the scenario's first sample (contig layout, whole reference)."""
    spans = [max(1, (L + SPAN - 1) // SPAN) for L in sc.lens]
    off = [0]
    for s in spans:
        off.append(off[-1] + s)
    cols, count = sc.samples[0].records, {}
    for i, t in enumerate(cols["tid"]):
        for k in range(cols["iv_begin"][i], cols["iv_begin"][i + 1]):
            s, n = int(cols["iv_start"][k]), int(cols["iv_len"][k])
            if s == ref.IV_PAD:
                continue
            for e in (s, s + n) if s + n < sc.lens[t] else (s,):
                w = (off[t] * SPAN + e) // WORD
                count[w] = count.get(w, 0) + 1
    return max(count.values())


def test_bucket_rows_model(tmp_path):
    """Rows of every round from word buckets, against the dense arena (ASan/UBSan build)."""
    src = os.path.join(ROOT, "tests", "native", "k2_buckets_check.cpp")
    exe = str(tmp_path / "k2_buckets_check")
    subprocess.run(["g++", "-O1", "-std=c++17", "-fsanitize=address,undefined", "-I", os.path.join(ROOT, "coverm_b200", "csrc"), src,
                    "-o", exe], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    m = re.search(r"\b1800 tests, 0 fails \((\d+) rounds sharing a word with the previous one, (\d+) words over 1024 events\)", out)
    assert m and int(m.group(1)) > 100 and int(m.group(2)) > 5, out


def test_scenarios_reach_what_they_claim():
    assert _word_events(dense_deep()) > 2 * STAGE_CODES
    assert _word_events(one_position()) > STAGE_CODES
    sc = dense_deep()
    assert ref.expected(sc.lens, sc.samples[0].params, sc.samples[0].records).load_counts(160)[1] == 1
    sc = straddle()
    assert ref.expected(sc.lens, sc.samples[0].params, sc.samples[0].records).load_counts(257)[0] == 40 + 70 + 33
    assert len(batches_grow().samples[0].records["tid"]) > 20 * 150
    assert ref.expected(*(lambda s: (s.lens, s.samples[1].params, s.samples[1].records))(after_failure())).error


@pytest.fixture(scope="module")
def emu():
    return coverm_b200.load_library(EMU_LIB)


@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_buckets_emulator(emu, name, want):
    ds.run_scenario(emu, SCENARIOS[name](), want)


def _dense_spans():
    src = open(os.path.join(ROOT, "coverm_b200", "csrc", "cmb_k2.cuh")).read()
    return int(re.search(r"#define CMB_K2_DENSE_SPANS (\d+)", src).group(1))


@pytest.mark.gpu
@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_buckets_gpu(name, want, monkeypatch, capfd):
    monkeypatch.setenv("CMB_PIPELINE_STATS", "1")
    sc = SCENARIOS[name]()
    for k, v in sc.env.items():
        monkeypatch.setenv(k, v)
    capfd.readouterr()

    def read_loads():
        err = capfd.readouterr().err.splitlines()
        fields = lambda tag: {k: int(v) for k, v in (f.split("=") for f in [ln for ln in err if ln.startswith(tag)][-1].split("\t")[1:])}
        ev = fields("#k2_events")
        assert ev["events"] <= ev["entries_read"] <= 2 * ev["events"], ev
        return fields("#k2_load")

    ds.run_scenario(coverm_b200.load_library(), sc, want, dense_spans=_dense_spans(), read_loads=read_loads)


PAIR_CONTIGS = [("c0", 3000), ("c1", CHUNK + 700)]


def _pair_bam(path):
    """Proper pairs piled on word and chunk edges, a third of them with an edit distance the identity threshold drops."""
    rng = random.Random(73)
    recs = []
    for i in range(400):
        tid = rng.randrange(2)
        L = PAIR_CONTIGS[tid][1]
        pos = min(L - 150, rng.choice([0, WORD - 10, 2 * WORD - 1, rng.randrange(L - 150)] + ([CHUNK - 60] if tid else [])))
        nm = rng.choice([0, 1, 9])
        mate = pos + rng.randint(0, 50)
        for p, flag in ((pos, 0x1 | 0x2 | 0x40), (mate, 0x1 | 0x2 | 0x80)):
            recs.append((tid, p, bw.record(tid, p, [("M", 100)], flag=flag, qname=f"p{i}", mtid=tid, mpos=pos + mate - p,
                                           tags=(("NM", "C", nm),))))
    recs.sort(key=lambda x: (x[0], x[1]))
    with open(path, "wb") as fh:
        fh.write(bw.bgzf(bw.bam_stream(PAIR_CONTIGS, [r for _, _, r in recs])))


@pytest.mark.gpu
def test_pair_filter_on_buckets(tmp_path):
    """`coverm contig --proper-pairs-only` with a pair identity threshold: the device path's table equals the oracle's."""
    bam = str(tmp_path / "pairs.bam")
    _pair_bam(bam)
    argv = ["contig", "-m", "count", "mean", "covered_bases", "variance", "trimmed_mean", "-b", bam, "-t", "4",
            "--proper-pairs-only", "--min-read-percent-identity-pair", "0.95"]
    want = subprocess.run([ORACLE_BIN] + argv, capture_output=True, text=True, timeout=300)
    got = subprocess.run([coverm_b200.COVERM_BIN] + argv, capture_output=True, text=True, timeout=300,
                         env=dict(os.environ, CMB_PIPELINE_STATS="1"))
    assert want.returncode == 0 and got.returncode == 0, got.stderr[-1500:]
    assert got.stdout == want.stdout
    assert any(ln.startswith("#k2_events") for ln in got.stderr.splitlines()), got.stderr[-1500:]
