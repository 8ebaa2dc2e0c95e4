"""K1 adds a warp's per-contig read counters once per run of counted records with the same contig; K3 finalises four contigs
per warp, eight lanes each, when all four have fewer than 8 depth bins, and walks them one after another with the whole warp
otherwise.  These scenarios put contig runs and K3's groups of four at their edges: warps whose 32 records fall in 1, 2, 31
and 32 contigs, runs with filtered-out records inside, across warp and CTA boundaries and across a shard's edges, warp sums of
`nm` and indels above 2^32, a partial last warp; groups with bin_hi 0/0/0/0, 7/7/7/7 and 0/7/8/3, a contig deeper than 32
beside shallow ones, contigs without a window or without reads inside a group, and a contig count that is not a multiple of
four, under several trim pairs.

They run on the CPU emulator of the ABI and, marked gpu, on the CUDA library through tests/device_scenarios.py's harness
(every row field, the histogram pairs and K2's load counts exactly, the identity sums to 1e-12)."""
import os
import random
import re
import subprocess
import sys

import pytest

import coverm_b200
import device_reference as ref
import device_scenarios as ds
from case_runner import ROOT

EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")
LIB_ENV, DENSE_ENV = "CMB_TEST_DEVICE_LIB", "CMB_TEST_K2_DENSE_SPANS"
K1_THREADS = 256
FLAGS = [0, 16, 0x2 | 0x40, 0x100, 0x800, 0x4, 16 | 0x800]


def _rec(recs, rng, tid, L, flag=0, mapq=60, nm=None, ins=0, dels=0):
    pos = rng.randrange(max(1, L - 60))
    n = rng.randint(1, 60)
    recs.add(tid, pos, n, flag=flag, mapq=mapq, nm=rng.randint(0, n // 4) if nm is None else nm, ins=ins, dels=dels)


def warp_runs():
    """Warps whose 32 records fall in 1, 2, 31 and 32 contigs, then one with lane 0 and lane 31 alone in their contigs, then
    a contig whose records run from lane 20 of one warp across the warp and CTA (256-record) boundaries, and a partial last
    warp.  Random flags; the second sample filters on MAPQ and identity, so that filtered-out records sit inside the runs."""
    rng = random.Random(41)
    recs, lens, counts = ds.Records(), [], []
    counts += [32]                      # warp 0: one contig
    counts += [5, 27]                   # warp 1: two
    counts += [2] + [1] * 30            # warp 2: 31
    counts += [1] * 32                  # warp 3: 32
    counts += [1, 30, 1]                # warp 4: lanes 0 and 31 alone
    counts += [20, 32 * 3 + 12 + 200, 7, 13]  # from lane 20 of warp 5 across the CTA boundary at record 256; 13 left over
    for t, c in enumerate(counts):
        L = rng.randint(100, 3000)
        lens.append(L)
        for _ in range(c):
            _rec(recs, rng, t, L, flag=rng.choice(FLAGS), mapq=rng.choice([0, 5, 30, 60, 255]))
    cols = recs.columns()
    assert len(cols["tid"]) % 32 and len(cols["tid"]) > K1_THREADS
    filt = ref.default_params(filtering=1, min_mapq=20, min_percent_identity_single=0.9, include_secondary=1)
    return ds.Scenario("warp_runs", lens, [ds.Sample(cols, ref.default_params()), ds.Sample(cols, filt),
                                           ds.Sample(cols, ref.default_params(include_secondary=1, include_supplementary=1))])


def shard_edges():
    """A shard [3, 7) whose first and last contigs share warps with records of contigs 2 and 7, which K1 drops."""
    rng = random.Random(43)
    counts = [40, 9, 20, 15, 1, 30, 17, 20, 50]
    lens = [rng.randint(200, 5000) for _ in counts]
    recs = ds.Records()
    for t, c in enumerate(counts):
        for _ in range(c):
            _rec(recs, rng, t, lens[t], flag=rng.choice(FLAGS))
    return ds.Scenario("shard_edges", lens, [ds.Sample(recs.columns(), ref.default_params(contig_end_exclusion=3))], shard=(3, 7))


def wide_sums():
    """`nm` near 2^32 and indels near 2^31 on every record of a warp: the warp's sums pass 2^32."""
    rng = random.Random(47)
    recs = ds.Records()
    for i in range(32 + 32 + 8):
        t = 0 if i < 40 else 1
        recs.add(t, rng.randrange(500), 50, nm=0xF0000000 + i, ins=0x70000000 + i, dels=0x6FFFFFFF - i)
    return ds.Scenario("wide_sums", [1000, 1000], [ds.Sample(recs.columns(), ref.default_params())])


# K3 groups: contig specs by window depth.  E = 5: depth d stacks d reads inside the window; 0 puts one read in the excluded
# end (a read, but bin_hi 0); None is a contig without reads; "nowin" one whose window is empty (2E >= L)
K3_E = 5
K3_GROUPS = [[0, 0, 0, 0], [7, 7, 7, 7], [0, 7, 8, 3], [40, 1, 2, 1], ["nowin", None, 3, 5], [33, None, 7, 0], [2, 31, 32]]


def k3_groups():
    """Warps of four contigs (the last one three) with the window depths of K3_GROUPS, under trim pairs whose indices fall
    inside, at the edge of and past the first 8 bins."""
    recs, lens = ds.Records(), []
    for t, d in enumerate(x for g in K3_GROUPS for x in g):
        if d == "nowin":
            lens.append(2 * K3_E)
            recs.add(t, 1, 3)
            continue
        L = 60 + 7 * t
        lens.append(L)
        if d == 0:
            recs.add(t, 0, K3_E)
        elif d is not None:
            for j in range(d):  # depths 1..d over [10, 50), stepping down from the middle
                recs.add(t, 10 + j % 5, 40 - j % 5 - j // 5 % 3, nm=j % 3)
    cols = recs.columns()
    trims = [(0.05, 0.95), (0.0, 1.0), (0.2, 0.3), (0.9, 1.0), (0.5, 0.51)]
    return ds.Scenario("k3_groups", lens, [ds.Sample(cols, ref.default_params(contig_end_exclusion=K3_E, trim_min=a, trim_max=b))
                                           for a, b in trims] + [ds.Sample(cols, ref.default_params())])


SCENARIOS = {f.__name__: f for f in (warp_runs, shard_edges, wide_sums, k3_groups)}


def test_k3_groups_reach_their_depths():
    sc = k3_groups()
    exp = ref.expected(sc.lens, dict(sc.samples[0].params, want=ref.WANT_HIST), sc.samples[0].records)
    want = [x for g in K3_GROUPS for x in g]
    assert len(want) % 4
    for t, d in enumerate(want):
        hp = exp.pairs[t]
        if d in ("nowin", None):
            assert hp is None or len(hp[0]) == 0 or exp.rows[t]["n_records"] == 0
        else:
            assert int(hp[0].max()) == d, (t, d, hp)


def test_wide_sums_pass_2_32():
    sc = wide_sums()
    exp = ref.expected(sc.lens, sc.samples[0].params, sc.samples[0].records)
    assert exp.rows[0]["sum_edit"] > 1 << 36 and exp.rows[0]["sum_indel"] > 1 << 36


@pytest.fixture(scope="module")
def emu():
    return coverm_b200.load_library(EMU_LIB)


@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_runs_groups_emulator(emu, name, want):
    ds.run_scenario(emu, SCENARIOS[name](), want)


def _dense_spans():
    if os.environ.get(DENSE_ENV):
        return int(os.environ[DENSE_ENV])
    src = open(os.path.join(ROOT, "coverm_b200", "csrc", "cmb_k2.cuh")).read()
    return int(re.search(r"#define CMB_K2_DENSE_SPANS (\d+)", src).group(1))


@pytest.mark.gpu
@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_runs_groups_gpu(name, want, monkeypatch, capfd):
    monkeypatch.setenv("CMB_PIPELINE_STATS", "1")
    capfd.readouterr()

    def read_loads():
        lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("#k2_load")]
        assert lines, "no #k2_load line on stderr"
        return {k: int(v) for k, v in (f.split("=") for f in lines[-1].split("\t")[1:])}

    lib = coverm_b200.load_library(os.environ.get(LIB_ENV) or None)
    ds.run_scenario(lib, SCENARIOS[name](), want, dense_spans=_dense_spans(), read_loads=read_loads)


@pytest.mark.gpu
@pytest.mark.skipif(bool(os.environ.get(LIB_ENV)), reason="already running on a variant")
@pytest.mark.parametrize("variant,dense", [("dense0", 0), ("dense257", 257), ("stages3", None)])
def test_runs_groups_variant(variant, dense):
    """The scenarios on the build variants, in a child process so that two builds of the library never share one."""
    so = os.path.join(ROOT, "variants", f"test_{variant}.so")
    if not os.path.exists(so):
        pytest.skip(f"{so} is built by tests/test_device_kernels.py::test_build_variant")
    env = dict(os.environ, **{LIB_ENV: so, DENSE_ENV: str(dense if dense is not None else _dense_spans())})
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, f"variant {variant}:\n{r.stdout[-6000:]}\n{r.stderr[-2000:]}"
