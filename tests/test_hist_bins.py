"""The window depth histogram's bin pool: every contig (or gene) owns read-count + 1 bins, K2 adds each window depth above 0
into bin `depth`, and K3 derives the depth-0 count, reads the bins in depth order and re-zeroes them.  These scenarios put depths exactly at that bound,
size the pool from a read-back in gene mode, reuse one context over samples that leave bins behind (a contig without reads,
samples that fail), and make the pool overflow so that cmb_grow_buffers has to size it in one step.

Each scenario runs on the CPU emulator of the ABI (checks the reference side without a GPU) and, marked gpu, on the CUDA
library: every integer field and histogram pair exactly, through tests/device_scenarios.py's harness."""
import os

import numpy as np
import pytest

import coverm_b200
import device_reference as ref
import device_scenarios as ds
from case_runner import ROOT

EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")
HIST_WANTS = {k: v for k, v in ds.WANTS.items() if v}


def _concat(*parts):
    """The records of several column sets, in that order (so that they can be out of order by tid)."""
    cols = {k: np.concatenate([p[k] for p in parts]) for k in parts[0] if k != "iv_begin"}
    ivb, base = [np.zeros(1, dtype=np.uint32)], 0
    for p in parts:
        ivb.append(p["iv_begin"][1:] + base)
        base += int(p["iv_begin"][-1])
    cols["iv_begin"] = np.concatenate(ivb).astype(np.uint32)
    return cols


def stacked():
    """Every read of contig 0 covers the same bases, so its window depth reaches its read count exactly; contig 1 has one
    read; contig 2 stacks reads that run past its end; contig 3 has a read count but no window (2E >= L)."""
    recs = ds.Records()
    for _ in range(300):
        recs.add(0, 100, 400)
    recs.add(1, 5, 10)
    for _ in range(40):
        recs.add(2, 900, 500)
    for _ in range(7):
        recs.add(3, 0, 20)
    return ds.Scenario("stacked", [1000, 64, 1000, 20], [ds.Sample(recs.columns(), ref.default_params(contig_end_exclusion=10))])


def genes_deep():
    """One read across 60 overlapping genes (it counts towards every gene it covers, also those it starts before), and a deep
    gene under 500 stacked reads that also covers the start of the next gene: the pool size is read back from the device."""
    gl = [(0, i * 7, 3000 + i * 7) for i in range(60)] + [(0, 5000, 5100), (0, 5090, 5300), (1, 0, 400)]
    recs = ds.Records()
    recs.add(0, 0, 4000)
    for _ in range(500):
        recs.add(0, 5020, 75)
    recs.add(1, 10, 50)
    return ds.Scenario("genes_deep", [6000, 400], [ds.Sample(recs.columns(), ref.default_params()),
                                                   ds.Sample(recs.columns(), ref.default_params(contig_end_exclusion=3))],
                       genes=sorted(gl, key=lambda g: (g[0], g[1])))


def reuse():
    """On one context: A covers contig 0 deep; B has no read on contig 0 (a window of depth 0 only, whose row K3 does not
    fill); A again; a sample rejected with CMB_E_BOUNDS; an unsorted one; then B and A.  A bin left behind by any of them
    changes a later sample's histogram."""
    lens = [3000, 2 * ds.CHUNK + 100, 500]
    a = ds.Records()
    for i in range(200):
        a.add(0, 10 + 3 * i, 1500)
    a.add(2, 0, 500)
    b = ds.Records().add(1, 10, 30).add(1, 20, 5000).add(2, 100, 50)
    bad = ds.Records().add(0, 5, 100).add(1, 10, 30).add(2, 500, 1)  # a block starting at the contig end
    unsorted = _concat(ds.Records().add(2, 10, 40).add(2, 11, 40).columns(), ds.Records().add(0, 10, 900).columns())
    p = ref.default_params(contig_end_exclusion=2)
    A, B = ds.Sample(a.columns(), p), ds.Sample(b.columns(), ref.default_params())
    return ds.Scenario("reuse", lens, [A, B, A, ds.Sample(bad.columns(), p), ds.Sample(unsorted, p), B, A])


SCENARIOS = {"stacked": stacked, "genes_deep": genes_deep, "reuse": reuse}


def test_scenarios_reach_what_they_claim():
    sc = stacked()
    smp = sc.samples[0]
    exp = ref.expected(sc.lens, dict(smp.params, want=ref.WANT_HIST | ref.WANT_HIST_CSR), smp.records)
    assert exp.pairs[0][0].max() == exp.rows[0]["n_records"] == 300
    assert exp.pairs[3] is None and exp.rows[3]["n_records"] == 7
    sc = reuse()
    errors = [ref.expected(sc.lens, s.params, s.records).error for s in sc.samples]
    assert errors == [0, 0, 0, ref.CMB_E_BOUNDS, ref.CMB_E_UNSORTED, 0, 0]
    b = ref.expected(sc.lens, sc.samples[1].params, sc.samples[1].records)
    assert b.rows[0]["n_records"] == 0
    sc = genes_deep()
    exp = ref.expected(sc.lens, dict(sc.samples[0].params, want=ref.WANT_HIST | ref.WANT_HIST_CSR), sc.samples[0].records,
                       genes=sc.genes)
    assert exp.pairs[60][0].max() == 500  # the deep gene


def _small_hist_run(lib, expect_retry):
    """CMB_TEST_SMALL_HIST starts the bin pool tiny and skips its sizing: the first end_sample fails with CMB_E_CAPACITY,
    cmb_grow_buffers grows the pool to the size that sample needed, and the same records then succeed at the first retry."""
    sc = stacked()
    smp = sc.samples[0]
    p = dict(smp.params, want=ref.WANT_HIST)
    exp = ref.expected(sc.lens, p, smp.records)
    ctx = coverm_b200.DeviceContext(lib=lib)
    try:
        ctx.set_reference(sc.lens)
        ctx.set_params(ds.to_params(p))
        retries = 0
        while True:
            ctx.begin_sample()
            ctx.submit_columns(smp.records)
            try:
                rows, pairs = ctx.end_sample(want_pairs=True)
                break
            except coverm_b200.CmbError as e:
                assert e.code == -7 and retries == 0, f"attempt {retries + 1}: {e}"
                retries += 1
                assert lib.cmb_grow_buffers(ctx._h) == 0
        assert retries == (1 if expect_retry else 0)
        ds._compare("small_hist", rows, pairs, exp, False)
    finally:
        ctx.close()


@pytest.fixture(scope="module")
def emu():
    return coverm_b200.load_library(EMU_LIB)


@pytest.mark.parametrize("want", list(HIST_WANTS.values()), ids=list(HIST_WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_hist_bins_emulator(emu, name, want):
    ds.run_scenario(emu, SCENARIOS[name](), want)


def test_small_hist_emulator(emu, monkeypatch):
    monkeypatch.setenv("CMB_TEST_SMALL_HIST", "1")
    _small_hist_run(emu, expect_retry=False)  # the emulator has no device buffers to outgrow


@pytest.mark.gpu
@pytest.mark.parametrize("want", list(HIST_WANTS.values()), ids=list(HIST_WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_hist_bins_gpu(name, want):
    ds.run_scenario(coverm_b200.load_library(os.environ.get("CMB_TEST_DEVICE_LIB") or None), SCENARIOS[name](), want)


@pytest.mark.gpu
def test_small_hist_grows_pool_in_one_retry(monkeypatch):
    monkeypatch.setenv("CMB_TEST_SMALL_HIST", "1")
    _small_hist_run(coverm_b200.load_library(os.environ.get("CMB_TEST_DEVICE_LIB") or None), expect_retry=True)
