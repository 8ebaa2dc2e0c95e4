"""The numpy reference of the kernel-level tests (tests/device_reference.py) and their harness against the CPU emulator of the
device ABI (oracle/libcoverm_hostcheck.so), on every scenario of tests/device_scenarios.py: row for row and pair for pair.
Needs no GPU, so that a failure of tests/test_device_kernels.py points at the kernels rather than at the reference.  The
emulator reports no load counts; the scenarios' load-path properties are checked on the reference alone."""
import os

import numpy as np
import pytest

import coverm_b200
import device_reference as ref
import device_scenarios as ds
from case_runner import ROOT

EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")


@pytest.fixture(scope="module")
def emu():
    return coverm_b200.load_library(EMU_LIB)


@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(ds.BUILDERS))
def test_reference_matches_emulator(emu, name, want):
    ds.run_scenario(emu, ds.build(name), want)


@pytest.mark.parametrize("seed", ds.SWEEP_SEEDS)
def test_reference_matches_emulator_seeded(emu, seed):
    ds.run_scenario(emu, ds.sweep(seed), None)


def test_reference_by_hand():
    """Depth 0 0 1 2 2 1 1 0 0 0 on a 10-base contig (blocks [2, 7) and [3, 5)) plus a block reaching the end of a 4-base one."""
    cols = ds.Records().add(0, 2, 5).add(0, 3, 2).add(1, 1, 3).columns()
    p = ref.default_params(contig_end_exclusion=1, trim_min=0.0, trim_max=1.0, want=ref.WANT_HIST)
    exp = ref.expected([10, 4], p, cols)
    r = exp.rows[0]
    assert (r["covered_full"], r["covered_window"], r["sum_depth_window"]) == (5, 5, 7)
    # window depths 0 1 2 2 1 1 0 0: histogram {0: 3, 1: 3, 2: 2}; indices 0 and ceil(1.0 * 8) = 8
    assert (r["trim_min_index"], r["trim_max_index"], r["var_k"], r["var_ex"], r["var_ex2"], r["hist_count"]) == (0, 8, 0, 7, 11, 3)
    assert r["trimmed_total"] == 7
    assert [x.tolist() for x in exp.pairs[0]] == [[0, 1, 2], [3, 3, 2]]
    r1 = exp.rows[1]  # depth 0 1 1 1, no -1 at the contig end
    assert (r1["covered_full"], r1["sum_depth_window"], r1["hist_count"]) == (3, 2, 1)
    # every event lies in span 0 of its contig; the second contig starts at span 1
    assert exp.occupied.tolist() == [0, 1] and exp.load_counts(2) == (256, 1) and exp.load_counts(3) == (2, 0)


def test_load_path_scenario_hits_each_occupancy():
    exp = ref.expected(*(lambda sc: (sc.lens, sc.samples[0].params, sc.samples[0].records))(ds.load_path()))
    sets = ds.load_path_span_sets()
    pop = exp.chunk_pop()
    assert pop[:len(sets)].tolist() == [len(s) for s in sets]
    assert pop[:len(ds.LOAD_POPS)].tolist() == ds.LOAD_POPS
    per_warp = [len(s) for s in ds.WARP_PATTERNS]
    assert pop[len(ds.LOAD_POPS):len(sets)].tolist() == per_warp
    for k, spans in enumerate(sets):
        got = exp.occupied[(exp.occupied >= k * 256) & (exp.occupied < (k + 1) * 256)] - k * 256
        assert got.tolist() == spans


def test_carry_scenario_reaches_the_k1b_walk_back():
    sc = ds.carries()
    exp = ref.expected(sc.lens, sc.samples[0].params, sc.samples[0].records)
    assert exp.n_chunks > 2 * 1024  # three K1b blocks, the last two without a contig start until the short last contig
    big_off = int(exp.seg_spans[:2].sum()) * ref.SPAN
    cols = sc.samples[0].records
    covers = (cols["tid"] == 2) & (cols["pos"] + big_off <= ds.K1B_BLOCK_ELEMS) & \
        (cols["pos"] + cols["aligned"] + big_off >= 2 * ds.K1B_BLOCK_ELEMS)
    assert covers.sum() >= 2
    assert int(np.float32(ds.BIG)) != ds.BIG  # T = L with E = 0 rounds in float32
    # chunks with depth but no event: the first one of the 100 000-base block of contig 1
    first = int(exp.seg_spans[0]) * ref.SPAN
    k = (first + 50_000 + 5 + ref.SPAN * ref.CHUNK_SPANS - 1) // (ref.SPAN * ref.CHUNK_SPANS)
    assert exp.chunk_pop()[k] == 0


def test_hist_scenarios_overflow_what_they_claim():
    sc = ds.hist_slots()
    exp = ref.expected(sc.lens, sc.samples[0].params, sc.samples[0].records)
    assert sum(r["covered_full"] > 0 for r in exp.rows[:12]) == 12 and exp.seg_spans[:12].sum() < ref.CHUNK_SPANS
    sc = ds.overflow_bins()
    d = ref.expected(sc.lens, dict(sc.samples[0].params, want=ref.WANT_HIST), sc.samples[0].records).pairs[0][0]
    assert {0, 128, 256} <= set(d.tolist())  # every depth change lies in the first chunk
    sc = ds.k3_windows()
    d = ref.expected(sc.lens, dict(sc.samples[0].params, want=ref.WANT_HIST), sc.samples[0].records).pairs[0][0]
    assert d.max() - d.min() > 2 * 512


def test_trim_scenario_has_float32_sensitive_indices():
    """At T = 10 the last two trim pairs give other indices when the product is taken in float64."""
    import math
    for lo, hi in ds.TRIMS[-2:]:
        f32 = ref.trim_indices(lo, hi, 10)
        f64 = (math.floor(float(np.float32(lo)) * 10), math.ceil(float(np.float32(hi)) * 10))
        assert f32 != f64
