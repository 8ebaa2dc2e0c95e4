"""K2 reduces only a chunk's slots (its occupied spans, or all 256 spans of a dense chunk) and closes the event-free stretch
after each slot's last event as one run, up to the next slot or the chunk's end; the stretch before a chunk's first slot has
the chunk's carry-in.  These scenarios put such stretches across spans, bitmap words and whole chunks, end them at a contig's
end and at the window's edges, and fill chunks with 31, 32, 33, 64 and 256 slots so that a contig goes on across rounds.

test_k2_slot_walk_model builds tests/native/k2_slots_check.cpp, the slot arithmetic as plain C++ against a per-position
prefix sum.  The scenarios run on the CPU emulator of the ABI and, marked gpu, on the CUDA library, with K2's load counts
checked (tests/device_scenarios.py's harness); on the dense0 / dense257 builds of scripts/build_variant.sh too when
test_device_kernels.py has built them."""
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
CHUNK, SPAN = ds.CHUNK, ref.SPAN


def _scenario(name, lens, recs, excl=(0, 37)):
    cols = recs.columns()
    return ds.Scenario(name, lens, [ds.Sample(cols, ref.default_params(contig_end_exclusion=e)) for e in excl])


def long_stretch():
    """Depth 1 and 2 over event-free stretches that cross many spans, a bitmap word (1024 elements) and two whole chunks
    without any event."""
    recs = ds.Records()
    recs.add(0, 100, 3 * CHUNK + 500)
    recs.add(0, 40, 3000)
    recs.add(0, 1020, 10)
    recs.add(0, 4 * CHUNK + 3, 2 * CHUNK)  # runs past the contig's end
    return _scenario("long_stretch", [5 * CHUNK + 77, 300], recs.add(1, 5, 20), excl=(0, 37, 1024))


def end_inside_chunk():
    """A stretch at depth 2 reaches its contig's end inside a chunk; the next contig has no event, the one after it has."""
    recs = ds.Records()
    recs.add(0, 2000, 1500).add(0, 2100, 900)
    recs.add(2, 700, 20)
    return _scenario("end_inside_chunk", [3000, 500, 2000], recs, excl=(0, 5, 999))


def window_edges():
    """Stretches that start or end exactly on E and on L - E, and one position to either side."""
    recs = ds.Records()
    L, E = 1000, 100
    recs.add(0, E, L - 2 * E)
    recs.add(0, E - 1, 400)
    recs.add(0, 500, L - E - 500 + 1)
    recs.add(1, E + 1, 200).add(1, 600, L - E - 600)
    return _scenario("window_edges", [L, L], recs, excl=(E,))


SLOT_COUNTS = [31, 32, 33, 64, 256]


def round_edges():
    """Chunks of one contig with exactly 31, 32, 33, 64 and 256 occupied spans under a read that covers them all, so that the
    contig's depth goes on across the rounds of 32 slots."""
    rng = random.Random(17)
    recs = ds.Records()
    L = len(SLOT_COUNTS) * CHUNK + 100
    recs.add(0, 1, L - 2)
    for k, n in enumerate(SLOT_COUNTS):  # chunk 0's span 0 holds the long read's start
        spans = [0] + rng.sample(range(1, ref.CHUNK_SPANS), n - 1) if k == 0 else rng.sample(range(ref.CHUNK_SPANS), n)
        for s in spans:
            off = rng.randrange(SPAN - 1)
            recs.add(0, k * CHUNK + s * SPAN + off, rng.randint(1, SPAN - 1 - off))  # both events in span s
    return _scenario("round_edges", [L, 64], recs.add(1, 0, 64))


def head_not_in_first_contig():
    """Chunk 1 starts inside contig 0, which carries depth 2 into it but has no event there; its first slot is in contig 1,
    and contig 2 starts in the same chunk without an event."""
    recs = ds.Records()
    L0 = CHUNK + 100
    recs.add(0, 50, L0 - 50).add(0, 60, L0)
    recs.add(1, 300, 40)
    return _scenario("head_not_in_first_contig", [L0, 5000, 900, 3000], recs.add(3, 10, 10))


def dense_gaps():
    """A dense chunk (200 occupied spans of 256) with empty spans between the occupied ones, at depths above 0."""
    rng = random.Random(23)
    recs = ds.Records()
    recs.add(0, CHUNK - 10, CHUNK + 20)
    for s in sorted(rng.sample(range(ref.CHUNK_SPANS), 200)):
        recs.add(0, CHUNK + s * SPAN + rng.randrange(SPAN), rng.randint(1, 90))
    return _scenario("dense_gaps", [3 * CHUNK], recs)


def padding():
    """Contig lengths that are not multiples of 32, with stretches at depth above 0 that run into the padding."""
    recs = ds.Records()
    lens = [1013, 77, 2049, 33]
    for t, L in enumerate(lens):
        recs.add(t, max(0, L - 40), 40).add(t, L // 2, L)
    return _scenario("padding", lens, recs)


SCENARIOS = {f.__name__: f for f in (long_stretch, end_inside_chunk, window_edges, round_edges, head_not_in_first_contig,
                                     dense_gaps, padding)}


def test_k2_slot_walk_model(tmp_path):
    """The slot lookup, range ends, depth seeding and clipped run closes of cmb_k2_slots.cuh (ASan/UBSan build)."""
    src = os.path.join(ROOT, "tests", "native", "k2_slots_check.cpp")
    exe = str(tmp_path / "k2_slots_check")
    subprocess.run(["g++", "-O1", "-std=c++17", "-fsanitize=address,undefined", "-I", os.path.join(ROOT, "coverm_b200", "csrc"), src,
                    "-o", exe], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    assert re.search(r"\b1800 tests, 0 fails", out), out


def test_scenarios_reach_what_they_claim():
    sc = round_edges()
    spans, _ = ref.expected(sc.lens, sc.samples[0].params, sc.samples[0].records).load_counts(257)
    assert spans == sum(SLOT_COUNTS) + 2  # + the long read's end and contig 1, both in the chunk after them
    sc = dense_gaps()
    assert ref.expected(sc.lens, sc.samples[0].params, sc.samples[0].records).load_counts(160)[1] == 1


@pytest.fixture(scope="module")
def emu():
    return coverm_b200.load_library(EMU_LIB)


@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_k2_slots_emulator(emu, name, want):
    ds.run_scenario(emu, SCENARIOS[name](), want)


def _dense_spans():
    if os.environ.get(DENSE_ENV):
        return int(os.environ[DENSE_ENV])
    src = open(os.path.join(ROOT, "coverm_b200", "csrc", "cmb_k2.cuh")).read()
    return int(re.search(r"#define CMB_K2_DENSE_SPANS (\d+)", src).group(1))


@pytest.mark.gpu
@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_k2_slots_gpu(name, want, monkeypatch, capfd):
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
@pytest.mark.parametrize("variant,dense", [("dense0", 0), ("dense257", 257)])
def test_k2_slots_variant(variant, dense):
    """The scenarios on a dense-threshold build, in a child process so that two builds of the library never share one."""
    so = os.path.join(ROOT, "variants", f"test_{variant}.so")
    if not os.path.exists(so):
        pytest.skip(f"{so} is built by tests/test_device_kernels.py::test_build_variant")
    env = dict(os.environ, **{LIB_ENV: so, DENSE_ENV: str(dense)})
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, f"variant {variant}:\n{r.stdout[-6000:]}\n{r.stderr[-2000:]}"
