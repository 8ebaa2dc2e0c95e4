"""K2 reads each chunk's slot -> span map from a table the warp builds when it enters the chunk, and (contig mode) each chunk's
contigs from a table of at most K2_CHUNK_CONTIGS entries; a chunk with more contigs finds them by bisection in global memory.

test_k2_span_table_model builds tests/native/k2_span_table_check.cpp (the table builder against k2_slot_span).  The scenarios
give chunks contig ranges of 16, 17, 18 and 42 entries (most of them one-span contigs), and a chunk whose first slot lies in
a contig that started two chunks earlier followed by short contigs, in contig mode and in gene mode, against
tests/device_reference.py: on the CPU emulator of the ABI and, marked gpu, on the CUDA library."""
import os
import re
import subprocess

import pytest

import coverm_b200
import device_reference as ref
import device_scenarios as ds
from case_runner import ROOT

EMU_LIB = os.path.join(ROOT, "oracle", "libcoverm_hostcheck.so")
CHUNK, SPAN = ds.CHUNK, ref.SPAN
CHUNK_CONTIGS = 16  # K2_CHUNK_CONTIGS (coverm_b200/csrc/cmb_k2.cuh)


def _lens_and_records(every_contig_seen=False):
    """Chunks 0..3: 14, 15, 16 and 40 one-span contigs (lengths 1..32), each followed by one that fills the chunk.
    Then a contig of 2.5 chunks, with reads that start in its first chunk and cover the next two, and eight short contigs in
    the chunk where it ends.  Every third contig has no read, or (every_contig_seen) only a one-base read at its start."""
    lens = []

    def chunk_of(n):  # n one-span contigs, then one contig that takes the chunk's remaining spans
        lens.extend(1 + (7 * i) % SPAN for i in range(n))
        lens.append((ref.CHUNK_SPANS - n) * SPAN)

    for n in (14, 15, 16, 40):
        chunk_of(n)
    long_t = len(lens)
    lens.append(2 * CHUNK + CHUNK // 2)
    lens.extend([100, 33, 64, 1, 500, 32, 31, 2000])
    recs = ds.Records()
    for t, L in enumerate(lens):
        if t == long_t:
            continue
        if t % 3 != 2:  # some contigs without events
            recs.add(t, 0, L)
            recs.add(t, L // 2, max(1, L - L // 2))
        elif every_contig_seen:
            recs.add(t, 0, 1)
    recs.add(long_t, 10, 2 * CHUNK + 100).add(long_t, 500, 2 * CHUNK)  # carried into chunks 5 and 6 without an event there
    recs.add(long_t, 2 * CHUNK + 3000, 1000)  # the first slot of the contig's last chunk
    return lens, recs


def _genes(lens):
    gl = []
    for t, L in enumerate(lens):
        gl.append((t, 0, L))
        if L > 64:
            gl.append((t, L // 3, L - 5))
    return gl


def contig_tables():
    lens, recs = _lens_and_records()
    cols = recs.columns()
    return ds.Scenario("k2_tables", lens, [ds.Sample(cols, ref.default_params(contig_end_exclusion=e)) for e in (0, 3, 700)])


def gene_tables():
    """Gene mode reports the genes of a contig without any record as zero-coverage entries on the host (genes.rs:434-465,
    cmb_fetch_gene_extras), so the device's rows of those genes are not results; here every contig has a record, and the
    second gene of a contig with only the one-base read has no event."""
    lens, recs = _lens_and_records(every_contig_seen=True)
    cols = recs.columns()
    return ds.Scenario("k2_tables_genes", lens, [ds.Sample(cols, ref.default_params())], genes=_genes(lens))


SCENARIOS = {"contig": contig_tables, "gene": gene_tables}


def test_k2_span_table_model(tmp_path):
    src = os.path.join(ROOT, "tests", "native", "k2_span_table_check.cpp")
    exe = str(tmp_path / "k2_span_table_check")
    subprocess.run(["g++", "-O1", "-std=c++17", "-fsanitize=address,undefined", "-I", os.path.join(ROOT, "coverm_b200", "csrc"), src,
                    "-o", exe], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    assert re.search(r"\b40000 tests, 0 fails", out), out


def test_scenario_reaches_both_contig_lookups():
    """Chunks whose contig range (chunk_first[k] .. chunk_first[k + 1], as K2 reads it) has 16 entries and more, and chunks
    entered at depth > 0 inside a contig that started one and two chunks before them."""
    src = open(os.path.join(ROOT, "coverm_b200", "csrc", "cmb_k2.cuh")).read()
    assert int(re.search(r"K2_CHUNK_CONTIGS = (\d+);", src).group(1)) == CHUNK_CONTIGS
    lens, _ = _lens_and_records()
    starts, s = [], 0
    for L in lens:
        starts.append(s)
        s += max(1, (L + SPAN - 1) // SPAN)
    n_chunks = (s + ref.CHUNK_SPANS - 1) // ref.CHUNK_SPANS
    first = [max(t for t, x in enumerate(starts) if x <= k * ref.CHUNK_SPANS) for k in range(n_chunks)] + [len(lens) - 1]
    entries = [first[k + 1] - first[k] + 1 for k in range(n_chunks)]
    assert entries[:4] == [CHUNK_CONTIGS, CHUNK_CONTIGS + 1, CHUNK_CONTIGS + 2, 42]
    long_t = 15 + 16 + 17 + 41
    assert starts[long_t] == 4 * ref.CHUNK_SPANS and first[5] == first[6] == long_t and entries[6] == 9


@pytest.fixture(scope="module")
def emu():
    return coverm_b200.load_library(EMU_LIB)


@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_k2_tables_emulator(emu, name, want):
    ds.run_scenario(emu, SCENARIOS[name](), want)


@pytest.mark.gpu
@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_k2_tables_gpu(name, want):
    ds.run_scenario(coverm_b200.load_library(), SCENARIOS[name](), want)
