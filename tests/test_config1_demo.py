"""BASELINE.json configs[0] -- "coverm contig -m mean on demo/ BAM (8 genomes, sample_1), plumbing only".  The reference's demo
directory ships reads and genomes but no BAM and no mapper is available here, so the BAM is synthesised over the
demo's own 1472 reference sequences (names and lengths in tests/golden/demo_contigs.tsv, extracted from demo/genome_*.fna by the
snippet in that file's commit) with 100 000 reads; the product's table must equal the oracle's: CLI -> decode -> device -> printer."""
import os
import subprocess

import pytest

import coverm_b200
from case_runner import ORACLE_BIN, ROOT

TABLE = os.path.join(ROOT, "tests", "golden", "demo_contigs.tsv")
HOSTCHECK = os.path.join(ROOT, "oracle", "coverm_hostcheck")
RUNS = [["contig", "-m", "mean"], ["genome", "-s", "~", "-m", "relative_abundance", "mean", "covered_fraction"], ["contig", "-m", "mean", "trimmed_mean", "covered_fraction", "--no-zeros"]]


@pytest.fixture(scope="module")
def demo_bam(tmp_path_factory):
    p = str(tmp_path_factory.mktemp("demo") / "demo_synth.bam")
    subprocess.check_call([coverm_b200.BAMGEN_BIN, "--out", p, "--contig-table", TABLE, "--reads", "100000", "--seed", "1", "--threads", "4"], stdout=subprocess.DEVNULL)
    return p


def _same(binary, argv, bam):
    a = subprocess.run([binary] + argv + ["-b", bam, "-t", "4", "--print-reads-mapped"], capture_output=True, text=True, timeout=600)
    o = subprocess.run([ORACLE_BIN] + argv + ["-b", bam, "--print-reads-mapped"], capture_output=True, text=True, timeout=600)
    assert a.returncode == o.returncode == 0, a.stderr[-500:]
    assert a.stdout == o.stdout
    assert o.stdout.count("\n") > 8
    assert [l for l in a.stderr.splitlines() if l.startswith("#reads")] == [l for l in o.stderr.splitlines() if l.startswith("#reads")]


@pytest.mark.parametrize("argv", RUNS, ids=[" ".join(r[:4]) for r in RUNS])
def test_config1_demo_plumbing_host(demo_bam, argv):
    _same(HOSTCHECK, argv, demo_bam)


@pytest.mark.gpu
@pytest.mark.parametrize("argv", RUNS, ids=[" ".join(r[:4]) for r in RUNS])
def test_config1_demo_plumbing_gpu(demo_bam, argv):
    _same(coverm_b200.COVERM_BIN, argv, demo_bam)
