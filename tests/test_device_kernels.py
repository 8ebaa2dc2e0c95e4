"""K1, K1b, K2 and K3 through the device ABI against the exact numpy reference (tests/device_reference.py), on the scenarios of
tests/device_scenarios.py: every integer field exactly, the identity sums to 1e-12, the histogram pairs exactly, and what K2
loaded (`#k2_load`, CMB_PIPELINE_STATS=1) exactly -- spans and whole-tile chunks.

CMB_TEST_DEVICE_LIB names another build of the library to test (a kernel variant of scripts/build_variant.sh) and
CMB_TEST_K2_DENSE_SPANS its dense-chunk threshold; test_build_variant runs this module once per variant that way, in a child
process so that two builds of the CUDA library never share one."""
import os
import re
import shutil
import subprocess
import sys

import pytest

import coverm_b200
import device_scenarios as ds
from case_runner import ROOT

pytestmark = pytest.mark.gpu

LIB_ENV, DENSE_ENV = "CMB_TEST_DEVICE_LIB", "CMB_TEST_K2_DENSE_SPANS"
CSRC = os.path.join(ROOT, "coverm_b200", "csrc")


def _default_dense_spans():
    src = open(os.path.join(CSRC, "cmb_k2.cuh")).read()
    return int(re.search(r"#define CMB_K2_DENSE_SPANS (\d+)", src).group(1))


DENSE_SPANS = int(os.environ.get(DENSE_ENV) or _default_dense_spans())


@pytest.fixture(scope="module")
def lib():
    return coverm_b200.load_library(os.environ.get(LIB_ENV) or None)


def _run(lib, sc, want, monkeypatch, capfd):
    monkeypatch.setenv("CMB_PIPELINE_STATS", "1")
    for k, v in sc.env.items():
        monkeypatch.setenv(k, v)
    capfd.readouterr()

    def read_loads():
        lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("#k2_load")]
        assert lines, "no #k2_load line on stderr"
        return {k: int(v) for k, v in (f.split("=") for f in lines[-1].split("\t")[1:])}

    ds.run_scenario(lib, sc, want, dense_spans=DENSE_SPANS, read_loads=read_loads)


@pytest.mark.parametrize("want", list(ds.WANTS.values()), ids=list(ds.WANTS))
@pytest.mark.parametrize("name", list(ds.BUILDERS))
def test_kernels_match_reference(lib, name, want, monkeypatch, capfd):
    _run(lib, ds.build(name), want, monkeypatch, capfd)


@pytest.mark.parametrize("seed", ds.SWEEP_SEEDS)
def test_kernels_match_reference_seeded(lib, seed, monkeypatch, capfd):
    _run(lib, ds.sweep(seed), None, monkeypatch, capfd)


# ------------------------------------------------------------------------------------------------------------ build variants
VARIANTS = {  # name: (nvcc flags, dense-chunk threshold or None for the default)
    "dense0": ("-DCMB_K2_DENSE_SPANS=0", 0),      # every chunk, even an empty one, through TMA
    "dense257": ("-DCMB_K2_DENSE_SPANS=257", 257),  # no chunk through TMA
    "stages3": ("-DCMB_K2_STAGES=3", None),       # cp.async.wait_group 1, three-stage ring
    "hist2": ("-DCMB_HIST_SLOTS=2", None),        # the overflow list in almost every chunk
}


def _nvcc():
    return shutil.which("nvcc") or next((p for p in ["/usr/local/cuda/bin/nvcc"] if os.path.exists(p)), None)


@pytest.fixture(scope="session")
def variant_libs():
    """variants/test_<name>.so, rebuilt with scripts/build_variant.sh when older than any kernel or host source."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc is not available to build the kernel variants")
    env = dict(os.environ, PATH=os.path.dirname(nvcc) + os.pathsep + os.environ.get("PATH", ""))
    sources = [os.path.join(d, f) for d in (CSRC, os.path.join(CSRC, "host"), os.path.join(ROOT, "include"))
               for f in os.listdir(d) if f.endswith((".cu", ".cuh", ".cpp", ".hpp", ".h"))]
    newest = max(os.path.getmtime(s) for s in sources)
    out, procs = {}, []
    subprocess.run(["make", "-C", CSRC], check=True, stdout=subprocess.DEVNULL)  # the objects every variant links
    for name, (flags, _) in VARIANTS.items():
        so = os.path.join(ROOT, "variants", f"test_{name}.so")
        out[name] = so
        if not os.path.exists(so) or os.path.getmtime(so) < newest:
            procs.append(subprocess.Popen(["bash", os.path.join(ROOT, "scripts", "build_variant.sh"), f"test_{name}", flags],
                                          env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    for p in procs:
        log = p.communicate()[0]
        assert p.returncode == 0, log[-3000:]
    return out


@pytest.mark.skipif(bool(os.environ.get(LIB_ENV)), reason="already running on a variant")
@pytest.mark.parametrize("name", list(VARIANTS))
def test_build_variant(variant_libs, name):
    dense = VARIANTS[name][1]
    env = dict(os.environ, **{LIB_ENV: variant_libs[name], DENSE_ENV: str(dense if dense is not None else DENSE_SPANS)})
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, f"variant {name}:\n{r.stdout[-6000:]}\n{r.stderr[-2000:]}"
