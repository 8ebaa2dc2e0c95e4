"""`coverm filter --device-deflate`: the output BAM compressed by the project's BGZF deflate encoder (coverm_b200/csrc/
cmb_deflate.cuh, run on the device by cmb_deflate.cu).

CPU: the encoder core's host build over the golden BAMs' record streams and synthetic buffers (tests/native/deflate_check.cpp:
zlib inflates every block to its input, header / BSIZE / CRC32 / ISIZE are right, codes are complete within their limits,
incompressible input is stored, runs repeat, and the t1 decoder's host build reads the blocks); `coverm filter
--device-deflate` on the CPU emulator of the ABI (tests/native/deflate_emulator.cpp) writes the file the encoder writes for the
default output's records, the same after a late decline, and no file after an error; the flag is a usage error elsewhere.
GPU (-m gpu): whole, sliced and host-decoded runs write one file, byte for byte, which holds the default run's records and
equals the host-built encoder's file; outputs beyond one 64 MB piece and empty outputs; `coverm contig` reads the file."""
import glob
import os
import re
import subprocess

import pytest

import coverm_b200
from case_runner import ROOT
from test_filter_slices import big_header_bam  # noqa: F401 (fixture)
from test_sliced_decode import _gen, _inflate, limit_for

NATIVE = os.path.join(ROOT, "tests", "native")
HOST = os.path.join(ROOT, "coverm_b200", "csrc", "host")
GOLDEN = os.path.join(ROOT, "tests", "golden", "data")
SANITIZE = ["-O1", "-g", "-fsanitize=address,undefined", "-fno-omit-frame-pointer", "-fno-sanitize-recover=undefined"]


@pytest.fixture(scope="module")
def recompress(tmp_path_factory):
    """the encoder core's host build as a tool: `exe --recompress in.bam out.bam` writes in's record stream as the encoder's
    BGZF file"""
    exe = str(tmp_path_factory.mktemp("deflate_check") / "deflate_check")
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(NATIVE, "deflate_check.cpp"), "-o", exe, "-lz"], check=True)
    return exe


def _recompressed(exe, bam, out):
    subprocess.run([exe, "--recompress", bam, out], check=True, timeout=1800)
    return open(out, "rb").read()


def test_encoder_core(tmp_path):
    exe = str(tmp_path / "deflate_check")
    subprocess.run(["g++", "-std=c++17"] + SANITIZE + [os.path.join(NATIVE, "deflate_check.cpp"), "-o", exe, "-lz"], check=True)
    bams = sorted(glob.glob(os.path.join(GOLDEN, "*.bam")))
    r = subprocess.run([exe] + bams, capture_output=True, text=True, timeout=1800, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert r.returncode == 0 and r.stdout.startswith("ok "), r.stdout + r.stderr[-3000:]
    m = re.search(r"t1 decoder read (\d+) of (\d+) blocks", r.stdout)
    assert m and m.group(1) == m.group(2), r.stdout
    print(r.stdout)


# ---------------------------------------------------------------------------------------------- CPU: the host's side
@pytest.fixture(scope="module")
def deflate_emu(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("deflate_emu") / "coverm_deflate_emu")
    subprocess.run(["g++", "-std=c++17", "-ffp-contract=off"] + SANITIZE + ["-o", exe, os.path.join(NATIVE, "deflate_emulator.cpp"),
                    os.path.join(HOST, "host_api.cpp"), os.path.join(HOST, "coverm_main.cpp"), "-lz", "-lpthread"], check=True)
    return exe


def _emu(exe, bam, out, extra, mode, sub="filter"):
    env = dict(os.environ, CMB_PIPELINE_STATS="1", ASAN_OPTIONS="detect_leaks=0")
    if mode == "host":
        env["CMB_HOST_DECODE"] = "1"
    elif mode:
        env["CMB_EMU_FILTER"] = mode
    return subprocess.run([exe, sub, "-b", bam] + (["-o", out] if out else []) + ["-t", "4", "--timing"] + extra, capture_output=True,
                          text=True, timeout=1800, env=env)


@pytest.mark.parametrize("extra", [["--min-read-percent-identity", "97"], ["--proper-pairs-only", "--min-read-aligned-length-pair", "100"]],
                         ids=["singles", "pairs"])
def test_device_deflate_on_the_emulator(deflate_emu, recompress, big_header_bam, tmp_path, extra):  # noqa: F811
    default = str(tmp_path / "default.bam")
    p = _emu(deflate_emu, big_header_bam, default, extra, "host")
    assert p.returncode == 0, p.stderr[-3000:]
    files = {}
    for mode in ("host", "", "decline_late"):
        out = str(tmp_path / f"out_{mode or 'declined'}.bam")
        p = _emu(deflate_emu, big_header_bam, out, extra + ["--device-deflate"], mode)
        assert p.returncode == 0 and "AddressSanitizer" not in p.stderr, p.stderr[-3000:]
        m = re.search(r"^#deflate\tsample=0\traw_bytes=(\d+)\tbgzf_bytes=(\d+)\tblocks=(\d+)\tstored_blocks=\d+\tsink_calls=(\d+)\t", p.stderr, re.M)
        assert m, p.stderr[-3000:]
        files[mode] = open(out, "rb").read()
        assert int(m.group(2)) == len(files[mode])
        if mode == "decline_late":  # the filler pieces were written, then the file was truncated and the stream begun again
            assert "#filter_declined\tslices_before=3\tsink_calls=3\n" in p.stderr, p.stderr[-3000:]
    assert files["decline_late"] == files["host"] == files[""]
    raw = _inflate(default)
    assert _inflate(str(tmp_path / "out_host.bam")) == raw
    assert files["host"] == _recompressed(recompress, default, str(tmp_path / "recompressed.bam"))
    assert files["host"].endswith(bytes([0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0] + [0] * 8))


@pytest.mark.parametrize("mode", ["nm", "sink_error"])
def test_device_deflate_error_leaves_no_file(deflate_emu, big_header_bam, tmp_path, mode):  # noqa: F811
    out = str(tmp_path / "out.bam")
    p = _emu(deflate_emu, big_header_bam, out, ["--min-read-percent-identity", "97", "--device-deflate"], mode)
    assert p.returncode != 0 and "AddressSanitizer" not in p.stderr, p.stderr[-3000:]
    assert ("does not have an 'NM' auxiliary tag" in p.stderr) == (mode == "nm"), p.stderr[-3000:]
    assert not os.path.exists(out)


@pytest.mark.parametrize("sub", ["contig", "genome", "filter-names"])
def test_device_deflate_is_a_usage_error_outside_filter(deflate_emu, tmp_path, sub):
    bam = os.path.join(GOLDEN, "7seqs.reads_for_seq1_and_seq2.bam")
    extra = ["--single-genome"] if sub == "genome" else []
    p = _emu(deflate_emu, bam, None, extra + ["--device-deflate"], "", sub=sub)
    assert p.returncode == 2 and "unexpected argument '--device-deflate'" in p.stderr, p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------- GPU
PAIRS = ["--proper-pairs-only", "--min-read-aligned-length-pair", "250", "--min-read-percent-identity-pair", "95"]
SINGLES = ["--min-read-percent-identity", "97", "--min-read-aligned-length", "100"]


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("device_deflate"))
    return {
        "small": _gen(d, "small", "--contigs", 3000, "--reads", 1_200_000, "--seed", 71, "--median-len", 2500, "--min-len", 200, "--max-len", 60000),
        "golden_pairs": os.path.join(GOLDEN, "7seqs.reads_for_seq1_and_seq2.bam"),
        "golden": os.path.join(GOLDEN, "2seqs.reads_for_seq1_and_seq2.bam"),
    }


def _filter(bam, out, extra, env=None):
    argv = [coverm_b200.COVERM_BIN, "filter", "-b", bam, "-o", out, "-t", "8", "--timing"] + extra
    p = subprocess.run(argv, capture_output=True, text=True, timeout=1800, env=dict(os.environ, CMB_PIPELINE_STATS="1", **(env or {})))
    assert p.returncode == 0, p.stderr[-2000:]
    return p


def _deflate_stats(p):
    m = re.search(r"^#deflate\tsample=0\traw_bytes=(\d+)\tbgzf_bytes=(\d+)\tblocks=(\d+)\tstored_blocks=(\d+)\tsink_calls=(\d+)\t", p.stderr, re.M)
    assert m, p.stderr[-2000:]
    return [int(g) for g in m.groups()]


def _device(p):
    m = re.search(r"^#filter\tsample=0\trecords_out=\d+\tdevice=(\d)$", p.stderr, re.M)
    return int(m.group(1)) if m else None


CASES = [("golden", ["--min-read-percent-identity", "95"]), ("golden_pairs", ["--proper-pairs-only"]),
         ("small", SINGLES), ("small", PAIRS), ("small", PAIRS + ["--inverse"]), ("small", ["--min-read-percent-identity", "97", "--inverse"]),
         ("small", ["--min-mapq", "30"])]


@pytest.mark.gpu
@pytest.mark.parametrize("which,extra", CASES, ids=[f"{w}:{' '.join(e)}#{i}" for i, (w, e) in enumerate(CASES)])
def test_routes_write_one_file(inputs, recompress, tmp_path, which, extra):
    bam = inputs[which]
    default = str(tmp_path / "default.bam")
    _filter(bam, default, extra)
    routes = {"whole": {}, "host": {"CMB_HOST_DECODE": "1"}}
    if which == "small":
        routes["sliced"] = {"CMB_DECODE_MEM_LIMIT_MB": limit_for(bam)}
    files = {}
    for route, env in routes.items():
        out = str(tmp_path / f"{route}.bam")
        p = _filter(bam, out, extra + ["--device-deflate"], env)
        files[route] = open(out, "rb").read()
        st = _deflate_stats(p)
        assert st[1] == len(files[route])
        if route == "whole" and which == "small":
            assert _device(p) == 1, p.stderr[-2000:]
        if route == "sliced":
            assert re.search(r"^#filter_slices\tslices=([4-9]|\d\d+)\t", p.stderr, re.M), p.stderr[-2000:]
    assert len(set(files.values())) == 1, {k: len(v) for k, v in files.items()}
    assert _inflate(str(tmp_path / "whole.bam")) == _inflate(default)
    assert files["whole"] == _recompressed(recompress, default, str(tmp_path / "recompressed.bam"))
    print(f"{which} {extra}: default {os.path.getsize(default)} B, device {len(files['whole'])} B, "
          f"ratio {len(files['whole']) / os.path.getsize(default):.4f}, deflate stats {st}")


@pytest.mark.gpu
def test_output_across_pieces_and_slices(inputs, tmp_path):
    """more than one 64 MB piece of BGZF bytes: the carry crosses pieces (and, sliced, slices)"""
    bam = inputs["small"]
    out, sliced, default = str(tmp_path / "out.bam"), str(tmp_path / "sliced.bam"), str(tmp_path / "default.bam")
    _filter(bam, default, ["--min-mapq", "0"])
    st = _deflate_stats(_filter(bam, out, ["--min-mapq", "0", "--device-deflate"]))
    _filter(bam, sliced, ["--min-mapq", "0", "--device-deflate"], {"CMB_DECODE_MEM_LIMIT_MB": limit_for(bam)})
    assert st[1] > 64 << 20 and st[4] >= 2, st
    assert open(out, "rb").read() == open(sliced, "rb").read()
    assert _inflate(out) == _inflate(default)


@pytest.mark.gpu
def test_empty_result_is_header_and_eof(inputs, tmp_path):
    bam = inputs["small"]
    out, default = str(tmp_path / "out.bam"), str(tmp_path / "default.bam")
    extra = ["--min-read-aligned-length", "100000000"]
    _filter(bam, default, extra)
    p = _filter(bam, out, extra + ["--device-deflate"])
    assert re.search(r"^#filter\tsample=0\trecords_out=0\t", p.stderr, re.M), p.stderr[-2000:]
    assert _inflate(out) == _inflate(default)
    assert open(out, "rb").read().endswith(bytes([0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0] + [0] * 8))


@pytest.mark.gpu
def test_contig_reads_the_device_deflated_file(inputs, tmp_path):
    """the project's own device decode reads the encoder's blocks: same table as on the default file; the blocks that went to
    the second inflate pass or to zlib are printed"""
    bam = inputs["small"]
    os.makedirs(tmp_path / "default")
    os.makedirs(tmp_path / "device")
    out, default = str(tmp_path / "device" / "out.bam"), str(tmp_path / "default" / "out.bam")  # one stem: the same column names
    _filter(bam, default, SINGLES)
    _filter(bam, out, SINGLES + ["--device-deflate"])
    tables = {}
    for name, path in (("default", default), ("device", out)):
        sess = coverm_b200.Session(device=0, threads=8)
        res = sess.run(["contig", "-m", "mean", "covered_fraction", "variance", "count", "-b", path, "-t", "8"])
        sess.close()
        assert res.status == 0, res.err
        s = res.samples[0]
        tables[name] = res.out
        print(f"{name}: second_pass_blocks={s['decode_second_pass_blocks']} host_blocks={s['decode_host_blocks']}")
    assert tables["device"] == tables["default"]
