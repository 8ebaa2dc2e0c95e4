"""`coverm filter` on samples that do not fit the device whole: cmb_filter_bgzf decodes and filters them in block slices and
the output BAM is written as the slices' records arrive (coverm_b200/csrc/host/bgzf_writer.hpp).

CPU: BgzfWriter fed a stream in arbitrary pieces writes the file a one-shot BGZF writer writes (tests/native/bgzf_writer_check.cpp);
on the CPU emulator with a scripted cmb_filter_bgzf (tests/native/filter_emulator.cpp), a decline after some pieces writes
the host loop's file, and a device error before any piece leaves no file and reads no freed buffer.
GPU (-m gpu): with CMB_DECODE_MEM_LIMIT_MB low enough for four or more slices, every case of test_gpu_parity.FILTER_RUNS
writes the file the unlimited run writes, byte for byte, holding the oracle's records; a late NM panic leaves no file; a late
decline ends like the host route; several inputs in one process, some sliced and some whole, each match the oracle."""
import os
import re
import struct
import subprocess

import pytest

import bam_writer as bw
import coverm_b200
from case_runner import ORACLE_BIN, ROOT
from test_gpu_parity import FILTER_RUNS
from test_sliced_decode import _gen, _inflate, _late_bad, _record_offsets, _reblock, limit_for

SRC = os.path.join(ROOT, "tests", "native", "bgzf_writer_check.cpp")


def test_bgzf_writer_matches_one_shot_writer(tmp_path):
    exe = str(tmp_path / "bgzf_writer_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "coverm_b200", "csrc"), SRC, "-o", exe, "-lz", "-lpthread"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.startswith("ok "), r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------- CPU: the host's side
EMU_SRC = os.path.join(ROOT, "tests", "native", "filter_emulator.cpp")
HOST = os.path.join(ROOT, "coverm_b200", "csrc", "host")


@pytest.fixture(scope="module")
def filter_emu(tmp_path_factory):
    """`coverm` on the CPU emulator with a cmb_filter_bgzf whose outcome CMB_EMU_FILTER picks, built with AddressSanitizer so
    that a piece read after its buffer is gone fails the run"""
    exe = str(tmp_path_factory.mktemp("filter_emu") / "coverm_filter_emu")
    subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address", "-fno-omit-frame-pointer", "-o", exe, EMU_SRC,
                    os.path.join(HOST, "host_api.cpp"), os.path.join(HOST, "coverm_main.cpp"), "-lz", "-lpthread"], check=True)
    return exe


@pytest.fixture(scope="module")
def big_header_bam(tmp_path_factory):
    """300 000 references (a header of about 14 MB, deflated in the background while the device works) and 3000 records"""
    contigs = [("contig_%06d" % k, 5000) for k in range(300_000)]
    path = str(tmp_path_factory.mktemp("big_header") / "big_header.bam")
    with open(path, "wb") as f:
        f.write(bw.bgzf(bw.bam_stream(contigs, bw.random_records(contigs[:20], 3000, seed=5)), level=1))
    return path


def _emu(exe, bam, out, extra, mode):
    env = dict(os.environ, CMB_PIPELINE_STATS="1", ASAN_OPTIONS="detect_leaks=0")
    if mode == "host":
        env["CMB_HOST_DECODE"] = "1"
    elif mode:
        env["CMB_EMU_FILTER"] = mode
    return subprocess.run([exe, "filter", "-b", bam, "-o", out, "-t", "4", "--timing"] + extra, capture_output=True, text=True, timeout=600, env=env)


@pytest.mark.parametrize("extra", [["--min-read-percent-identity", "97"], ["--proper-pairs-only", "--min-read-aligned-length-pair", "100"]],
                         ids=["singles", "pairs"])
def test_decline_after_pieces_writes_the_host_loops_file(filter_emu, big_header_bam, tmp_path, extra):
    files = {}
    for mode in ("host", "", "decline_late"):
        out = str(tmp_path / f"out_{mode or 'declined'}.bam")
        p = _emu(filter_emu, big_header_bam, out, extra, mode)
        assert p.returncode == 0, p.stderr[-3000:]
        assert "#filter\tsample=0\t" in p.stderr and "device=0" in p.stderr, p.stderr[-3000:]
        files[mode] = open(out, "rb").read()
        if mode == "decline_late":  # the pieces before the decline were written, then dropped
            assert "#filter_declined\tslices_before=3\tsink_calls=3\n" in p.stderr, p.stderr[-3000:]
    assert files["decline_late"] == files["host"] == files[""]


@pytest.mark.parametrize("mode", ["nm", "sink_error"])
def test_device_error_leaves_no_file(filter_emu, big_header_bam, tmp_path, mode):
    out = str(tmp_path / "out.bam")
    p = _emu(filter_emu, big_header_bam, out, ["--min-read-percent-identity", "97"], mode)
    assert p.returncode != 0 and "AddressSanitizer" not in p.stderr, p.stderr[-3000:]
    assert ("does not have an 'NM' auxiliary tag" in p.stderr) == (mode == "nm"), p.stderr[-3000:]
    assert not os.path.exists(out)


# ---------------------------------------------------------------------------------------------- GPU
PAIRS = ["--proper-pairs-only", "--min-read-aligned-length-pair", "250", "--min-read-percent-identity-pair", "95"]


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("filter_slices"))
    out = {
        "small": _gen(d, "small", "--contigs", 3000, "--reads", 1_200_000, "--seed", 71, "--median-len", 2500, "--min-len", 200, "--max-len", 60000),
        "deep": _gen(d, "deep", "--contigs", 40, "--reads", 1_500_000, "--seed", 74, "--median-len", 9000, "--min-len", 2000, "--max-len", 40000),
        "mags": _gen(d, "mags", "--contigs", 2500, "--genomes", 60, "--reads", 1_000_000, "--seed", 75, "--median-len", 8000),
        "one_ref": _gen(d, "one_ref", "--contigs", 1, "--reads", 1_000_000, "--seed", 76, "--median-len", 3000000, "--min-len", 3000000,
                        "--max-len", 3000000),
        "fits": _gen(d, "fits", "--contigs", 500, "--reads", 100_000, "--seed", 77, "--median-len", 5000),
    }
    # small blocks, many of them per reference's run: slice ends fall inside pairs and inside reference runs
    out["reblocked"] = _reblock(out["small"], os.path.join(d, "small_reblocked.bam"), (600, 5000))
    return out


def _filter(bams, outs, extra, env=None, sub="filter"):
    argv = [coverm_b200.COVERM_BIN, sub, "-b"] + bams + (["-o"] + outs if outs else []) + ["-t", "8", "--timing"] + extra
    return subprocess.run(argv, capture_output=True, text=True, timeout=1800, env=dict(os.environ, CMB_PIPELINE_STATS="1", **(env or {})))


def _oracle_names(bam, extra):
    p = subprocess.run([ORACLE_BIN, "filter-names", "-b", bam] + extra, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-500:]
    return p.stdout.split("\n")[:-1]


def _names(path):
    stream = _inflate(path)
    return [stream[o + 36:o + 36 + stream[o + 12] - 1].decode() for o in _record_offsets(stream)]


def filter_slices(p):
    m = re.search(r"^#filter_slices\tslices=(\d+)\tmax_slice_bytes=(\d+)\thalvings=(\d+)\tpair_cut_records=(\d+)$", p.stderr, re.M)
    return tuple(int(g) for g in m.groups()) if m else None


def _device(p, k=0):
    m = re.search(rf"^#filter\tsample={k}\trecords_out=\d+\tdevice=(\d)$", p.stderr, re.M)
    return int(m.group(1)) if m else None


def _sliced_equals_whole(inputs, tmp_path, which, extra, pair_cuts=False):
    bam = inputs[which]
    whole, sliced = str(tmp_path / "whole.bam"), str(tmp_path / "sliced.bam")
    w = _filter([bam], [whole], extra)
    s = _filter([bam], [sliced], extra, {"CMB_DECODE_MEM_LIMIT_MB": limit_for(bam)})
    for p in (w, s):
        assert p.returncode == 0, p.stderr[-2000:]
        assert _device(p) == 1, p.stderr[-2000:]
    assert filter_slices(w) is None
    st = filter_slices(s)
    assert st and st[0] >= 4, s.stderr[-2000:]
    if pair_cuts:
        assert st[3] > 0, s.stderr[-2000:]
    assert open(sliced, "rb").read() == open(whole, "rb").read()
    assert _names(sliced) == _oracle_names(bam, extra)


@pytest.mark.gpu
@pytest.mark.parametrize("which,extra", FILTER_RUNS, ids=[f"{w}:{' '.join(e)}#{i}" for i, (w, e) in enumerate(FILTER_RUNS)])
def test_sliced_filter_writes_the_whole_runs_file(inputs, tmp_path, which, extra):
    _sliced_equals_whole(inputs, tmp_path, which, extra, pair_cuts="--proper-pairs-only" in extra)


@pytest.mark.gpu
@pytest.mark.parametrize("inverse", [False, True], ids=["kept", "inverse"])
def test_slice_ends_inside_pairs_and_reference_runs(inputs, tmp_path, inverse):
    _sliced_equals_whole(inputs, tmp_path, "reblocked", PAIRS + (["--inverse"] if inverse else []), pair_cuts=True)


def _without_nm_late(src, dst):
    """`src` with the NM tag of a mapped primary proper-pair record at 85 % of the records renamed to XM"""
    stream = bytearray(_inflate(src))
    offs = _record_offsets(stream)
    for o in offs[int(len(offs) * 0.85):]:
        flag = struct.unpack_from("<H", stream, o + 18)[0]
        if flag & 0x904 or not flag & 0x2:
            continue
        l_name, n_cig, l_seq = stream[o + 12], struct.unpack_from("<H", stream, o + 16)[0], struct.unpack_from("<i", stream, o + 20)[0]
        a = o + 36 + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq
        end = o + 4 + struct.unpack_from("<i", stream, o)[0]
        while a < end:  # the aux fields
            tag, typ = bytes(stream[a:a + 2]), chr(stream[a + 2])
            if tag == b"NM":
                stream[a:a + 2] = b"XM"
                with open(dst, "wb") as f:
                    f.write(bw.bgzf(bytes(stream), level=1))
                return dst
            size = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}.get(typ)
            if size is not None:
                a += 3 + size
            elif typ in "ZH":
                a = stream.index(0, a + 3) + 1
            else:  # B
                sub, n = chr(stream[a + 3]), struct.unpack_from("<i", stream, a + 4)[0]
                a += 8 + n * {"c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}[sub]
    raise AssertionError("no mapped primary proper-pair record with an NM tag")


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [["--min-read-percent-identity", "97"], PAIRS], ids=["singles", "pairs"])
def test_late_nm_panic_leaves_no_file(inputs, tmp_path, extra):
    """the oracle's exit status, and the message the host route gives (the oracle's, but for its final full stop)"""
    bam = _without_nm_late(inputs["small"], str(tmp_path / "no_nm.bam"))
    out = str(tmp_path / "out.bam")
    p = _filter([bam], [out], extra, {"CMB_DECODE_MEM_LIMIT_MB": limit_for(inputs["small"])})
    host = _filter([bam], [str(tmp_path / "host.bam")], extra, {"CMB_HOST_DECODE": "1"})
    o = subprocess.run([ORACLE_BIN, "filter-names", "-b", bam] + extra, capture_output=True, text=True, timeout=1800)
    assert o.returncode != 0 and p.returncode == o.returncode == host.returncode, (p.stderr[-2000:], o.stderr[-2000:])
    last = lambda g: [l for l in g.stderr.splitlines() if l.strip() and not l.startswith("#")][-1:]
    assert last(p) == last(host)
    assert last(p)[0].rstrip(".") == last(o)[0].rstrip(".")
    assert not any(l.startswith("#device_decode\tdeclined") for l in p.stderr.splitlines()), p.stderr[-2000:]
    assert not os.path.exists(out)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,extra", [("corrupt_block", ["--min-read-percent-identity", "97"]), ("unsorted", PAIRS), ("one_ref", PAIRS)])
def test_late_decline_ends_like_the_host_route(inputs, tmp_path, kind, extra):
    bam = inputs["one_ref"] if kind == "one_ref" else _late_bad(inputs, str(tmp_path), kind)
    out, host_out = str(tmp_path / "out.bam"), str(tmp_path / "host.bam")
    p = _filter([bam], [out], extra, {"CMB_DECODE_MEM_LIMIT_MB": limit_for(inputs[kind if kind == "one_ref" else "small"])})
    host = _filter([bam], [host_out], extra, {"CMB_HOST_DECODE": "1"})
    assert p.returncode == host.returncode, (p.stderr[-2000:], host.stderr[-2000:])
    assert any(l.startswith("#device_decode\tdeclined") for l in p.stderr.splitlines()), p.stderr[-2000:]
    m = re.search(r"^#filter_declined\tslices_before=(\d+)\tsink_calls=(\d+)$", p.stderr, re.M)
    assert m, p.stderr[-2000:]
    if kind == "one_ref":  # the first slice already holds one reference's run and nothing else
        assert re.search(r"^#device_decode\tdeclined: .*proper-pair records of reference 0 do not fit in one decode slice", p.stderr, re.M)
        assert m.groups() == ("0", "0")
    else:  # the fault lies at 40 % (unsorted) or 85 % of the records: earlier slices were handed over and are dropped
        assert int(m.group(1)) >= 2 and int(m.group(2)) >= 2, m.group(0)
    assert os.path.exists(out) == os.path.exists(host_out)
    if p.returncode == 0:
        assert _device(p) == 0 and _device(host) == 0
        assert open(out, "rb").read() == open(host_out, "rb").read()
    else:
        last = lambda g: [l for l in g.stderr.splitlines() if l.strip() and not l.startswith("#")][-1:]
        assert last(p) == last(host)
        assert not os.path.exists(out)


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [PAIRS, ["--min-read-percent-identity", "97", "--inverse"]], ids=["pairs", "singles_inverse"])
def test_inputs_that_fit_and_inputs_in_slices_in_one_process(inputs, tmp_path, extra):
    which = ["fits", "small", "fits", "mags"]
    outs = [str(tmp_path / f"{k}_{w}.bam") for k, w in enumerate(which)]
    p = _filter([inputs[w] for w in which], outs, extra, {"CMB_DECODE_MEM_LIMIT_MB": limit_for(inputs["small"])})
    assert p.returncode == 0, p.stderr[-2000:]
    assert len(re.findall(r"^#filter_slices\t", p.stderr, re.M)) == 2, p.stderr[-2000:]
    for k, (w, out) in enumerate(zip(which, outs)):
        assert _device(p, k) == 1, p.stderr[-2000:]
        assert _names(out) == _oracle_names(inputs[w], extra), w


@pytest.mark.gpu
def test_filter_names_in_slices(inputs):
    p = _filter([inputs["small"]], None, PAIRS, {"CMB_DECODE_MEM_LIMIT_MB": limit_for(inputs["small"])}, sub="filter-names")
    assert p.returncode == 0, p.stderr[-2000:]
    assert filter_slices(p)[0] >= 4
    assert p.stdout.split("\n")[:-1] == _oracle_names(inputs["small"], PAIRS)
