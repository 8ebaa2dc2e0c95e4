"""The decoded record columns, exactly: what the device record chain (kd_guess, kd_walk, kd_verify, kd_scan_items, kd_offsets)
and kd_extract make of a BAM file, column by column of cmb_read_batch, against tests/record_reference.py.

The coverage table sees these columns only through sums and filters, so it misses many errors in them: `ins` and `del`
swapped (only their sum reaches the table), an aligned block split into two adjacent intervals (same depth), a bad value
in an unused interval slot (K1 skips those), fields no filter reads, and wrong record boundaries that make the device
decline to the host decoder (the table is then still right).  Here:

- CPU half: the reference parser against the host decoder (cmbh_extract_tuples on the emulator build) on every corpus file,
  per record and per interval list (the host packs intervals tightly; the device reserves one slot per CIGAR operation);
  and every corpus file is a valid `coverm contig` input (the host decoder's table equals the oracle's).
- GPU half: `contig -m mean` in-process, then the resident device columns (cmb_last_bgzf_batch) against the reference:
  every per-record column, iv_begin as the running sum of n_cigar_op, each record's intervals first in its slots in CIGAR
  order and (CMB_IV_PAD, 0) in the rest.  Files the reference says the device must decline are declined and still give
  the oracle's table.  Once with the blocks as inflated, once with every 7th block re-inflated by the second pass or zlib
  (CMB_DECODE_RETRY_TEST), and in child processes with small copy windows and with the thread-per-block inflate kernel.

The corpus is built here with tests/bam_writer.py: block cuts at every offset 0..36 after record starts, runs of 1-byte
blocks, headers that fill block 0 exactly or span many blocks, empty blocks, decoy record headers at block starts,
records longer than kd_guess's 1 MiB scan, block and record counts at the scan and warp edges, and records that exercise
each kd_extract field.  Records that need coordinates outside their contig are flagged unmapped (0x4): both decoders
compute their intervals regardless of the flag, and K1 and the oracle skip them."""
import os
import re
import struct
import subprocess
import sys

import numpy as np
import pytest

import bam_writer as bw
import record_reference as rr
from case_runner import ORACLE_BIN, ROOT
from test_host_input import _extract

try:  # imported before anything loads libcoverm_b200, whose NCCL would otherwise shadow the one libtorch_cuda needs
    import torch
except ImportError:  # the CPU half does without it
    torch = None

HOSTCHECK = os.path.join(ROOT, "oracle", "coverm_hostcheck")
CONTIGS = [("c0", 300000), ("c1", 5000), ("c2", 4000000)]
UNMAPPED = 0x4
I32MAX = 2 ** 31 - 1
L28 = 2 ** 28 - 1  # the longest CIGAR operation

# A plausible record header by kd_guess's rules (block_size >= 32, tid in [-1, n_ref), l_name >= 1 with its NUL in place,
# fixed fields <= block_size): an empty record of 37 bytes.  Eight in a row make a decoy chain.
FAKE = struct.pack("<IiiBBHHHIiii", 33, 0, 0, 1, 0, 0, 0, 0, 0, -1, -1, 0) + b"\0"
DECOY = FAKE * 8


def _starts(stream, recs):
    """Stream offset of each record of `recs`, the last ones of `stream`."""
    at = len(stream) - sum(len(r) for r in recs)
    out = []
    for r in recs:
        out.append(at)
        at += len(r)
    return out


def _tid_pos(r):
    return struct.unpack_from("<ii", r, 4)


def _fill(n, seed, contigs=CONTIGS[:1], **kw):
    return bw.random_records(contigs, n, seed, rich_tags=True, **kw)


def _with_aux(rec, raw):
    """`rec` with raw aux bytes appended (and its block_size grown)."""
    r = bytearray(rec) + raw
    r[0:4] = struct.pack("<I", len(r) - 4)
    return bytes(r)


def _qual_offset(rec):
    l_name, n_cig, l_seq = rec[12], struct.unpack_from("<H", rec, 16)[0], struct.unpack_from("<I", rec, 20)[0]
    return 36 + l_name + 4 * n_cig + (l_seq + 1) // 2


# ---------------------------------------------------------------------------------------------- the record chain
def _cuts_near_record_starts():
    recs = _fill(500, 11, read_len=(20, 150))
    s = bw.bam_stream(CONTIGS, recs)
    st = _starts(s, recs)
    cuts = {a + k % 37 for k, a in enumerate(st)}            # every offset 0..36 after a record start, many times over
    cuts |= set(range(st[250], st[250] + 90))                # a run of 1-byte blocks across a record start
    return bw.bgzf_cuts(s, sorted(cuts))


def _header_fills_block0():
    recs = _fill(300, 12)
    s = bw.bam_stream(CONTIGS, recs)
    at = _starts(s, recs)[0]
    return bw.bgzf_cuts(s, [at] + list(range(at + 3000, len(s), 3000)))


def _header_many_blocks():
    contigs = [("contig_%05d" % i, 1000 + i % 700) for i in range(6000)]
    return bw.bgzf(bw.bam_stream(contigs, bw.random_records(contigs, 1500, 13, read_len=(30, 100))), block_sizes=4096)


def _empty_blocks_no_eof():
    recs = _fill(600, 14)
    s = bw.bam_stream(CONTIGS, recs)
    st = _starts(s, recs)
    cuts = [st[0], st[0]]                                        # an empty block first in the record section
    for k, a in enumerate(st[1:], 1):
        cuts += [a, a] if k % 25 == 0 else [a + 5] if k % 7 == 0 else []  # and between records
    return bw.bgzf_cuts(s, cuts, eof=False)


def _decoys(resync):
    """Records whose QUAL bytes or B:C array carry a decoy chain, each at the start of a block.  resync: the decoy ends the
    record, so that a walk from it reaches the next true record start."""
    recs = _fill(900, 15, read_len=(30, 120))
    host = {}
    for k in range(40):
        pos = 1000 + 7000 * k
        if resync:
            r = bw.record(0, pos, [("M", 60)], qname="d%d" % k, tags=[("NM", "C", 1), ("XB", "B", ("C", list(DECOY)))])
            host[r] = len(r) - len(DECOY)
        elif k % 2:
            r = bw.record(0, pos, [("M", 400)], qname="dq%d" % k, qual=DECOY + b"\x1e" * (400 - len(DECOY)))
            host[r] = _qual_offset(r)
        else:
            r = bw.record(0, pos, [("M", 80)], qname="db%d" % k, tags=[("XB", "B", ("C", list(DECOY))), ("NM", "C", 2)])
            host[r] = _qual_offset(r) + 80 + 3 + 5
        recs.append(r)
    recs.sort(key=_tid_pos)
    s = bw.bam_stream(CONTIGS, recs)
    cuts = [a + host[r] for r, a in zip(recs, _starts(s, recs)) if r in host]
    return bw.bgzf_cuts(s, cuts)


def _long(mb):
    l_seq = int(mb * 1e6 / 1.5)
    return lambda pos, q: bw.record(2, pos, [("M", l_seq)], qname=q)


def _long_records():
    """1.5-3 MB records, back to back and between short ones: most of their blocks are over 1 MiB from a record start."""
    layout = [None] * 5 + [3, 2] + [None] * 3 + [1.5] + [None] * 5 + [3] + [None] * 7
    recs = [(_long(m) if m else lambda pos, q: bw.record(2, pos, [("M", 80)], qname=q))(100 + 1000 * k, "L%d" % k) for k, m in enumerate(layout)]
    return bw.bgzf(bw.bam_stream(CONTIGS, recs), level=1)


def _long_record_small_blocks():
    """A 3 MB record in 4 KB blocks: ~500 blocks without a findable record start.  The chain's repairs advance one block
    per round from the first of them to the end of the stream, so it needs more than its 256 rounds and declines."""
    recs = [bw.record(2, 100 + k, [("M", 80)], qname="s%d" % k) for k in range(8)]
    recs.insert(4, _long(3)(103, "big"))
    return bw.bgzf(bw.bam_stream(CONTIGS, recs), level=1, block_sizes=4096)


def _walked_blocks(n):
    """Header alone in block 0, the records in n - 1 blocks, the EOF block: the chain walks exactly n blocks."""
    recs = _fill(2500, 16)
    s = bw.bam_stream(CONTIGS, recs)
    at, L = _starts(s, recs)[0], len(s) - _starts(s, recs)[0]
    return bw.bgzf_cuts(s, [at] + [at + (k * L) // (n - 1) for k in range(1, n - 1)])


def _tiny_blocks():
    s = bw.bam_stream(CONTIGS, bw.random_records(CONTIGS, 1200, 17, read_len=(20, 60), homopolymer=True))
    return bw.bgzf(s, level=1, block_sizes=max(1, len(s) // 40000))


def _n_records(n):
    return bw.bgzf(bw.bam_stream(CONTIGS, bw.random_records(CONTIGS, n, 18 + n, rich_tags=True)), block_sizes=(500, 5000), seed=n)


# ---------------------------------------------------------------------------------------------- kd_extract's fields
def _field_records():
    R = bw.record
    every_op = [("H", 5), ("S", 3), ("M", 10), ("I", 2), ("D", 3), ("N", 20), ("P", 1), ("=", 5), ("X", 4), ("M", 6), ("S", 2), ("H", 1)]
    all_aux = [("XA", "A", "x"), ("Xc", "c", -5), ("XC", "C", 200), ("Xs", "s", -300), ("XS", "S", 60000), ("Xi", "i", -70000),
               ("XI", "I", 4000000000), ("Xf", "f", 1.5), ("XZ", "Z", ""), ("XH", "H", ""), ("Xz", "Z", "abc"), ("Xh", "H", "1AE3")]
    all_aux += [("B" + sub, "B", (sub, vals)) for sub, vals in (("c", [-1, 2]), ("C", [1]), ("s", [-3]), ("S", [7, 8]), ("i", [-9]),
                                                                   ("I", [10]), ("f", [1.0]))]
    all_aux += [("E1", "B", ("i", [])), ("E2", "B", ("C", []))]
    long_ops = [("M", 1), ("I", 1)] * 32767 + [("M", 1)]  # 65 535 operations
    m, u = [], []  # mapped records of c0 in position order; unmapped ones
    m += [R(0, 100, every_op, qname="every_op", tags=[("NM", "C", 7)]),
          R(0, 200, [("M", 0), ("I", 0), ("D", 0), ("M", 5), ("N", 0), ("M", 0)], qname="zero_len_ops"),
          R(0, 300, long_ops, qname="ops65535", tags=[("NM", "S", 32767)]),
          R(0, 400, [], l_seq=10, qname="no_cigar_mapped"),
          R(0, 500, [("M", 50)], l_seq=0, qname="l_seq0"),
          R(0, 600, [("M", 7)], qname="l_seq_odd"),
          R(0, 700, [("M", 30)], mapq=0, qname="mapq0"),
          R(0, 800, [("M", 30)], mapq=255, qname="mapq255")]
    m += [R(0, 900 + 10 * k, [("M", 40)], qname="nm_%s_%d" % (ty, v), tags=[("NM", ty, v)]) for k, (ty, v) in
          enumerate((("C", 0), ("C", 255), ("S", 0), ("S", 65535), ("I", 0)))]
    m += [R(0, 1000 + 10 * k, [("M", 40), ("D", 1), ("M", 3)], flag=1 << k, qname="flag%d" % k) for k in range(16) if not (1 << k) & UNMAPPED]
    m += [R(0, 1200, [("M", 40)], qname="nm_twice", tags=[("NM", "C", 3), ("NM", "S", 9)]),
          R(0, 1300, [("M", 40)], qname="nm_after_all", tags=all_aux + [("NM", "S", 4)]),
          R(0, 1400, [("M", 40)], qname="nm_I_last", tags=[("XZ", "Z", "q"), ("NM", "I", 5)]),
          R(0, 1500, [("M", 10)], qname="cg_not_placeholder", tags=[("NM", "C", 0), ("CG", "B", ("I", [(10 << 4) | 0]))]),
          R(0, 1600, [("S", 50), ("N", 500)], qname="placeholder_no_cg"),
          R(1, 10, [("I", 5), ("M", 20), ("D", 7), ("M", 4), ("I", 3)], qname="ins_del_c1", tags=[("NM", "C", 15)])]
    u += [R(0, 50, [("M", 5)], flag=UNMAPPED, qname="nm_absent", tags=()),
          R(0, 50, [("M", 5)], flag=UNMAPPED, qname="nm_I_max", tags=[("NM", "I", 2 ** 32 - 1)])]
    u += [R(0, 60, [("M", 5)], flag=UNMAPPED, qname="nm_type_" + ty, tags=[("NM", ty, v)]) for ty, v in
          (("c", -1), ("s", 7), ("i", 70000), ("A", "z"), ("f", 2.5), ("Z", "12"), ("H", "0F"), ("B", ("C", [1])))]
    u += [R(0, 70, [("M", 5)], flag=UNMAPPED, qname="nm_twice_wrong_first", tags=[("NM", "c", 1), ("NM", "C", 5)]),
          R(0, 80, [("M", 5)], flag=0xFFFF, qname="flag_all"),
          R(0, 90, [("M", 5)], flag=UNMAPPED, qname="flag4"),
          R(0, -1, [("M", 1), ("M", 3)], flag=UNMAPPED, qname="pos_m1"),
          R(0, -1, [("S", 2), ("M", 5), ("D", 3), ("M", 4)], flag=UNMAPPED, qname="pos_m1_del"),
          R(0, -3, [("M", 1), ("N", 1), ("M", 4), ("M", 2)], flag=UNMAPPED, qname="pos_m3"),
          R(0, I32MAX - 1, [("M", 1), ("M", 1), ("M", 1), ("D", L28), ("M", L28), ("N", L28), ("X", 3)], l_seq=0, flag=UNMAPPED,
            qname="clamp"),
          R(0, I32MAX, [("M", 5)], flag=UNMAPPED, qname="pos_max"),
          R(0, 2 ** 31 - 2 ** 28, [("M", L28), ("=", L28), ("M", L28), ("X", 1)], l_seq=0, flag=UNMAPPED, qname="long_ops_to_clamp"),
          R(0, 40, [], l_seq=3, flag=UNMAPPED, qname="no_cigar_unmapped"),
          R(-1, -1, [("S", 7), ("N", 6)], l_seq=7, flag=UNMAPPED, qname="placeholder_cg_unplaced",
            tags=[("NM", "C", 0), ("CG", "B", ("I", [(3 << 4) | 0, (1 << 4) | 1, (3 << 4) | 0]))])]
    tail = [R(-1, -1, [], l_seq=30, flag=UNMAPPED | 1 | 0x40, qname="tail1"), R(-1, -1, [("M", 10)], flag=UNMAPPED, qname="tail2"),
            R(-1, -1, [], l_seq=0, flag=UNMAPPED, qname="tail3")]
    # unmapped records between the mapped ones of c0
    out = []
    for k, r in enumerate(m):
        out.append(r)
        if k < len(u):
            out.append(u[k])
    return out + u[len(m):] + tail


def _fields():
    return bw.bgzf(bw.bam_stream(CONTIGS, _field_records()), block_sizes=(200, 3000), seed=19)


def _cg_placeholder():
    """CG:B,I behind the `<l_seq>S<reflen>N` placeholder of a mapped read: its real CIGAR has more operations than the
    record's n_cigar_op, so the device declines the stream."""
    cg = [(3 << 4) | 0, (1 << 4) | 1, (3 << 4) | 0]
    recs = _fill(200, 20)
    recs.append(bw.record(0, 150000, [("S", 7), ("N", 6)], l_seq=7, qname="ultralong", tags=[("NM", "C", 1), ("CG", "B", ("I", cg))]))
    recs.sort(key=_tid_pos)
    return bw.bgzf(bw.bam_stream(CONTIGS, recs), block_sizes=(500, 4000), seed=20)


def _unknown_aux():
    recs = _fill(300, 21)
    recs[150] = _with_aux(recs[150], b"XXQ\0")  # 'Q' is no SAM aux type
    return bw.bgzf(bw.bam_stream(CONTIGS, recs), block_sizes=(500, 4000), seed=21)


def _overrun_fixed_fields():
    recs = _fill(300, 22)
    victim = bytearray(recs[150])
    victim[16:18] = struct.pack("<H", 40000)  # n_cigar_op far past block_size
    recs[150] = bytes(victim)
    return bw.bgzf(bw.bam_stream(CONTIGS, recs), block_sizes=(500, 4000), seed=22)


# name -> (builder, what the device does with it): "exact" (decoded, every column exact), "decline" (the reference
# parser flags a record), "chain_decline" (the chain needs more repair rounds than it allows)
CORPUS = {
    "cuts_near_record_starts": (_cuts_near_record_starts, "exact"),
    "header_fills_block0": (_header_fills_block0, "exact"),
    "header_many_blocks": (_header_many_blocks, "exact"),
    "empty_blocks_no_eof": (_empty_blocks_no_eof, "exact"),
    "decoys": (lambda: _decoys(False), "exact"),
    "decoys_resync": (lambda: _decoys(True), "exact"),
    "long_records": (_long_records, "exact"),
    "long_record_small_blocks": (_long_record_small_blocks, "chain_decline"),
    "walked_blocks_1023": (lambda: _walked_blocks(1023), "exact"),
    "walked_blocks_1024": (lambda: _walked_blocks(1024), "exact"),
    "walked_blocks_1025": (lambda: _walked_blocks(1025), "exact"),
    "walked_blocks_2049": (lambda: _walked_blocks(2049), "exact"),
    "tiny_blocks_40k": (_tiny_blocks, "exact"),
    "records_0": (lambda: _n_records(0), "exact"),
    "records_1": (lambda: _n_records(1), "exact"),
    "records_255": (lambda: _n_records(255), "exact"),
    "records_256": (lambda: _n_records(256), "exact"),
    "records_257": (lambda: _n_records(257), "exact"),
    "fields": (_fields, "exact"),
    "cg_placeholder": (_cg_placeholder, "decline"),
    "unknown_aux": (_unknown_aux, "decline"),
    "overrun_fixed_fields": (_overrun_fixed_fields, "decline"),
}
NAMES = list(CORPUS)
EXACT = [n for n in NAMES if CORPUS[n][1] == "exact"]
DECLINE = [n for n in NAMES if CORPUS[n][1] != "exact"]
DECOYS = {"decoys", "decoys_resync"}
READ_ERRORS = {"unknown_aux", "overrun_fixed_fields"}  # the reference panics: "Error reading BAM record"


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("tuples")
    out = {}
    for name, (build, _) in CORPUS.items():
        out[name] = str(d / (name + ".bam"))
        with open(out[name], "wb") as f:
            f.write(build())
    return out


_parsed = {}


def _ref(path):
    if path not in _parsed:
        _parsed[path] = rr.parse(path)
    return _parsed[path]


def _same(name, got, want):
    got, want = np.asarray(got).astype(np.int64), np.asarray(want).astype(np.int64)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{name}: {bad.size} differ, first at {bad[0]}: got {got[bad[0]]}, want {want[bad[0]]}"


def _table(binary, path):
    return subprocess.run([binary, "contig", "-m", "mean", "-b", path], capture_output=True, text=True, timeout=600)


# ---------------------------------------------------------------------------------------------- CPU half
def test_corpus_is_what_it_claims(corpus):
    """The files have the shapes the device tests rely on: expected declines flagged by the reference and nowhere else,
    the walked block counts, a decoy chain at the start of blocks in the decoy files, records over 1 MiB."""
    for name in NAMES:
        ref = _ref(corpus[name])
        assert bool(ref.declines) == (CORPUS[name][1] == "decline"), (name, ref.declines[:3])
    for n in (1023, 1024, 1025, 2049):
        data = open(corpus["walked_blocks_%d" % n], "rb").read()
        assert data.count(b"\x1f\x8b\x08\x04") - 1 == n  # every block but the header's
    assert _ref(corpus["records_0"]).n_records == 0 and _ref(corpus["records_257"]).n_records == 257
    assert _ref(corpus["tiny_blocks_40k"]).n_records == 1200 and open(corpus["tiny_blocks_40k"], "rb").read().count(b"BC\x02\x00") > 40000
    assert _ref(corpus["fields"]).n_cigar_op.max() == 65535
    assert (_ref(corpus["long_records"]).cols["l_seq"].astype(np.int64) * 3 // 2 > 1 << 20).sum() == 4  # SEQ + QUAL bytes
    for name in DECOYS:
        stream = rr.inflate_bgzf(open(corpus[name], "rb").read())
        assert stream.count(DECOY) == 40


@pytest.mark.parametrize("name", NAMES)
def test_reference_parser_matches_the_host_decoder(corpus, name):
    """The reference against cmbh_extract_tuples: every column, and each record's interval list."""
    ref, host = _ref(corpus[name]), _extract(corpus[name])
    reasons = {why.split(" ")[0] for _, why in ref.declines}
    if reasons & {"unknown", "fixed"}:  # the host decoder raises the reference's read error
        assert host is None
        return
    assert host is not None
    n = ref.n_records
    keep = np.ones(n, dtype=bool)
    keep[np.array([i for i, _ in ref.declines], dtype=np.int64)] = False  # CG behind a placeholder: the host restores the real CIGAR from the tag
    for col, _ in rr.COLUMNS:
        _same(f"{name}: {col}", host[col][keep], ref.cols[col][keep])
    hb = host["iv_begin"].astype(np.int64)
    assert hb.size == n + 1 and hb[0] == 0
    _same(f"{name}: intervals per record", np.diff(hb)[keep], ref.iv_count[keep])
    pick = lambda begin, count: np.concatenate([np.arange(b, b + c) for b, c in zip(begin[keep], count[keep])] or [np.zeros(0, int)])
    rb = np.concatenate([[0], np.cumsum(ref.iv_count)])
    hi, ri = pick(hb[:-1], np.diff(hb)), pick(rb[:-1], ref.iv_count)
    _same(f"{name}: iv_start", host["iv_start"][hi], ref.iv_start[ri])
    _same(f"{name}: iv_len", host["iv_len"][hi], ref.iv_len[ri])


@pytest.mark.parametrize("name", NAMES)
def test_corpus_is_a_valid_contig_input(corpus, name):
    """The host decoder's table equals the oracle's; it fails only where the reference raises a read error."""
    a, o = _table(HOSTCHECK, corpus[name]), _table(ORACLE_BIN, corpus[name])
    assert a.returncode == o.returncode, (a.stderr[-400:], o.stderr[-400:])
    assert a.stdout == o.stdout
    assert o.returncode == (101 if name in READ_ERRORS else 0), o.stderr[-300:]


# ---------------------------------------------------------------------------------------------- GPU half
class _Dev:
    """A device pointer as a byte array (__cuda_array_interface__) for torch to copy."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def _device_columns(batch, n, ni):
    torch.cuda.synchronize()
    out = {}
    for col, dt, cnt in [(c, d, n) for c, d in rr.COLUMNS] + [("iv_begin", np.uint32, n + 1), ("iv_start", np.int32, ni), ("iv_len", np.int32, ni)]:
        nbytes = cnt * np.dtype(dt).itemsize
        raw = torch.as_tensor(_Dev(getattr(batch, col), nbytes), device="cuda").cpu().numpy() if nbytes else np.zeros(0, np.uint8)
        out[col] = raw.view(dt)
    return out


@pytest.fixture(scope="module")
def session():
    import coverm_b200
    s = coverm_b200.Session(device=0, threads=4)
    yield s
    s.close()


def _run(session, path, capfd, monkeypatch):
    monkeypatch.setenv("CMB_PIPELINE_STATS", "1")
    capfd.readouterr()
    res = session.run(["contig", "-m", "mean", "-b", path])
    err = capfd.readouterr().err
    o = _table(ORACLE_BIN, path)
    assert res.status == o.returncode, (res.status, o.returncode, res.err[-400:])
    assert res.out == o.stdout
    return res, [l for l in err.splitlines() if l.startswith("#device_decode")]


@pytest.mark.gpu
@pytest.mark.parametrize("retry", [False, True], ids=["first_pass", "retry_blocks"])
@pytest.mark.parametrize("name", EXACT)
def test_device_columns(corpus, session, capfd, monkeypatch, name, retry):
    import coverm_b200
    if retry:
        monkeypatch.setenv("CMB_DECODE_RETRY_TEST", "1")
    ref = _ref(corpus[name])
    res, lines = _run(session, corpus[name], capfd, monkeypatch)
    s = res.samples[0]
    assert s["device_decode"] == 1 and len(lines) == 1 and lines[0].startswith("#device_decode\tblocks="), lines
    assert s["n_records"] == ref.n_records and s["num_reads"] == ref.n_primary, (s["n_records"], s["num_reads"])
    if ref.n_records == 0:  # nothing to extract: no tuples are left resident
        with pytest.raises(coverm_b200.CmbError):
            session.device_context().last_bgzf_batch()
        return
    batch, n, ni = session.device_context().last_bgzf_batch()
    assert (n, ni) == (ref.n_records, ref.n_intervals)
    got = _device_columns(batch, n, ni)
    for col, _ in rr.COLUMNS:
        _same(f"{name}: {col}", got[col], ref.cols[col])
    _same(f"{name}: iv_begin", got["iv_begin"], np.concatenate([[0], np.cumsum(ref.n_cigar_op)]))
    want_start, want_len = ref.slots()
    _same(f"{name}: iv_start", got["iv_start"], want_start)
    _same(f"{name}: iv_len", got["iv_len"], want_len)
    repairs = int(re.search(r"\trepairs=(\d+)", lines[0]).group(1))
    print(f"{name}: {n} records, {ni} interval slots, repairs={repairs}")
    if name in DECOYS:
        assert repairs > 0, lines  # kd_guess took the decoys; the chain repaired them
    if name == "long_records":
        assert repairs > 0, lines


@pytest.mark.gpu
@pytest.mark.parametrize("name", DECLINE)
def test_device_declines(corpus, session, capfd, monkeypatch, name):
    """Streams the device cannot vouch for go to the host decoder: the table (or the read error) is the oracle's."""
    import coverm_b200
    # a run that ends in the read error leaves its session mid-sample: those get a session of their own
    own = coverm_b200.Session(device=0, threads=4) if name in READ_ERRORS else None
    res, lines = _run(own or session, corpus[name], capfd, monkeypatch)
    assert all(s["device_decode"] == 0 for s in res.samples)
    assert any(l.startswith("#device_decode\tdeclined") for l in lines), lines
    if name == "long_record_small_blocks":
        assert any("record chain did not settle" in l for l in lines), lines
    with pytest.raises(coverm_b200.CmbError):
        (own or session).device_context().last_bgzf_batch()
    if own:
        own.close()


VARIANTS = {"window64": {"CMB_DECODE_WINDOW_KB": "64", "CMB_INFLATE_SERIAL": "0"}, "t1": {"CMB_INFLATE": "t1"}}


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_variant_in_child(variant):
    """The inflate settings are read once per process: each variant runs the corpus in a child process."""
    env = dict(os.environ, **VARIANTS[variant])
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not variant_in_child and not retry_blocks"], env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, f"variant {variant}:\n{r.stdout[-6000:]}\n{r.stderr[-2000:]}"
