"""An exact parser of the record decoder's contract: what the device decode (cmb_decode.cuh: the record chain and kd_extract)
and the host decoder must make of a BAM file's records, column by column of cmb_read_batch (include/coverm_b200.h).

Written from SAMv1 §4.1-4.2 and the cmb_read_batch comments, in plain Python integers (no overflow anywhere) and numpy; it
shares no code with either decoder.  parse(path) inflates the BGZF file with zlib, skips the header and returns, per record:

- the columns tid, pos, flag, mapq, nm_state, nm, l_seq, aligned, del_, ins (the names of tests/device_scenarios.py);
- n_cigar_op, the record's share of the interval slots the device reserves (one per CIGAR operation);
- its M/=/X intervals (start, len) in CIGAR order, flattened into iv_start / iv_len with iv_count per record.

Interval rules: the cursor starts at pos; M, = and X add an interval at the cursor, then advance the cursor and `aligned`;
D advances the cursor, `del` and `aligned`; N advances the cursor; I adds to `ins` and `aligned`; S, H and P do nothing.  An
interval whose cursor is below 0 starts at -1 (K1's bounds check rejects it); a start above INT32_MAX is clamped to it.

NM: the first NM tag wins.  Types C, S and I give nm_state 1 and the value, any other type nm_state 2, no NM tag 0.

Records the device must decline (the whole stream then goes to the host decoder) are listed in `declines` as (record index,
reason): an unknown aux type, fixed fields (name, CIGAR, SEQ, QUAL) that overrun block_size, and a CG:B tag behind the
`<l_seq>S...` placeholder CIGAR of a mapped record (tid >= 0 and pos >= 0): its real CIGAR (SAMv1 §4.2.2, more than 65 535
operations) does not fit the n_cigar_op slot reservation."""
import struct
import zlib
from dataclasses import dataclass

import numpy as np

INT32_MAX = 2 ** 31 - 1
IV_PAD = -2 ** 31  # CMB_IV_PAD: an unused interval slot

AUX_FIXED = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}
B_ELEM = {"c": 1, "C": 1, "s": 2, "S": 2}  # every other subtype: 4 bytes
COLUMNS = [("tid", np.int32), ("pos", np.int32), ("flag", np.uint16), ("mapq", np.uint8), ("nm_state", np.uint8),
           ("nm", np.uint32), ("l_seq", np.uint32), ("aligned", np.uint32), ("del_", np.uint32), ("ins", np.uint32)]


def inflate_bgzf(data):
    """The uncompressed stream of a BGZF file (SAMv1 §4.1), block by block, each checked against its CRC-32 and ISIZE."""
    out, o = [], 0
    while o < len(data):
        assert data[o:o + 4] == b"\x1f\x8b\x08\x04", f"no BGZF block header at {o}"
        xlen = struct.unpack_from("<H", data, o + 10)[0]
        x, bsize = o + 12, None
        while x < o + 12 + xlen:
            si1, si2, slen = data[x], data[x + 1], struct.unpack_from("<H", data, x + 2)[0]
            if (si1, si2, slen) == (66, 67, 2):
                bsize = struct.unpack_from("<H", data, x + 4)[0]
            x += 4 + slen
        assert bsize is not None, f"gzip member at {o} has no BC field"
        end = o + bsize + 1
        payload = zlib.decompressobj(-15).decompress(data[o + 12 + xlen:end - 8])
        crc, isize = struct.unpack_from("<II", data, end - 8)
        assert len(payload) == isize and zlib.crc32(payload) == crc, f"BGZF block at {o} does not check"
        out.append(payload)
        o = end
    return b"".join(out)


def records_start(stream):
    """(n_ref, offset of the first record) of an uncompressed BAM stream."""
    assert stream[:4] == b"BAM\1"
    l_text = struct.unpack_from("<I", stream, 4)[0]
    o = 8 + l_text
    n_ref = struct.unpack_from("<I", stream, o)[0]
    o += 4
    for _ in range(n_ref):
        l_name = struct.unpack_from("<I", stream, o)[0]
        o += 8 + l_name
    return n_ref, o


def _aux_size(body, p, end, ty):
    """Bytes of the value of an aux field of type `ty` at body[p:], or None for an unknown type.  A Z / H string without
    its NUL, or a B array header cut short, takes the rest of the record."""
    if ty in AUX_FIXED:
        return AUX_FIXED[ty]
    if ty in "ZH":
        nul = body.find(b"\0", p, end)
        return end - p if nul < 0 else nul - p + 1
    if ty == "B":
        if p + 5 > end:
            return end - p
        sub, count = chr(body[p]), struct.unpack_from("<I", body, p + 1)[0]
        return 5 + B_ELEM.get(sub, 4) * count
    return None


def parse_record(body, start, end):
    """One record whose fields are body[start:end] (after block_size): (fields dict, intervals, decline reason or None)."""
    tid, pos, l_name, mapq, _bin, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHI", body, start)
    rec = dict(tid=tid, pos=pos, flag=flag, mapq=mapq, l_seq=l_seq, n_cigar_op=n_cig, nm_state=0, nm=0, aligned=0, del_=0,
               ins=0)
    cig = start + 32 + l_name
    aux = cig + 4 * n_cig + (l_seq + 1) // 2 + l_seq
    if aux > end:
        return rec, [], "fixed fields overrun block_size"
    ops = struct.unpack_from("<%dI" % n_cig, body, cig)
    ivs, cursor = [], pos
    for v in ops:
        op, n = v & 0xF, v >> 4
        if op in (0, 7, 8):  # M = X
            ivs.append((-1 if cursor < 0 else min(cursor, INT32_MAX), n))
            cursor += n
            rec["aligned"] += n
        elif op == 2:  # D
            cursor += n
            rec["del_"] += n
            rec["aligned"] += n
        elif op == 3:  # N
            cursor += n
        elif op == 1:  # I
            rec["ins"] += n
            rec["aligned"] += n
    placeholder = n_cig > 0 and ops[0] & 0xF == 4 and ops[0] >> 4 == l_seq and tid >= 0 and pos >= 0
    p, decline = aux, None
    while p + 3 <= end:
        tag, ty = body[p:p + 2], chr(body[p + 2])
        p += 3
        size = _aux_size(body, p, end, ty)
        if size is None:
            decline = "unknown aux type %r" % ty
            break
        if tag == b"NM" and rec["nm_state"] == 0:
            if ty in "CSI":
                rec["nm_state"], rec["nm"] = 1, int.from_bytes(body[p:p + AUX_FIXED[ty]], "little")
            else:
                rec["nm_state"] = 2
        if tag == b"CG" and ty == "B" and placeholder:
            decline = decline or "CG:B behind a placeholder CIGAR"
        p += size
    return rec, ivs, decline


@dataclass
class Parsed:
    n_ref: int
    records_at: int
    cols: dict          # COLUMNS, numpy arrays
    n_cigar_op: np.ndarray
    iv_count: np.ndarray  # M/=/X intervals per record
    iv_start: np.ndarray  # all records' intervals in record and CIGAR order (int64)
    iv_len: np.ndarray
    declines: list      # (record index, reason)

    @property
    def n_records(self):
        return len(self.n_cigar_op)

    @property
    def n_intervals(self):  # interval slots the device reserves: one per CIGAR operation
        return int(self.n_cigar_op.sum())

    @property
    def n_primary(self):  # neither secondary nor supplementary
        return int(((self.cols["flag"].astype(np.int64) & 0x900) == 0).sum())

    def slots(self, iv_begin=None):
        """(iv_start, iv_len) of the device's interval slots: record i owns [iv_begin[i], iv_begin[i + 1]) (by default the
        running sum of n_cigar_op); its intervals come first in CIGAR order, every other slot is (CMB_IV_PAD, 0)."""
        if iv_begin is None:
            iv_begin = np.concatenate([[0], np.cumsum(self.n_cigar_op, dtype=np.int64)])
        iv_begin = np.asarray(iv_begin, dtype=np.int64)
        start = np.full(int(iv_begin[-1]), IV_PAD, dtype=np.int64)
        length = np.zeros(int(iv_begin[-1]), dtype=np.int64)
        rec = np.repeat(np.arange(self.n_records), self.iv_count)
        first = np.concatenate([[0], np.cumsum(self.iv_count, dtype=np.int64)])[:-1]
        at = iv_begin[:-1][rec] + (np.arange(len(rec)) - first[rec])
        start[at] = self.iv_start
        length[at] = self.iv_len
        return start, length


def parse(path_or_bytes):
    data = path_or_bytes
    if isinstance(path_or_bytes, str):
        with open(path_or_bytes, "rb") as f:
            data = f.read()
    stream = inflate_bgzf(data)
    n_ref, o = records_start(stream)
    records_at = o
    recs, counts, starts, lens, declines = [], [], [], [], []
    while o < len(stream):
        assert o + 4 <= len(stream), "a record's block_size is cut short"
        block_size = struct.unpack_from("<I", stream, o)[0]
        assert block_size >= 32 and o + 4 + block_size <= len(stream), f"record at {o} runs past the stream"
        rec, ivs, decline = parse_record(stream, o + 4, o + 4 + block_size)
        if decline:
            declines.append((len(recs), decline))
        recs.append(rec)
        counts.append(len(ivs))
        starts += [s for s, _ in ivs]
        lens += [n for _, n in ivs]
        o += 4 + block_size
    cols = {name: np.array([r[name] for r in recs], dtype=dt) for name, dt in COLUMNS}
    return Parsed(n_ref, records_at, cols, np.array([r["n_cigar_op"] for r in recs], dtype=np.int64), np.array(counts, dtype=np.int64),
                  np.array(starts, dtype=np.int64), np.array(lens, dtype=np.int64), declines)
