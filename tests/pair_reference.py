"""Exact expected results of ReferenceSortedBamFilter::read (filter.rs:86-234) over decoded BAM records, in plain Python.

Restated from the reference's lines -- never from the kernels -- so that the device's mate matching (cmb_pairs.cuh), its
`coverm filter` layout (cmb_filter.cuh) and the pair branch of K1 can be checked against it:
  * singles path (filter.rs:88-116) when only the single-read thresholds apply (filter.rs:48-61);
  * pair path (filter.rs:117-233): an unmapped record is returned at once when filter_out is false (133-135) and never reaches
    the set; secondary and supplementary records are skipped (138-140); an improper pair is returned when filter_out is false
    (141-147); the set of stored first mates is cleared whenever a record reaching it has a new tid (150-162); a record whose
    name is not stored is stored only when its mtid is the current tid (168-184); a record whose name is stored completes
    the pair whatever its mtid (185-223), and a third record of the name is stored again;
  * the predicates (filter.rs:243-336) in float32, with `&&` short-circuiting exactly as written, which decides whether nm()
    (lib.rs:138-158) is reached and panics on a record without an NM tag of type C, S or I.
`run` returns the emitted records in the reference's order (a passing pair as stored mate then second mate, at the second
mate's position) and whether nm() panicked (the records emitted before the panic are then meaningless to the CLI).
"""
import struct
import zlib

import numpy as np

from device_reference import filter_mode

NM_PANIC = "Mapping record encountered that does not have an 'NM' auxiliary tag"
AUX_SIZE = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}


class Record:
    """The fields of one BAM record (SAMv1 4.2) the filter reads."""

    def __init__(self, raw):
        self.raw = raw  # with its 4-byte block_size
        (self.tid, self.pos, l_name, self.mapq, _bin, n_cig, self.flag, self.l_seq, self.mtid, _mpos,
         _tlen) = struct.unpack_from("<iiBBHHHIiii", raw, 4)
        self.qname = raw[36:36 + l_name - 1]
        o = 36 + l_name
        ops = struct.unpack_from("<%dI" % n_cig, raw, o)
        o += 4 * n_cig + (self.l_seq + 1) // 2 + self.l_seq
        # aligned length with D (filter.rs:259-266: M I D X =) and without (filter.rs:302-309: M I X =)
        self.aligned = sum(v >> 4 for v in ops if v & 15 in (0, 1, 2, 7, 8))
        self.aligned_pair = sum(v >> 4 for v in ops if v & 15 in (0, 1, 7, 8))
        self.nm = None  # None: nm() panics
        while o < len(raw):
            tag, ty = raw[o:o + 2], chr(raw[o + 2])
            o += 3
            if ty in "ZH":
                end = raw.index(b"\0", o)
                size = end + 1 - o
            elif ty == "B":
                sub, cnt = chr(raw[o]), struct.unpack_from("<I", raw, o + 1)[0]
                size = 5 + AUX_SIZE[sub] * cnt
            else:
                size = AUX_SIZE[ty]
            if tag == b"NM" and ty in "CSI":
                self.nm = int.from_bytes(raw[o:o + size], "little")
            o += size

    @property
    def name(self):
        return self.qname.decode()


def read_bam(path):
    """(header bytes, [Record]) of a BGZF BAM file, via zlib."""
    raw = open(path, "rb").read()
    data, o = bytearray(), 0
    while o < len(raw):
        bsize = struct.unpack_from("<H", raw, o + 16)[0] + 1
        data += zlib.decompress(raw[o + 18:o + bsize - 8], -15)
        o += bsize
    l_text = struct.unpack_from("<I", data, 4)[0]
    n_ref = struct.unpack_from("<I", data, 8 + l_text)[0]
    p = 12 + l_text
    for _ in range(n_ref):
        p += 8 + struct.unpack_from("<I", data, p)[0]
    header, recs = bytes(data[:p]), []
    while p < len(data):
        bs = struct.unpack_from("<I", data, p)[0]
        recs.append(Record(bytes(data[p:p + 4 + bs])))
        p += 4 + bs
    return header, recs


class NmPanic(Exception):
    pass


def _nm(r):  # lib.rs:138-158
    if r.nm is None:
        raise NmPanic(NM_PANIC)
    return r.nm


def single_read_passes(r, p):  # filter.rs:243-279
    f32 = np.float32
    if p["min_mapq"] != 255 and (r.mapq < p["min_mapq"] or r.mapq == 255):
        return False
    edit = _nm(r)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (r.aligned >= p["min_aligned_length_single"]
                and f32(r.aligned) / f32(r.l_seq) >= f32(p["min_aligned_percent_single"])
                and f32(1.0) - f32(edit) / f32(r.aligned) >= f32(p["min_percent_identity_single"]))


def read_pair_passes(r1, r2, p):  # filter.rs:281-336
    f32 = np.float32
    m = p["min_mapq"]
    if m != 255 and (r1.mapq < m or r2.mapq < m or r1.mapq == 255 or r2.mapq == 255):
        return False
    e1, e2 = _nm(r1), _nm(r2)
    aligned = r1.aligned_pair + r2.aligned_pair
    with np.errstate(divide="ignore", invalid="ignore"):
        return (aligned >= p["min_aligned_length_pair"]
                and f32(aligned) / f32(r1.l_seq + r2.l_seq) >= f32(p["min_aligned_percent_pair"])
                and f32(1.0) - f32(e1 + e2) / f32(aligned) >= f32(p["min_percent_identity_pair"]))


def run(recs, p, filter_out):
    """(emitted record indices in the reference's order, nm_panicked) of ReferenceSortedBamFilter::read over `recs`.
    p: device_reference.default_params(...) with filtering = 1."""
    filter_single, filter_pairs = filter_mode(p)
    out = []
    try:
        if filter_single and not filter_pairs:  # filter.rs:88-116
            for i, r in enumerate(recs):
                unmapped = r.flag & 0x4
                if unmapped and not filter_out:
                    out.append(i)
                    continue
                passes1 = (not unmapped and (p["include_supplementary"] or not r.flag & 0x800)
                           and (p["include_secondary"] or not r.flag & 0x100))
                if passes1 and single_read_passes(r, p) == filter_out:
                    out.append(i)
            return out, False
        first_set, current_reference = {}, -1  # filter.rs:65-66
        for i, r in enumerate(recs):
            if r.flag & 0x4 and not filter_out:  # 133-135
                out.append(i)
                continue
            if r.flag & 0x900:  # 138-140
                continue
            if not r.flag & 0x2:  # 141-147
                if not filter_out:
                    out.append(i)
                continue
            if r.tid != current_reference:  # 150-162
                current_reference = r.tid
                first_set = {}
            j = first_set.pop(r.qname, None)
            if j is None:  # 169-184
                if r.mtid == current_reference:
                    first_set[r.qname] = i
                continue
            stored = recs[j]  # 185-223
            passes = ((not filter_single or (single_read_passes(stored, p) and single_read_passes(r, p)))
                      and read_pair_passes(r, stored, p))
            if passes == filter_out:
                out += [j, i]
        return out, False
    except NmPanic:
        return out, True


def contig_read_counts(recs, p, n_contigs):
    """Per tid, the records `coverm contig` counts (contig.rs:119-159) behind the pair filter (filter_out = true): the emitted
    records that pass the flag filter (lib.rs:59-79) and are mapped.  None when nm() panics, in the filter or on a counted
    record."""
    emitted, panicked = run(recs, p, True)
    if panicked:
        return None
    counts = [0] * n_contigs
    for i in emitted:
        r = recs[i]
        f = r.flag
        if f & 0x4 or (f & 0x100 and not p["include_secondary"]) or (f & 0x800 and not p["include_supplementary"]):
            continue
        if not f & 0x2 and not p["include_improper_pairs"]:
            continue
        if r.nm is None:  # nm(&record), contig.rs:206
            return None
        counts[r.tid] += 1
    return counts

