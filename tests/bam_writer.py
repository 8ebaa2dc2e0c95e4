"""A small BAM/BGZF writer for tests: full control over the things a decoder can trip on — deflate level (0 = stored
blocks), BGZF block sizes (records straddling many blocks, blocks holding no record start at all), empty blocks, a
missing EOF marker, long reads, aux tags of every type in front of NM.  Written from the SAM/BAM specification (SAMv1
§4.1-4.2); not derived from any htslib code."""
import random
import struct
import zlib

CIGAR_OPS = "MIDNSHP=X"


def bgzf_block(payload, level):
    co = zlib.compressobj(level, zlib.DEFLATED, -15)
    data = co.compress(payload) + co.flush()
    bsize = 12 + 6 + len(data) + 8 - 1
    assert bsize < 65536, "payload too large for one BGZF block at this level"
    return (b"\x1f\x8b\x08\x04" + b"\0\0\0\0" + b"\0\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, bsize) + data +
            struct.pack("<II", zlib.crc32(payload) & 0xFFFFFFFF, len(payload)))


BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def bgzf(stream, level=6, block_sizes=None, eof=True, empty_block_every=0, seed=0):
    """Cut `stream` into BGZF blocks.  block_sizes: None (0xff00 bytes each), an int, or (lo, hi) for random sizes."""
    rng = random.Random(seed)
    out, o, k = [], 0, 0
    while o < len(stream):
        if block_sizes is None:
            n = 0xFF00
        elif isinstance(block_sizes, int):
            n = block_sizes
        else:
            n = rng.randint(*block_sizes)
        if level == 0:
            n = min(n, 65000)  # stored blocks add 5 bytes per 65535
        out.append(bgzf_block(stream[o:o + n], level))
        o += n
        k += 1
        if empty_block_every and k % empty_block_every == 0:
            out.append(bgzf_block(b"", level))
    if eof:
        out.append(BGZF_EOF)
    return b"".join(out)


def bgzf_cuts(stream, cuts, level=6, eof=True):
    """Cut `stream` into BGZF blocks that end at each offset of the sorted list `cuts` (a repeated offset gives an empty
    block there), then into blocks of 0xff00 bytes after the last cut."""
    out, o = [], 0
    for c in list(cuts) + list(range(cuts[-1] + 0xFF00 if cuts else 0xFF00, len(stream), 0xFF00)) + [len(stream)]:
        assert o <= c <= len(stream), (o, c)
        if c > o or (c == o and out and c < len(stream)):
            out.append(bgzf_block(stream[o:c], level))
        o = c
    if eof:
        out.append(BGZF_EOF)
    return b"".join(out)


def aux_bytes(tags):
    """tags: list of (tag, type, value); type in AcCsSiIfZHB (B takes (subtype, [values]))."""
    out = bytearray()
    for tag, ty, val in tags:
        out += tag.encode() + ty.encode()
        if ty == "A":
            out += val.encode()
        elif ty in "cCsSiIf":
            out += struct.pack("<" + {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}[ty], val)
        elif ty in "ZH":
            out += val.encode() + b"\0"
        elif ty == "B":
            sub, vals = val
            out += sub.encode() + struct.pack("<I", len(vals))
            out += struct.pack("<%d%s" % (len(vals), {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}[sub]), *vals)
        else:
            raise ValueError(ty)
    return bytes(out)


def record(tid, pos, cigar, flag=0, mapq=60, qname="r", l_seq=None, mtid=-1, mpos=-1, tlen=0, tags=(("NM", "C", 0),), seq_byte=0x11,
           qual_byte=30, rng=None, qual=None):
    """cigar: list of (op_char, len).  qual: the QUAL bytes (l_seq of them) instead of `qual_byte` repeated."""
    ops = [(CIGAR_OPS.index(c), n) for c, n in cigar]
    if l_seq is None:
        l_seq = sum(n for o, n in ops if o in (0, 1, 4, 7, 8))
    name = qname.encode() + b"\0"
    body = struct.pack("<iiBBHHHIiii", tid, pos, len(name), mapq, 4680, len(ops), flag, l_seq, mtid, mpos, tlen)
    body += name + b"".join(struct.pack("<I", (n << 4) | o) for o, n in ops)
    if qual is not None:
        assert len(qual) == l_seq
        body += bytes([seq_byte]) * ((l_seq + 1) // 2) + bytes(qual)
    elif rng is None:
        body += bytes([seq_byte]) * ((l_seq + 1) // 2) + bytes([qual_byte]) * l_seq
    else:  # incompressible-ish SEQ, QUAL from a 40-letter alphabet
        body += rng.randbytes((l_seq + 1) // 2) + bytes(b % 40 for b in rng.randbytes(l_seq))
    body += aux_bytes(list(tags))
    return struct.pack("<I", len(body)) + body


def bam_stream(contigs, records, text=""):
    """contigs: list of (name, length); records: list of record() byte strings (already sorted)."""
    if not text:
        text = "@HD\tVN:1.6\tSO:coordinate\n" + "".join(f"@SQ\tSN:{n}\tLN:{l}\n" for n, l in contigs)
    t = text.encode()
    out = bytearray(b"BAM\1" + struct.pack("<I", len(t)) + t + struct.pack("<I", len(contigs)))
    for n, l in contigs:
        nb = n.encode() + b"\0"
        out += struct.pack("<I", len(nb)) + nb + struct.pack("<I", l)
    for r in records:
        out += r
    return bytes(out)


def random_records(contigs, n, seed, read_len=(50, 300), long_every=0, long_len=120000, rich_tags=False, homopolymer=False):
    """Sorted records with a mix of CIGAR shapes; every `long_every`-th read is `long_len` bases (spans BGZF blocks)."""
    rng = random.Random(seed)
    recs = []
    for i in range(n):
        tid = rng.randrange(len(contigs))
        L = contigs[tid][1]
        rl = long_len if long_every and i % long_every == long_every - 1 else rng.randint(*read_len)
        rl = max(10, min(rl, L))
        shape = rng.random()
        if shape < 0.6:
            cig = [("M", rl)]
        elif shape < 0.7:
            a = rng.randint(1, rl - 2)
            cig = [("M", a), ("D", rng.randint(1, 5)), ("M", rl - a)]
        elif shape < 0.8:
            a = rng.randint(1, rl - 3)
            cig = [("M", a), ("I", 2), ("M", rl - a - 2)]
        elif shape < 0.9:
            s = rng.randint(1, rl // 2)
            cig = [("S", s), ("=", rl - s)]
        else:
            a = rng.randint(1, rl - 2)
            cig = [("X", a), ("N", rng.randint(1, 50)), ("M", rl - a)]
        # every aligned block must START inside the contig (the reference indexes ups_and_downs[cursor]); ends may overhang
        ref_before_last = sum(n for c, n in cig[:-1] if c in "MDN=X")
        if ref_before_last >= L:
            cig, ref_before_last = [("M", rl)], 0
        pos = rng.randrange(0, L - ref_before_last)
        flag = rng.choice([0, 16, 99, 147, 83, 163, 65, 129, 256, 2048, 2064, 0, 0, 16])
        nm = rng.randint(0, 5)
        if rich_tags:
            tags = [("RG", "Z", "grp%d" % (i % 3)), ("XA", "A", "q"), ("ZB", "B", ("S", [1, 2, 3, i % 65536])), ("XS", "i", -i),
                    ("XF", "f", 1.5), ("MD", "Z", "10A5^AC6" * rng.randint(1, 4)), ("NM", rng.choice("CSI"), nm), ("XH", "H", "1AE301")]
        else:
            tags = [("NM", "C", nm)]
        recs.append((tid, pos, record(tid, pos, cig, flag=flag, mapq=rng.choice([0, 3, 20, 30, 60, 255]), qname="q%07d" % i, tags=tags,
                                      rng=None if homopolymer else rng)))
    recs.sort(key=lambda r: (r[0], r[1]))
    return [r[2] for r in recs]
