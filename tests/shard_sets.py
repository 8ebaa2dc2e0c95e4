"""Seeded sets of sharded BAMs for `--sharded`: one read set "mapped" to K disjoint reference shards, each shard a
read-name-sorted BAM holding every pair.

rich_set: small and varied -- ties, unmapped mates and pairs, secondary and supplementary records between the primaries,
AS of type C and S, genomes meant for exclusion.  big_set: fixed-size records laid out with numpy, for millions of pairs."""
import os
import random

import numpy as np

import bam_writer as bw


def shard_contigs(k, n_genomes=2, contigs_per_genome=2, seed=0):
    rng = random.Random(seed * 1000 + k)
    return [(f"s{k}g{g}~c{c}", rng.randint(3000, 12000)) for g in range(n_genomes) for c in range(contigs_per_genome)]


def rich_set(out_dir, K, n_pairs, seed, exclude_genomes=("s0g1",)):
    """Writes shard0.bam .. shard{K-1}.bam, an exclusion list, a genome definition and a GFF; returns their paths.
    Shards other than the last may hold excluded genomes, so every pair keeps a candidate."""
    rng = random.Random(seed)
    contigs = [shard_contigs(k, seed=seed) for k in range(K)]
    recs = [[] for _ in range(K)]

    def aligned(k, rlen):
        tid = rng.randrange(len(contigs[k]))
        pos = rng.randrange(0, contigs[k][tid][1] - rlen - 10)
        shape = rng.choice([[("M", rlen)], [("S", 5), ("M", rlen - 5)], [("M", 40), ("I", 2), ("M", rlen - 42)],
                            [("M", 30), ("D", 3), ("M", rlen - 30)]])
        return tid, pos, shape

    def as_tag(score):
        return ("AS", "S", score) if (score > 255 or rng.random() < 0.3) else ("AS", "C", score)

    for i in range(n_pairs):
        name = "q%08d" % i
        rlen = rng.choice([100, 150])
        tie_score = rng.choice([60, 80, 100, 300])
        for k in range(K):
            mates = []
            for m in range(2):
                r = rng.random()
                if r < 0.08:
                    mates.append(None)  # unmapped
                else:
                    mates.append(aligned(k, rlen))
            if rng.random() < 0.04:
                mates = [None, None]
            for m in range(2):
                me, other = mates[m], mates[1 - m]
                flag = 0x1 | (0x40 if m == 0 else 0x80)
                if me is None:
                    flag |= 0x4
                if other is None:
                    flag |= 0x8
                if me and other and me[0] == other[0]:
                    flag |= 0x2
                tags = []
                if me is not None:
                    score = tie_score if rng.random() < 0.5 else rng.randint(20, 320)
                    tags = [("NM", "C", rng.randint(0, 6)), as_tag(score)]
                    tid, pos, cig = me
                else:
                    tid, pos, cig = (other[0], other[1], []) if other else (-1, -1, [])
                    if rng.random() < 0.5:
                        tags = [("AS", "C", 0)]
                recs[k].append(bw.record(tid, pos, cig, flag=flag, qname=name, l_seq=rlen if cig else 0, tags=tags))
                if me is not None and rng.random() < 0.06:  # a secondary or supplementary between the primaries
                    t2, p2, c2 = aligned(k, rlen)
                    extra = 0x100 if rng.random() < 0.5 else 0x800
                    recs[k].append(bw.record(t2, p2, c2, flag=(flag & ~0x2) | extra, qname=name,
                                             tags=[("AS", "i", 5), ("NM", "S", 1)]))
    paths = []
    for k in range(K):
        p = os.path.join(out_dir, f"shard{k}.bam")
        with open(p, "wb") as f:
            f.write(bw.bgzf(bw.bam_stream(contigs[k], recs[k], text="@HD\tVN:1.6\tSO:queryname\n"), seed=seed + k))
        paths.append(p)
    excl = os.path.join(out_dir, "excluded.txt")
    with open(excl, "w") as f:
        f.write("\n".join(exclude_genomes) + "\n\n")
    definition = os.path.join(out_dir, "shards.definition")
    gff = os.path.join(out_dir, "shards.gff")
    with open(definition, "w") as d, open(gff, "w") as g:
        g.write("##gff-version 3\n")
        for k in range(K):
            for n, length in contigs[k]:
                d.write(f"{n.split('~')[0]}\t{n}\n")
                g.write(f"{n}\ttest\tgene\t1\t{length // 2}\t.\t+\t.\tID={n}_a\n")
                g.write(f"{n}\ttest\tgene\t{length // 3}\t{length}\t.\t-\t.\tID={n}_b\n")
    return dict(shards=paths, excluded=excl, definition=definition, gff=gff)


REC_BYTES = 60  # fixed layout of big_set's records: 32 B core, 12 B name, one CIGAR op, AS:C, NM:C, no SEQ / QUAL


def big_records(tid, pos, flag, name_idx, as_val, nm, read_len):
    """n fixed-size BAM records (numpy columns of equal length) as one byte string."""
    n = len(tid)
    dt = np.dtype([("bs", "<u4"), ("tid", "<i4"), ("pos", "<i4"), ("lname", "u1"), ("mapq", "u1"), ("bin", "<u2"), ("ncig", "<u2"),
                   ("flag", "<u2"), ("lseq", "<u4"), ("mtid", "<i4"), ("mpos", "<i4"), ("tlen", "<i4"), ("name", "S12"), ("cig", "<u4"),
                   ("as_tag", "S3"), ("as", "u1"), ("nm_tag", "S3"), ("nm", "u1")])
    assert dt.itemsize == REC_BYTES
    a = np.zeros(n, dt)
    a["bs"] = REC_BYTES - 4
    a["tid"] = tid
    a["pos"] = pos
    a["lname"] = 12
    a["mapq"] = 60
    a["ncig"] = 1
    a["flag"] = flag
    a["mtid"] = -1
    a["mpos"] = -1
    a["name"] = np.char.add(b"p", np.char.zfill(name_idx.astype("S10"), 10))
    a["cig"] = (read_len << 4) | 0
    a["as_tag"] = b"ASC"
    a["as"] = as_val
    a["nm_tag"] = b"NMC"
    a["nm"] = nm
    return a.tobytes()


def big_set(out_dir, K, n_pairs, seed, contig_len=2_000_000, contigs_per_shard=8, block_bytes=0xFF00, level=1):
    """K shards of n_pairs proper pairs (100-base mates, AS in 60..100 so that ties are common); returns the shard paths."""
    rng = np.random.default_rng(seed)
    paths = []
    names = np.repeat(np.arange(n_pairs, dtype=np.int64), 2)
    for k in range(K):
        tid = np.repeat(rng.integers(0, contigs_per_shard, n_pairs, dtype=np.int32), 2)
        pos = rng.integers(0, contig_len - 400, 2 * n_pairs, dtype=np.int32)
        flag = np.tile(np.array([0x1 | 0x2 | 0x40, 0x1 | 0x2 | 0x80], np.uint16), n_pairs)
        as_val = rng.integers(6, 11, 2 * n_pairs).astype(np.uint8) * 10
        nm = rng.integers(0, 5, 2 * n_pairs).astype(np.uint8)
        body = big_records(tid, pos, flag, names, as_val, nm, 100)
        contigs = [(f"s{k}g{c // 2}~c{c}", contig_len) for c in range(contigs_per_shard)]
        stream = bw.bam_stream(contigs, [], text="@HD\tVN:1.6\tSO:queryname\n") + body
        p = os.path.join(out_dir, f"big{k}.bam")
        with open(p, "wb") as f:
            f.write(bw.bgzf(stream, level=level, block_sizes=block_bytes))
        paths.append(p)
    return paths
