"""The oracle side of `--sharded`: the reference's reader restated (oracle/shard_oracle) writes the winners of the shards as one
BAM named after the shards' stems joined with '|', and oracle/coverm_oracle reads it like any sample -- as the reference feeds
its desharded stream through `samtools sort` into the ordinary coverage loop (coverm.rs:187-239, 565-578).  With a read filter
the reference ignores --sharded (coverm.rs:168-187): every BAM is then its own sample."""
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_BIN = os.path.join(ROOT, "oracle", "coverm_oracle")
SHARD_ORACLE_BIN = os.path.join(ROOT, "oracle", "shard_oracle")

_THRESHOLDS = ("--min-read-aligned-length", "--min-read-percent-identity", "--min-read-aligned-percent", "--min-read-aligned-length-pair",
               "--min-read-percent-identity-pair", "--min-read-aligned-percent-pair")


def _value(argv, *names):
    for i, a in enumerate(argv[:-1]):
        if a in names:
            return argv[i + 1]
    return None


def doing_filtering(argv):
    """FilterParameters::doing_filtering (coverm.rs:1695-1703), with metabat's identity threshold (coverm.rs:1680-1693)"""
    if any(v is not None and float(v) > 0 for v in (_value(argv, t) for t in _THRESHOLDS)):
        return True
    if _value(argv, "--min-mapq") is not None:
        return True
    return argv[0] == "contig" and "metabat" in argv


def _split(argv):
    """argv without --sharded / --exclude-genomes-from-deshard FILE, the BAM list, and the position the list stood at"""
    rest, bams, exclude, at, i = [], [], None, None, 0
    while i < len(argv):
        a = argv[i]
        if a == "--sharded":
            i += 1
        elif a == "--exclude-genomes-from-deshard":
            exclude = argv[i + 1]
            i += 2
        elif a in ("-b", "--bam-files"):
            at = len(rest)
            i += 1
            while i < len(argv) and not (argv[i].startswith("-") and len(argv[i]) > 1):
                bams.append(argv[i])
                i += 1
        else:
            rest.append(a)
            i += 1
    return rest, bams, exclude, at


def run_oracle(argv, timeout=1800):
    """`coverm <argv>` as the reference computes it, --sharded included"""
    rest, bams, exclude, at = _split(argv)
    if "--sharded" not in argv or doing_filtering(argv):
        return subprocess.run([ORACLE_BIN] + rest[:at] + ["-b"] + bams + rest[at:], capture_output=True, text=True, timeout=timeout)
    with tempfile.TemporaryDirectory() as td:
        stem = "|".join(os.path.splitext(os.path.basename(b))[0] for b in bams)
        desharded = os.path.join(td, stem + ".bam")
        cmd = [SHARD_ORACLE_BIN, "--out", desharded]
        if argv[0] == "genome":
            for flag in ("-s", "--separator", "--genome-definition"):
                v = _value(argv, flag)
                if v is not None:
                    cmd += [flag, v]
            if "--single-genome" in argv:
                cmd.append("--single-genome")
            if exclude is not None:
                cmd += ["--exclude-genomes-from-deshard", exclude]
        p = subprocess.run(cmd + bams, capture_output=True, text=True, timeout=timeout)
        if p.returncode:
            return p
        return subprocess.run([ORACLE_BIN] + rest[:at] + ["-b", desharded] + rest[at:], capture_output=True, text=True, timeout=timeout)
