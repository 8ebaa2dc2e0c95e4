"""Cost of decoding a sample in block slices: `bin/coverm contig -m mean trimmed_mean covered_fraction --timing` on a
generated config-2 file (bench.py --config 2: 500 000 contigs, 10 M reads) decoded whole, forced into 2, 4 and 8 slices
(CMB_DECODE_MEM_LIMIT_MB), and on the host pipeline (CMB_HOST_DECODE=1), which is where such a sample went before slicing.  The
runs alternate, `--rounds` times each; every output must be identical.  Prints one JSON line with each way's decode and total
seconds (median and all rounds, from the #timing line), its slice count, and the card's name and power limit, read in the same
run.

    python scripts/sliced_decode_bench.py [--reads 10000000] [--contigs 500000] [--rounds 3] [--bam FILE] [--out DIR]

Needs a GPU and a built tree (__graft_entry__.build()).  The generated file goes to a temporary directory and is removed."""
import argparse
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

COVERM = os.path.join(ROOT, "coverm_b200", "bin", "coverm")
BAMGEN = os.path.join(ROOT, "coverm_b200", "bin", "bamgen")
GEN_CONTIG = ["--median-len", "4000", "--sigma", "0.8", "--min-len", "1000", "--max-len", "2000000"]  # bench.py's config 2


def inflated_bytes(path):
    """the file's inflated size: the ISIZE footers of its BGZF blocks"""
    import struct
    raw, o, n = open(path, "rb").read(), 0, 0
    while o < len(raw):
        bsize = struct.unpack_from("<H", raw, o + 16)[0] + 1
        n += struct.unpack_from("<I", raw, o + bsize - 4)[0]
        o += bsize
    return n


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(bam, env):
    argv = [COVERM, "contig", "-m", "mean", "trimmed_mean", "covered_fraction", "--timing", "-t", "16", "-b", bam]
    p = subprocess.run(argv, capture_output=True, text=True, env=dict(os.environ, CMB_PIPELINE_STATS="1", **env))
    if p.returncode:
        raise SystemExit(f"coverm failed ({p.returncode}): {p.stderr[-2000:]}")
    t = re.search(r"^#timing\t.*\ttotal_s=([0-9.e+-]+)\tdecode_s=([0-9.e+-]+)", p.stderr, re.M)
    s = re.search(r"^#decode_slices\tslices=(\d+)", p.stderr, re.M)
    host = bool(re.search(r"^#pipeline\t", p.stderr, re.M))
    return p.stdout, float(t.group(1)), float(t.group(2)), int(s.group(1)) if s else (0 if host else 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--contigs", type=int, default=500_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bam", default=None, help="an existing file instead of a generated one")
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/sliced_decode_bench.json")
    args = ap.parse_args()
    tmp = None
    try:
        bam = args.bam
        if not bam:
            tmp = tempfile.mkdtemp(prefix="sliced_bench_")
            bam = os.path.join(tmp, "c2.bam")
            subprocess.run([BAMGEN, "--out", bam, "--contigs", str(args.contigs), "--reads", str(args.reads), "--seed", "1",
                            "--threads", "16"] + GEN_CONTIG, check=True, capture_output=True)
        whole_bytes = os.path.getsize(bam) + inflated_bytes(bam)
        # the first slice takes half the room and the others about 1/1.2 of it: room for n slices
        ways = {"whole": {}}
        for n in (2, 4, 8):
            ways[f"slices_{n}"] = {"CMB_DECODE_MEM_LIMIT_MB": str(max(64, int(whole_bytes / (n - 0.5) / 1.15 / (1 << 20))))}
        ways["host"] = {"CMB_HOST_DECODE": "1"}
        res = {w: {"total_s": [], "decode_s": [], "slices": None} for w in ways}
        want = None
        for _ in range(args.rounds):
            for w, env in ways.items():
                out, total, decode, n = run(bam, env)
                if want is None:
                    want = out
                if out != want:
                    raise SystemExit(f"{w}: output differs from the first run")
                res[w]["total_s"].append(round(total, 4))
                res[w]["decode_s"].append(round(decode, 4))
                res[w]["slices"] = n
        for w in res:
            res[w]["total_median_s"] = statistics.median(res[w]["total_s"])
            res[w]["decode_median_s"] = statistics.median(res[w]["decode_s"])
        line = {"what": "coverm contig -m mean trimmed_mean covered_fraction --timing, decoded whole / in n slices / on the host",
                "reads": args.reads, "contigs": args.contigs, "bam_bytes": os.path.getsize(bam), "whole_decode_bytes": whole_bytes,
                "card": card(), "ways": res, "limits_mb": {w: e.get("CMB_DECODE_MEM_LIMIT_MB") for w, e in ways.items()}}
        print(json.dumps(line))
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "sliced_decode_bench.json"), "w") as f:
                f.write(json.dumps(line) + "\n")
    finally:
        if tmp:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
