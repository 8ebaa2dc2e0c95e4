"""Cost of `coverm filter` on a sample decoded whole, in block slices, on the host, and with the output compressed on the GPU:
`bin/coverm filter --proper-pairs-only --min-read-percent-identity-pair 95 --timing` on a generated config-2 file (bench.py
--config 2: 500 000 contigs, 10 M reads) decoded whole, under CMB_DECODE_MEM_LIMIT_MB limits that give about 3 and about 8
slices, on the host (CMB_HOST_DECODE=1), which is where such a sample went before the filter took slices, and decoded whole
with `--device-deflate` (the output BAM deflated on the GPU).  The ways alternate, `--rounds` times each; every output file of
the default writer must be byte-identical, and so must every `--device-deflate` file.  Prints one JSON line with each way's
wall seconds, output file bytes, peak resident memory of the coverm process, its `#filter` / `#filter_slices` / `#deflate`
lines, and the card's name and power limit, read in the same run; for the device way also the file's size over the default
file's, the deflate kernels' milliseconds and the raw GB/s through them.

    python scripts/filter_bench.py [--reads 10000000] [--contigs 500000] [--rounds 2] [--ways whole,device_deflate] [--bam FILE] [--out DIR]

Needs a GPU and a built tree (__graft_entry__.build()).  Generated and written files go to a temporary directory and are
removed."""
import argparse
import hashlib
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sliced_decode_bench import BAMGEN, COVERM, GEN_CONTIG, card, inflated_bytes  # noqa: E402

FILTER = ["--proper-pairs-only", "--min-read-percent-identity-pair", "95"]


def run(bam, out, env, tmp, extra=()):
    """wall seconds, peak RSS (MB), the #filter, #filter_slices and #deflate lines, and the output's digest and bytes"""
    err_path = os.path.join(tmp, "stderr.txt")
    with open(err_path, "w") as err:
        t0 = time.perf_counter()
        p = subprocess.Popen([COVERM, "filter", "-b", bam, "-o", out, "--timing", "-t", "16"] + FILTER + list(extra), stdout=subprocess.DEVNULL, stderr=err,
                             env=dict(os.environ, CMB_PIPELINE_STATS="1", **env))
        _, status, ru = os.wait4(p.pid, 0)
        wall = time.perf_counter() - t0
    text = open(err_path).read()
    if status:
        raise SystemExit(f"coverm filter failed ({status}): {text[-2000:]}")
    lines = [l for l in text.splitlines() if l.startswith("#filter") or l.startswith("#deflate")]
    s = re.search(r"^#filter_slices\tslices=(\d+)", text, re.M)
    with open(out, "rb") as f:
        data = f.read()
    os.remove(out)
    return wall, ru.ru_maxrss / 1024.0, lines, int(s.group(1)) if s else None, hashlib.sha256(data).hexdigest(), len(data)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--contigs", type=int, default=500_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--ways", default=None, help="comma-separated subset of whole,slices_3,slices_8,host,device_deflate")
    ap.add_argument("--bam", default=None, help="an existing file instead of a generated one")
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/filter_bench.json")
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="filter_bench_")
    try:
        bam = args.bam
        if not bam:
            bam = os.path.join(tmp, "c2.bam")
            subprocess.run([BAMGEN, "--out", bam, "--contigs", str(args.contigs), "--reads", str(args.reads), "--seed", "1",
                            "--threads", "16"] + GEN_CONTIG, check=True, capture_output=True)
        whole_bytes = os.path.getsize(bam) + inflated_bytes(bam)
        # a slice also holds its tuples, mate arrays and filter output: about 1.2 times its compressed + inflated bytes beside
        # them, so n slices need about 2.2 / n of the whole decode's bytes (the counts reached are reported)
        ways = {"whole": {}}
        for n in (3, 8):
            ways[f"slices_{n}"] = {"CMB_DECODE_MEM_LIMIT_MB": str(max(64, int(whole_bytes * 2.2 / n / (1 << 20))))}
        ways["host"] = {"CMB_HOST_DECODE": "1"}
        ways["device_deflate"] = {}
        if args.ways:
            ways = {w: ways[w] for w in args.ways.split(",")}
        res = {w: {"wall_s": [], "peak_rss_mb": [], "file_bytes": None, "slices": None, "lines": None} for w in ways}
        want = {}
        out = os.path.join(tmp, "out.bam")
        for _ in range(args.rounds):
            for w, env in ways.items():
                dev = w == "device_deflate"
                wall, rss, lines, n, digest, size = run(bam, out, env, tmp, ["--device-deflate"] if dev else [])
                want.setdefault(dev, digest)
                if digest != want[dev]:
                    raise SystemExit(f"{w}: output file differs from the first run's")
                res[w]["wall_s"].append(round(wall, 3))
                res[w]["peak_rss_mb"].append(round(rss, 1))
                res[w]["file_bytes"] = size
                res[w]["slices"] = n
                res[w]["lines"] = lines
        for w in res:
            res[w]["wall_median_s"] = statistics.median(res[w]["wall_s"])
        if "device_deflate" in res:
            r = res["device_deflate"]
            z = dict(kv.split("=") for l in r["lines"] if l.startswith("#deflate") for kv in l.split("\t")[1:])
            r["deflate_ms"] = float(z["deflate_ms"])
            r["d2h_ms"] = float(z["d2h_ms"])
            r["raw_gb_per_s"] = round(int(z["raw_bytes"]) / (float(z["deflate_ms"]) * 1e6), 2) if float(z["deflate_ms"]) else None
            default = next((res[w]["file_bytes"] for w in res if w != "device_deflate"), None)
            r["size_over_default"] = round(r["file_bytes"] / default, 4) if default else None
        line = {"what": "coverm filter " + " ".join(FILTER) + ", decoded whole / in slices / on the host / deflated on the device",
                "reads": args.reads, "contigs": args.contigs, "bam_bytes": os.path.getsize(bam), "inflated_bytes": whole_bytes - os.path.getsize(bam),
                "card": card(), "ways": res, "limits_mb": {w: e.get("CMB_DECODE_MEM_LIMIT_MB") for w, e in ways.items()}}
        print(json.dumps(line))
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "filter_bench.json"), "w") as f:
                f.write(json.dumps(line) + "\n")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
