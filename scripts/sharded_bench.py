"""`coverm contig --sharded` on a generated set of 3 shards x 10 M read pairs (tests/shard_sets.big_set): the device times of
decode, choice of each pair's shard (plus the counting sort) and coverage, from CUDA events; the end-to-end wall time against the
CPU oracle's (oracle/shard_oracle, then oracle/coverm_oracle) on the same files; and the card's name and power limit, read in the same run.  Prints one JSON line.
With --gpus N the shards are spread over N GPUs (`coverm --sharded --gpus N`): the line then also holds every rank's decode,
choice, score exchange and sort times and its shards (from the #shard_exchange lines); coverage times are rank 0's.

    python scripts/sharded_bench.py [--pairs 10000000] [--shards 3] [--gpus 1] [--skip-oracle] [--out DIR]

Needs a GPU and a built tree (__graft_entry__.build()).  The shards are written to a temporary directory and removed."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import shard_sets  # noqa: E402
from sharded_oracle import run_oracle  # noqa: E402

COVERM = os.path.join(ROOT, "coverm_b200", "bin", "coverm")


def fields(line):
    return dict(kv.split("=", 1) for kv in line.split("\t")[1:] if "=" in kv)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=10_000_000)
    ap.add_argument("--shards", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--skip-oracle", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/sharded_bench.json")
    a = ap.parse_args()
    cards = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           check=True).stdout.strip().splitlines()
    if len(cards) < a.gpus:
        sys.exit(f"--gpus {a.gpus}: only {len(cards)} GPU(s) present")
    gpu = cards[0] if a.gpus == 1 else cards[:a.gpus]
    tmp = tempfile.mkdtemp(prefix="sharded_bench_")
    try:
        t = time.time()
        shards = shard_sets.big_set(tmp, a.shards, a.pairs, seed=1)
        gen_s = time.time() - t
        base = ["contig", "-m", "mean", "variance", "--sharded", "-b"] + shards + ["-t", str(a.threads)]
        argv = base + ["--timing", "-q"] + (["--gpus", str(a.gpus)] if a.gpus > 1 else [])
        runs = []
        for _ in range(2):  # the first run also warms the page cache and the driver
            t = time.time()
            p = subprocess.run([COVERM] + argv, capture_output=True, text=True, env=dict(os.environ, CMB_PIPELINE_STATS="1"))
            wall = time.time() - t
            if p.returncode:
                sys.exit(p.stderr[-3000:])
            runs.append((wall, p))
        wall, p = runs[-1]
        sh = fields(next(l for l in p.stderr.splitlines() if l.startswith("#sharded")))
        tm = fields(next(l for l in p.stderr.splitlines() if l.startswith("#timing\tsample=")))
        ranks = [fields(l) for l in p.stderr.splitlines() if l.startswith("#shard_exchange")]
        if a.gpus > 1:
            sh = dict(decode_ms=max(float(r["decode_ms"]) for r in ranks), choose_ms=max(float(r["choose_ms"]) for r in ranks),
                      sort_ms=max(float(r["sort_ms"]) for r in ranks))
        res = dict(gpu=gpu, gpus=a.gpus, shards=a.shards, pairs=a.pairs, records=2 * a.pairs * a.shards,
                   decode_ms=float(sh["decode_ms"]), choose_ms=float(sh["choose_ms"]), sort_ms=float(sh["sort_ms"]),
                   coverage_ms=float(tm["k1_ms"]) + float(tm["k2_ms"]) + float(tm["k3_ms"]),
                   end_to_end_s=round(wall, 3), end_to_end_first_s=round(runs[0][0], 3), generate_s=round(gen_s, 1))
        if ranks:  # per rank; the top-level decode / choose / sort are then the slowest rank's
            res["ranks"] = sorted(({k: (v if k in ("shards", "rank") else float(v)) for k, v in r.items()} for r in ranks), key=lambda r: int(r["rank"]))
        if not a.skip_oracle:
            t = time.time()
            o = run_oracle(base, timeout=7200)
            res["oracle_cpu_s"] = round(time.time() - t, 3)
            res["same_output"] = o.stdout == p.stdout
        line = json.dumps(res)
        print(line)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "sharded_bench.json"), "w") as f:
                f.write(line + "\n")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
