#!/usr/bin/env python
"""Where the device step of bench.py's workload spends its time, K2 first: per-kernel times with the histogram on (the
workload's own `want`) and off (`want = 0`), and the grid K2 launched with.

    python scripts/k2_breakdown.py [--config 2|ns|3] [--steps 50] [--warmup 5] [--lib variants/<name>.so]

The input is the file bench.py times (same generator, arguments, seed and work directory, so a file bench.py generated is
reused), and the tuples stay in HBM as in bench.py's device arm: one end-to-end run, then cmb_last_bgzf_batch.  Each case
times --steps device steps; K1 / K2 / K3 are the library's CUDA-event times per step (K1 includes K1b and K1c, as in
bench.py's breakdown), `step` is CUDA events around all the steps.  The histogram's share of the step is the difference of
the two cases: K2's histogram adds and record flushes, and K3.  One JSON line goes to stdout.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (CONFIGS, gen_bam, coverm_argv: the same workload as bench.py)


def gpu_info(index):
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        o = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=10).stdout.strip()
        return dict(zip(q.split(","), (v.strip() for v in o.split(","))))
    except Exception as e:  # the timings do not depend on it; say why it is missing
        return {"error": repr(e)}


def stats_lines(fn):
    """Run fn() with CMB_PIPELINE_STATS=1 and return the '#k2_grid' / '#k2_load' lines the library printed on stderr."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as tmp:
        os.dup2(tmp.fileno(), 2)
        os.environ["CMB_PIPELINE_STATS"] = "1"
        try:
            fn()
        finally:
            del os.environ["CMB_PIPELINE_STATS"]
            libc = ctypes.CDLL(None)
            libc.fflush(None)
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        text = tmp.read()
    out = {}
    for ln in text.splitlines():
        if ln.startswith(("#k2_grid", "#k2_load")):
            f = ln.split("\t")
            out[f[0][1:]] = {k: int(v) for k, v in (x.split("=") for x in f[1:])}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="2", choices=sorted(bench.CONFIGS))
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seed", type=int, default=20260925)
    ap.add_argument("--lib", default=None, help="bind another build of libcoverm_b200.so")
    ap.add_argument("--workdir", default=os.environ.get("CMB_BENCH_DIR", "/tmp/coverm_b200_bench"))
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    import coverm_b200
    if args.lib:
        coverm_b200.LIB_PATH = os.path.abspath(args.lib)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("k2_breakdown.py needs a CUDA device")
    cfg = bench.CONFIGS[args.config]
    contigs, reads = cfg["contigs"], cfg["reads"]
    ncpu = bench.effective_cpus()
    os.makedirs(args.workdir, exist_ok=True)
    bam = os.path.join(args.workdir, f"sample_c{args.config}_r0_{contigs}_{reads}.bam")
    info = bench.gen_bam(bam, cfg, contigs, reads, args.seed, ncpu)
    argv = bench.coverm_argv(cfg, bam, ncpu)
    torch.cuda.set_device(0)
    gpu = gpu_info(0)

    sess = coverm_b200.Session(device=0, threads=ncpu)
    res = sess.run(argv)
    if res.status != 0:
        raise SystemExit(f"coverm_b200 failed: {res.err}")
    if not res.samples[0]["device_decode"]:
        raise SystemExit("the device-side decoder declined the file; the tuples must be left in HBM")
    ctx = sess.device_context()
    ctx.n_contigs = contigs
    batch, n_rec, n_iv = ctx.last_bgzf_batch()
    stream = torch.cuda.ExternalStream(ctx.stream())
    params = coverm_b200.plan_params(argv)

    def step():
        ctx.begin_sample()
        ctx.submit_device_batch(batch, n_rec, n_iv)
        ctx.end_sample_device()

    cases = {}
    for name, want in (("hist", params.want), ("nohist", 0)):
        p = coverm_b200.Params.from_buffer_copy(params)
        p.want = want
        ctx.set_params(p)
        for _ in range(args.warmup):
            step()
        launch = stats_lines(step)
        torch.cuda.synchronize()
        k1, k2, k3 = [], [], []
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            ev0.record()
        for _ in range(args.steps):
            step()
            t = ctx.timing()
            k1.append(t["ms_accumulate"]); k2.append(t["ms_scan"]); k3.append(t["ms_finalize"])
        with torch.cuda.stream(stream):
            ev1.record()
        torch.cuda.synchronize()
        cases[name] = {"want": want, "step_ms": ev0.elapsed_time(ev1) / args.steps,
                       "k1_ms": statistics.mean(k1), "k2_ms": statistics.mean(k2), "k3_ms": statistics.mean(k3),
                       "k2_ms_min": min(k2), "k2_ms_max": max(k2), **launch}
    ctx.set_params(params)
    sess.close()
    h, n = cases["hist"], cases["nohist"]
    line = {"config": args.config, "records": n_rec, "bases": int(info["bases"]), "steps": args.steps, "gpu": gpu,
            "lib": os.path.abspath(coverm_b200.LIB_PATH), "cases": cases,
            "histogram_share_ms": {"k2": h["k2_ms"] - n["k2_ms"], "k3": h["k3_ms"] - n["k3_ms"],
                                   "step": h["step_ms"] - n["step_ms"]}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
