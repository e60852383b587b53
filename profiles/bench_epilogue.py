"""Builds of the scan kernel against each other, on one GPU, in one job: each arm is a source tree (this one, and a copy
of the parent commit's tree made beforehand, e.g. `git archive HEAD~1 | tar -x -C /tmp/parent`), built in place before
the first run.  Alternating `bench.py --no-also --no-cpu-baseline` headline runs per arm, byte comparison of
`--dump-outputs` for the listed workloads against the first arm, optionally one full default `bench.py` line per arm and
NK_TC_DEBUG=64 timelines of one launch at the headline (int8 image and BF16 shadow), Q = 1 and Q = 1024 k = 10.  Prints
the card and its power limit (read in the same job), the TRUE bytes one headline launch streams from the int8 image
(n * dimpad8 + 12 n; bench.py's roofline counts BF16 shadow bytes for the `shadow` path) and the scan rate over them,
and one JSON summary line; `--out` appends the bench lines (labelled) and the summary to a jsonl file.

  python profiles/bench_epilogue.py --arm parent=/tmp/parent --arm this=. --pairs 5 --full --timeline \
      --out profiles/epilogue_h100.jsonl
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMP_ARGS = {"c4": ["--workload", "c4", "--q", "64"]}  # c4 at Q = 64 runs the 16-bit pass; Q = 1 would not
TIMELINES = {  # label: (bench.py arguments, NK_SHADOW)
    "headline_int8": ([], None),
    "headline_bf16": ([], "bf16"),
    "q1": (["--workload", "q1"], None),
    "q1024_k10": (["--q", "1024"], None),
}


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def build(tree: str) -> None:
    subprocess.run([sys.executable, "-c", "from nornicdb_b200 import build; print(build.build())"], cwd=tree, check=True)


def bench(tree: str, args: list[str], env_extra: dict | None = None) -> tuple[dict | None, str]:
    env = dict(os.environ, **(env_extra or {}))
    p = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), *args], cwd=tree, env=env, capture_output=True, text=True)
    line = None
    for s in p.stdout.splitlines()[::-1]:
        if s.startswith("{"):
            line = json.loads(s)
            break
    if p.returncode != 0 or line is None:
        sys.stderr.write(f"bench.py {' '.join(args)} ({tree}) failed rc={p.returncode}\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}\n")
    return line, p.stderr


def int8_bytes(n: int, d: int) -> int:
    """HBM bytes one scan launch streams from the int8 image: the rows plus |x|^2, |dx|^2 and the scale per row."""
    return n * ((d + 127) // 128 * 128) + 12 * n


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", action="append", required=True, help="label=source tree (the first arm is the dump reference)")
    ap.add_argument("--pairs", type=int, default=5, help="alternating headline runs per arm")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump", default="headline,q1,c2,clustered,c3,c4", help="workloads whose outputs must be byte-identical")
    ap.add_argument("--full", action="store_true", help="also one full default bench.py line per arm (the also grid)")
    ap.add_argument("--timeline", default="", help="arms to take NK_TC_DEBUG=64 timelines of (comma list)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    arms = dict(s.split("=", 1) for s in a.arm)
    arms = {k: os.path.abspath(v) for k, v in arms.items()}
    gpu = gpu_info()
    print(f"[gpu] {gpu}", file=sys.stderr)
    for tree in arms.values():
        build(tree)
    nbytes = int8_bytes(10_000_000, 1024)
    print(f"[bytes] headline int8 image per launch: {nbytes} B", file=sys.stderr)
    # the headline runs below use the default image choice, which is the int8 image at this shape (k <= 16, a large shard)
    common = ["--gpus", "1", "--steps", str(a.steps), "--warmup", str(a.warmup)]
    runs: dict[str, list[dict]] = {k: [] for k in arms}
    lines = []
    order = list(arms)
    for i in range(a.pairs):
        for arm in (order if i % 2 == 0 else order[::-1]):
            line, _ = bench(arms[arm], [*common, "--no-also", "--no-cpu-baseline"])
            if line:
                ms = line.get("roofline", {}).get("avg_launch_ms")
                cfg = line.get("config", {})
                b = int8_bytes(cfg["N"], cfg["dim"]) if "N" in cfg and "dim" in cfg else nbytes
                int8 = os.environ.get("NK_SHADOW", "") != "bf16"  # NK_SHADOW=bf16 keeps the BF16 shadow: no int8 figure
                line["int8_scan"] = {"bytes_per_launch": b if int8 else None, "avg_launch_ms": ms,
                                     "tbs": b / ms / 1e9 if ms and int8 else None}
                runs[arm].append(line)
                lines.append(dict(line, run=f"epilogue_ab_{arm}", gpu=gpu))
                print(f"[ab] {arm} ms_per_step={line.get('ms_per_step'):.4f} value={line.get('value'):.1f} scan_ms={ms} "
                      f"int8_TB/s={line['int8_scan']['tbs']} retries={line.get('filter_retries')} "
                      f"parity={line.get('parity_check', {}).get('ok')}", file=sys.stderr)
    identical = {}
    for wl in [w for w in a.dump.split(",") if w]:
        got = {}
        for arm, tree in arms.items():
            d = tempfile.mkdtemp(prefix=f"nk_dump_{wl}_{arm}_")
            bench(tree, ["--gpus", "1", "--steps", "1", "--warmup", "1", *DUMP_ARGS.get(wl, ["--workload", wl]), "--no-also",
                         "--no-cpu-baseline", "--no-parity", "--dump-outputs", d])
            got[arm] = {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}
        ref = got[order[0]]
        identical[wl] = bool(ref) and all(g == ref for g in got.values())
        print(f"[dump] {wl}: byte-identical={identical[wl]} files={sorted(ref)}", file=sys.stderr)
    if a.full:
        for arm, tree in arms.items():
            line, _ = bench(tree, common)
            if line:
                lines.append(dict(line, run=f"epilogue_full_{arm}", gpu=gpu))
                print(f"[full] {arm} {json.dumps(line)}", file=sys.stderr)
    timelines = {}
    for arm in [t for t in a.timeline.split(",") if t]:
        for label, (extra, shadow) in TIMELINES.items():
            env = {"NK_TC_DEBUG": "64", **({"NK_SHADOW": shadow} if shadow else {})}
            _, err = bench(arms[arm], ["--gpus", "1", "--steps", "1", "--warmup", "1", *extra, "--no-also", "--no-cpu-baseline",
                                       "--no-parity"], env)
            prof = [s for s in err.splitlines() if s.startswith("[shadow prof")][-4:]
            timelines[f"{arm}/{label}"] = prof
            print(f"[timeline] {arm} {label}\n" + "\n".join(prof), file=sys.stderr)
    med = {k: statistics.median([r["ms_per_step"] for r in v]) for k, v in runs.items() if v}
    rng = {k: [min(r["ms_per_step"] for r in v), max(r["ms_per_step"] for r in v)] for k, v in runs.items() if v}
    scan = {k: statistics.median([r["int8_scan"]["avg_launch_ms"] for r in v]) for k, v in runs.items() if v}
    summary = {"run": "epilogue_summary", "gpu": gpu, "arms": order, "median_ms_per_step": med, "range_ms_per_step": rng,
               "median_scan_ms": scan, "int8_bytes_per_launch_headline": nbytes,
               "int8_scan_tbs": {k: statistics.median([r["int8_scan"]["tbs"] for r in v]) for k, v in runs.items()
                                 if v and all(r["int8_scan"]["tbs"] for r in v)},
               "filter_retries": {k: [r.get("filter_retries", {}).get("exact_stage_rate") for r in v] for k, v in runs.items()},
               "parity_ok": {k: [r.get("parity_check", {}).get("ok") for r in v] for k, v in runs.items()},
               "outputs_identical": identical, "timelines": timelines}
    print(json.dumps(summary))
    if a.out:
        with open(a.out, "a") as f:
            for l in lines + [summary]:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
