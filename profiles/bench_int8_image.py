"""The default image choice (NK_SHADOW unset: both images, the int8 one wherever it serves the search; arm "int8") against
the BF16 shadow alone (NK_SHADOW=bf16; arm "bf16"), on one GPU, in one job: alternating
`bench.py --no-also --no-cpu-baseline` runs of the headline under both settings, byte comparison of `--dump-outputs` for
the listed workloads, optionally one full default `bench.py` line and one NK_TC_DEBUG=64 timeline per setting.  Prints the
card and its power limit (read in the same job), the true bytes one scan launch streams under each image, and one JSON
summary line; `--out` appends the bench lines (labelled) and the summary to a jsonl file.

  python profiles/bench_int8_image.py --pairs 5 --dump headline,q1,c2,clustered,c3 --full --timeline --out profiles/bench_h100.jsonl
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
SETTINGS = {"int8": "1", "bf16": "bf16"}


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def bench(setting: str, args: list[str], env_extra: dict | None = None) -> tuple[dict | None, str]:
    env = dict(os.environ, NK_SHADOW=SETTINGS[setting], **(env_extra or {}))
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], cwd=ROOT, env=env, capture_output=True, text=True)
    line = None
    for s in p.stdout.splitlines()[::-1]:
        if s.startswith("{"):
            line = json.loads(s)
            break
    if p.returncode != 0 or line is None:
        sys.stderr.write(f"bench.py {' '.join(args)} ({setting}) failed rc={p.returncode}\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}\n")
    return line, p.stderr


def image_bytes(n: int, d: int) -> dict:
    """Algorithmic HBM bytes of one scan launch: the image rows plus the per-row side arrays it reads."""
    dimpad8, dimpad = (d + 127) // 128 * 128, (d + 63) // 64 * 64
    return {"int8": n * dimpad8 + 12 * n, "bf16": n * dimpad * 2 + 8 * n}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=5, help="alternating headline runs per setting")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump", default="headline,q1,c2,clustered,c3", help="workloads whose outputs must be byte-identical ('' = none)")
    ap.add_argument("--full", action="store_true", help="also one full default bench.py line per setting (the also grid)")
    ap.add_argument("--timeline", action="store_true", help="also one NK_TC_DEBUG=64 timeline per setting (headline, 2 steps)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = gpu_info()
    print(f"[gpu] {gpu}", file=sys.stderr)
    common = ["--gpus", "1", "--steps", str(a.steps), "--warmup", str(a.warmup)]
    runs = {"int8": [], "bf16": []}
    lines = []
    for i in range(a.pairs):
        for setting in (("int8", "bf16") if i % 2 == 0 else ("bf16", "int8")):
            line, _ = bench(setting, [*common, "--no-also", "--no-cpu-baseline"])
            if line:
                runs[setting].append(line)
                lines.append(dict(line, run=f"int8_image_ab_{setting}", gpu=gpu))
                print(f"[ab] {setting} value={line.get('value')} retries={line.get('filter_retries')} "
                      f"parity={line.get('parity_check', {}).get('ok')}", file=sys.stderr)
    identical = {}
    for wl in [w for w in a.dump.split(",") if w]:
        got = {}
        for setting in SETTINGS:
            d = tempfile.mkdtemp(prefix=f"nk_dump_{wl}_{setting}_")
            bench(setting, ["--gpus", "1", "--steps", "1", "--warmup", "1", "--workload", wl, "--no-also", "--no-cpu-baseline",
                            "--no-parity", "--dump-outputs", d])
            got[setting] = {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}
        identical[wl] = bool(got["int8"]) and got["int8"] == got["bf16"]
        print(f"[dump] {wl}: byte-identical={identical[wl]} files={sorted(got['int8'])}", file=sys.stderr)
    if a.full:
        for setting in SETTINGS:
            line, _ = bench(setting, common)
            if line:
                lines.append(dict(line, run=f"int8_image_full_{setting}", gpu=gpu))
                print(f"[full] {setting} {json.dumps(line)}", file=sys.stderr)
    if a.timeline:
        for setting in SETTINGS:
            _, err = bench(setting, ["--gpus", "1", "--steps", "2", "--warmup", "1", "--no-also", "--no-cpu-baseline", "--no-parity"],
                           {"NK_TC_DEBUG": "64"})
            prof = [s for s in err.splitlines() if s.startswith("[shadow prof")]
            print(f"[timeline] {setting}\n" + "\n".join(prof[-3:]), file=sys.stderr)
    med = {s: statistics.median([r["value"] for r in v]) for s, v in runs.items() if v}
    rng = {s: [min(r["value"] for r in v), max(r["value"] for r in v)] for s, v in runs.items() if v}
    summary = {"run": "int8_image_summary", "gpu": gpu, "median_value": med, "range": rng,
               "speedup": med["int8"] / med["bf16"] if len(med) == 2 else None,
               "disjoint": len(rng) == 2 and rng["int8"][0] > rng["bf16"][1],
               "bytes_per_launch_headline": image_bytes(10_000_000, 1024),
               "filter_retries": {s: [r.get("filter_retries") for r in v] for s, v in runs.items()},
               "parity_ok": {s: [r.get("parity_check", {}).get("ok") for r in v] for s, v in runs.items()},
               "outputs_identical": identical}
    print(json.dumps(summary))
    if a.out:
        with open(a.out, "a") as f:
            for l in lines + [summary]:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
