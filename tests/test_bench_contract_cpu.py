"""bench.py's output contract, checked without a GPU: helpers import, every workload BASELINE.json names is defined, and
the committed bench lines (profiles/bench_h100.jsonl: the default command and `--impl reference`, produced by bench.py on an
H100) carry every key a reader of the results relies on, the in-run parity check and the north_star grid included."""
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REQUIRED = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
            "dtype", "data", "config", "roofline", "e2e", "clocks", "gpu_launches"]


def test_bench_helpers_and_workloads():
    import bench
    assert set(["headline", "c1", "c2", "c3", "c4", "c5", "q1"]) <= set(bench.WORKLOADS)
    n, d, dt, Q, k, metric, _ = bench.WORKLOADS["headline"]
    assert (n, d, dt, Q, k, metric) == (10_000_000, 1024, "f32", 64, 10, "cosine")   # BASELINE.json metric shape
    assert bench.WORKLOADS["c3"][:6] == (10_000_000, 1024, "f32", 1024, 100, "dot")
    assert bench.WORKLOADS["c4"][:6] == (10_000_000, 768, "f16", 1, 10, "euclidean")
    assert bench.WORKLOADS["c5"][:6] == (100_000_000, 1024, "f32", 1024, 10, "cosine")
    peak, src = bench.load_peaks()
    assert 3000 < peak < 9000 and ("measured" in src or "fallback" in src)
    tf32, _ = bench.load_tensor_peak()
    bf16, _ = bench.load_tensor_peak(bf16=True)
    assert abs(bf16 - 2 * tf32) < 1e-6


def test_committed_bench_lines_follow_the_contract():
    lines = [json.loads(l) for l in open(os.path.join(ROOT, "profiles", "bench_h100.jsonl"))]
    ours = [d for d in lines if d.get("impl") != "reference"]
    ref = [d for d in lines if d.get("impl") == "reference"]
    assert ours and ref
    for d in ours:
        for key in REQUIRED:
            assert key in d, (d.get("run"), key)
        assert d["metric"] == "kNN queries/sec" and d["unit"] == "queries/s" and d["higher_is_better"] is True
        assert d["vs_baseline"] is None and d["data"] == "synthetic" and d["scaling"] == "strong"
        r = d["roofline"]
        assert r["bound"] in ("hbm", "tensor") and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and r["unit"] in ("GB/s", "TFLOP/s")
        e = d["e2e"]
        assert e["unit"] == "queries/s" and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and e["value"] > 0
        assert d["gpu_launches"] > 0 and "workload" in d["config"] and "model" not in d["config"]
        assert "sm_mhz" in d["clocks"] and "reasons" in d["clocks"]
        assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    default = [d for d in ours if d.get("run", "").startswith("default")][0]
    cb = default["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["unit"] == "queries/s" and "sample" in cb
    for d in ref:
        assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["cpu_baseline"]["value"] == d["value"]


def test_round2_bench_lines_carry_parity_check_and_grid():
    lines = [json.loads(l) for l in open(os.path.join(ROOT, "profiles", "bench_h100.jsonl")) if json.loads(l).get("impl") != "reference"]
    by = {d["run"]: d for d in lines}
    for d in lines:
        for key in REQUIRED + ["scan", "timing"]:
            assert key in d, (d["run"], key)
        assert "scan" not in d["config"]  # moved to the top level so the two arms' configs compare equal
        pc = d.get("parity_check")
        if pc is None:  # the NCCL-exchange comparison run was taken with --no-parity
            assert "nccl" in d["run"], d["run"]
            continue
        # every returned score is recomputed (bounded at 4096 row read-backs per rank for the Q=1024, k=100 shape)
        assert pc["ok"] is True and pc["scores_recomputed_fp64"] >= min(d["config"]["Q"] * d["config"]["k"], 4096 * d["n_gpus"]), (d["run"], pc)
        assert d["e2e"]["value"] <= d["value"] * 1.02, d["run"]  # one clock per quantity: e2e never beats device-resident
        r = d["roofline"]
        assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    one = by["default_1gpu"]
    want = {"c3", "c3_k10", "q1", "k100", "headline_filter", "q1_simt", "headline_clustered", "c4", "c4_q64", "c2", "c1"}
    assert want <= set(one["also"]), sorted(set(one["also"]))
    for name, e in one["also"].items():
        assert "error" not in e, (name, e)
        assert e["ms_per_step"] > 0 and 0 < e["roofline_frac"] < 1.25 and e["bound"] in ("hbm", "tensor")
    assert one["also"]["headline_clustered"]["filter_retries"]["first_stage_retry_rate"] <= 0.05  # the round-1 cliff
    assert one["also"]["headline_clustered"]["filter_retries"]["exact_stage_rate"] <= 0.05
    st = one["cpu_baseline"]["single_thread"]
    assert st["cores"] == 1 and st["value"] > 0 and one["cpu_baseline"]["value"] >= st["value"] * 0.9
