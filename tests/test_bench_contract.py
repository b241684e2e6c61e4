"""CPU: the bench.py contract the driver relies on, as far as it can be checked without a GPU - the reference (CPU) arm's
JSON line, its behaviour on non-zero ranks, and the workload table against BASELINE.json / SURVEY.md §8d."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None, timeout=400):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, env=e,
                          timeout=timeout, cwd=ROOT)


def test_reference_arm_json_line_and_rank_behaviour():
    r = _run(["--impl", "reference", "--gpus", "1", "--steps", "1", "--warmup", "1"])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "samples/s" and d["value"] > 0 and d["higher_is_better"] is True
    assert d["n_gpus"] == 1 and d["steps"] == 1 and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["data"] == "synthetic" and "workload" in d["config"] and d["ms_per_step"] > 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    baseline = json.load(open(os.path.join(ROOT, "BASELINE.json")))
    assert baseline["metric"].startswith(d["metric"])            # the same metric string the GPU arm prints
    # under torchrun only rank 0 works and prints; the other ranks exit 0 without output
    r = _run(["--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1"], env={"RANK": "1", "WORLD_SIZE": "2",
                                                                                        "LOCAL_RANK": "1"}, timeout=120)
    assert r.returncode == 0 and not [ln for ln in r.stdout.splitlines() if ln.startswith("{")]


def test_workload_table_matches_survey():
    sys.path.insert(0, ROOT)
    import bench
    assert set(bench.WORKLOADS) == {"cfg2", "cfg4", "cfg5"}
    # algorithmic fwd+bwd GFLOP per sample of SURVEY.md §8d (the roofline numerator) and the per-GPU batch of BASELINE.json
    expect = {"cfg2": (65.41e9, 128, "base", 224, 98), "cfg4": (196.40e9, 64, "large", 224, 98),
              "cfg5": (287.0e9, 32, "base", 448, 392)}
    for k, (flop, batch, size, image, visible) in expect.items():
        w = bench.WORKLOADS[k]
        assert (w["flop"], w["batch"], w["size"], w["image"], w["visible"]) == (flop, batch, size, image, visible), k
    assert bench.WORKLOADS["cfg2"]["metric"] == bench.METRIC


def test_encoder_tensor_core_figure_from_a_gemm_table():
    """bench.encoder_tc_from_table on a per-shape table of one MultiMAE-B step (bs 128, 99 encoder rows per sample): the
    144 encoder GEMM launches (12 blocks x {QKV, proj, fc1, fc2} x {forward, dgrad, wgrad}) and nothing from the decoders /
    embedding.  Every encoder launch is timed at exactly 500 TFLOP/s."""
    sys.path.insert(0, ROOT)
    import bench
    R, D = 128 * 99, 768
    fwd = [(R, 3 * D, D), (R, D, D), (R, 4 * D, D), (R, D, 4 * D)]
    shapes = [(m, n, k, 0) for m, n, k in fwd] + [(R, k, n, 2) for _, n, k in fwd] + [(n, k, R, 3) for _, n, k in fwd]
    agg = {(m, n, k, maj, 1): [12, 12 * 2.0 * m * n * k / 500e12 * 1e3] for m, n, k, maj in shapes}
    agg[(25088, 256, 256, 0, 1)] = [17, 0.3]                 # decoder / embedding shapes are not counted
    agg[(R, 256, D, 0, 1)] = [4, 0.2]
    r = bench.encoder_tc_from_table(agg, R, D, 989.0)
    assert r["launches_per_step"] == 144
    assert abs(r["encoder_gemm_tflops"] - 500.0) < 0.1 and abs(r["frac_of_measured_peak"] - 500.0 / 989.0) < 1e-3
    assert bench.encoder_tc_from_table({(25088, 256, 256, 0, 1): [17, 0.3]}, R, D, 989.0) is None
