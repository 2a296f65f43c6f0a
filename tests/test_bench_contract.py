"""CPU: the JSON line of bench.py's reference arm carries the keys of the benchmark's contract (run on the smallest model)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_contract():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--model", "tiny.en", "--steps", "1", "--warmup", "0",
                          "--cpu-sample-tokens", "2"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
                "config", "e2e", "cpu_baseline", "impl"):
        assert key in line, key
    assert line["impl"] == "reference" and line["higher_is_better"] is True and line["vs_baseline"] is None
    assert "workload" in line["config"] and line["value"] > 0
    assert set(line["e2e"]) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} and line["e2e"]["value"] == line["value"]
    assert set(line["cpu_baseline"]) >= {"value", "unit", "cores", "kind", "sample"} and line["cpu_baseline"]["kind"] == "port"


def test_reference_arm_is_silent_on_other_ranks():
    env = dict(os.environ, RANK="1", LOCAL_RANK="1", WORLD_SIZE="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"], capture_output=True, text=True,
                         timeout=120, cwd=ROOT, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_committed_bench_line_of_our_arm_meets_the_contract():
    """The GPU arm cannot run without a GPU; the line recorded on an H100 (the last line of profiles/h100_bench_default.jsonl, written by bench.py itself)
    must carry every key of the benchmark's contract and be internally consistent."""
    with open(os.path.join(ROOT, "profiles", "h100_bench_default.jsonl")) as f:
        line = json.loads(f.read().strip().splitlines()[-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
                "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"):
        assert key in line, key
    with open(os.path.join(ROOT, "BASELINE.json")) as f:
        assert line["metric"] == json.load(f)["metric"].split(" @")[0]
    assert line["higher_is_better"] is True and line["scaling"] == "weak" and line["vs_baseline"] is None and line["data"] == "synthetic"
    assert line["warmup"] >= 3 and line["n_gpus"] == 1 and line["gpu_launches"] > 0 and "workload" in line["config"] and "l2" in line["config"]
    # value = audio seconds of one step / step time (16 chunks of 30 s)
    assert abs(line["value"] - 16 * 30.0 / (line["ms_per_step"] / 1e3)) < 1e-6 * line["value"]
    e2e = line["e2e"]
    assert e2e["h2d_bytes_per_step"] == 16 * 480000 * 4 and e2e["d2h_bytes_per_step"] > 0 and 0 < e2e["value"] <= line["value"] * 1.001
    assert not set(line["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    r = line["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert abs(r["achieved"] - r["alg_bytes_per_step"] / (r["ms_per_decode_step"] * 1e-3) / 1e9) < 1e-6 * r["achieved"]
    assert set(line["cpu_baseline"]) >= {"value", "unit", "cores", "kind", "sample"}


def test_dump_outputs_files_dtypes_and_size():
    """bench.py --dump-outputs: one .npy per returned array, float32 / float64 only, a fixed seeded encoder sample, < 64 MB in all."""
    import tempfile
    from types import SimpleNamespace

    import numpy as np

    sys.path.insert(0, ROOT)
    import bench

    rng = np.random.default_rng(0)
    enc_array = rng.standard_normal((16, 1500, 1280)).astype(np.float16)  # large-v3 encoder output of 16 chunks
    enc = SimpleNamespace(numpy=lambda: enc_array.astype(np.float32))
    res = [SimpleNamespace(sequences_ids=[list(range(i, i + 128))], scores=[-0.5 * i], no_speech_prob=0.01 * i) for i in range(16)]
    with tempfile.TemporaryDirectory() as d1, tempfile.TemporaryDirectory() as d2:
        bench.dump_outputs(d1, "batched", enc, res)
        bench.dump_outputs(d2, "batched", enc, res)
        names = sorted(os.listdir(d1))
        assert names == ["batched_encoder_output_sample.npy", "batched_no_speech_prob.npy", "batched_scores.npy", "batched_tokens.npy"]
        assert sum(os.path.getsize(os.path.join(d1, n)) for n in names) < 64 * 2**20
        for n in names:
            a, b = np.load(os.path.join(d1, n)), np.load(os.path.join(d2, n))
            assert a.dtype in (np.float32, np.float64) and np.array_equal(a, b), n
        assert np.load(os.path.join(d1, "batched_tokens.npy")).tolist()[3][:2] == [3.0, 4.0]
        assert np.load(os.path.join(d1, "batched_encoder_output_sample.npy")).shape == (1 << 22,)
