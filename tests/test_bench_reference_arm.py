"""`bench.py --impl reference` (the CPU arm the driver runs beside ours) on the small CPU-runnable workload: the JSON
line carries every key of the contract, and under a multi-rank launch only rank 0 prints."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(extra_env=None):
    env = dict(os.environ)
    env.update(extra_env or {})
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "c0", "--steps", "2",
                        "--warmup", "1", "--cpu-seconds", "1"], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout.strip()


def test_reference_arm_line():
    out = run()
    line = json.loads(out.splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "Mrays/s" and line["unit"] == "Mrays/s"
    for key in ("value", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
                "config", "cpu_baseline", "e2e", "gpu_launches"):
        assert key in line, key
    assert line["value"] > 0 and line["steps"] == 2 and line["gpu_launches"] == 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["cpu_baseline"]["value"] == line["value"] == line["e2e"]["value"]
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
    assert "workload" in line["config"]


def test_reference_arm_other_ranks_stay_silent():
    assert run({"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"}) == ""


def test_reference_arm_dump_outputs(tmp_path):
    """--dump-outputs writes the last timed step's pixels as float32 .npy files, with the frame rows they belong to."""
    import numpy as np
    out = tmp_path / "out"
    run_args = [sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "c0", "--steps", "1",
                "--warmup", "0", "--cpu-seconds", "1", "--dump-outputs", str(out)]
    r = subprocess.run(run_args, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    srgb, rows = np.load(out / "srgb8.npy"), np.load(out / "srgb8_frame_rows.npy")
    assert srgb.dtype == np.float32 and rows.dtype == np.float64
    assert srgb.shape == (256 * len(rows), 4) and srgb.min() >= 0 and srgb.max() <= 255
    assert (srgb[:, 3] == 255).all()
    assert sum(f.stat().st_size for f in out.iterdir()) <= 64 * 10**6
