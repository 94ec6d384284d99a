"""bench.py contract checks that need no GPU: the reference arm (CPU port of the reference's path) prints ONE JSON line
with the keys a caller reads, and the CUDA arm refuses to run without a CUDA device (no CPU fallback)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(*args, timeout=600):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True,
                          timeout=timeout, env=env, cwd=ROOT)


def test_reference_arm_prints_one_json_line():
    r = run("--impl", "reference", "--workload", "lift_splat", "--steps", "1", "--warmup", "0")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "bev_frames_per_sec" and d["unit"] == "frames/s"
    assert d["higher_is_better"] is True and d["value"] > 0 and d["vs_baseline"] is None
    # "reference" = the unmodified reference package (oracle/_ref); "port" only where it does not exist
    assert d["cpu_baseline"]["kind"] in ("reference", "port")
    assert d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and d["config"]["samples_per_gpu_per_step"] == 4


def test_reference_arm_uses_the_installed_reference_when_present():
    """oracle/_ref (oracle/build_ref.py) present -> the arm times the reference's own modules."""
    sys.path.insert(0, ROOT)
    from oracle import ref_loader
    if not ref_loader.reference_available():
        import pytest
        pytest.skip("no reference install on this machine")
    r = run("--impl", "reference", "--workload", "lift_splat", "--steps", "1", "--warmup", "0")
    d = json.loads([l for l in r.stdout.splitlines() if l.strip()][0])
    assert d["cpu_baseline"]["kind"] == "reference"


def test_b200_arm_has_no_cpu_fallback():
    r = run("--steps", "1", "--warmup", "3", "--no-cpu-baseline", timeout=300)
    assert r.returncode != 0 and "no CPU fallback" in (r.stderr + r.stdout)


def test_extras_watchdog_prints_the_line_it_has():
    """Once the timed regions are done the contract line exists; if the explanatory part (sustained loop, stage graphs,
    latency mode ...) never comes back, rank 0 prints that line with a note and every rank exits 0."""
    import io
    import time
    sys.path.insert(0, ROOT)
    import bench
    exits = []
    for rank in (0, 1):
        bench._LINE["line"] = {"metric": "bev_frames_per_sec", "value": 1.0}
        buf = io.StringIO()
        dog = bench.extras_watchdog(0.05, rank, exit_fn=exits.append, out=buf)
        dog.join(5)
        time.sleep(0.05)
        lines = [l for l in buf.getvalue().splitlines() if l.strip()]
        if rank == 0:
            assert len(lines) == 1
            d = json.loads(lines[0])
            assert d["value"] == 1.0 and "timed out" in d["extras"]["unavailable"]
        else:
            assert lines == []
    assert exits == [0, 0]
    # cancelled in time: nothing is printed, nobody exits
    buf = io.StringIO()
    dog = bench.extras_watchdog(0.2, 0, exit_fn=exits.append, out=buf)
    dog.cancel()
    time.sleep(0.4)
    assert buf.getvalue() == "" and exits == [0, 0]
