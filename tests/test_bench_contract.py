"""bench.py's reference arm (`--impl reference`: the CPU restatement timed on the host cores) runs without a GPU, so its JSON line --
the part of the benchmark contract the driver parses for both arms -- is checked here; the GPU arm prints the same keys plus `roofline`,
`kernel_ms`, `clocks` and `device` (profiles/bench_h100.json is a committed example)."""

import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _line(*extra):
  out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1", "--cpu-sample-worlds", "32", *extra],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
  assert out.returncode == 0, out.stderr[-2000:]
  lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
  assert len(lines) == 1, out.stdout
  return json.loads(lines[0])


def test_reference_arm_prints_the_contract_line():
  d = _line()
  assert d["impl"] == "reference" and d["higher_is_better"] is True and d["unit"] == "env-steps/s" and d["scaling"] == "weak"
  assert d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 1 and d["value"] > 0 and d["ms_per_step"] > 0
  assert "humanoid.xml" in d["metric"] and "nworld=8192" in d["metric"] and "workload" in d["config"]
  cb, e2e = d["cpu_baseline"], d["e2e"]
  assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "worlds x 2 steps" in cb["sample"]
  assert e2e["value"] == d["value"] and e2e["unit"] == d["unit"] and e2e["h2d_bytes_per_step"] == 0 and e2e["d2h_bytes_per_step"] == 0
  assert d["gpu_launches"] == 0 and d["vs_baseline"] is None


def test_reference_arm_other_ranks_exit_quietly():
  env = dict(os.environ, RANK="1", WORLD_SIZE="2")
  out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "2", "--warmup", "1"], capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
  assert out.returncode == 0 and out.stdout.strip() == ""


def test_committed_gpu_line_has_the_contract_keys():
  d = json.load(open(os.path.join(ROOT, "profiles", "bench_h100.json")))
  for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "cpu_baseline", "clocks", "device"):
    assert k in d, k
  r = d["roofline"]
  assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and r["unit"] == "GB/s"
  assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["value"] <= d["value"] * 1.02
  assert d["gpu_launches"] > 0 and d["dtype"] == "f32" and d["clocks"]["reasons"] == []
