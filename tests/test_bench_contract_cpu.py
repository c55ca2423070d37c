"""bench.py's reference arm runs on the host cores alone (oracle/c, C++/OpenMP): its JSON line is checked here against the
driver's contract on a small grid (the GPU arm prints the same keys; it needs an H100)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--grid", "256", "--steps", "2", "--warmup", "3",
                        "--ref-batches", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1                                   # ONE JSON line
    d = json.loads(lines[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "impl", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["unit"] == "steps/s" and d["higher_is_better"] is True and d["dtype"] == "f64"
    assert d["steps"] == 2 and d["warmup"] == 3 and d["vs_baseline"] is None and d["data"] == "synthetic"
    assert "workload" in d["config"] and "model" not in d["config"] and d["config"]["grid"] == [256, 256]
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["value"] == d["value"] and cb["cores"] >= 1 and "sample" in cb
    assert d["e2e"] == {"value": d["value"], "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["details"]["sample_steps"] == 10 and d["value"] > 0
    hr = cb["host_roofline"]
    assert hr["unit"] == "GB/s" and hr["achieved"] > 0 and hr["peak"] > 0 and hr["blas1_gbytes"] > hr["spmv_gbytes"] > 0


def test_reference_arm_other_ranks_exit_without_work():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--grid", "256"],
                       capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_dump_outputs_layout_and_size_cap(tmp_path, monkeypatch):
    """--dump-outputs: one float64 row per continuation step (param, x, itnewton, itlinear, ds, step), the final state -- a
    seeded sample of it above DUMP_MAX_VALUES -- and the final parameter; the whole dump stays under 64 MB."""
    import types
    import numpy as np
    import bench
    assert bench.DUMP_MAX_VALUES * 8 + 1024 * 1024 <= 64 * 1024 * 1024
    rows = [dict(param=-0.1 - 1e-3 * k, x=2.0 + k, itnewton=k % 3, itlinear=10 * k, ds=-1e-3, step=k, n_unstable=-1) for k in range(5)]
    st = types.SimpleNamespace(z_u=np.linspace(0.0, 1.0, 1000), z_p=-0.104)
    bench.dump_outputs(str(tmp_path / "full"), rows, st)
    br = np.load(tmp_path / "full" / "branch.npy")
    assert br.dtype == np.float64 and br.shape == (5, 6) and br[3].tolist() == [rows[3][k] for k in ("param", "x", "itnewton", "itlinear", "ds", "step")]
    assert np.array_equal(np.load(tmp_path / "full" / "u_final.npy"), st.z_u)
    assert np.load(tmp_path / "full" / "p_final.npy").tolist() == [-0.104]
    monkeypatch.setattr(bench, "DUMP_MAX_VALUES", 100)
    for d in ("s1", "s2"):
        bench.dump_outputs(str(tmp_path / d), rows, st)
    u1, u2 = np.load(tmp_path / "s1" / "u_final.npy"), np.load(tmp_path / "s2" / "u_final.npy")
    assert u1.dtype == np.float64 and u1.shape == (100,) and np.array_equal(u1, u2) and np.all(np.diff(u1) > 0)
    assert sorted(os.listdir(tmp_path / "s1")) == ["branch.npy", "p_final.npy", "u_final.npy"]


def test_reference_arm_refuses_dump_outputs(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--dump-outputs", str(tmp_path)],
                       capture_output=True, text=True, timeout=60, cwd=ROOT)
    assert r.returncode == 2 and "--dump-outputs" in r.stderr and os.listdir(tmp_path) == []
