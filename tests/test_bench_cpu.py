"""bench.py contract checks that need no GPU: the reference arm (`--impl reference`) must print ONE JSON line with the
GPU arm's metric / unit / config for the same workload, so that the two arms' results form a ratio."""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def _run(*extra):
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", *extra],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip().startswith("{")]
    assert len(lines) == 1
    return json.loads(lines[0])


def test_reference_arm_clip_workload_line():
    sys.path.insert(0, str(ROOT))
    import bench

    d = _run("--evals", "50", "--clips", "32")
    assert d["impl"] == "reference" and d["metric"] == "clips/sec" and d["unit"] == "clips/s" and d["higher_is_better"]
    assert d["config"] == bench.clip_config(50, 50, 32)          # identical to the GPU arm's config for these flags
    assert d["value"] > 0 and d["cpu_baseline"]["value"] == d["value"] and d["cpu_baseline"]["kind"] in ("port", "reference")
    assert d["e2e"] == {"value": d["value"], "unit": "clips/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["gpu_launches"] == 0 and "sample" in d["cpu_baseline"] and d["cpu_baseline"]["cores"] >= 1


def test_reference_arm_other_ranks_print_nothing(monkeypatch):
    import os

    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1"],
                       capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_workload_configs_and_eval_counts():
    """the img2img start-point arithmetic bench.py extrapolates with equals the reference's (riffusion_pipeline.py:358-396,
    SURVEY Appendix B: 38 evaluations at denoising 0.75, 50 at 1.0, 26 at 0.5) and the product scheduler's"""
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "riffusion-hobby_b200"))
    import bench
    from riffusion.scheduler_b200 import PNDMSchedulerB200

    assert [bench.n_evals_for(50, s) for s in (0.75, 1.0, 0.5)] == [38, 50, 26]
    sch = PNDMSchedulerB200()
    for steps, s in ((50, 0.75), (50, 1.0), (20, 0.7499999999999999), (8, 1.0)):
        sch.set_timesteps(steps)
        init = min(int(steps * s) + 1, steps)
        assert bench.n_evals_for(steps, s) == len(sch.timesteps[max(steps - init + 1, 0):])
    rt = bench.clip_config(50, 50, 16, "roundtrip")
    rf = bench.clip_config(50, 38, 1, "riffuse", 0.75)
    assert "configs[4]" in rt["workload"] and "configs[2]" in rf["workload"] and rt["clips_per_gpu"] == 16
