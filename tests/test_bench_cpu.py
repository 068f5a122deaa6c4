"""CPU-only: the CPU legs of bench.py (cpu_baseline / --impl reference) run and speak the JSON contract."""
import json
import subprocess
import sys


def test_cpu_pipeline_leg_runs_on_a_tiny_sample():
    import bench
    from sonar_slam_b200 import synth
    d = synth.make_trajectory_frames(6, seed=1)
    bench._cpu_init(d["bearings"])
    secs = bench.cpu_pipeline(d["frames"].numpy(), d["poses_odom"], d["bearings"])
    assert 0.0 < secs < 60.0


def test_reference_arm_prints_one_json_line(monkeypatch, capsys):
    import bench
    monkeypatch.setattr(bench, "host_cores", lambda: (2, 8))   # usable (affinity mask), reported by the OS
    monkeypatch.setattr(sys, "argv", ["bench.py", "--impl", "reference", "--steps", "1", "--warmup", "0"])
    a = bench.parse()
    bench.run_reference(a)
    out = [l for l in capsys.readouterr().out.splitlines() if l.startswith("{")]
    assert len(out) == 1
    line = json.loads(out[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "impl", "cpu_baseline", "e2e"):
        assert k in line, k
    assert line["impl"] == "reference" and line["unit"] == "frames/s" and line["value"] > 0
    assert line["cpu_baseline"]["cores"] == 2 and line["e2e"]["h2d_bytes_per_step"] == 0
    assert line["cpu_baseline"]["cores_reported_by_os"] == 8 and len(line["config"]["step_seconds"]) == 1


def test_host_cores_follow_the_affinity_mask():
    import os
    import bench
    usable, reported = bench.host_cores()
    assert 1 <= usable <= reported and usable == len(os.sched_getaffinity(0))


def test_bench_refuses_to_run_the_product_path_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        return
    r = subprocess.run([sys.executable, "bench.py", "--steps", "1", "--warmup", "0"], capture_output=True, text=True)
    assert r.returncode != 0 and "no CUDA device" in (r.stderr + r.stdout)


def test_clock_sampler_keeps_the_load_until_samples_arrive(tmp_path, monkeypatch):
    """nvidia-smi that starts slower than the timed region (eight of them at N = 8): the sampler keeps the workload
    running, untimed, until it has its samples instead of reporting none."""
    import stat
    import time
    import bench
    fake = tmp_path / "nvidia-smi"
    fake.write_text("#!/bin/bash\nsleep 0.4\nwhile true; do echo '0, 1965, 1965, 700.0, Not Active, Not Active, "
                    "Not Active, Active'; sleep 0.05; done\n")
    fake.chmod(fake.stat().st_mode | stat.S_IEXEC)
    monkeypatch.setenv("PATH", f"{tmp_path}:" + __import__("os").environ["PATH"])
    c = bench.ClockSampler(0)
    c.start()
    extra = c.keep_load_until(3, lambda: time.sleep(0.01))
    out = c.stop()
    assert extra > 0 and out["samples"] >= 3 and out["sm_mhz"] == 1965.0 and out["reasons"] == ["sw_power_cap"]


def test_clock_sampler_counts_only_lines_after_the_mark(tmp_path, monkeypatch):
    """The sampler is started before the data is rendered (nvidia-smi's start-up is over when the timed region
    begins); what it printed before mark() -- idle clocks -- is not part of the report."""
    import stat
    import time
    import bench
    fake = tmp_path / "nvidia-smi"
    fake.write_text("#!/bin/bash\nfor i in 1 2 3; do echo '0, 120, 1965, 90.0, Not Active, Not Active, Not Active, "
                    "Not Active'; sleep 0.03; done\nsleep 0.3\nwhile true; do echo '0, 1965, 1965, 700.0, Not Active, "
                    "Not Active, Not Active, Not Active'; sleep 0.03; done\n")
    fake.chmod(fake.stat().st_mode | stat.S_IEXEC)
    monkeypatch.setenv("PATH", f"{tmp_path}:" + __import__("os").environ["PATH"])
    c = bench.ClockSampler(0)
    c.start()
    time.sleep(0.25)          # "rendering + warm-up": the three idle lines arrive
    c.mark()
    c.keep_load_until(3, lambda: time.sleep(0.01))
    out = c.stop()
    assert out["lines_before_timed_region_not_counted"] == 3
    assert out["samples"] >= 3 and out["sm_mhz"] == 1965.0 and out["reasons"] == []


def test_rank_binding_near_its_gpu(tmp_path):
    """bench.py under torchrun: a rank restricts itself to its GPU's local CPUs (sysfs local_cpulist) before it pins
    host memory; without the entry, or when the list is not narrower than what it may use, nothing changes."""
    import os
    import bench
    assert bench.parse_cpulist("0-3,8,10-11\n") == [0, 1, 2, 3, 8, 10, 11] and bench.parse_cpulist("") == []
    before = os.sched_getaffinity(0)
    try:
        assert bench.bind_near_gpu(0, 0x1b, 0, sysfs=str(tmp_path))["bound"] is False          # no such device
        dev = tmp_path / "0000:1b:00.0"
        dev.mkdir()
        (dev / "local_cpulist").write_text(",".join(map(str, sorted(before))) + "\n")
        assert bench.bind_near_gpu(0, 0x1b, 0, sysfs=str(tmp_path))["bound"] is False          # not narrower
        if len(before) > 1:
            one = sorted(before)[0]
            (dev / "local_cpulist").write_text(f"{one},100000\n")
            r = bench.bind_near_gpu(0, 0x1b, 0, sysfs=str(tmp_path))
            assert r["bound"] and r["cpus"] == 1 and os.sched_getaffinity(0) == {one}
    finally:
        os.sched_setaffinity(0, before)


def test_dump_outputs_writes_float_arrays_within_the_budget(tmp_path, monkeypatch):
    """--dump-outputs: every array is float32 / float64 and integers survive exactly; when all clouds would pass the
    byte budget, those of a fixed, seeded subset of frames are written, the same subset on every run."""
    import os
    import numpy as np
    import bench
    rng = np.random.default_rng(3)
    n, stride = 64, 100
    dev = {"T": rng.random((n, 3, 3), dtype=np.float32), "iterations": rng.integers(0, 40, n, dtype=np.int32),
           "inliers": rng.integers(0, 500, n, dtype=np.int32), "status": rng.integers(0, 8, n, dtype=np.int32),
           "cloud_count": rng.integers(0, stride, n, dtype=np.int32),
           "cloud_xy": rng.random((n, stride, 2), dtype=np.float32)}
    names = list(dev)

    class FakeCtx:
        def to_host(self, p, shape, dtype):
            a = dev[names[p]]
            assert a.dtype == dtype
            return a.reshape(shape).copy()

    r = dict({k: i for i, k in enumerate(names)}, cloud_stride=stride)

    def load(d):
        return {f[:-4]: np.load(d / f) for f in sorted(os.listdir(d))}

    bench.dump_outputs(str(tmp_path / "all"), FakeCtx(), r, n)
    a = load(tmp_path / "all")
    assert all(v.dtype in (np.float32, np.float64) for v in a.values())
    assert np.array_equal(a["status"], dev["status"]) and np.array_equal(a["T"], dev["T"])
    assert np.array_equal(a["cloud_frames"], np.arange(n))
    want = np.concatenate([dev["cloud_xy"][i, :dev["cloud_count"][i]] for i in range(n)])
    assert np.array_equal(a["cloud_points"], want)

    monkeypatch.setattr(bench, "DUMP_BYTES", 20000)
    for tag in ("s1", "s2"):
        bench.dump_outputs(str(tmp_path / tag), FakeCtx(), r, n)
    s1, s2 = load(tmp_path / "s1"), load(tmp_path / "s2")
    assert sum(v.nbytes for v in s1.values()) <= 20000
    assert all(np.array_equal(s1[k], s2[k]) for k in s1)
    fr = s1["cloud_frames"].astype(int)
    assert 0 < len(fr) < n and np.all(np.diff(fr) > 0)
    off = s1["cloud_offsets"].astype(int)
    for j, i in enumerate(fr):
        assert np.array_equal(s1["cloud_points"][off[j]:off[j + 1]], dev["cloud_xy"][i, :dev["cloud_count"][i]])
