"""
Cost of the time limit (include/locosim.h locosim_set_time_limit) on one GPU, measured the way bench.py measures its
workloads (it reuses bench.Workload): CUDA events around each step, an L2 flush between steps, 40 untimed steps after the
mass reset, then --warmup and --steps timed steps of seeded U(-1, 1) actions with auto-reset.

In ONE invocation, for UnitreeA1.simple and HumanoidTorque.run at --envs envs, --rounds rounds alternate three settings:
  off             no limit: the step kernels' epilogue keeps the per-episode statistics, bit 1 of `done` is never set
  never-reached   time_limit = 10**6: the limit test runs and never fires (same work, same bits as `off`)
  limit-50        time_limit = 50: reported, not judged - it resets envs the other two leave alone, which changes the mix of
                  episode ages and therefore the work
`off` against `never-reached` is the comparison: their difference has to stay inside the spread of the rounds of each.

One JSON line per measurement, then one summary line with the device name and its power limit (read-only nvidia-smi query).
    python tools/bench_time_limit.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")
import bench                                                               # noqa: E402

TASKS = ["UnitreeA1.simple", "HumanoidTorque.run"]
SETTINGS = [("off", {}), ("never-reached", dict(time_limit=10 ** 6)), ("limit-50", dict(time_limit=50))]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    ma = types.SimpleNamespace(steps=a.steps, warmup=a.warmup, no_flush=False, gather_chunk=0)
    sampler = bench.ClockSampler(0)
    sampler.start()
    results = []
    for task in TASKS:
        for rnd in range(a.rounds):
            for name, kw in SETTINGS:
                w = bench.Workload(task, [(task, a.envs, kw)], rank=0, world=1, local=0)
                res = w.measure(ma, 0, gather=False)
                out = {"task": task, "setting": name, "round": rnd, "envs": a.envs, "env_steps_per_s": res["value"],
                       "ms_per_step": res["ms_per_step"], "kernel_ms_per_step": res["kernel_ms_per_step"],
                       "resets_in_run": res["resets_in_run"], "nonfinite_in_run": res["nonfinite_in_run"]}
                print(json.dumps(out), flush=True)
                results.append(out)
                del w
                torch.cuda.empty_cache()
    clocks = sampler.stop()
    summary = {}
    for task in TASKS:
        for name, _ in SETTINGS:
            v = [r["env_steps_per_s"] for r in results if r["task"] == task and r["setting"] == name]
            summary["%s / %s" % (task, name)] = {"min": min(v), "median": sorted(v)[len(v) // 2], "max": max(v)}
    meta = {"device": torch.cuda.get_device_name(0), "power_limit_w": clocks.get("power_limit_w"),
            "sm_mhz_median": clocks.get("sm_mhz"), "clock_reasons": clocks.get("reasons"),
            "method": "bench.Workload.measure: CUDA events, L2 flush between steps, %d-step pre-roll, %d warm-up, %d timed, "
                      "%d alternating rounds" % (bench.PREROLL, a.warmup, a.steps, a.rounds),
            "env_steps_per_s": summary}
    print(json.dumps(meta), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(meta, results=results), f, indent=1)


if __name__ == "__main__":
    main()
