"""
Speed of the inverse dynamics (include/locosim.h locosim_inverse / locosim_create_dataset_inverse; LocoEnv.inverse_dynamics /
create_dataset_inverse) on one GPU, with bench.py's method: CUDA events around each call, an L2 flush between calls, a warm-up
of --warmup calls, then --steps timed calls.

In ONE invocation, for UnitreeA1.simple, HumanoidTorque.run (its bone-bone MPR pairs) and Atlas.walk with arms at --envs
envs, --rounds alternating rounds of:
  inverse   one inverse call over all envs at states of a 40-step random-action rollout (contacts active), random qacc
  dataset   create_dataset_inverse over the task's whole dataset
One JSON line per measurement (inverse evaluations per second), then one summary line with the device name and its power
limit (read-only nvidia-smi query).
    python tools/bench_inverse.py [--envs 4096] [--steps 100] [--warmup 10] [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")
# Atlas with arms is a test fixture (tools/build_assets.py), not a bundled asset
os.environ["LOCO_MUJOCO_B200_ASSET_PATH"] = os.pathsep.join(
    [p for p in (os.environ.get("LOCO_MUJOCO_B200_ASSET_PATH"), os.path.join(ROOT, "tests", "golden", "full_body")) if p])

TASKS = {"UnitreeA1.simple": ("UnitreeA1.simple", {}), "HumanoidTorque.run": ("HumanoidTorque.run", {}),
         "Atlas.walk+arms": ("Atlas.walk", dict(disable_arms=False))}
VARIANTS = ["inverse", "dataset"]
PREROLL = 40


def measure(task, variant, n, steps, warmup, seed=0):
    import torch
    from loco_mujoco_b200 import LocoEnv
    base, kw = TASKS[task]
    env = LocoEnv.make(base + ".real", num_envs=n, seed=seed, copy_outputs=False, **kw)
    eng = env._get_engine()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.uint8, device="cuda")      # > the H100's 50 MB L2
    env.reset()
    act = torch.empty((n, eng.action_dim), device="cuda")
    for _ in range(PREROLL):
        act.uniform_(-1, 1, generator=gen)
        eng.step(act, auto_reset=True)
    qacc = torch.randn((n, eng.nq), device="cuda", generator=gen)
    out = torch.empty_like(qacc)
    rows = n if variant == "inverse" else int(eng.lib.locosim_dataset_rows(eng.h))
    call = (lambda: eng.inverse(qacc, out)) if variant == "inverse" else eng.create_dataset_inverse
    times = []
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in range(warmup + steps):
        flush.zero_()
        t0.record()
        call()
        t1.record()
        t1.synchronize()
        if k >= warmup:
            times.append(t0.elapsed_time(t1))
    ms = sum(times) / len(times)
    eng.close()
    return {"task": task, "variant": variant, "rows": rows, "evals_per_s": rows / (ms * 1e-3), "ms_per_call": ms}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, watts = out[0].split(",")
        return name.strip(), float(watts)
    except Exception:
        return None, None


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=100)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    results = []
    for task in TASKS:
        for rnd in range(a.rounds):
            for var in VARIANTS:
                r = dict(measure(task, var, a.envs, a.steps, a.warmup), round=rnd)
                print(json.dumps(r), flush=True)
                results.append(r)
                torch.cuda.empty_cache()
    summary = {}
    for task in TASKS:
        for var in VARIANTS:
            v = sorted(r["evals_per_s"] for r in results if r["task"] == task and r["variant"] == var)
            rows = next(r["rows"] for r in results if r["task"] == task and r["variant"] == var)
            summary["%s / %s" % (task, var)] = {"rows": rows, "min": v[0], "median": statistics.median(v), "max": v[-1]}
    name, watts = gpu_info()
    meta = {"device": torch.cuda.get_device_name(0), "nvidia_smi_name": name, "power_limit_w": watts,
            "method": "CUDA events per call, L2 flush between calls, %d-step rollout, %d warm-up, %d timed, %d alternating "
                      "rounds" % (PREROLL, a.warmup, a.steps, a.rounds),
            "evals_per_s": summary}
    print(json.dumps(meta), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(meta, results=results), f, indent=1)


if __name__ == "__main__":
    main()
