"""
Speed of the forward dynamics under an action (include/locosim.h locosim_forward; LocoEnv.forward_dynamics) on one GPU,
with bench.py's method: CUDA events around each call, an L2 flush between calls, a warm-up of --warmup calls, then --steps
timed calls.

In ONE invocation, for UnitreeA1.simple, HumanoidTorque.run and Atlas.walk with arms at --envs envs at the states of a
40-step random-action rollout, under one fixed random action, --rounds alternating rounds of:
  dof       the dof row alone (qfrc_actuator, qfrc_constraint, qacc)
  all       all four outputs (dof, body_acc, cfrc_int, cfrc_ext)
Each call is one full mj_forward per env (collision and the Newton solve included) in a one-warp block, plus
mj_rnePostConstraint for "all". One JSON line per measurement (evaluations, i.e. envs, per second), then one summary line
with the medians, the device name and its power limit (read-only nvidia-smi query).
    python tools/bench_forward.py [--envs 4096] [--steps 50] [--warmup 10] [--rounds 3] [--out FILE]
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
VARIANTS = {"dof": dict(dof=True, body_acc=False, cfrc_int=False, cfrc_ext=False),
            "all": dict(dof=True, body_acc=True, cfrc_int=True, cfrc_ext=True)}
PREROLL = 40


def make(task, n, seed):
    import torch
    from loco_mujoco_b200 import LocoEnv
    base, kw = TASKS[task]
    env = LocoEnv.make(base + ".real", num_envs=n, seed=seed, copy_outputs=False, **kw)
    eng = env._get_engine()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    env.reset()
    act = torch.empty((n, eng.action_dim), device="cuda")
    for _ in range(PREROLL):
        act.uniform_(-1, 1, generator=gen)
        eng.step(act, auto_reset=True)
    act.uniform_(-1, 1, generator=gen)
    return env, act


def measure(env, act, variant, steps, warmup):
    import torch
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.uint8, device="cuda")      # > the H100's 50 MB L2
    out = env.forward_dynamics(act, **VARIANTS[variant])
    times = []
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in range(warmup + steps):
        flush.zero_()
        t0.record()
        env.forward_dynamics(act, **VARIANTS[variant], out=out)
        t1.record()
        t1.synchronize()
        if k >= warmup:
            times.append(t0.elapsed_time(t1))
    ms = statistics.median(times)
    return {"variant": variant, "envs": env.num_envs, "evals_per_s": env.num_envs / (ms * 1e-3), "ms_per_call": ms,
            "output_mb": sum(x.numel() * 4 for x in out.values()) / 1e6}


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
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    results = []
    for task in TASKS:
        env, act = make(task, a.envs, 0)
        for rnd in range(a.rounds):
            for var in VARIANTS:
                r = dict(measure(env, act, var, a.steps, a.warmup), task=task, round=rnd)
                print(json.dumps(r), flush=True)
                results.append(r)
        env._get_engine().close()
        torch.cuda.empty_cache()
    summary = {}
    for task in TASKS:
        for var in VARIANTS:
            v = sorted(r["evals_per_s"] for r in results if r["task"] == task and r["variant"] == var)
            summary["%s / %s" % (task, var)] = {"min": v[0], "median": statistics.median(v), "max": v[-1]}
    name, watts = gpu_info()
    meta = {"device": torch.cuda.get_device_name(0), "nvidia_smi_name": name, "power_limit_w": watts,
            "method": "CUDA events per call, L2 flush between calls, %d-step rollout, %d warm-up, median of %d timed calls, "
                      "%d alternating rounds" % (PREROLL, a.warmup, a.steps, a.rounds),
            "evals_per_s": summary}
    print(json.dumps(meta), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(meta, results=results), f, indent=1)


if __name__ == "__main__":
    main()
