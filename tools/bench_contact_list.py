"""
Cost of the contact list (include/locosim.h locosim_set_contact_list_outputs, LocoEnv.contacts) on one GPU, with
bench.py's method: CUDA events around each step, an L2 flush between steps, 40 untimed steps after the mass reset, then
--warmup and --steps timed steps of seeded U(-1, 1) actions with auto-reset.

In ONE invocation, for UnitreeA1.simple (its default launch path: the persistent kernel), HumanoidTorque.run (RK4, bone-bone
self contacts) and Atlas.walk with arms (the 31-dof RK4 configuration) at --envs envs, --rounds rounds alternate two variants:
  off         nothing registered (the default path)
  registered  the contact list registered: after the last sub-step each contact's lane writes its row, every other lane an
              empty one

One JSON line per measurement, then one summary line with the device name and its power limit (read-only nvidia-smi query).
    python tools/bench_contact_list.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
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
VARIANTS = ["off", "registered"]
PREROLL = 40


def measure(task, variant, n, steps, warmup, seed=0):
    import torch
    from loco_mujoco_b200 import LocoEnv
    base, kw = TASKS[task]
    env = LocoEnv.make(base + ".real", num_envs=n, seed=seed, copy_outputs=False, **kw)
    eng = env._get_engine()
    nu = eng.action_dim
    gen = torch.Generator(device="cuda").manual_seed(seed)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.uint8, device="cuda")      # > the H100's 50 MB L2
    if variant == "registered":
        env.contacts
    env.reset()
    act = torch.empty((n, nu), device="cuda")

    def one():
        act.uniform_(-1, 1, generator=gen)
        return eng.step(act, auto_reset=True)

    for _ in range(PREROLL):
        one()
    times = []
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in range(warmup + steps):
        flush.zero_()
        t0.record()
        one()
        t1.record()
        t1.synchronize()
        if k >= warmup:
            times.append(t0.elapsed_time(t1))
    ms = sum(times) / len(times)
    eng.close()
    return {"task": task, "variant": variant, "envs": n, "env_steps_per_s": n / (ms * 1e-3), "ms_per_step": ms}


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return float(out[0])
    except Exception:
        return None


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
            v = sorted(r["env_steps_per_s"] for r in results if r["task"] == task and r["variant"] == var)
            summary["%s / %s" % (task, var)] = {"min": v[0], "median": v[len(v) // 2], "max": v[-1]}
    meta = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit(),
            "method": "CUDA events per step, L2 flush between steps, %d-step pre-roll, %d warm-up, %d timed, %d alternating "
                      "rounds" % (PREROLL, a.warmup, a.steps, a.rounds),
            "env_steps_per_s": summary}
    print(json.dumps(meta), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(meta, results=results), f, indent=1)


if __name__ == "__main__":
    main()
