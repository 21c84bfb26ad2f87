"""
Speed of the saved simulation states (include/locosim.h locosim_save_state / locosim_load_state) on one GPU, with bench.py's
method: CUDA events around each call, an L2 flush between calls, a warm-up of --warmup calls, then --steps timed calls.

In ONE invocation, for UnitreeA1.simple, HumanoidTorque.run and Atlas.walk with arms at --envs envs at the states of a
40-step random-action rollout, --rounds alternating rounds of:
  step         one control step (auto-reset), for scale
  save         save_state of every env
  load         load_state of every env (identity rows)
  save+out / load+out / step+out   the same with body, reference, contact and dof outputs registered (the load then
               rewrites the next body and reference rows: one more kernel)
and, for UnitreeA1.simple, a predictive-sampling planner captured in one CUDA graph: --robots robots x --samples samples
(= the envs), horizon --horizon. Per planning step: fork (every sample env loads its robot's row), roll out the horizon
under fixed perturbed action sequences summing the rewards, pick each robot's best first action, load the robots' rows
into one env each, apply the chosen actions with one more step, and save the robots' new rows. Planning steps per second
= graph replays per second (each advances every robot by one control step).
One JSON line per measurement, then one summary line with the medians, the device name, its power limit and SM clocks
(read-only nvidia-smi query), and the row bytes each call moves.
    python tools/bench_state.py [--envs 4096] [--steps 50] [--warmup 10] [--rounds 3] [--out FILE]
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
PREROLL = 40


def make(task, n, seed):
    import torch
    from loco_mujoco_b200 import LocoEnv
    base, kw = TASKS[task]
    # (the end-of-trajectory limit lets the reference outputs be registered for the "+out" variants)
    env = LocoEnv.make(base + ".real", num_envs=n, seed=seed, copy_outputs=False, truncate_at_trajectory_end=True, **kw)
    eng = env._get_engine()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    env.reset()
    act = torch.empty((n, eng.action_dim), device="cuda")
    for _ in range(PREROLL):
        act.uniform_(-1, 1, generator=gen)
        eng.step(act, auto_reset=True)
    return env, act


def timed(fn, steps, warmup):
    import torch
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.uint8, device="cuda")      # > the H100's 50 MB L2
    times = []
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in range(warmup + steps):
        flush.zero_()
        t0.record()
        fn()
        t1.record()
        t1.synchronize()
        if k >= warmup:
            times.append(t0.elapsed_time(t1))
    return statistics.median(times)


def measure_calls(env, act, steps, warmup, suffix):
    import torch
    eng = env._get_engine()
    S = torch.empty((eng.n_envs, eng.state_words), dtype=torch.int32, device="cuda")
    obs = eng.next_obs.clone()
    eng.save_state(obs, out=S)
    calls = {"step": lambda: eng.step(act, auto_reset=True), "save": lambda: eng.save_state(obs, out=S),
             "load": lambda: eng.load_state(S, obs_out=obs)}
    out = []
    for name, fn in calls.items():
        ms = timed(fn, steps, warmup)
        out.append({"call": name + suffix, "envs": eng.n_envs, "us_per_call": ms * 1e3,
                    "row_mb": S.numel() * 4 / 1e6 if name != "step" else None})
    return out


def planner(robots, samples, horizon, steps, warmup):
    """graph-captured predictive sampling on UnitreeA1.simple: returns ms per planning step"""
    import torch
    env, _ = make("UnitreeA1.simple", robots * samples, 0)
    eng = env._get_engine()
    n, nu = eng.n_envs, eng.action_dim
    g = torch.Generator(device="cuda").manual_seed(1)
    plans = (torch.rand((horizon, n, nu), device="cuda", generator=g) * 2 - 1).contiguous()
    S = torch.empty((n, eng.state_words), dtype=torch.int32, device="cuda")
    obs = eng.next_obs.clone()
    eng.save_state(obs, out=S)
    R = S[::samples].contiguous()                                       # the robots' rows
    fork = (torch.arange(n, device="cuda", dtype=torch.int32) // samples).contiguous()
    i = torch.arange(n, device="cuda", dtype=torch.int32)
    one = torch.where(i % samples == 0, i // samples, -1).to(torch.int32).contiguous()   # robot r -> env r * samples
    ret = torch.zeros(n, device="cuda")
    act = torch.zeros((n, nu), device="cuda")
    ar = torch.arange(robots, device="cuda")

    def plan_step():
        eng.load_state(R, fork, obs_out=obs)
        ret.zero_()
        for h in range(horizon):
            eng.step(plans[h], auto_reset=True)
            ret.add_(eng.reward)
        best = ret.view(robots, samples).argmax(1)
        act[::samples] = plans[0].view(robots, samples, nu)[ar, best]
        eng.load_state(R, one, obs_out=obs)
        eng.step(act, auto_reset=True)
        eng.save_state(eng.next_obs, out=S)
        R.copy_(S[::samples])

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        plan_step()                                                     # (warm-up outside the capture)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan_step()
    ms = timed(graph.replay, steps, warmup)
    eng.close()
    return ms


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, watts, sm, sm_max = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return dict(nvidia_smi_name=name, power_limit_w=float(watts), sm_clock_mhz=float(sm), sm_clock_max_mhz=float(sm_max))
    except Exception:
        return dict(nvidia_smi_name=None, power_limit_w=None, sm_clock_mhz=None, sm_clock_max_mhz=None)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--robots", type=int, default=64)
    p.add_argument("--samples", type=int, default=64)
    p.add_argument("--horizon", type=int, default=16)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    results = []
    for task in TASKS:
        env, act = make(task, a.envs, 0)
        for rnd in range(a.rounds):
            for r in measure_calls(env, act, a.steps, a.warmup, ""):
                results.append(dict(r, task=task, round=rnd))
                print(json.dumps(results[-1]), flush=True)
        for name in ("body_state", "reference_body_state", "contact_wrench", "dof_outputs"):
            getattr(env, name)
        for rnd in range(a.rounds):
            for r in measure_calls(env, act, a.steps, a.warmup, "+out"):
                results.append(dict(r, task=task, round=rnd))
                print(json.dumps(results[-1]), flush=True)
        env._get_engine().close()
        torch.cuda.empty_cache()
    plan = []
    for rnd in range(a.rounds):
        ms = planner(a.robots, a.samples, a.horizon, max(10, a.steps // 5), 3)
        plan.append(ms)
        print(json.dumps({"planner": "%d robots x %d samples, horizon %d" % (a.robots, a.samples, a.horizon),
                          "ms_per_planning_step": ms, "planning_steps_per_s": 1e3 / ms, "round": rnd}), flush=True)
    summary = {}
    for r in results:
        summary.setdefault("%s / %s" % (r["task"], r["call"]), []).append(r["us_per_call"])
    summary = {k: {"median_us": statistics.median(v), "min_us": min(v), "max_us": max(v)} for k, v in summary.items()}
    row_mb = {t: next(r["row_mb"] for r in results if r["task"] == t and r["call"] == "save") for t in TASKS}
    meta = dict(gpu_info(), device=torch.cuda.get_device_name(0),
                method="CUDA events per call, L2 flush between calls, %d-step rollout, %d warm-up, median of %d timed calls, "
                       "%d alternating rounds; planner: CUDA-graph replays, same timing" % (PREROLL, a.warmup, a.steps, a.rounds),
                us_per_call=summary, row_mb_per_call=row_mb,
                planner={"robots": a.robots, "samples": a.samples, "horizon": a.horizon,
                         "median_ms_per_planning_step": statistics.median(plan),
                         "median_planning_steps_per_s": 1e3 / statistics.median(plan)})
    print(json.dumps(meta), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(meta, results=results), f, indent=1)


if __name__ == "__main__":
    main()
