"""Where the SMs' time goes in one control step of the headline workload (UnitreeA1.simple, 4096 envs, random actions).

The persistent sub-step kernel records one timeline entry per group (locosim_set_timeline: SM, chunk, envs, pop start, group
start and end from %globaltimer, the group's Newton iterations). Per step this reports
  busy       = sum of group durations / (SMs x span)                 (span: first pop to last group end)
  pop        = sum of time blocks spent popping or waiting for a group / (SMs x span)
  tail_us    = from the first SM going idle for good to the end of the step
  lockstep   = sum of per-env iterations / (warps x the group's largest iteration count), over all groups
and, for the fused kernel, the separate sub-step launches and the persistent kernel, the step time from CUDA events around
each step. The work the SMs have to do is the same on every path, so `step time - work / SMs` (work: the persistent
kernel's summed group durations) estimates the idle SM time of the other two paths.

Usage: python tools/sm_timeline.py [--steps 20] [--out DIR]   (writes DIR/sm_timeline.json with the GPU's name and power
limit)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")

PATHS = {"fused": {"LOCOSIM_RESORT": "100", "LOCOSIM_PERSIST": "0"},
         "split_launches": {"LOCOSIM_RESORT": "2", "LOCOSIM_PERSIST": "0"},
         "persistent": {}}
KNOBS = ("LOCOSIM_RESORT", "LOCOSIM_PERSIST")


def make(task, n, knobs):
    from loco_mujoco_b200 import LocoEnv
    saved = {k: os.environ.get(k) for k in KNOBS}
    for k in KNOBS:
        os.environ.pop(k, None)
    os.environ.update(knobs)
    try:
        env = LocoEnv.make(task + ".real", debug=True, num_envs=n, seed=0)
        eng = env._get_engine()
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v
    return eng


def step_times(eng, acts, warm):
    import torch
    eng.reset()
    for k in range(warm):
        eng.step(acts[k % len(acts)])
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in acts]
    for (a, b), act in zip(ev, acts):
        a.record()
        eng.step(act)
        b.record()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def timeline(eng, acts, warm, cap=8192):
    import numpy as np
    import torch
    buf = torch.zeros((1 + cap, 8), dtype=torch.int64, device=eng.device)
    eng.reset()
    for k in range(warm):
        eng.step(acts[k % len(acts)])
    if eng.lib.locosim_set_timeline(eng.h, buf.data_ptr(), cap) != 0:
        raise RuntimeError(eng.lib.locosim_last_error(eng.h).decode())
    wpb = eng.launch_info()["warps_per_block"]
    steps = []
    for act in acts:
        buf.zero_()
        eng.step(act)
        torch.cuda.synchronize()
        r = buf.cpu().numpy()
        n = int(r[0, 0])
        assert n <= cap, "timeline buffer too small"
        rec = r[1:1 + n]
        sm, t_pop, t0, t1, it_sum, it_max = rec[:, 0], rec[:, 3], rec[:, 4], rec[:, 5], rec[:, 6], rec[:, 7]
        start, end = t_pop.min(), t1.max()
        span = float(end - start)
        sms = np.unique(sm)
        last_end = np.array([t1[sm == s].max() for s in sms])
        steps.append({"span_us": span / 1e3, "groups": n, "sms": int(len(sms)),
                      "busy": float((t1 - t0).sum()) / (len(sms) * span),
                      "pop": float((t0 - t_pop).sum()) / (len(sms) * span),
                      "tail_us": float(end - last_end.min()) / 1e3,
                      "lockstep": float(it_sum.sum()) / max(1.0, float((wpb * it_max).sum())),
                      "work_us": float((t1 - t0).sum()) / 1e3,
                      "envs_per_group": float(rec[:, 2].mean())})
    eng.lib.locosim_set_timeline(eng.h, None, 0)
    return steps


def main():
    import numpy as np
    import torch
    import __graft_entry__
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="UnitreeA1.simple")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--out", default=".", help="directory for sm_timeline.json (default: the working directory)")
    a = ap.parse_args()
    __graft_entry__.build()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    gen = torch.Generator(device="cuda").manual_seed(1234)
    engs = {k: make(a.task, a.envs, v) for k, v in PATHS.items()}
    nu = engs["fused"].action_dim
    acts = [torch.rand((a.envs, nu), device="cuda", generator=gen) * 2 - 1 for _ in range(a.steps)]
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    res = {"gpu": gpu[0] if gpu else None, "task": a.task, "envs": a.envs, "sms": n_sm, "paths": {}}
    tl = timeline(engs["persistent"], acts, a.warmup)
    work_ms = float(np.mean([s["work_us"] for s in tl])) / 1e3
    for k, eng in engs.items():
        t = step_times(eng, acts, a.warmup)
        ms = float(np.median(t))
        res["paths"][k] = {"kernels_per_step": eng.kernels_per_step, "step_ms_median": ms,
                           "sm_idle_estimate": 1.0 - work_ms / n_sm / ms}
    keys = ("span_us", "busy", "pop", "tail_us", "lockstep", "envs_per_group", "groups", "sms")
    res["persistent_timeline"] = {k: float(np.median([s[k] for s in tl])) for k in keys}
    res["work_ms_per_step"] = work_ms
    print(json.dumps(res, indent=1))
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "sm_timeline.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
