"""
Throughput of the full-body robot humanoids (arms, and for Atlas the back joint) on one GPU, measured the way bench.py
measures its workloads (it reuses bench.Workload): CUDA events around each step, an L2 flush between steps, 40 untimed
steps after the mass reset, then --warmup and --steps timed steps of U(-1, 1) actions with auto-reset.

Workloads: each variant alone at --envs envs, and Atlas with arms + Talos with arms, both with their bundled DR pools,
as one MixedBatch of --envs / 4 + --envs / 4 envs (the full-body analogue of bench.py's config 4). Next to each, the
CPU oracle's rate on the same model (bench.cpu_rollout: the fp64 C restatement on pinned host threads).

One JSON line per workload on stdout, and all of them with the device name and power limit in --out (optional).
    python tools/bench_full_body.py [--envs 4096] [--steps 200] [--warmup 20] [--cpu-seconds 5] [--out FILE]
"""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")
# the compiled variants and their DR pools (tools/build_assets.py, tools/build_dr_pools.py)
os.environ["LOCO_MUJOCO_B200_ASSET_PATH"] = os.pathsep.join(
    [p for p in (os.environ.get("LOCO_MUJOCO_B200_ASSET_PATH"), os.path.join(ROOT, "tests", "golden", "full_body")) if p])
import bench                                                               # noqa: E402

ARMS = dict(disable_arms=False)
DR = lambda robot: dict(ARMS, domain_randomization_config="domain_randomization_%s.yaml" % robot)   # noqa: E731


def workloads(n):
    return [("Atlas.walk+arms", [("Atlas.walk", n, ARMS)]),
            ("Atlas.walk+arms+back", [("Atlas.walk", n, dict(ARMS, disable_back_joint=False))]),
            ("Talos.walk+arms", [("Talos.walk", n, ARMS)]),
            ("UnitreeH1.walk+arms", [("UnitreeH1.walk", n, ARMS)]),
            ("Atlas.walk+arms + Talos.walk+arms, DR, MixedBatch",
             [("Atlas.walk", n // 4, DR("atlas")), ("Talos.walk", n // 4, DR("talos"))])]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--cpu-seconds", type=float, default=5.0, help="oracle timing per model (0: skip)")
    p.add_argument("--out", default=None)
    a = p.parse_args()
    import torch
    from loco_mujoco_b200 import LocoEnv
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures the GPU")
    ma = types.SimpleNamespace(steps=a.steps, warmup=a.warmup, no_flush=False, gather_chunk=0)
    sampler = bench.ClockSampler(0)
    sampler.start()
    results, cpu = [], {}
    for name, members in workloads(a.envs):
        w = bench.Workload(name, members, rank=0, world=1, local=0)
        res = w.measure(ma, 0, gather=False)
        wpb = [e.launch_info()["warps_per_block"] for e in w.engines]
        rates = {}
        for task, _, kw in members:
            variant = {k: v for k, v in kw.items() if k.startswith("disable_")}
            label = LocoEnv._registered_envs[task.split(".")[0]].variant_suffix(**variant)
            label = task + label
            if a.cpu_seconds > 0 and label not in cpu:
                cpu[label] = bench.cpu_rollout(LocoEnv.make(task + ".real", debug=True, **variant), a.cpu_seconds,
                                               bench.host_cores()[0])
            rates[label] = cpu[label]["value"] if label in cpu else None
        out = {"workload": name, "envs": sum(n for _, n, _ in members), "env_steps_per_s": res["value"],
               "ms_per_step": res["ms_per_step"], "kernel_ms_per_step": res["kernel_ms_per_step"],
               "gpu_launches": res["gpu_launches"], "resets_in_run": res["resets_in_run"],
               "nonfinite_in_run": res["nonfinite_in_run"], "warps_per_block": wpb, "cpu_oracle_env_steps_per_s": rates}
        print(json.dumps(out), flush=True)
        results.append(out)
        del w
        torch.cuda.empty_cache()
    clocks = sampler.stop()
    meta = {"device": torch.cuda.get_device_name(0), "power_limit_w": clocks.get("power_limit_w"),
            "sm_mhz_median": clocks.get("sm_mhz"), "clock_reasons": clocks.get("reasons"),
            "method": "bench.Workload.measure: CUDA events, L2 flush between steps, %d-step pre-roll, %d warm-up, %d timed"
                      % (bench.PREROLL, a.warmup, a.steps),
            "cpu_oracle": cpu}
    print(json.dumps(meta), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(meta, results=results), f, indent=1)


if __name__ == "__main__":
    main()
