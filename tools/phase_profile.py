"""Where a warp's time goes inside one sub-step of the headline workload (UnitreeA1.simple, 4096 envs, random actions).

Builds a diagnostic copy of the engine library with -DLOCOSIM_PHASE_CLOCK into a temporary directory (the in-tree library is
not touched) and runs it by bench.py's method: mass reset, 40 untimed pre-roll steps, --warmup untimed steps, then --steps
timed steps with the 256 MiB L2 flush before each. In that build lane 0 of every warp adds the clock64() cycles of each phase
of its env to a device-side table (locosim_core.cuh, PH_*); a phase's figure is the warp's own latency, i.e. what the env
waits for, and the Newton loop's block barrier (`BLOCK_ANY`, lock-step) is reported apart from the work. Cycles are SM
cycles per env and sub-step (summed over warps, divided by the env-sub-steps run); shares are of the warp's whole sub-step.

Usage: python tools/phase_profile.py [--steps 50] [--warmup 20] [--out DIR]   (writes DIR/phase_profile.json with the GPU's
name, power limit and SM clock)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")

# the order of the PH_* enum in locosim_core.cuh
PHASES = ["kinematics", "com_pos", "crb_factor", "smooth_forces", "collision", "convex_queue", "make_constraint", "warmstart",
          "newton_wait", "newton_trips", "newton_iters", "make_hessian", "chol_factor", "chol_solve", "line_search", "ls_eval",
          "ls_evals", "update_constraint", "update_gradient", "newton_tail", "integrator", "substep", "substeps", "prologue",
          "epilogue", "groups",
          # collision() split: primitive filter rounds, primitive narrow phase + fill_contact, convex bounding spheres, box
          # (and capsule-hull) tests, the job queue's first barrier, own jobs, the wait for the block's other jobs,
          # convex_consume; counts of box-test survivors, of jobs published, of primitive pairs that pass the filter and
          # of primitive narrow sets (rounds) run
          "col_prim_filter", "col_prim_narrow", "col_spheres", "col_obb", "col_queue_wait", "col_jobs", "col_jobs_wait",
          "col_consume", "col_obb_survivors", "col_jobs_published", "col_prim_candidates", "col_prim_sets"]
COUNTS = {"newton_trips", "newton_iters", "ls_evals", "substeps", "groups", "col_obb_survivors", "col_jobs_published",
          "col_prim_candidates", "col_prim_sets"}
COLLISION_SPLIT = ["col_prim_filter", "col_prim_narrow", "col_spheres", "col_obb", "col_queue_wait", "col_jobs",
                   "col_jobs_wait", "col_consume"]


def build_diagnostic(tmp):
    from __graft_entry__ import NVCC_FLAGS
    so = os.path.join(tmp, "liblocosim_cuda.so")
    cmd = [os.environ.get("NVCC", "nvcc")] + [f for f in NVCC_FLAGS if f != "-Xptxas" and f != "-v"] + \
          ["-DLOCOSIM_PHASE_CLOCK", "-o", so, os.path.join(ROOT, "loco_mujoco_b200", "csrc", "locosim.cu")]
    print("[phase_profile]", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return so


def table(raw):
    """Per env-sub-step cycles of every phase, the derived split of make_hessian and line_search, and the shares."""
    c = dict(zip(PHASES, raw))
    n = max(1, c["substeps"])
    cyc = {k: c[k] / n for k in PHASES if k not in COUNTS}
    cyc["hessian_assembly"] = cyc["make_hessian"] - cyc["chol_factor"]
    cyc["line_search_other"] = cyc["line_search"] - cyc["ls_eval"]
    cyc["collision_other"] = cyc["collision"] - cyc["convex_queue"]
    newton_work = sum(cyc[k] for k in ("make_hessian", "chol_solve", "line_search", "update_constraint", "update_gradient"))
    sub = cyc["substep"]
    iters = max(1, c["newton_iters"])
    return {
        "cycles_per_env_substep": cyc,
        "share_of_substep": {k: v / sub for k, v in cyc.items() if k != "substep"},
        "newton_work_share": newton_work / sub,
        "newton_wait_share": cyc["newton_wait"] / sub,
        "newton_share": (newton_work + cyc["newton_wait"]) / sub,
        "per_newton_iteration_cycles": {k: c[k] / iters for k in ("make_hessian", "chol_factor", "chol_solve", "line_search",
                                                                   "ls_eval", "update_constraint", "update_gradient")},
        "iterations_per_solve": c["newton_iters"] / n,
        "lockstep_trips_per_solve": c["newton_trips"] / n,
        "lockstep_efficiency": c["newton_iters"] / max(1, c["newton_trips"]),
        "ls_evals_per_iteration": c["ls_evals"] / iters,
        "collision_split_cycles": {k: cyc[k] for k in COLLISION_SPLIT},
        "collision_unsplit_cycles": cyc["collision"] - sum(cyc[k] for k in COLLISION_SPLIT),
        "convex_jobs_per_env_substep": c["col_jobs_published"] / n,
        "box_test_survivors_per_env_substep": c["col_obb_survivors"] / n,
        "primitive_candidates_per_env_substep": c["col_prim_candidates"] / n,
        "primitive_narrow_sets_per_env_substep": c["col_prim_sets"] / n,
        "env_substeps": c["substeps"], "groups": c["groups"],
        "prologue_epilogue_cycles_per_group": (c["prologue"] + c["epilogue"]) / max(1, c["groups"]),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="UnitreeA1.simple")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=".", help="directory for phase_profile.json (default: the working directory)")
    a = ap.parse_args()
    import torch
    from loco_mujoco_b200 import engine
    with tempfile.TemporaryDirectory(prefix="locosim_phase_") as tmp:
        engine._LIB_PATH = build_diagnostic(tmp)
        lib = engine.load_library()
        lib.locosim_phase_clock.restype = ctypes.c_int
        lib.locosim_phase_clock.argtypes = [ctypes.c_void_p]
        import bench
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()
        wl = bench.Workload(a.task, [(a.task, a.envs, {})], 0, 1, 0)
        dev = wl.dev
        total = bench.PREROLL + a.warmup + a.steps
        gen = torch.Generator(device=dev).manual_seed(1234)
        eng = wl.engines[0]
        acts = torch.rand((total, eng.n_envs, eng.action_dim), device=dev, generator=gen) * 2 - 1
        flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
        wl.batch.reset()
        for k in range(bench.PREROLL + a.warmup):
            wl.step([acts[k]])
        torch.cuda.synchronize()
        raw = (ctypes.c_ulonglong * len(PHASES))()
        if lib.locosim_phase_clock(raw) != len(PHASES):      # (clears the table)
            raise RuntimeError("phase clock: %d phases expected" % len(PHASES))
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.steps)]
        for k in range(a.steps):
            flush.fill_(k & 0xff)
            ev[k][0].record()
            wl.step([acts[bench.PREROLL + a.warmup + k]])
            ev[k][1].record()
        torch.cuda.synchronize()
        lib.locosim_phase_clock(raw)
        res = {"gpu": gpu[0] if gpu else None, "gpu_query": "name, power.limit, clocks.sm, clocks.max.sm",
               "task": a.task, "envs": a.envs, "steps": a.steps, "launch_info": eng.launch_info(),
               "kernel_ms_per_step_with_clock": sum(x.elapsed_time(y) for x, y in ev) / a.steps,
               "raw": dict(zip(PHASES, [int(x) for x in raw]))}
        res.update(table(list(raw)))
        del wl
    print(json.dumps(res, indent=1))
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "phase_profile.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
