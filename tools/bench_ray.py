"""Ray casting (include/locosim.h locosim_ray; LocoEnv.ray_cast / camera) on the GPU: rays/s of a legged-gym-style height
scan (11 x 17 rays in the root's heading frame, 4096 envs) and of a 128 x 128 follow camera (256 envs), each next to the
time of one step() of the same env. Prints one JSON line per task, and the card's name and power limit first.

    python tools/bench_ray.py [--tasks UnitreeA1.simple Atlas.walk ...] [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")


def timed(fn, reps):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def main():
    import torch
    from loco_mujoco_b200 import LocoEnv
    ap = argparse.ArgumentParser()
    ap.add_argument("--tasks", nargs="+", default=["UnitreeA1.simple", "Atlas.walk", "HumanoidTorque.run",
                                                   "UnitreeG1.walk"])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=smi)), flush=True)
    for task in args.tasks:
        row = dict(task=task)
        # height scan: 11 x 17 grid, 0.1 m spacing, from 0.5 m above the root, straight down, heading frame
        n = 4096
        env = LocoEnv.make(task + ".real", num_envs=n, debug=True, copy_outputs=False)
        env.reset()
        gx, gy = torch.meshgrid(torch.linspace(-0.8, 0.8, 17), torch.linspace(-0.5, 0.5, 11), indexing="ij")
        pnt = torch.stack([gx.flatten(), gy.flatten(), torch.full((187,), 0.5)], dim=1).cuda()
        vec = torch.tensor([[0.0, 0.0, -1.0]]).expand(187, 3).contiguous().cuda()
        out = env.ray_cast(pnt, vec, mode="heading")
        act = torch.zeros((n, env._model.nu), device="cuda")
        t_scan = timed(lambda: env.ray_cast(pnt, vec, mode="heading", out=out), args.reps)
        t_step = timed(lambda: env.step(act), args.reps)
        row.update(scan_envs=n, scan_rays=187, scan_ms=t_scan * 1e3, scan_rays_per_s=n * 187 / t_scan,
                   step_ms_4096=t_step * 1e3, scan_hit_fraction=float((out["geom"] >= 0).float().mean()))
        del env
        torch.cuda.empty_cache()
        # follow camera, 128 x 128, 256 envs
        n = 256
        env = LocoEnv.make(task + ".real", num_envs=n, debug=True, copy_outputs=False)
        env.reset()
        cam = env.camera(128, 128)
        act = torch.zeros((n, env._model.nu), device="cuda")
        t_cam = timed(lambda: env.camera(128, 128, out=cam), args.reps)
        t_step = timed(lambda: env.step(act), args.reps)
        row.update(camera_envs=n, camera_ms=t_cam * 1e3, camera_rays_per_s=n * 128 * 128 / t_cam, step_ms_256=t_step * 1e3,
                   camera_robot_fraction=float((cam["body"] > 0).float().mean()))
        print(json.dumps(row), flush=True)
        del env
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
