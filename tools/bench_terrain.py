"""UnitreeA1 on height-field terrain (include/locosim.h locosim_set_terrain_origin) on the GPU, with bench.py's method (U(-1,1)
actions, auto-reset, warm-up, CUDA events around the timed steps): env-steps/s at 4096 envs without a terrain, on a flat
field and on the rough tiled field of loco_mujoco_b200.terrain.tiled_terrain (envs spread over its tiles), with the mean
number of terrain contacts per env in the contact list after a step and the mean number of terrain MPR runs per env and
control step (counted by the fp64 reference, tests/terrain_ref.py, on a sample of envs from their engine states). Prints
the card's name, power limit and SM clock first, then one JSON line per field.

    python tools/bench_terrain.py [--envs 4096] [--steps 200] [--warmup 20] [--sample 32]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ.setdefault("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")


def run(name, hf, args):
    import numpy as np
    import torch
    from loco_mujoco_b200 import LocoEnv, modelpack
    n = args.envs
    kw = {} if hf is None else dict(terrain=hf)
    env = LocoEnv.make("UnitreeA1.simple.real", num_envs=n, debug=True, copy_outputs=False, seed=0, **kw)
    origins = None
    if hf is not None and hf.tiles is not None:
        o = hf.tile_origins()
        origins = o[np.arange(n) % len(o)]
        env.terrain_origin.copy_(torch.as_tensor(origins, dtype=torch.float32))
    cl = env.contacts
    env.reset()
    g = torch.Generator(device="cuda").manual_seed(0)
    nu = env._model.nu

    def step():
        env.step(torch.rand((n, nu), generator=g, device="cuda") * 2 - 1)
    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        step()
    b.record()
    b.synchronize()
    dt = a.elapsed_time(b) * 1e-3 / args.steps
    row = dict(field=name, envs=n, env_steps_per_s=n / dt, ms_per_step=dt * 1e3)
    if hf is not None:
        tg = env._model.ngeom - 1
        k = torch.arange(cl.geom.shape[1], device=cl.geom.device)[None, :] < cl.ncon[:, None]
        row["terrain_contacts_per_env"] = float(((cl.geom[..., 0] == tg) & k).sum()) / n
        import terrain_ref
        lib = terrain_ref.load()
        blobs = modelpack.pack(env._model)
        spec = env.task_spec()
        q, v = (t.cpu().numpy().astype(np.float64) for t in env._get_engine().get_state()[:2])
        c0 = lib.reft_mpr_calls()
        for i in range(min(args.sample, n)):
            rs = terrain_ref.Sim(lib, blobs)
            if origins is not None:
                rs.set_origin(origins[i])
            rs.reset(q[i], v[i])
            ctrl = np.zeros(nu)
            ctrl[spec.act_idx] = np.random.RandomState(i).uniform(-1, 1, nu) * spec.act_delta + spec.act_mean
            rs.step(ctrl, spec.n_substeps)
            rs.close()
        row["reference_terrain_mpr_per_env_step"] = (lib.reft_mpr_calls() - c0) / min(args.sample, n)
    print(json.dumps(row), flush=True)
    del env
    torch.cuda.empty_cache()


def main():
    import numpy as np
    from loco_mujoco_b200 import terrain
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--sample", type=int, default=32)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=smi)), flush=True)
    run("none", None, args)
    run("flat", terrain.HeightField(np.zeros((161, 161)), (8.0, 8.0), base=0.2), args)
    run("rough", terrain.tiled_terrain(n_rows=4, n_cols=4, tile_size=4.0, resolution=0.05, base=0.2, seed=0), args)


if __name__ == "__main__":
    main()
