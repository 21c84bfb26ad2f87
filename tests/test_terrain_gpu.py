"""Height-field terrain on the GPU (include/locosim.h locosim_set_terrain_origin): UnitreeA1 with distinct per-env origins on a
tiled rough field against the fp64 reference (tests/csrc/terrain_ref.c) on every launch path, state and contact list;
bit-identical reruns and CUDA graph replays; the dataset inverse with fewer envs than dataset rows; rays and the camera;
and the refusals."""
import os

import numpy as np
import pytest

import terrain_ref
from helpers import make_env

pytestmark = pytest.mark.gpu


def _env(n, **kw):
    from loco_mujoco_b200 import terrain
    hf = terrain.tiled_terrain(n_rows=2, n_cols=4, tile_size=2.0, resolution=0.05, max_rough=0.04, max_slope=0.25,
                               max_step=0.06, step_width=0.2, platform=0.4, seed=1)
    return make_env("UnitreeA1.simple", num_envs=n, seed=3, terrain=hf, **kw), hf


@pytest.mark.parametrize("path", ["fused", "substep", "persist"])
def test_engine_matches_the_reference_with_per_env_origins(bundled_only, monkeypatch, path):
    import torch
    from loco_mujoco_b200 import modelpack
    if path == "fused":
        monkeypatch.setenv("LOCOSIM_RESORT", "100")
    elif path == "substep":
        monkeypatch.setenv("LOCOSIM_RESORT", "2")
    else:
        monkeypatch.setenv("LOCOSIM_PERSIST", "1")
    n = 16
    env, hf = _env(n)
    eng = env._get_engine()
    origins = hf.tile_origins()
    env.terrain_origin.copy_(torch.as_tensor(origins[np.arange(n) % len(origins)], dtype=torch.float32))
    cl = env.contacts
    env.reset()
    spec = env.task_spec()
    mg, gp = np.asarray(env._model.geom_margin), np.asarray(env._model.geom_gap)
    same, total = 0, 0
    lib = terrain_ref.load()
    blobs = modelpack.pack(env._model)
    g = torch.Generator().manual_seed(0)
    worst = 0.0
    for k in range(5):
        q0, v0 = (t.cpu().numpy().astype(np.float64) for t in eng.get_state()[:2])
        act = (torch.rand((n, env._model.nu), generator=g) * 2 - 1) * 0.3
        env.step(act.to(eng.device))
        q1, v1 = (t.cpu().numpy().astype(np.float64) for t in eng.get_state()[:2])
        for i in range(n):
            rs = terrain_ref.Sim(lib, blobs)
            rs.set_origin(origins[i % len(origins)])
            rs.reset(q0[i], v0[i])
            ctrl = np.zeros(env._model.nu)
            ctrl[spec.act_idx] = act[i].numpy() * spec.act_delta + spec.act_mean
            # the contact list after the step is the last sub-step's, at its start state: the reference's forward there
            rs.step(ctrl, spec.n_substeps - 1)
            rs.forward(ctrl)
            incl = lambda a, b: max(mg[a], mg[b]) - max(gp[a], gp[b])
            cr = [r for r in rs.contacts() if r[0] < incl(int(r[7]), int(r[8]))]
            nc = int(cl.ncon[i])
            ce, de = cl.geom[i, :nc].cpu().numpy(), cl.dist[i, :nc].cpu().numpy()
            if nc == 16 or len(cr) > 16:
                continue                                 # (a cap binds: which contacts fall off depends on the drift)
            # contacts within 2 mm of their inclusion distance may be in one list only (the drift of nine sub-steps)
            ke = [(int(a), int(b)) for (a, b), d in zip(ce, de) if d < incl(a, b) - 2e-3]
            kr = [(int(r[7]), int(r[8])) for r in cr if r[0] < incl(int(r[7]), int(r[8])) - 2e-3]
            total += 1
            same += ke == kr
            rs.reset(q0[i], v0[i])
            rs.step(ctrl, spec.n_substeps)
            q, _ = rs.state()
            worst = max(worst, float(np.abs(q - q1[i]).max()))
            rs.close()
    # (five control steps of fp32 against fp64 on rough terrain: DESIGN.md section 6)
    assert worst < 1e-2, worst
    # the contact list in order, where no cap binds and away from the inclusion distance
    # (measured on an H100: 61 of 69 env-steps identical on every launch path)
    assert total >= 20 and same >= 0.8 * total, (same, total)


def test_two_runs_and_a_graph_replay_are_bit_identical(bundled_only):
    import torch
    outs = []
    for _ in range(2):
        env, hf = _env(64, copy_outputs=False)
        o = hf.tile_origins()
        env.terrain_origin.copy_(torch.as_tensor(o[np.arange(64) % len(o)], dtype=torch.float32))
        env.reset()
        eng = env._get_engine()
        a = torch.zeros((64, env._model.nu), device=eng.device)
        for _ in range(10):
            env.step(a)
        outs.append(torch.cat([t.flatten() for t in eng.get_state()[:2]]).cpu())
    assert torch.equal(outs[0], outs[1])
    # a step captured in a CUDA graph replays bit for bit
    env, hf = _env(64, copy_outputs=False)
    o = hf.tile_origins()
    env.terrain_origin.copy_(torch.as_tensor(o[np.arange(64) % len(o)], dtype=torch.float32))
    env.reset()
    eng = env._get_engine()
    a = torch.zeros((64, env._model.nu), device=eng.device)
    saved = env.save_state()
    env.step(a)
    ref_state = torch.cat([t.flatten() for t in eng.get_state()[:2]]).clone()
    env.load_state(saved)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            eng.step(a, auto_reset=False)
    env.load_state(saved)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([t.flatten() for t in eng.get_state()[:2]]), ref_state)


def test_refusals(bundled_only):
    import torch
    env, _ = _env(8)
    eng = env._get_engine()
    with pytest.raises(ValueError):
        eng.set_terrain_origin(torch.zeros((8, 3), device=eng.device))
    plain = make_env("UnitreeA1.simple", num_envs=8)
    with pytest.raises(RuntimeError, match="no terrain"):
        plain._get_engine().set_terrain_origin(torch.zeros((8, 2), device=eng.device))


def test_rays_and_camera_see_the_field(bundled_only):
    """Vertical and slanted rays of every env against the fp64 brute force (terrain_ref.ray_hfield), each env at its own
    terrain origin; the robot is lifted out of the way. camera() sees the terrain too."""
    import torch
    n = 8
    env, hf = _env(n)
    eng = env._get_engine()
    o = hf.tile_origins()[:n] + np.array([0.37, -0.21])          # (off the platforms)
    env.terrain_origin.copy_(torch.as_tensor(o, dtype=torch.float32))
    env.reset()
    cam = env.camera(32, 24)
    assert (cam["geom"] == env._model.ngeom - 1).any()
    q, v = (t.clone() for t in eng.get_state()[:2])
    q[:, env._model.joint_id("trunk_tz")] += 5.0
    eng.set_state(q, v)
    rng = np.random.RandomState(0)
    pnt = np.c_[rng.uniform(-0.9, 0.9, (64, 2)), np.full(64, 1.0)]
    vec = np.c_[rng.uniform(-0.3, 0.3, (64, 2)), -np.ones(64)]
    P = torch.as_tensor(pnt, dtype=torch.float32, device=eng.device)
    V = torch.as_tensor(vec, dtype=torch.float32, device=eng.device)
    d = torch.zeros((n, 64), device=eng.device)
    g = torch.zeros((n, 64), dtype=torch.int32, device=eng.device)
    nr = torch.zeros((n, 64, 3), device=eng.device)
    eng.ray(P, V, d, g, nr, flags=1)
    d, g, nr = d.cpu().numpy(), g.cpu().numpy(), nr.cpu().numpy()
    tg = env._model.ngeom - 1
    checked = 0
    for i in range(n):
        for k in range(64):
            x, nn = terrain_ref.ray_hfield(hf, o[i], pnt[k], vec[k])
            if x < 0 or x > 1.0 - 1e-4:             # (at or below z = 0 the floor plane comes first or ties)
                continue
            assert g[i, k] == tg and abs(d[i, k] - x) < 2e-5, (i, k, d[i, k], x)
            np.testing.assert_allclose(nr[i, k], nn, atol=1e-4)
            checked += 1
    assert checked > 50


def test_dataset_inverse_with_fewer_envs_than_rows_takes_the_zero_origin(bundled_only):
    """locosim_create_dataset_inverse evaluates dataset rows, not envs: with an origin registered for 8 envs and ~300 rows,
    every row is computed at the zero terrain origin (as on a handle whose origin was never registered)."""
    import torch
    env, hf = _env(8)
    a = env.create_dataset_inverse().clone()
    o = hf.tile_origins()
    env.terrain_origin.copy_(torch.as_tensor(o[np.arange(8) % len(o)] + 0.3, dtype=torch.float32))
    b = env.create_dataset_inverse()
    torch.cuda.synchronize()
    assert a.shape[0] > 8 and torch.equal(a, b)
