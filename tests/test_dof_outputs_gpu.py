"""Per-dof outputs on the GPU (include/locosim.h locosim_set_dof_outputs; LocoEnv.dof_outputs): registering them changes no
other bit, parity with the fp64 reference (tests/dof_outputs_ref.py) from the engine's own pre-step states for every kernel
family and for UnitreeA1 in position mode, the three launch paths bit for bit, terminal steps of auto-reset envs, non-finite
envs, CUDA graphs (one captured before the registration included), sharding, MixedBatch members, and a push seen in qacc."""
import os

import numpy as np
import pytest
import torch

import dof_outputs_ref as dor
from full_body import make_variant
from helpers import blobs, make_env
from position_mode import make_position
from test_dof_outputs import within

pytestmark = pytest.mark.gpu

# launch paths of UnitreeA1 (environment variables read when an engine is created, locosim.cu setup_cfg)
PATHS = {"fused": {"LOCOSIM_RESORT": "10"}, "substeps": {"LOCOSIM_RESORT": "2"},
         "persistent": {"LOCOSIM_RESORT": "2", "LOCOSIM_PERSIST": "1"}}
# one task per kernel family: CfgEllEuler (three launch paths, torque and position control), CfgPyrEuler, CfgPyrRK4,
# CfgPyrEuler29, CfgPyrRK4_31, CfgPyrEuler31
FAMILIES = [("UnitreeA1.simple", "fused"), ("UnitreeA1.simple", "substeps"), ("UnitreeA1.simple", "persistent"),
            ("UnitreeA1.simple+position", "fused"), ("UnitreeA1.simple+position", "substeps"),
            ("UnitreeA1.simple+position", "persistent"),
            ("Talos.walk", None), ("HumanoidTorque.run", None), ("UnitreeG1.walk", None), ("Atlas.walk+arms", None),
            ("Talos.walk+arms", None)]


@pytest.fixture(scope="module")
def ref():
    return dor.load()


def _with_env(vars_, fn):
    old = {k: os.environ.get(k) for k in vars_}
    os.environ.update(vars_)
    try:
        return fn()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _make(task, path=None, **kw):
    if task.endswith("+position"):
        build = lambda: make_position(task[:-len("+position")], **kw)          # noqa: E731
    else:
        build = lambda: make_variant(task, **kw)                                # noqa: E731
    env = _with_env(PATHS[path] if path else {}, build)
    _with_env(PATHS[path] if path else {}, env._get_engine)
    return env


@pytest.mark.parametrize("task,path", FAMILIES)
def test_registered_outputs_change_no_other_bit(ref, bundled_only, task, path):
    """512 envs: an engine with dof outputs registered steps bit for bit like one without (auto-resets included); from the
    engine's own pre-step state and warm start, sampled rows match the fp64 reference's sub-step mean within the tolerance of
    tests/test_dof_outputs.py (or within 10x the oracle's own jump where a contact switches within the step)."""
    n = 512
    a, b = _make(task, path, num_envs=n, seed=7), _make(task, path, num_envs=n, seed=7)
    d = b.dof_outputs
    assert torch.equal(a.reset(), b.reset())
    eng = b._get_engine()
    mb, tb = blobs(b)
    user = b._model_user_features[0]
    gen = torch.Generator().manual_seed(0)
    nu = a.info.action_space.shape[0]
    checked, allowed, constrained = 0, 0, 0
    for k in range(4):
        act = (torch.rand((n, nu), generator=gen) * 2 - 1).cuda()
        q0, v0, w0 = (x.cpu().numpy().astype(np.float64) for x in eng.get_state())
        ra, rb = a.step(act), b.step(act)
        for x, y in zip(ra[:3], rb[:3]):
            assert torch.equal(x, y)
        assert torch.equal(ra[3]["next_obs"], rb[3]["next_obs"])
        rows = d.cpu().numpy()
        an = act.cpu().numpy().astype(np.float64)
        for i in range(k, n, 43):
            oe = ref.env(mb, tb)
            oe.set_user(user)
            oe.set_state(q0[i], v0[i], w0[i])
            want, _, _ = dor.env_step(ref, oe, an[i])
            oe.close()
            constrained += int(np.abs(want[:, 1]).max() > 1.0)
            ok, err, tol = within(rows[i], want)
            if not ok:
                gap = dor.sensitivity(ref, mb, tb, q0[i], v0[i], an[i], want, warmstart=w0[i], eps=1e-6, n_probe=8,
                                      user=user)
                ok, err, tol = within(rows[i], want, gap)
                assert ok, (task, k, i, err, tol, gap)
                allowed += 1
            checked += 1
    for x, y in zip(a._get_engine().get_state(), eng.get_state()):
        assert torch.equal(x, y)
    assert constrained > checked // 4, (constrained, checked)
    assert allowed <= max(2, checked // 20), (allowed, checked)


@pytest.mark.parametrize("task", ["UnitreeA1.simple", "UnitreeA1.simple+position"])
def test_launch_paths_agree_bit_for_bit(bundled_only, task):
    n = 512
    envs = [_make(task, p, num_envs=n, seed=3) for p in PATHS]
    for e in envs:
        e.dof_outputs
    obs = [e.reset() for e in envs]
    assert all(torch.equal(obs[0], o) for o in obs[1:])
    gen = torch.Generator().manual_seed(2)
    resets = 0
    for _ in range(8):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        outs = [e.step(act) for e in envs]
        resets += int(outs[0][2].bool().sum())
        for e, o in zip(envs[1:], outs[1:]):
            assert torch.equal(outs[0][0], o[0])
            assert torch.equal(envs[0].dof_outputs, e.dof_outputs)
    assert resets > 0 and float(envs[0].dof_outputs.abs().max()) > 0


@pytest.mark.parametrize("task,path", FAMILIES)
def test_terminal_rows_of_auto_reset_envs(bundled_only, task, path):
    """In lock-step from the same state, a twin engine steps with auto_reset=False: the dof rows of the two are equal bit for
    bit, those of the envs the first one ended and reset included. The twin then resets exactly those envs and the two agree
    again."""
    n = 512
    a, b = _make(task, path, num_envs=n, seed=13), _make(task, path, num_envs=n, seed=13)
    ea, eb = a._get_engine(), b._get_engine()
    da_, db_ = a.dof_outputs, b.dof_outputs
    assert torch.equal(ea.reset(), eb.reset())
    gen = torch.Generator().manual_seed(8)
    ended = 0
    for k in range(8):
        act = (torch.rand((n, ea.action_dim), generator=gen) * 2 - 1).cuda()
        _, _, da, _ = ea.step(act, auto_reset=True)
        _, _, db, _ = eb.step(act, auto_reset=False)
        assert torch.equal(da, db)
        assert torch.equal(da_, db_)
        done = da.bool()
        ended += int(done.sum())
        if bool(done.any()):
            q, _, _ = eb.get_state()
            fin = torch.isfinite(q).all(dim=1)
            eb.reset(mask=(done & fin).to(torch.uint8))
        for x, y in zip(ea.get_state(), eb.get_state()):
            assert torch.equal(x, y)
    assert ended > 0, "no env ended: the terminal rows were not exercised"


def test_a_non_finite_env_gets_a_zero_row(bundled_only):
    """a NaN in one env's qpos (set_state: a value, not a fault): the step reports it done with all-zero obs and dof rows"""
    for task in ("UnitreeA1.simple", "UnitreeA1.simple+position"):
        for path in PATHS:
            n = 64
            env = _make(task, path, num_envs=n, seed=9)
            eng = env._get_engine()
            env.reset()
            d = env.dof_outputs
            d.fill_(7.0)
            q, v, _ = eng.get_state()
            q[5, 3] = float("nan")
            eng.set_state(q.contiguous(), v.contiguous())
            obs, _, done, _ = env.step(torch.zeros((n, 12), device="cuda"))
            assert bool(done[5]) and float(obs[5].abs().max()) == 0.0
            assert float(d[5].abs().max()) == 0.0 and bool(torch.isfinite(d).all())
            assert not bool((d == 7.0).all(dim=2).all(dim=1).any())        # every env's row was written


def test_reset_and_set_state_leave_the_rows_alone(bundled_only):
    n = 64
    env = make_env("UnitreeA1.simple", num_envs=n, seed=4)
    eng = env._get_engine()
    env.reset()
    d = env.dof_outputs
    env.step(torch.zeros((n, 12), device="cuda"))
    keep = d.clone()
    env.reset()
    q, v, _ = eng.get_state()
    eng.set_state(q, v)
    torch.cuda.synchronize()
    assert torch.equal(d, keep)


def test_graphs_captured_before_and_after_registering(bundled_only):
    """the step kernels read the registration when they run: a graph captured while nothing was registered writes the
    buffer at replays after the registration, as an eager engine does; registering None stops it"""
    n, steps = 256, 6
    eager = make_position(num_envs=n, seed=21)
    early = make_position(num_envs=n, seed=21)
    de = eager.dof_outputs
    assert torch.equal(eager.reset(), early.reset())
    warm = make_position(num_envs=n, seed=99)
    warm.reset()
    static_act = torch.zeros((n, 12), device="cuda")
    warm._get_engine().step(static_act)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                               # nothing registered yet
        early._get_engine().step(static_act)
    dg = early.dof_outputs                                      # registered after the capture
    eager._get_engine().step(torch.zeros((n, 12), device="cuda"))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(de, dg)
    gen = torch.Generator().manual_seed(5)
    for _ in range(steps):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        eager.step(act)
        static_act.copy_(act)
        dg.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(de, dg) and float(dg.abs().max()) > 0
    # a graph captured after the registration
    graph2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph2):
        early._get_engine().step(static_act)
    act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
    eager.step(act)
    static_act.copy_(act)
    graph2.replay()
    torch.cuda.synchronize()
    assert torch.equal(de, dg)
    early._get_engine().set_dof_outputs(None)
    dg.zero_()
    graph.replay()
    graph2.replay()
    torch.cuda.synchronize()
    assert float(dg.abs().max()) == 0.0


def test_two_shards_equal_one_batch(bundled_only):
    n, steps = 64, 6
    full = make_position(num_envs=n, seed=11)
    a = make_position(num_envs=n // 2, seed=11, env_id_offset=0)
    b = make_position(num_envs=n // 2, seed=11, env_id_offset=n // 2)
    for e in (full, a, b):
        e.dof_outputs
    assert torch.equal(full.reset(), torch.cat([a.reset(), b.reset()]))
    gen = torch.Generator().manual_seed(1)
    for _ in range(steps):
        act = (torch.rand((n, 12), generator=gen) * 2 - 1).cuda()
        full.step(act)
        a.step(act[:n // 2].contiguous())
        b.step(act[n // 2:].contiguous())
        assert torch.equal(full.dof_outputs, torch.cat([a.dof_outputs, b.dof_outputs]))


def test_mixed_batch_members_expose_their_own_rows(bundled_only):
    from loco_mujoco_b200.parallel import MixedBatch
    n = 48
    mb = MixedBatch([("Atlas.walk.real", n, {}), ("Talos.walk.real", n, {})], device="cuda:0", seed=3, debug=True)
    solo = [make_env("Atlas.walk", num_envs=n, seed=3, env_id_offset=0), make_env("Talos.walk", num_envs=n, seed=3, env_id_offset=n)]
    for e in mb.envs + solo:
        e.dof_outputs
    mb.reset()
    for e in solo:
        e.reset()
    gen = torch.Generator().manual_seed(4)
    for _ in range(4):
        acts = [(torch.rand((n, e.action_dim), generator=gen) * 2 - 1).cuda() for e in mb.engines]
        mb.step(acts)
        for e, a in zip(solo, acts):
            e.step(a)
        torch.cuda.synchronize()
        for m, s in zip(mb.envs, solo):
            assert m.dof_outputs.shape[1] == s._model.nq
            assert torch.equal(m.dof_outputs, s.dof_outputs)
    assert float(mb.envs[0].dof_outputs.abs().max()) > 0


def test_a_push_shows_in_qacc(bundled_only):
    """UnitreeA1 in position mode, half of the envs pushed by a horizontal force +F x on the trunk's CoM for one control step
    from the same states: the trunk's x slide accelerates more in +x (its qacc mean rises), and the push changes neither the
    actuator forces' clamp nor the other envs"""
    n, F = 16, 200.0
    env = make_position(num_envs=2 * n, seed=1)
    eng = env._get_engine()
    m = env._model
    env.reset()
    q, v, _ = eng.get_state()
    eng.set_state(torch.cat([q[:n], q[:n]]).contiguous(), torch.cat([v[:n], v[:n]]).contiguous())
    d = env.dof_outputs
    tx = m.jnt_names.index("trunk_tx")
    env.xfrc_applied.zero_()
    env.xfrc_applied[n:, env.body_index("trunk"), 0] = F
    eng.step(torch.zeros((2 * n, m.nu), device="cuda"), auto_reset=False)
    acc = d[:, tx, 2].cpu().numpy()
    shift = acc[n:] - acc[:n]
    total, trunk = float(m.body_mass.sum()), float(m.body_mass[env.body_index("trunk")])
    # (the contacts resist part of the push, and the legs lag behind the trunk: the shift is positive, and at most what the
    #  trunk alone would get)
    assert np.all(shift > 0.05 * F / total) and np.all(shift < F / trunk), (shift, F / total, F / trunk)
    assert float(d[:, :, 0].abs().max()) <= 33.5 * (1 + 1e-6)            # (a mean of forces clamped to +-33.5)
