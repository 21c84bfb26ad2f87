"""Full-body robot humanoids on the 31-dof configurations, GPU tier (H100): the engine against the fp64 oracle (one batched
step, whole drop-in episodes, foot forces, DR pools), the stage probe on both new configurations, long auto-resetting
runs at 4096 envs, and bitwise scheduling identities (sub-step launches, the persistent kernel, MixedBatch).

The existing checks are reused with their tolerances: their tasks are resolved through full_body.make_variant, and the
batched comparison runs 8 envs per block (the new configurations hold 8 envs per SM, not 12)."""
import copy
import ctypes

import numpy as np
import pytest

import stage_probe as sp
import test_gpu_parity as gpu_parity
import test_gpu_stages as gpu_stages
import test_persistent_kernel as persistent
from full_body import (FP32_ROWS, VARIANTS, build_probe_cuda, build_probe_emu, make_variant, oracle_episode,
                       use_variants_in_stage_probe)
from helpers import oracle_step_sensitivity

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

NEW_CFG = ["Atlas.walk+arms+back", "Talos.walk+arms"]       # one model per new configuration (RK4_31, Euler31)


@pytest.fixture
def variants(monkeypatch):
    use_variants_in_stage_probe(monkeypatch)
    monkeypatch.setattr(gpu_parity, "make_env", lambda task, **kw: make_variant(task, **dict(kw, warps_per_block=8)))
    monkeypatch.setattr(persistent, "make_env", make_variant)


@pytest.fixture(scope="module")
def probe_cuda():
    return sp._bind(ctypes.CDLL(build_probe_cuda()))


@pytest.fixture(scope="module")
def probe_emu():
    return build_probe_emu()


@pytest.mark.parametrize("name", list(VARIANTS))
def test_batched_steps_match_oracle(oracle, bundled_only, variants, name):
    """test_gpu_parity.test_batched_steps_match_oracle on each variant (tolerances, done-flag rule and the
    oracle_step_sensitivity allowance as there)."""
    env = gpu_parity._batched_vs_oracle(oracle, name)
    assert env._get_engine().launch_info()["warps_per_block"] == 8


def test_foot_forces_match_oracle(oracle, bundled_only, variants):
    """use_foot_forces on Atlas with arms and back: a 60 + 12 = 72-wide observation (MAXOBS of the new configurations)."""
    env = gpu_parity._batched_vs_oracle(oracle, "Atlas.walk+arms+back", n_steps=4, use_foot_forces=True)
    assert env.task_spec().obs_dim == env.info.observation_space.shape[0] == 72
    obs = env.reset()
    assert float(obs[:, -12:].abs().max()) == 0.0
    seen = 0.0
    for _ in range(10):
        obs, _, _, _ = env.step(torch.zeros((env.num_envs, env.info.action_space.shape[0]), device="cuda"))
        seen = max(seen, float(obs[:, -12:].abs().max()))
    assert seen > 1e-3, "no ground reaction force ever observed"


@pytest.mark.parametrize("name", list(VARIANTS))
def test_dropin_single_env_follows_oracle_episode(oracle, bundled_only, name):
    """The reference test's protocol through the drop-in API against the oracle's episode: same length, within 5e-3
    (UnitreeH1: over full_body.FP32_ROWS)."""
    want = oracle_episode(oracle, make_variant(name))[0]
    np.random.seed(0)
    env = make_variant(name)
    rows = [env.reset()]
    absorbing = False
    while not absorbing and len(rows) < 1001:
        obs, _, absorbing, _ = env.step(np.random.randn(env.info.action_space.shape[0]) * 0.1)
        rows.append(obs)
    rows = np.array(rows)
    assert np.abs(rows[0] - want[0]).max() < 1e-6
    if name in FP32_ROWS:
        n = FP32_ROWS[name]
        rows, want = rows[:n], want[:n]
    assert rows.shape == want.shape, "episode length %d vs the oracle's %d" % (len(rows), len(want))
    assert np.allclose(rows, want, rtol=5e-3, atol=5e-3), "max abs err %.3e" % np.abs(rows - want).max()


def test_A_cholesky_register_variant_nv31(probe_cuda):
    gpu_stages.test_A_cholesky_register_variant(probe_cuda, 31)


@pytest.mark.parametrize("name", NEW_CFG)
def test_D_structure_matches_serial_build(probe_cuda, probe_emu, oracle, bundled_only, variants, name):
    gpu_stages.test_D_structure_matches_serial_build(probe_cuda, probe_emu, oracle, bundled_only, name)


@pytest.mark.parametrize("name", NEW_CFG)
def test_B_C_E_cuda_record_against_fp64(probe_cuda, probe_emu, oracle, bundled_only, variants, name):
    env, S, e, g, cfg = gpu_stages._records(name, probe_cuda, probe_emu, oracle)
    assert cfg in (4, 5) and int(g["cfg_nv"][0]) == 31
    gpu_stages.test_B_C_E_cuda_record_against_fp64(probe_cuda, probe_emu, oracle, bundled_only, name)


@pytest.mark.parametrize("name", NEW_CFG)
def test_F_scheduling_invariance(probe_cuda, oracle, bundled_only, variants, name):
    gpu_stages.test_F_scheduling_invariance(probe_cuda, oracle, bundled_only, name)


def _model_with_pool_row(m, row):
    """A copy of model m carrying the parameters of one pool row (domain_randomization.POOL_FIELDS layout)."""
    from loco_mujoco_b200.domain_randomization import POOL_FIELDS
    m = copy.deepcopy(m)
    off = 0
    for field, _, _ in POOL_FIELDS:
        shape = np.shape(getattr(m, field))
        n = int(np.prod(shape))
        setattr(m, field, np.asarray(row[off:off + n], dtype=np.float64).reshape(shape))
        off += n
    m.stat_meaninertia = float(row[off])
    return m


@pytest.mark.parametrize("name", ["Atlas.walk+arms", "Talos.walk+arms"])
def test_dr_pool_matches_oracle(oracle, bundled_only, name):
    """The bundled DR pool of each arm variant (tools/build_dr_pools.py from the shipped YAML): every env steps with the
    parameters of the pool row it drew, as the oracle does with a model carrying the same row (tolerance and the
    oracle_step_sensitivity allowance of test_domain_randomization.test_pooled_parameters_match_oracle)."""
    from loco_mujoco_b200 import modelpack
    from loco_mujoco_b200.domain_randomization import pool_row
    robot = name.split(".")[0].lower()
    n = 48
    env = make_variant(name, num_envs=n, seed=4, domain_randomization_config="domain_randomization_%s.yaml" % robot)
    eng = env._get_engine()
    pool = env.domain_randomization_pool()
    assert pool.shape[1] == len(pool_row(env._model))
    assert np.array_equal(pool_row(_model_with_pool_row(env._model, pool[-1])), pool[-1])
    rng = np.random.RandomState(0)
    tr = np.zeros(n, dtype=np.int32)
    st = rng.randint(0, env.trajectories.trajectory_length, n).astype(np.int32)
    eng.reset(traj_no=torch.tensor(tr, device=eng.device), step_no=torch.tensor(st, device=eng.device))
    rows = eng.param_rows().cpu().numpy()
    assert len(pool) == 1 or len(set(rows.tolist())) > 1, "every env drew the same pool row"
    tb = env.task_spec().pack()
    mbs = {int(r): modelpack.pack(_model_with_pool_row(env._model, pool[r])) for r in set(rows.tolist())}
    oes = [oracle.env(mbs[int(r)], tb) for r in rows]
    for i in range(n):
        oes[i].reset_to(tr[i], st[i])
    alive, n_switch = np.ones(n, dtype=bool), 0
    for k in range(2):
        act = rng.uniform(-1, 1, (n, eng.action_dim)).astype(np.float32)
        obs, _, _, _ = eng.step(torch.tensor(act, device=eng.device), auto_reset=False)
        obs = obs.cpu().numpy()
        for i in range(n):
            if not alive[i]:
                continue
            q, v = oes[i].get_state()
            o, _, d = oes[i].step(act[i].astype(np.float64))
            if not np.allclose(obs[i], o, rtol=3e-3 * (k + 1), atol=3e-3 * (k + 1)):
                err = np.abs(obs[i] - o).max()
                gap = oracle_step_sensitivity(oracle, mbs[int(rows[i])], tb, tr[i], st[i], q, v, act[i], o)
                assert err < 2.0 * gap, (k, i, err, gap)
                n_switch += 1
                alive[i] = False
            elif d:
                alive[i] = False
    for oe in oes:
        oe.close()
    assert n_switch <= n // 16, "too many envs disagree with the oracle: %d" % n_switch


@pytest.mark.parametrize("name", list(VARIANTS))
def test_4096_envs_auto_reset_stay_finite(bundled_only, name):
    """4096 envs, 200 auto-resetting steps under U(-1, 1) actions: no non-finite state, and episodes end and restart."""
    n = 4096
    env = make_variant(name, num_envs=n, seed=9)
    eng = env._get_engine()
    env.reset()
    g = torch.Generator(device="cuda").manual_seed(0)
    n_done = 0
    for _ in range(200):
        obs, rew, done, info = env.step(torch.rand((n, eng.action_dim), device="cuda", generator=g) * 2 - 1)
        n_done += int(done.sum())
    q, v, _ = eng.get_state()
    cnt = eng.counters()
    assert bool(torch.isfinite(q).all() and torch.isfinite(v).all() and torch.isfinite(obs).all() and torch.isfinite(rew).all())
    assert int(cnt[:, 4].sum()) == 0, "non-finite states counted by the engine"
    assert n_done > 0 and int(cnt[:, 1].sum()) > 0, "no env reset"


@pytest.mark.parametrize("knobs", [{"LOCOSIM_RESORT": 2, "LOCOSIM_PERSIST": 0}, {"LOCOSIM_RESORT": 2, "LOCOSIM_PERSIST": 1}],
                         ids=["substep-launches", "persistent"])
def test_talos_arms_scheduling_paths_are_bitwise_identical(bundled_only, variants, monkeypatch, knobs):
    """Talos with arms over 50 auto-resetting steps: the sub-step launches and the persistent kernel (forced; the default
    is the fused kernel) equal the fused kernel bit for bit (test_persistent_kernel._rollout's outputs)."""
    ref, n_done, kps, _ = persistent._rollout({"LOCOSIM_RESORT": 100, "LOCOSIM_PERSIST": 0}, "Talos.walk+arms", 2000, 50, {}, monkeypatch)
    assert n_done > 0 and kps == 2
    got, _, kps, cnt = persistent._rollout(knobs, "Talos.walk+arms", 2000, 50, {}, monkeypatch)
    assert kps == (1 if knobs["LOCOSIM_PERSIST"] else 5)
    assert bool((cnt[:, 0] == 50).all())
    for i, (a, b) in enumerate(zip(ref, got)):
        assert torch.equal(a, b), "%s differs from the fused kernel in output %d" % (knobs, i)


def test_full_body_mixed_batch_equals_separate_engines(bundled_only):
    """Atlas with arms and Talos with arms, both with their DR pools, as one MixedBatch (the full-body analogue of the
    benchmark's config 4) behave bit for bit like the same envs stepped on separate engines."""
    from loco_mujoco_b200.parallel import MixedBatch
    n, steps = 256, 50
    kw = [dict(disable_arms=False, domain_randomization_config="domain_randomization_%s.yaml" % r) for r in ("atlas", "talos")]
    mb = MixedBatch([("Atlas.walk.real", n, kw[0]), ("Talos.walk.real", n, kw[1])], device="cuda:0", seed=3, debug=True)
    solo = [make_variant("Atlas.walk", num_envs=n, seed=3, env_id_offset=0, **kw[0]),
            make_variant("Talos.walk", num_envs=n, seed=3, env_id_offset=n, **kw[1])]
    o_mb, o_solo = mb.reset(), [e.reset() for e in solo]
    for a, b in zip(o_mb, o_solo):
        assert torch.equal(a, b)
    g = torch.Generator(device="cpu").manual_seed(0)
    n_done = 0
    for _ in range(steps):
        acts = [(torch.rand((n, e.action_dim), generator=g) * 2 - 1).cuda() for e in mb.engines]
        out = mb.step(acts)
        torch.cuda.synchronize()
        for i, env in enumerate(solo):
            o, r, d, info = env.step(acts[i])
            assert torch.equal(out[i][0], o) and torch.equal(out[i][1], r) and torch.equal(out[i][2], d)
            n_done += int(d.sum())
    assert n_done > 0
