"""The full-body model variants of the robot humanoids (arms, and for Atlas the back joint) that run on the 31-dof kernel
configurations, and what their tests share. Test infrastructure only.

A variant is named like its asset: task + BaseRobotHumanoid.variant_suffix, e.g. "Atlas.walk+arms+back". The compiled
variant assets and their DR pools are data fixtures under tests/golden/full_body (tools/build_assets.py,
tools/build_dr_pools.py); importing this module adds that directory to LOCO_MUJOCO_B200_ASSET_PATH. No reference golden
covers these variants: their tests compare the engine with the fp64 oracle, which is pinned on the goldens of every
element these models use (hinge trees, joint limits, plane contacts against boxes, cylinders and meshes, RK4 and Euler)."""
import ctypes
import os
import subprocess

import numpy as np

import stage_probe as sp
from helpers import GOLDEN, make_env, oracle_env, reference_draws

FIXTURES = os.path.join(GOLDEN, "full_body")
if FIXTURES not in os.environ.get("LOCO_MUJOCO_B200_ASSET_PATH", "").split(os.pathsep):
    os.environ["LOCO_MUJOCO_B200_ASSET_PATH"] = os.pathsep.join(
        [p for p in (os.environ.get("LOCO_MUJOCO_B200_ASSET_PATH"), FIXTURES) if p])
CONFIGS31 = os.path.join(sp.CSRC, "locosim_configs31.cu")

VARIANTS = {"Atlas.walk+arms": ("Atlas.walk", dict(disable_arms=False)),
            "Atlas.walk+arms+back": ("Atlas.walk", dict(disable_arms=False, disable_back_joint=False)),
            "Talos.walk+arms": ("Talos.walk", dict(disable_arms=False)),
            "UnitreeH1.walk+arms": ("UnitreeH1.walk", dict(disable_arms=False))}
# configuration index of locosim_host.h select_cfg: 4 CfgPyrRK4_31, 5 CfgPyrEuler31, 3 CfgPyrEuler29
CFG = {"Atlas.walk+arms": 4, "Atlas.walk+arms+back": 4, "Talos.walk+arms": 5, "UnitreeH1.walk+arms": 3}
# (nv, nbody, ngeom, nu) after static-body fusion
SIZES = {"Atlas.walk+arms": (28, 24, 99, 22), "Atlas.walk+arms+back": (31, 27, 99, 25), "Talos.walk+arms": (30, 26, 52, 24),
         "UnitreeH1.walk+arms": (25, 21, 21, 19)}

# Rows of the oracle episode the fp32 engine is compared on, where not the whole episode. UnitreeH1: as for UnitreeH1.walk
# (helpers.FP32_ROWS), the swing leg's hip cylinder meets the thigh mesh (an MPR self contact) and the feet are meshes on
# the floor; there an fp32 and an fp64 rollout take different, equally valid branches. With arms that happens at row 7
# (serial build: |obs - oracle| <= 6e-6 up to row 6, 5e-3 at row 7).
FP32_ROWS = {"UnitreeH1.walk+arms": 7}


def make_variant(name, **kw):
    """make_env for a variant name (plain task names pass through)."""
    base, variant_kw = VARIANTS.get(name, (name, {}))
    return make_env(base, **variant_kw, **kw)


def use_variants_in_stage_probe(monkeypatch):
    """Let stage_probe.states (and the checks built on it) take variant names."""
    monkeypatch.setattr(sp, "make_env", make_variant)


def obs_from_state(spec, q, v):
    """Observation of a (qpos, qvel) state through the TaskSpec's observation gather (joint positions / velocities)."""
    assert set(np.unique(spec.obs_src_type)) <= {0, 1}
    return np.array([q[i] if t == 0 else v[i] for t, i in zip(spec.obs_src_type, spec.obs_src_idx)])


def oracle_episode(oracle, env, max_len=1001):
    """The reference test's protocol on the fp64 oracle (tests/test_environments.py of loco-mujoco): np.random.seed(0),
    reset draws, then randn(nu) * 0.1 actions until has_fallen. Returns (observations, actions, reset qpos, reset qvel)."""
    traj_no, step_no = reference_draws(env)
    oe = oracle_env(oracle, env)
    rows = [oe.reset_to(traj_no, step_no)]
    q0, v0 = oe.get_state()
    acts, done = [], False
    while not done and len(rows) < max_len:
        a = np.random.randn(env.info.action_space.shape[0]) * 0.1
        obs, _, done = oe.step(a)
        rows.append(obs)
        acts.append(a)
    oe.close()
    return np.array(rows), np.array(acts), np.array(q0), np.array(v0)


def build_probe_emu():
    """The serial stage probe with the 31-dof configurations (tests/cuda/stage_probe_emu_full_body.cpp)."""
    so = os.path.join(sp.BUILD, "libstage_probe_emu_full_body.so")
    src = os.path.join(sp.CUDA_DIR, "stage_probe_emu_full_body.cpp")
    deps = sp.CORE_SRCS + [src] + [os.path.join(sp.CUDA_DIR, f) for f in ("stage_probe_emu.cpp", "stage_probe.h")]
    if sp._stale(so, deps):
        os.makedirs(sp.BUILD, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-o", so, src, "-lm"])
    return sp._bind(ctypes.CDLL(so))


def build_probe_cuda(so=None):
    """The CUDA stage probe with the 31-dof configurations: tests/cuda/stage_probe_full_body.cu and the engine's second
    translation unit, with the product's nvcc flags."""
    import __graft_entry__
    so = so or os.path.join(sp.BUILD, "libstage_probe_cuda_full_body.so")
    srcs = [os.path.join(sp.CUDA_DIR, "stage_probe_full_body.cu"), CONFIGS31]
    deps = sp.CORE_SRCS + srcs + [os.path.join(sp.CUDA_DIR, f) for f in ("stage_probe.cu", "stage_probe.h")]
    if sp._stale(so, deps):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        r = subprocess.run([os.environ.get("NVCC", "nvcc")] + __graft_entry__.NVCC_FLAGS + ["-o", so] + srcs,
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
    return so
