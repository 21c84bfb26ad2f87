"""Full-body robot humanoids on the 31-dof configurations, CPU tier: configuration routing, bundled variant assets, the
oracle's reset rows, the serial build against the oracle (whole episodes and the stage checks of stage_probe.py), and
the cross-compiled kernels of the two new configurations.

No reference golden covers these variants (see full_body.py): the oracle episode under the reference test's protocol
stands in for the golden."""
import ctypes
import glob
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import stage_probe as sp
from full_body import (CFG, CONFIGS31, FIXTURES, FP32_ROWS, SIZES, VARIANTS, build_probe_emu, make_variant, obs_from_state,
                       oracle_episode, use_variants_in_stage_probe)
from helpers import ROOT, blobs, reference_draws

ASSETS = os.path.join(ROOT, "loco_mujoco_b200", "assets")
# the configuration every model bundled before the full-body variants runs in (unchanged by them: select_cfg is first-fit
# and the 31-dof configurations come last)
EXISTING_CFG = {"Atlas.carry": 2, "Atlas.walk": 2, "HumanoidTorque.run": 2, "HumanoidTorque.walk": 2,
                **{"HumanoidTorque4Ages.%s.%d" % (t, k): 2 for t in ("run", "walk") for k in (1, 2, 3, 4)},
                "Talos.carry": 1, "Talos.walk": 1, "UnitreeA1.hard": 0, "UnitreeA1.simple": 0, "UnitreeG1.run": 3,
                "UnitreeG1.walk": 3, "UnitreeH1.carry": 1, "UnitreeH1.run": 1, "UnitreeH1.walk": 1}
SMEM_PER_SM = 232448        # dynamic shared memory of one block on sm_90 (227 KB)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _asset_models(path):
    from loco_mujoco_b200 import modelpack
    a = np.load(path, allow_pickle=False)
    n = int(a["n_models"]) if "n_models" in a.files else 1
    prefixes = ["model%d_" % i for i in range(n)] if n > 1 else ["model_"]
    return [modelpack.from_npz_dict({k[len(pf):]: a[k] for k in a.files if k.startswith(pf)}) for pf in prefixes]


def _select(emu, m):
    from loco_mujoco_b200 import modelpack
    emu.emu_select_cfg.restype = ctypes.c_int
    emu.emu_select_cfg.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    mi, mr = [np.ascontiguousarray(x) for x in modelpack.pack(m)]
    return emu.emu_select_cfg(_p(mi), len(mi), _p(mr), len(mr))


def test_select_cfg_routes_variants_and_keeps_existing_models(emu):
    """Atlas with arms (and back) -> CfgPyrRK4_31, Talos with arms -> CfgPyrEuler31, H1 with arms stays on CfgPyrEuler29;
    every other bundled model keeps its configuration."""
    seen = set()
    for path in sorted(glob.glob(os.path.join(ASSETS, "*.npz")) + glob.glob(os.path.join(FIXTURES, "*.npz"))):
        name = os.path.basename(path)[:-4]
        want = CFG[name] if name in VARIANTS else EXISTING_CFG[name]
        for m in _asset_models(path):
            assert _select(emu, m) == want, name
        if name in VARIANTS:
            assert (m.nv, m.nbody, m.ngeom, m.nu) == SIZES[name], name
        seen.add(name)
    assert seen == set(VARIANTS) | set(EXISTING_CFG)


def test_new_configurations_hold_8_envs_per_sm(emu):
    """sizeof(EnvS) of the serial build less its emulation-only scratch (Y[6][NV]) is the CUDA layout: 8 envs per SM
    (the static_asserts of locosim.cu), not 9."""
    emu.emu_sizeof_env.restype = ctypes.c_int
    emu.emu_sizeof_env.argtypes = [ctypes.c_int]
    for k in (4, 5):
        cuda_bytes = emu.emu_sizeof_env(k) - 6 * 31 * 4
        assert 8 * cuda_bytes <= SMEM_PER_SM < 9 * cuda_bytes, (k, cuda_bytes)


def test_default_kwargs_keep_todays_asset_names(monkeypatch):
    from loco_mujoco_b200.environments.robot_humanoids import Atlas, Talos, UnitreeG1, UnitreeH1
    assert Atlas.variant_suffix() == Talos.variant_suffix() == UnitreeH1.variant_suffix() == UnitreeG1.variant_suffix() == ""
    assert Atlas.variant_suffix(disable_arms=False) == "+arms"
    assert Atlas.variant_suffix(disable_arms=False, disable_back_joint=False) == "+arms+back"
    assert Talos.variant_suffix(disable_back_joint=True) == "-back"
    monkeypatch.setenv("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")
    assert make_variant("Atlas.walk")._task_id == "Atlas.walk"
    for name in VARIANTS:
        assert make_variant(name)._task_id == name


def test_variant_without_bundled_asset_raises(monkeypatch):
    """Without a loco_mujoco checkout a variant that has no bundled asset is an error, never the default model."""
    from loco_mujoco_b200 import LocoEnv
    monkeypatch.setenv("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")
    with pytest.raises(FileNotFoundError, match=r"no bundled asset for Atlas\.walk\+back"):
        LocoEnv.make("Atlas.walk.real", debug=True, disable_back_joint=False)
    with pytest.raises(FileNotFoundError, match=r"no bundled asset for Talos\.walk-back"):
        LocoEnv.make("Talos.walk.real", debug=True, disable_back_joint=True)
    with pytest.raises(AssertionError, match="disable the arms"):
        LocoEnv.make("Talos.carry.real", debug=True, disable_arms=False)
    monkeypatch.delenv("LOCO_MUJOCO_B200_ASSET_PATH")          # the package itself bundles the default models only
    with pytest.raises(FileNotFoundError, match=r"no bundled asset for Talos\.walk\+arms"):
        LocoEnv.make("Talos.walk.real", debug=True, disable_arms=False)


def test_variant_assets_equal_a_fresh_compile(monkeypatch):
    """With a loco_mujoco checkout, every bundled variant asset holds the same ModelPack and TaskSpec blobs as a fresh
    compile of the same variant (tools/build_assets.py is reproducible)."""
    from loco_mujoco_b200.environments.base import reference_data_root
    monkeypatch.delenv("LOCO_MUJOCO_B200_FORCE_BUNDLED", raising=False)
    if reference_data_root() is None:
        pytest.skip("no loco_mujoco checkout (LOCO_MUJOCO_PATH)")
    for name in VARIANTS:
        fresh = blobs(make_variant(name))
        monkeypatch.setenv("LOCO_MUJOCO_B200_FORCE_BUNDLED", "1")
        bundled = blobs(make_variant(name))
        monkeypatch.delenv("LOCO_MUJOCO_B200_FORCE_BUNDLED")
        for (fi, fr), (bi, br) in zip(fresh, bundled):
            assert np.array_equal(fi, bi) and np.array_equal(fr, br), name


@pytest.mark.parametrize("name", list(VARIANTS))
def test_oracle_reset_row_is_the_trajectory_sample(oracle, bundled_only, name):
    """The oracle's reset row (built from the TaskSpec table) equals the host Trajectory's sample mapped through the
    observation specification, arm joints included."""
    env = make_variant(name)
    traj_no, step_no = reference_draws(env)
    oe = oracle.env(*blobs(env))
    row = oe.reset_to(traj_no, step_no)
    oe.close()
    sample = env.trajectories.reset_trajectory(substep_no=step_no, traj_no=traj_no)
    spec = env.obs_helper.observation_spec
    want = np.array([float(np.asarray(sample[env.trajectories.get_idx(key)]).reshape(-1)[0]) for key, _, _ in spec])[2:]
    assert len(want) == len(row) and any(key.startswith("q_l_arm") or key.startswith("q_left") for key, _, _ in spec)
    assert np.abs(row - want).max() <= 1e-12


@pytest.mark.parametrize("name", list(VARIANTS))
def test_serial_build_follows_the_oracle_episode(emu, oracle, bundled_only, name):
    """The reference test's episode, oracle as the golden: the serial fp32 build from the same reset state, with the
    same actions, falls at the same step and stays within 2e-3 + 2e-3 |obs| (UnitreeH1: over full_body.FP32_ROWS)."""
    from loco_mujoco_b200 import modelpack
    env = make_variant(name)
    rows, acts, q0, v0 = oracle_episode(oracle, env)
    m, spec = env._model, env.task_spec()
    ints, reals = modelpack.pack(m)
    sim = emu.emu_create(_p(ints), len(ints), _p(reals), len(reals))
    assert sim
    q, v = np.ascontiguousarray(q0, dtype=np.float64), np.ascontiguousarray(v0, dtype=np.float64)
    emu.emu_reset(sim, _p(q), _p(v))
    got = [obs_from_state(spec, q, v)]
    for a in acts:
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = a * spec.act_delta + spec.act_mean
        emu.emu_step(sim, _p(ctrl), spec.n_substeps)
        emu.emu_get_state(sim, _p(q), _p(v))
        got.append(obs_from_state(spec, q, v))
        if env._has_fallen(got[-1]):
            break
    emu.emu_destroy(sim)
    got = np.array(got)
    if name in FP32_ROWS:
        got, rows = got[:FP32_ROWS[name]], rows[:FP32_ROWS[name]]
    err = np.abs(got[:len(rows)] - rows[:len(got)])
    print(name, "episode length", len(rows), "max |obs - oracle| %.3e" % err.max())
    assert got.shape == rows.shape, "episode length %d vs the oracle's %d" % (len(got), len(rows))
    assert np.all(err <= 2e-3 + 2e-3 * np.abs(rows)), "max abs err %.3e" % err.max()


@pytest.mark.parametrize("name", list(VARIANTS))
def test_serial_stages_against_fp64(monkeypatch, oracle, bundled_only, name):
    """C, B, E and D-against-the-oracle (stage_probe.py, bounds in DESIGN section 6) on >= 256 states of each variant,
    in the configuration the CUDA engine picks."""
    use_variants_in_stage_probe(monkeypatch)
    probe = build_probe_emu()
    env, S = sp.states(name, oracle)
    assert len(S["qpos"]) >= 256
    rec, cfg = sp.emu_record(probe, blobs(env)[0], S)
    assert cfg == CFG[name] and int(rec["cfg_nv"][0]) == (31 if cfg in (4, 5) else 29)
    print(name, "C", sp.check_smooth_vs_oracle(rec, env, oracle, S))
    stats = sp.check_hessians(rec, 0)
    print(name, "B", stats)
    assert stats["helper_region"] > 0
    compared, knife, ncmp = sp.check_contacts_vs_oracle(rec, env, oracle, S)
    print(name, "D-vs-oracle: %d envs compared, %d knife-edge, %d primitive contacts" % (compared, knife, ncmp))
    assert ncmp > 0 and knife <= 0.1 * len(S["qpos"])
    worst, n_con, n_cap = sp.check_optimality(rec, env, oracle, S, 0)
    print(name, "E: worst gap / bound %.3g over %d envs with constraints, %d at the iteration cap" % (worst, n_con, n_cap))
    assert n_con > 0 and n_cap <= 0.05 * n_con


def _ptxas(stderr):
    """{mangled function: (registers or None, stack frame, spill stores, spill loads)} from nvcc -Xptxas -v."""
    out, cur = {}, None
    for line in stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = [None] + [int(x) for x in m.groups()]
            continue
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur in out:
            out[cur][0] = int(m.group(1))
    return out


def _kernel(rep, kernel, cfg):
    """ptxas entry of kernel<cfg>, in the engine's first unit (global scope) or in locosim_configs31.cu (namespace locosim31)"""
    pre = ("_Z%d%sI%d%sE" % (len(kernel), kernel, len(cfg), cfg), "_ZN9locosim31%d%sINS_%d%sE" % (len(kernel), kernel, len(cfg), cfg))
    hits = [v for k, v in rep.items() if k.startswith(pre)]
    assert len(hits) == 1, (kernel, cfg, len(hits))
    return hits[0]


@pytest.mark.skipif(shutil.which(os.environ.get("NVCC", "nvcc")) is None and not os.path.exists("/usr/local/cuda/bin/nvcc"),
                    reason="nvcc not installed")
def test_new_kernels_cross_compile_without_new_spills(tmp_path):
    """The engine's second translation unit (locosim_configs31.cu) and the full-body CUDA stage probe (the first unit +
    the probe kernels) for sm_90a with the product's flags. The second unit holds the step, sub-step and persistent
    kernels of the two 31-dof configurations and of no other. They use <= 128 registers; each sub-step kernel fits its
    fused kernel's registers and stack; their stack and spills are those of the existing kernel of the same family (the
    saves around the __noinline__ stages). The NV-31 Cholesky and the wide Hessian spill nothing."""
    import __graft_entry__
    nvcc = shutil.which(os.environ.get("NVCC", "nvcc")) or "/usr/local/cuda/bin/nvcc"
    flags = [f for f in __graft_entry__.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    procs = [subprocess.Popen([nvcc] + flags + ["-cubin", "-o", str(tmp_path / ("%d.cubin" % k)), src], stderr=subprocess.PIPE,
                              stdout=subprocess.DEVNULL, text=True)
             for k, src in enumerate((CONFIGS31, os.path.join(sp.CUDA_DIR, "stage_probe_full_body.cu")))]
    outs = [p.communicate()[1] for p in procs]
    assert all(p.returncode == 0 for p in procs), [o[-4000:] for o in outs]
    new, rep = _ptxas(outs[0]), _ptxas(outs[0] + outs[1])
    assert sorted(k for k in new if "step_kernelI" in k and "substep" not in k) == sorted(
        "_ZN9locosim3111step_kernelINS_%sEEEviNS_7DevTaskENS_10SolverOptsENS_11EngineStateEPKfPfS7_PhS7_iimliiPKhi" % c
        for c in ("12CfgPyrRK4_31", "13CfgPyrEuler31"))
    for cfg, old in (("CfgPyrRK4_31", "CfgPyrRK4"), ("CfgPyrEuler31", "CfgPyrEuler29")):
        for kernel in ("step_kernel", "substep_kernel", "persist_kernel"):
            a, b = _kernel(rep, kernel, cfg), _kernel(rep, kernel, old)
            assert a[0] is not None and a[0] <= 128, (kernel, cfg, a)
            assert a[1] <= b[1] and a[2] <= b[2] and a[3] <= b[3], (kernel, cfg, a, old, b)
        fused, split = _kernel(rep, "step_kernel", cfg), _kernel(rep, "substep_kernel", cfg)
        assert split[0] <= fused[0] and split[1] <= fused[1], (cfg, fused, split)
    nv31 = {k: v for k, v in rep.items()
            if re.search(r"(chol_factor|chol_solve)ILi31ELi32E|make_hessian_wide\w*CfgPyr(RK4_31|Euler31)|probe_chol_kernelILi31E", k)}
    assert len(nv31) >= 5, sorted(nv31)
    for k, v in nv31.items():
        assert v[2] == 0 and v[3] == 0, (k, v)
