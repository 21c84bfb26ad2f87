"""Sub-step launches (LOCOSIM_RESORT): the control step runs as several launches of the step kernel, each over a range of
sub-steps, with the envs regrouped by solver effort between launches (loco_mujoco_b200/csrc/locosim.cu, substep_kernel).
Regrouping is pure scheduling, so every split of the step must give the bits of the fused kernel.

CPU tier: (i) the serial build of the core loses its working set between sub-steps except the fields the CUDA engine carries
in HBM (emu_poison) and must still reproduce the uninterrupted trajectory bit for bit - nothing else may be read before it is
written in a sub-step; (ii) the sub-step kernel compiles for sm_90a with the same registers and stack as the fused kernel.
GPU tier: bitwise identity of everything the engine returns for LOCOSIM_RESORT in {10, 1, 2, 3} (3: uneven launches)."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from helpers import ROOT, make_env


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("task,kw", [("UnitreeA1.simple", {}), ("UnitreeA1.simple", {"use_foot_forces": True}),
                                     ("HumanoidTorque.run", {}), ("Talos.walk", {})])
def test_carried_fields_are_the_whole_sub_step_state(emu, bundled_only, task, kw):
    from loco_mujoco_b200 import modelpack
    emu.emu_poison.argtypes = [ctypes.c_void_p]
    emu.emu_poison.restype = None
    emu.emu_set_grf.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    emu.emu_get_grf.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    emu.emu_iter.argtypes = [ctypes.c_void_p]
    env = make_env(task, **kw)
    m, spec = env._model, env.task_spec()
    ints, reals = modelpack.pack(m)
    sims = [emu.emu_create(_p(ints), len(ints), _p(reals), len(reals)) for _ in range(2)]
    grp = np.ascontiguousarray(spec.grf_group, dtype=np.int32)
    for s in sims:
        assert s
        if spec.n_grf:
            emu.emu_set_grf(s, _p(grp), len(grp), spec.n_grf)
    table = spec.table.reshape(-1, spec.table.shape[-1])
    nv = m.nq
    rng = np.random.default_rng(0)
    q, v = [np.zeros(nv) for _ in sims], [np.zeros(nv) for _ in sims]
    grf = [np.zeros(12) for _ in sims]
    iters = 0
    for step in range(60):
        if step % 20 == 0:                      # a fresh episode from a table row
            row = table[rng.integers(len(table))]
            for s in sims:
                emu.emu_reset(s, _p(np.ascontiguousarray(row[:nv])), _p(np.ascontiguousarray(row[nv:2 * nv])))
        ctrl = np.zeros(m.nu)
        ctrl[spec.act_idx] = rng.uniform(-1, 1, m.nu) * spec.act_delta + spec.act_mean
        emu.emu_step(sims[0], _p(ctrl), spec.n_substeps)
        for _ in range(spec.n_substeps):
            emu.emu_step(sims[1], _p(ctrl), 1)
            emu.emu_poison(sims[1])
        for i, s in enumerate(sims):
            emu.emu_get_state(s, _p(q[i]), _p(v[i]))
            emu.emu_get_grf(s, _p(grf[i]), 0)
        assert np.array_equal(q[0], q[1]) and np.array_equal(v[0], v[1]), "step %d" % step
        assert np.array_equal(grf[0], grf[1]), "step %d" % step
        iters += emu.emu_iter(sims[0])
    assert iters > 0
    for s in sims:
        emu.emu_destroy(s)


def _ptxas_report(text, kernel):
    """(registers, stack frame, spill stores) of every instantiation of `kernel`, by configuration"""
    out = {}
    for m in re.finditer(r"Compiling entry function '_Z\d+%sI(\w+?)Evi\S*' for 'sm_90a'\n((?:.*\n){3})" % kernel, text):
        frame = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores", m.group(2))
        regs = re.search(r"Used (\d+) registers", m.group(2))
        out[m.group(1)] = (int(regs.group(1)), int(frame.group(1)), int(frame.group(2)))
    return out


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="no nvcc")
def test_substep_kernel_cross_compiles_for_sm90a(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(ROOT, "loco_mujoco_b200", "csrc", "locosim.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-prec-div=false",
                        "-prec-sqrt=false", "-ftz=true", "-Xptxas", "-v", "-cubin", "-o", str(tmp_path / "locosim.cubin"), src],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    fused, split = _ptxas_report(r.stderr, "step_kernel"), _ptxas_report(r.stderr, "substep_kernel")
    assert set(fused) == set(split) == {"11CfgEllEuler", "11CfgPyrEuler", "13CfgPyrEuler29", "9CfgPyrRK4"}, (fused, split)
    for cfg in fused:
        # one resident block of up to 16 warps per SM: the sub-step kernel must fit the fused kernel's register budget, and
        # its stack (spills of the __noinline__ phases) must not grow
        assert split[cfg][0] <= 128 and split[cfg][0] <= fused[cfg][0], (cfg, fused[cfg], split[cfg])
        assert split[cfg][1] <= fused[cfg][1], (cfg, fused[cfg], split[cfg])


# ---------------------------------------------------------------------------------------------------------------------
# GPU tier
# ---------------------------------------------------------------------------------------------------------------------
def _rollout(resort, task, n, steps, kw, monkeypatch):
    import torch
    monkeypatch.setenv("LOCOSIM_RESORT", str(resort))
    env = make_env(task, num_envs=n, seed=5, **kw)
    eng = env._get_engine()
    nsub = env.task_spec().n_substeps
    launches = -(-nsub // min(resort, nsub)) if resort < nsub else 2
    assert eng.kernels_per_step == launches
    geo = eng.launch_info()
    nu = env.info.action_space.shape[0]
    out = [env.reset().clone()]
    g = torch.Generator(device="cpu").manual_seed(7)
    n_done = 0
    for _ in range(steps):
        act = (torch.rand((n, nu), generator=g) * 2 - 1).cuda()
        obs, rew, done, info = env.step(act)
        out += [obs.clone(), rew.clone(), done.clone(), info["next_obs"].clone()]
        n_done += int(done.sum())
    q, v, w = eng.get_state()
    out += [q.clone(), v.clone(), w.clone(), eng.counters()[:, 0:5].clone()]
    torch.cuda.synchronize()
    monkeypatch.delenv("LOCOSIM_RESORT")
    return out, n_done, geo


CASES = [("UnitreeA1.simple", 2000, {"warps_per_block": 15}),       # full blocks, more blocks than SMs, ghost warps
         ("HumanoidTorque.run", 512, {}),                             # RK4 + MPR (separating-direction cache across launches)
         ("Talos.walk", 512, {"domain_randomization_config": "domain_randomization_talos.yaml"}),   # DR pool rows per reset
         ("UnitreeA1.simple", 512, {"use_foot_forces": True}),       # foot forces summed over the sub-steps
         ("UnitreeA1.simple", 512, {"reward_type": "tracking"})]     # tracking reward + cursor


@pytest.mark.gpu
@pytest.mark.parametrize("task,n,kw", CASES, ids=["A1-2000", "HumanoidTorque", "Talos-DR", "A1-foot-forces", "A1-tracking"])
def test_substep_launches_are_bitwise_identical(bundled_only, monkeypatch, task, n, kw):
    import torch
    ref, n_done, geo = _rollout(10, task, n, 50, kw, monkeypatch)
    assert n_done > 0, "the rollout should reach the auto-reset path"
    if n == 2000:
        # the geometry the sub-step launches run by default: 134 blocks of 15 warps (133 x 15 + 5 envs), so the last block
        # has 10 ghost warps, and more blocks than the 132 SMs of an H100 SXM
        assert geo["warps_per_block"] == 15 and geo["blocks"] == 134, geo
    for resort in (1, 2, 3):
        got, _, _ = _rollout(resort, task, n, 50, kw, monkeypatch)
        for i, (a, b) in enumerate(zip(ref, got)):
            assert torch.equal(a, b), "LOCOSIM_RESORT=%d differs from the fused kernel in output %d" % (resort, i)
