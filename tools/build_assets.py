"""
Generate the bundled task assets (compiled ModelPack + interpolated reset trajectories) from a loco_mujoco
checkout (default: /root/reference/loco_mujoco). The GPU box has no reference tree, so tests / bench there use
these files. Re-run after changing mjcf.py or the task definitions:   python tools/build_assets.py
A task may name a model variant of a robot humanoid: "Atlas.walk+arms" is Atlas(disable_arms=False),
"Atlas.walk+arms+back" also enables the back joint (see BaseRobotHumanoid.variant_suffix).
"UnitreeA1.simple+position" is UnitreeA1(action_mode="position"), the PD position-control model.
Variants are written to tests/golden/full_body/ and tests/golden/position/ (data fixtures, found through
LOCO_MUJOCO_B200_ASSET_PATH), the default models to the package's assets. The variants are built with:
    python tools/build_assets.py Atlas.walk+arms Atlas.walk+arms+back Talos.walk+arms UnitreeH1.walk+arms
    python tools/build_assets.py UnitreeA1.simple+position UnitreeA1.hard+position
"""
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from loco_mujoco_b200 import LocoEnv, modelpack                                   # noqa: E402
from loco_mujoco_b200.environments.base import processed_trajectory_dict, ASSET_DIR  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
TASKS = sys.argv[1:] or ["UnitreeA1.simple", "UnitreeA1.hard"]
VARIANT_KWARGS = {"+arms": ("disable_arms", False), "-arms": ("disable_arms", True),
                  "+back": ("disable_back_joint", False), "-back": ("disable_back_joint", True),
                  "+position": ("action_mode", "position")}


def variant_kwargs(task):
    """"Atlas.walk+arms+back" -> ("Atlas.walk", dict(disable_arms=False, disable_back_joint=False))"""
    base, parts = re.fullmatch(r"([\w.]+?)((?:[+-](?:arms|back)|\+position)*)", task).groups()
    return base, dict(VARIANT_KWARGS[p] for p in re.findall(r"[+-](?:arms|back)|\+position", parts))


for task in TASKS:
    base, kw = variant_kwargs(task)
    env = LocoEnv.make(base + ".real", debug=True, **kw)
    variant_dir = os.path.join(GOLDEN, "position" if "action_mode" in kw else "full_body")
    if kw and "action_mode" not in kw:
        assert env._task_id == task, (env._task_id, task)
    if len(env._models) > 1:        # multi-model env (carry): every model, prefix model<i>_
        d = {"n_models": np.int32(len(env._models))}
        for i, m in enumerate(env._models):
            d.update({"model%d_%s" % (i, k): v for k, v in modelpack.to_npz_dict(m).items()})
    else:
        d = {"model_" + k: v for k, v in modelpack.to_npz_dict(env._model).items()}
    d.update({"traj_" + k: v for k, v in processed_trajectory_dict(env.trajectories).items()})
    os.makedirs(variant_dir if kw else ASSET_DIR, exist_ok=True)
    path = os.path.join(variant_dir if kw else ASSET_DIR, task + ".npz")
    np.savez_compressed(path, **d)
    print(task, "->", path, os.path.getsize(path), "bytes")
