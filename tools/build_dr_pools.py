"""
Pre-built, seeded domain-randomisation parameter pools for the reference's SHIPPED YAML configs
(/root/reference/loco_mujoco/environments/data/{atlas,talos}/domain_randomization_*.yaml), stored under
loco_mujoco_b200/assets/dr_pools/ so that a box without the MJCF sources (the GPU box) can run BASELINE config 4
(Atlas.walk + Talos.walk with domain randomisation).  Run here:  python tools/build_dr_pools.py

Each pool = K consecutive randomised recompilations (np.random.seed(SEED); the draws compound from row to row exactly
like consecutive reference resets, utils/domain_randomization.py:530).

Talos: the shipped YAML asks for `Inertial.leg_right_5_link.fullinertia`, but that body's <inertial> carries
`diaginertia` (talos.xml:379); the reference asserts at the first reset ("Randomizing fullinertia not allowed if not
specified in the xml", domain_randomization.py:502) and so does this package.  What a reference user does to get past
it -- drop that one entry -- is what is done here (recorded in the pool's metadata); everything else is the shipped file.
"""
import copy
import json
import os
import sys

import numpy as np
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from loco_mujoco_b200 import LocoEnv                                  # noqa: E402
from loco_mujoco_b200.environments.base import ASSET_DIR              # noqa: E402

REF = os.environ.get("LOCO_MUJOCO_PATH", "/root/reference/loco_mujoco")
K, SEED = 64, 0
TALOS_DROP = [("Inertial", "leg_right_5_link", "fullinertia")]
# (pool name = task + model variant, shipped YAML, dropped entries, model-variant kwargs)
JOBS = [("Atlas.walk", "atlas/domain_randomization_atlas.yaml", [], {}),
        ("Talos.walk", "talos/domain_randomization_talos.yaml", TALOS_DROP, {}),
        ("Atlas.walk+arms", "atlas/domain_randomization_atlas.yaml", [], dict(disable_arms=False)),
        ("Talos.walk+arms", "talos/domain_randomization_talos.yaml", TALOS_DROP, dict(disable_arms=False))]

VARIANT_DIR = os.path.join(ROOT, "tests", "golden", "full_body")       # pools of model variants: data fixtures
for task, rel, drop, variant in JOBS:
    conf = yaml.safe_load(open(os.path.join(REF, "environments", "data", rel)))
    shipped = copy.deepcopy(conf)
    for sec, name, key in drop:
        del conf[sec][name][key]
        if not conf[sec][name]:
            del conf[sec][name]
    np.random.seed(SEED)
    env = LocoEnv.make(task.split("+")[0] + ".real", debug=True, domain_randomization_config=conf,
                       domain_randomization_pool_size=K, **variant)
    assert env._task_id == task, (env._task_id, task)
    pool = env.domain_randomization_pool()
    meta = dict(task=task, yaml=os.path.basename(rel), seed=SEED, rows=K, dropped=[list(d) for d in drop],
                config_used=conf, config_shipped=shipped)
    out = os.path.join(VARIANT_DIR if variant else ASSET_DIR, "dr_pools", task + ".npz")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    np.savez_compressed(out, pool=pool, meta=np.array(json.dumps(meta)))
    spread = np.abs(pool - pool[0]).max(axis=0)
    print(task, pool.shape, "columns that vary:", int((spread > 0).sum()), "->", out, os.path.getsize(out), "bytes")
