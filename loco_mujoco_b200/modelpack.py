"""
ModelPack serialisation: Model (mjcf.py) <-> the two flat blobs described in include/locosim_modelpack.h.
Also (de)serialises to .npz so compiled models can ship with the package (the GPU box has no
/root/reference, see tools/build_assets.py).
"""
import numpy as np

MAGIC = 0x4C4F434F
VERSION = 3

INT_FIELDS = ["body_parentid", "body_jntadr", "body_jntnum", "body_lastdof", "body_rootid",
              "jnt_type", "jnt_bodyid", "jnt_limited", "dof_parentid",
              "geom_type", "geom_bodyid", "geom_condim", "geom_priority", "geom_meshadr", "geom_meshnum",
              "pair_geom",
              "actuator_dof", "actuator_ctrllimited", "actuator_forcelimited"]
REAL_FIELDS = ["body_pos", "body_quat", "body_ipos", "body_iquat", "body_mass", "body_inertia", "body_invweight0",
               "jnt_pos", "jnt_axis", "jnt_range", "jnt_stiffness", "jnt_margin", "jnt_solref", "jnt_solimp",
               "qpos0", "qpos_spring",
               "dof_armature", "dof_damping", "dof_frictionloss", "dof_solref", "dof_solimp", "dof_invweight0",
               "geom_size", "geom_pos", "geom_quat", "geom_friction", "geom_margin", "geom_gap", "geom_solref",
               "geom_solimp", "geom_solmix", "geom_rbound", "geom_invweight0",
               "mesh_vert",
               "actuator_gear", "actuator_ctrlrange", "actuator_forcerange", "actuator_gain", "actuator_bias"]
SCALARS = ["nbody", "njnt", "nq", "nv", "ngeom", "nu", "npair", "opt_timestep", "opt_integrator", "opt_cone",
           "opt_impratio", "opt_iterations", "opt_tolerance", "stat_meaninertia"]
NAME_LISTS = ["body_names", "jnt_names", "geom_names", "actuator_names", "site_names"]
EXTRA_ARRAYS = ["opt_gravity", "body_weldid", "body_dofadr", "body_dofnum", "dof_bodyid", "geom_contype",
                "geom_conaffinity", "site_bodyid", "site_pos", "site_quat"]


GEOM_PLANE, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE, GEOM_BOX, GEOM_MESH = 0, 1, 2, 3, 6, 7
PRIMITIVE_PAIRS = {(GEOM_SPHERE, GEOM_SPHERE), (GEOM_SPHERE, GEOM_CAPSULE), (GEOM_CAPSULE, GEOM_CAPSULE), (GEOM_SPHERE, GEOM_BOX)}


def convex_pair_mask(m):
    """True for the candidate pairs that go through the general convex routine (mjc_Convex / MPR): everything that is
    neither a plane pair, nor a terrain pair, nor one of the dedicated primitive routines (same rule as
    csrc/locosim_host.h parse_model)."""
    pg = np.asarray(m.pair_geom).reshape(-1, 2)
    t = np.asarray(m.geom_type)
    return np.array([t[a] not in (GEOM_PLANE, GEOM_HFIELD) and (int(t[a]), int(t[b])) not in PRIMITIVE_PAIRS for a, b in pg],
                    dtype=bool).reshape(-1)


def terrain_pair_mask(m):
    """True for the pairs (terrain, g) of a height field (loco_mujoco_b200/terrain.py attach)."""
    pg = np.asarray(m.pair_geom).reshape(-1, 2)
    return (np.asarray(m.geom_type)[pg[:, 0]] == GEOM_HFIELD) if len(pg) else np.zeros(0, dtype=bool)


def pack(m, convex_pairs=True):
    """Model -> (ints int32[], reals float64[]). convex_pairs=False leaves the general convex (MPR) candidate pairs out of
    the pair table (LocoEnv kwarg `convex_collisions=False`: the round-1 feature set, without bone-bone contacts)."""
    pair_geom = np.asarray(m.pair_geom).reshape(-1, 2)
    # wire order of the candidate pairs: primitive pairs first, general convex pairs next, the terrain's pairs last, model
    # order within each part (the engine runs a lean bounding-sphere loop over the convex part and the terrain pass after
    # it; contact lists are ordered accordingly)
    cm, tm = convex_pair_mask(m), terrain_pair_mask(m)
    parts = [pair_geom[~cm & ~tm]] + ([pair_geom[cm]] if convex_pairs else []) + [pair_geom[tm]]
    pair_geom = np.concatenate(parts)
    hf = getattr(m, "hfield", None)
    ih = np.zeros(16, dtype=np.int32)
    ih[:11] = [MAGIC, VERSION, m.nbody, m.nv, m.ngeom, m.nu, len(pair_geom), len(m.mesh_vert), m.opt_integrator,
               m.opt_cone, m.opt_iterations]
    rh = np.zeros(16, dtype=np.float64)
    rh[:7] = [m.opt_timestep, m.opt_gravity[0], m.opt_gravity[1], m.opt_gravity[2], m.opt_impratio,
              m.opt_tolerance, m.stat_meaninertia]
    if hf is not None:      # (header slots MPI_HF_NROW / MPI_HF_NCOL, MPR_HF_SIZE; zeros without a terrain)
        ih[11:13] = hf.data.shape
        rh[7:11] = hf.size4
    ints = [ih] + [np.ascontiguousarray(pair_geom if f == "pair_geom" else getattr(m, f), dtype=np.int32).ravel()
                   for f in INT_FIELDS]
    reals = [rh] + [np.ascontiguousarray(getattr(m, f), dtype=np.float64).ravel() for f in REAL_FIELDS]
    if hf is not None:      # the trailing hfield_data[nrow * ncol]
        reals.append(np.ascontiguousarray(hf.data, dtype=np.float64).ravel())
    return np.concatenate(ints), np.concatenate(reals)


def to_npz_dict(m):
    d = {}
    for f in INT_FIELDS + REAL_FIELDS + EXTRA_ARRAYS:
        d[f] = np.asarray(getattr(m, f))
    for s in SCALARS:
        d["scalar_" + s] = np.asarray(getattr(m, s))
    for n in NAME_LISTS:
        d["names_" + n] = np.array(getattr(m, n), dtype=object).astype(str)
    fused = getattr(m, "fused_bodies", None)
    if fused:      # (optional: which body each static body was fused into, for Model.body_index's message)
        d["names_fused_from"] = np.array(list(fused), dtype=object).astype(str)
        d["names_fused_into"] = np.array(list(fused.values()), dtype=object).astype(str)
    return d


def from_npz_dict(d):
    from .mjcf import Model
    m = Model()
    for f in INT_FIELDS + REAL_FIELDS + EXTRA_ARRAYS:
        setattr(m, f, np.asarray(d[f]))
    for s in SCALARS:
        v = d["scalar_" + s]
        setattr(m, s, v.item())
    for n in NAME_LISTS:
        setattr(m, n, [str(x) for x in d["names_" + n]])
    if "names_fused_from" in d:
        m.fused_bodies = {str(a): str(b) for a, b in zip(d["names_fused_from"], d["names_fused_into"])}
    return m
