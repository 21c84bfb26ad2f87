/*
 * ModelPack wire format: the flat, compiled robot model handed across the C-ABI.
 *
 * Produced by loco_mujoco_b200/mjcf.py + modelpack.py from the reference's MJCF files
 * (/root/reference/loco_mujoco/environments/data/...), consumed by the CUDA engine
 * (loco_mujoco_b200/csrc/locosim.cu) and by the CPU oracle (oracle/locosim_ref.c).
 * It replaces what the reference gets from `mujoco.MjModel.from_xml_path` inside
 * mushroom_rl's MuJoCo.__init__ (called at /root/reference/loco_mujoco/environments/base.py:109-111).
 *
 * Two blobs: `ints` (int32) and `reals` (float64), each = fixed header followed by the arrays below,
 * tightly packed in the order listed. Sizes are functions of the header counts.
 * This is a data-format description only: no algorithm lives here.
 */
#ifndef LOCOSIM_MODELPACK_H
#define LOCOSIM_MODELPACK_H

#define LOCOSIM_MP_MAGIC   0x4C4F434F
#define LOCOSIM_MP_VERSION 3

/* int header slots */
enum {
  MPI_MAGIC = 0, MPI_VERSION, MPI_NBODY, MPI_NV, MPI_NGEOM, MPI_NU, MPI_NPAIR, MPI_NMESHVERT,
  MPI_INTEGRATOR /*0 Euler,1 RK4*/, MPI_CONE /*0 pyramidal,1 elliptic*/, MPI_ITERATIONS,
  MPI_HF_NROW /*height field rows, 0 = no terrain*/, MPI_HF_NCOL /*height field columns*/,
  MPI_HEADER_LEN = 16
};
/* real header slots */
enum {
  MPR_TIMESTEP = 0, MPR_GRAV_X, MPR_GRAV_Y, MPR_GRAV_Z, MPR_IMPRATIO, MPR_TOLERANCE, MPR_MEANINERTIA,
  MPR_HF_SIZE /*4 slots: the height field's size (rx, ry, elevation, base)*/,
  MPR_HEADER_LEN = 16
};

/* X(name, count-expression) ; nb=nbody nv=nv ng=ngeom nu=nu np=npair nm=nmeshvert
 * pair_geom: candidate geom pairs (g1, g2) with type(g1) <= type(g2); the pairs handled by a dedicated primitive routine
 * (plane-X, sphere-sphere, sphere-capsule, capsule-capsule, sphere-box) MUST come first, the general convex pairs
 * (mjc_Convex / MPR) next, and the pairs (terrain, g) of the height field last (none without a terrain); model order
 * inside each part (loco_mujoco_b200/modelpack.py pack()). */
#define LOCOSIM_MP_INT_FIELDS(X) \
  X(body_parentid, nb) X(body_jntadr, nb) X(body_jntnum, nb) X(body_lastdof, nb) X(body_rootid, nb) \
  X(jnt_type, nv) X(jnt_bodyid, nv) X(jnt_limited, nv) X(dof_parentid, nv) \
  X(geom_type, ng) X(geom_bodyid, ng) X(geom_condim, ng) X(geom_priority, ng) X(geom_meshadr, ng) X(geom_meshnum, ng) \
  X(pair_geom, 2 * np) \
  X(actuator_dof, nu) X(actuator_ctrllimited, nu) X(actuator_forcelimited, nu)

#define LOCOSIM_MP_REAL_FIELDS(X) \
  X(body_pos, 3 * nb) X(body_quat, 4 * nb) X(body_ipos, 3 * nb) X(body_iquat, 4 * nb) X(body_mass, nb) \
  X(body_inertia, 3 * nb) X(body_invweight0, 2 * nb) \
  X(jnt_pos, 3 * nv) X(jnt_axis, 3 * nv) X(jnt_range, 2 * nv) X(jnt_stiffness, nv) X(jnt_margin, nv) \
  X(jnt_solref, 2 * nv) X(jnt_solimp, 5 * nv) X(qpos0, nv) X(qpos_spring, nv) \
  X(dof_armature, nv) X(dof_damping, nv) X(dof_frictionloss, nv) X(dof_solref, 2 * nv) X(dof_solimp, 5 * nv) \
  X(dof_invweight0, nv) \
  X(geom_size, 3 * ng) X(geom_pos, 3 * ng) X(geom_quat, 4 * ng) X(geom_friction, 3 * ng) X(geom_margin, ng) \
  X(geom_gap, ng) X(geom_solref, 2 * ng) X(geom_solimp, 5 * ng) X(geom_solmix, ng) X(geom_rbound, ng) \
  X(geom_invweight0, 2 * ng) \
  X(mesh_vert, 3 * nm) \
  X(actuator_gear, nu) X(actuator_ctrlrange, 2 * nu) X(actuator_forcerange, 2 * nu) X(actuator_gain, nu) \
  X(actuator_bias, 3 * nu)

/* Height field (terrain): present when ints[MPI_HF_NROW] > 0. Its elevation samples follow the real fields as one
 * trailing array, hfield_data[nrow * ncol] (row major, normalised to [0, 1]); its size is reals[MPR_HF_SIZE .. + 4). The
 * terrain is the model's LAST geom (type LS_GEOM_HFIELD, on the world body). A pack without a terrain has zeros in these
 * slots and no trailing array: it is the same bytes as before the terrain existed, and keeps LOCOSIM_MP_VERSION.
 * The terrain's semantics are include/locosim.h's (locosim_set_terrain_origin). */

/* geom / joint type codes (MuJoCo's numbering) */
enum { LS_GEOM_PLANE = 0, LS_GEOM_HFIELD, LS_GEOM_SPHERE, LS_GEOM_CAPSULE, LS_GEOM_ELLIPSOID, LS_GEOM_CYLINDER,
       LS_GEOM_BOX, LS_GEOM_MESH };
enum { LS_JNT_SLIDE = 2, LS_JNT_HINGE = 3 };

#endif
