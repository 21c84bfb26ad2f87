// locosim_core.cuh -- warp-per-environment rigid-body + soft-contact step, fp32, sm_100a.
//
// One warp owns one environment for the whole control step (n_substeps physics steps + observation /
// reward / termination / auto-reset); all per-env state lives in shared memory (struct EnvS) and never
// touches HBM between the initial load and the final store.  Loops whose iterations are independent are
// strided over the 32 lanes (PAR_FOR) and separated by __syncwarp(); scalar control flow (solver iterations,
// line-search bracketing) is warp-uniform because every reduction is an all-lanes butterfly.
//
// What is computed is the reference's LocoEnv.step() hot path: mushroom_rl MuJoCo.step ->
// mujoco.mj_step(model, data, n_substeps) (/root/reference/loco_mujoco/environments/base.py:25,32-33,109-111)
// plus the hooks listed in include/locosim_task.h.  The algorithmic spec is MuJoCo 2.3.7's mj_step pipeline;
// the fp64 restatement that pins it against the reference's golden rollouts is oracle/locosim_ref.c (test only).
//
// The same source compiles as a *serial emulation* with -DLS_EMULATE (lanes executed one after another):
// a development aid to debug numerics on a CPU-only box; it is never part of the product path.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/locosim.h"            // (LS_BODY_DIM, LS_CONTACT_DIM)
#include "../../include/locosim_modelpack.h"
#include "../../include/locosim_task.h"

#ifdef LS_EMULATE
struct alignas(16) float4 { float x, y, z, w; };
#define LS_DEV static inline
#define LS_FN static
#define PAR_FOR(i, n) for (int i = 0; i < (n); i++)
#define PAR_FOR4(i, n) for (int i = 0; i < (n); i++)
#define SYNC() ((void)0)
#define WARP_SUM(x) (x)
#define WARP_MIN(x) (x)
#define WARP_ARGMAX(v, i) ((void)0)
#define LANE0
#define LS_LANE 0
#define LS_FFS(x) __builtin_ffs((int)(x))
#define LS_CLZ(x) __builtin_clz((unsigned)(x))
#define BLOCK_ANY(flag, pred) (pred)
#define BLOCK_SYNC(flag) ((void)0)
#define LS_LDG(p) (*(p))
#define LS_LDCG(p) (*(p))
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
#else
#define LS_DEV __device__ __forceinline__
#define LS_FN __device__ __noinline__
#define PAR_FOR(i, n) _Pragma("unroll 1") for (int i = (int)(threadIdx.x & 31); i < (n); i += 32)
#define PAR_FOR4(i, n) _Pragma("unroll 4") for (int i = (int)(threadIdx.x & 31); i < (n); i += 32)   // (loops that wait on global loads)
#define SYNC() __syncwarp()
#define WARP_SUM(x) warp_sum(x)
#define LANE0 if ((threadIdx.x & 31) == 0)
#define LS_LANE ((int)(threadIdx.x & 31))
#define LS_FFS(x) __ffs((int)(x))
#define LS_CLZ(x) __clz((int)(x))
#define LS_LDG(p) __ldg(p)           // read-only path (caller-owned inputs that no warp writes before its last read)
#define LS_LDCG(p) __ldcg(p)         // past L1 (rows another SM of the same launch may have written)
// OR-reduction that doubles as a barrier: keeps warps in the same solver iteration (flag = 0: plain predicate).
// flag = number of consecutive warps that iterate in lock-step (a GROUP): flag >= warps per block -> the whole block
// (__syncthreads_or); smaller groups use one named barrier each (barrier.red with a thread count), so a group only waits
// for the slowest of its own envs while all groups still execute the same (solver) code region.
__device__ __forceinline__ bool group_any(int group_warps, bool pred) {
  const int nw = (int)(blockDim.x >> 5);
  if (group_warps >= nw) return __syncthreads_or(pred ? 1 : 0) != 0;
  const int g = (int)(threadIdx.x >> 5) / group_warps;
  const int first = g * group_warps, cnt = (first + group_warps <= nw ? group_warps : nw - first) * 32;
  unsigned out, p = pred ? 1u : 0u, id = (unsigned)(1 + g), n = (unsigned)cnt;
  asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 p, %1, 0;\n\tbarrier.cta.red.or.pred q, %2, %3, p;\n\tselp.u32 %0, 1, 0, q;\n\t}"
               : "=r"(out) : "r"(p), "r"(id), "r"(n) : "memory");
  return out != 0;
}
#define BLOCK_ANY(flag, pred) ((flag) ? group_any((flag), (pred)) : (pred))
#define BLOCK_SYNC(flag) do { if (flag) __syncthreads(); } while (0)
LS_DEV float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// all lanes end up with the largest v and its index i; ties go to the smaller index (= the first maximum of a serial scan)
#define WARP_ARGMAX(v, i)                                                                  \
  do {                                                                                     \
    _Pragma("unroll") for (int o_ = 16; o_ > 0; o_ >>= 1) {                                \
      const float ov_ = __shfl_xor_sync(0xffffffffu, (v), o_);                             \
      const int oi_ = __shfl_xor_sync(0xffffffffu, (i), o_);                               \
      if (ov_ > (v) || (ov_ == (v) && oi_ < (i))) { (v) = ov_; (i) = oi_; }                \
    }                                                                                      \
  } while (0)
#endif

#define NOUNROLL _Pragma("unroll 1")
#define LS_MINVAL 1e-15f
#define LS_MINIMP 0.0001f
#define LS_MAXIMP 0.9999f

enum { ROW_FRICTION = 1, ROW_LIMIT = 3, ROW_CON_FRICTIONLESS = 5, ROW_CON_PYRAMIDAL = 6, ROW_CON_ELLIPTIC = 7 };
enum { ST_SATISFIED = 0, ST_QUADRATIC = 1, ST_LINEARNEG = 2, ST_LINEARPOS = 3, ST_CONE = 4 };

// ----------------------------------------------------------------------------------------------------------
// device-side model view: pointers into the fp32 / int32 device copies of the ModelPack blobs
// ----------------------------------------------------------------------------------------------------------
struct DevModel {
  int nb, nv, ng, nu, np, nm, integrator, cone, iterations, nlevel, nfric;
  float timestep, gravity[3], impratio, tolerance, meaninertia;
  int has_damping;
  int np_prim;               // the first np_prim candidate pairs are primitive (plane / sphere / capsule routines), the rest general convex
  int pk_n;                  // entries of the table EnvS::pk_tab points to (np: the model's; np_prim: the block's TMA-staged copy)
#define X(name, cnt) const int* name;
  LOCOSIM_MP_INT_FIELDS(X)
#undef X
#define X(name, cnt) const float* name;
  LOCOSIM_MP_REAL_FIELDS(X)
#undef X
  // engine-only derived tables (built in locosim.cu from the ModelPack)
  const int* body_level;     // [nb] depth in the tree (world = 0)
  const int* body_dofmask;   // [nb] bit d set if dof d is on the path root..body
  const int* dof_frow;       // [nv] index of the frictionloss row of dof d, or -1
  const int* tri_ij;         // [nv(nv+1)/2] packed (i << 8) | j of the lower triangle, row major
  const int* pair_packed;    // [np] g1 | g2 << 12 | flags << 24 (1: plane pair, 2: convex pair, 4: capsule-hull test) of pair p
  const float* pair_bound;   // [np] bound of the bounding-sphere / plane mid-phase test of pair p
  // per-env parameter pool (domain randomisation): float offsets of each field inside one pool row
  int po_dof_damping, po_dof_frictionloss, po_dof_armature, po_jnt_stiffness, po_dof_invweight0, po_body_mass,
      po_body_inertia, po_body_ipos, po_body_iquat, po_geom_friction, po_geom_invweight0, po_meaninertia, po_user, pool_P;
};

// applied forces of a handle (locosim_set_applied_forces): caller-owned [N, nb, 6] body wrenches (force, torque; world frame,
// at the body's CoM) and [N, nv] generalised forces, row EnvS::env; NULL = none. The engine zeroes the rows of an env it resets.
struct DevApplied {
  float* xfrc;
  float* qfrc;
};

// body outputs of a handle (locosim_set_body_outputs): caller-owned [N, nb, LS_BODY_DIM] rows (xpos, xquat, angular and linear
// velocity of the body-frame origin, world frame) of the returned state (`body`) and of the state to act on next
// (`next_body`); NULL = not written. reset_mark [N] (engine-owned): set where a step's reset_env wrote the env's `body` rows.
struct DevBodyOut {
  float* body;
  float* next_body;
  int* reset_mark;
};

// contact outputs of a handle (locosim_set_contact_outputs): caller-owned [N, nb, LS_CONTACT_DIM] per-body contact wrenches
// (force, torque about xpos; world frame), row EnvS::env, the mean over the n_substeps sub-steps of a control step (the
// task's); NULL = not written
struct DevContact {
  float* wrench;
  int n_substeps;
};

// per-dof outputs of a handle (locosim_set_dof_outputs): caller-owned [N, nv, LS_DOF_DIM] (qfrc_actuator, qfrc_constraint,
// qacc), row EnvS::env, the mean over the n_substeps sub-steps of a control step; NULL = not written. The layout and size
// of DevContact: physics_substeps tests both pointers, and with a 24-byte stride the extra address arithmetic grew the
// CfgPyrRK4 step kernel's stack frame with nothing registered.
struct DevDof {
  float* out;
  int n_substeps;
};

// contact list of a handle (locosim_set_contact_list_outputs): caller-owned [N] contact counts, [N, MAXCON, LS_CONLIST_DIM]
// rows (dist, pos, frame, contact-frame force) and [N, MAXCON, LS_CONLIST_ID_DIM] ids (geom1, geom2, body1, body2, dim),
// row EnvS::env, the contacts of the control step's last sub-step; NULL = not written. Two tables of DevDof's 16-byte
// layout: physics_substeps tests `ncon`, and a 32-byte stride grew the CfgPyrRK4 step kernel's stack frame by 16 bytes.
struct DevConList {
  int* ncon;
  int n_substeps;
};
struct DevConRows {
  float* con;
  int* id;
};

struct DevTask {
  int obs_dim, n_done, reward_type, n_substeps, n_traj, traj_len, n_goal, recenter0, recenter1, ri[4], use_absorbing;
  int n_grf;                      // foot-force groups (use_foot_forces), 0 = off
  int po_user;                    // offset of the user features inside a parameter-pool row (LS_OBS_PARAM)
  int rot[3];                     // setup_random_rot: qpos index of the yaw, dof indices of root vx / vy (-1: off)
  float rp[2];
  float track[4];                 // LS_REWARD_TRACKING: w_pose, k_pose, w_vel, k_vel
  const int *obs_src_type, *obs_src_idx, *done_obs_idx, *act_idx, *grf_group;
  const float *act_mean, *act_delta, *done_lo, *done_hi, *table;
};


// Model descriptors live in __constant__ memory (16 slots, one per live handle): every warp reads them uniformly.
#define LS_MAX_SLOTS 16
#ifdef LS_EMULATE
static DevModel c_models[LS_MAX_SLOTS];
static DevApplied c_applied[LS_MAX_SLOTS];
static DevBodyOut c_bodyout[LS_MAX_SLOTS];
static DevContact c_contact[LS_MAX_SLOTS];
static DevDof c_dof[LS_MAX_SLOTS];
static float* c_dof_act[LS_MAX_SLOTS];
static DevConList c_conlist[LS_MAX_SLOTS];
static DevConRows c_conrows[LS_MAX_SLOTS];
static int c_debug = 0;
#else
__constant__ DevModel c_models[LS_MAX_SLOTS];
__constant__ DevApplied c_applied[LS_MAX_SLOTS];   // (a table of its own: DevModel's layout, and the code reading it, stay as they are)
__constant__ DevBodyOut c_bodyout[LS_MAX_SLOTS];  // (likewise)
__constant__ DevContact c_contact[LS_MAX_SLOTS];  // (likewise)
__constant__ int c_debug;      // diagnostic switches (LOCOSIM_DEBUG): 1 skip MPR, 2 skip the OBB filter, 4 drop convex pairs,
                               // 8 count MPR runs / support calls (locosim_debug_counters), 16 no separating-direction cache,
                               // 32 no capsule-hull test of sphere | capsule | cylinder pairs, 64 primitive pairs in
                               // rounds of 32 (filter, then narrow phase) also where C::PRIMLEAN
__constant__ DevDof c_dof[LS_MAX_SLOTS];          // (a table of its own, like c_contact)
// the dof outputs' [N, nu] scratch of the force per actuator, written by every dynamics evaluation while c_dof[ms].out is
// registered (the actuator force is folded into qfrc_smooth, and the Euler state it was evaluated at is gone after the
// integrator), read by dof_outputs
__constant__ float* c_dof_act[LS_MAX_SLOTS];
__constant__ DevConList c_conlist[LS_MAX_SLOTS];  // (a table of its own, like c_contact)
__constant__ DevConRows c_conrows[LS_MAX_SLOTS];  // (likewise)
__device__ unsigned long long g_dbg[8];      // (LOCOSIM_DEBUG & 8) MPR statistics: calls, support pairs, hits, cap exits
#endif

#ifdef LOCOSIM_TERRAIN
// height field (terrain) of a handle, read by terrain_pass: only the translation unit of the terrain configuration
// (locosim_terrain.cu) and the serial build define LOCOSIM_TERRAIN, so no other unit compiles any of this.
// data: the ModelPack's hfield_data [nrow * ncol] (fp32, in the model's device copy); origin: the caller-owned [N, 2] terrain
// origin per env (locosim_set_terrain_origin), row EnvS::env, NULL = zeros. The terrain pairs are pair_geom[p0, p0 + npair).
struct DevTerrain {
  const float* data;
  const float* origin;
  int nrow, ncol, geom, p0, npair;
  float size[4], pos[3];
};
#ifdef LS_EMULATE
static DevTerrain c_terrain[LS_MAX_SLOTS];
#else
__constant__ DevTerrain c_terrain[LS_MAX_SLOTS];
#endif
#endif

// Phase clock: a diagnostic build (-DLOCOSIM_PHASE_CLOCK, tools/phase_profile.py) in which lane 0 of every warp adds the
// clock64() cycles its env spends in each phase (or a count) to g_phase[slot][phase], one slot per (block mod 256, warp).
// Without the macro the hooks expand to nothing, so the product library's code is the same as without them.
enum {
  PH_KINEMATICS, PH_COM_POS, PH_CRB_FACTOR, PH_SMOOTH_FORCES, PH_COLLISION, PH_CONVEX_QUEUE, PH_MAKE_CONSTRAINT, PH_WARMSTART,
  PH_NEWTON_WAIT, PH_NEWTON_TRIPS, PH_NEWTON_ITERS, PH_MAKE_HESSIAN, PH_CHOL_FACTOR, PH_CHOL_SOLVE, PH_LINE_SEARCH, PH_LS_EVAL,
  PH_LS_EVALS, PH_UPDATE_CONSTRAINT, PH_UPDATE_GRADIENT, PH_NEWTON_TAIL, PH_INTEGRATOR, PH_SUBSTEP, PH_SUBSTEPS, PH_PROLOGUE,
  PH_EPILOGUE, PH_GROUPS,
  // collision() split: primitive filter rounds, primitive narrow phase + fill_contact, convex bounding-sphere loop, box (and
  // capsule-hull) tests, the job queue's first barrier, the warp's own jobs, the barrier that waits for the block's other
  // jobs, convex_consume; then counts of the box-test survivors, of the jobs published, of the primitive pairs that pass
  // the filter and of the primitive narrow sets (rounds) run
  PH_COL_PRIM_FILTER, PH_COL_PRIM_NARROW, PH_COL_SPHERES, PH_COL_OBB, PH_COL_QWAIT, PH_COL_JOBS, PH_COL_JOBS_WAIT,
  PH_COL_CONSUME, PH_COL_NOBB, PH_COL_NJOBS, PH_COL_NPRIM, PH_COL_PRIM_SETS, PH_N
};
#if defined(LOCOSIM_PHASE_CLOCK) && !defined(LS_EMULATE)
#define LS_PH_SLOTS (256 * 16)
__device__ unsigned long long g_phase[LS_PH_SLOTS][PH_N];
__device__ __forceinline__ void ph_add(int ph, long long v) {
  if ((threadIdx.x & 31) == 0) atomicAdd(&g_phase[(blockIdx.x & 255) * 16 + (threadIdx.x >> 5)][ph], (unsigned long long)v);
}
#define PH_T0(t) long long t = clock64()
#define PH_LAP(ph, t) do { const long long n_ = clock64(); ph_add((ph), n_ - (t)); (t) = n_; } while (0)
#define PH_CNT(ph, n) ph_add((ph), (n))
#else
#define PH_T0(t) ((void)0)
#define PH_LAP(ph, t) ((void)0)
#define PH_CNT(ph, n) ((void)0)
#endif

struct SolverOpts {
  float tolerance;     // Newton termination (scaled improvement / gradient), fp32-appropriate
  float ls_tolerance;  // relative line-search gradient tolerance
  int max_iter;        // Newton iterations cap
  int ls_iter;         // line-search evaluations cap
  int sync_iters;      // warps per lock-step group of the Newton iterations (0: none; >= warps per block: the whole block)
  int sync_phases;     // bit mask of extra block barriers at phase boundaries of forward()
};

// ----------------------------------------------------------------------------------------------------------
// per-environment working set (shared memory, one per warp)
// ----------------------------------------------------------------------------------------------------------
template <class C>
struct alignas(16) EnvS {
  enum { NV = C::NV, NB = C::NB, NG = C::NG, NVP = C::NV + 1, JS = (C::NV + 3) & ~3, MAXCON = C::MAXCON, MAXROW = C::MAXROW,
         MAXUNIT = 2 * C::NV, MAXEFC = 2 * C::NV + C::MAXROW, NRK = C::RK4 ? C::NV : 1, NSEP = C::CONVEX ? 4 : 1 };
  // state + per-sub-step vectors
  float qpos[NV], qvel[NV], qacc[NV], qacc_ws[NV], ctrl[NV];
  float qfrc_smooth[NV], qacc_smooth[NV];
  float x0q[NRK], x0v[NRK], accq[NRK], accv[NRK];           // RK4 accumulators (RK4 configurations only)
  // kinematics that stays alive through collision / constraint assembly
  float xpos[NB][3], xquat[NB][4], xmat[NB][9];
  float gxpos[NG][3];
  float com[3];
  int substep;             // contact / dof outputs, contact list: index within the control step of the next sub-step (-1: a
                           // warp that shadows another env, which writes no outputs); set by the kernels, advanced by
                           // contact_wrench (or by dof_outputs when it is not registered, or by contact_list when neither is)
  float cdof[NV][6];
  float M[NV][NVP], H[NV][NVP];                              // H: chol(M) during smooth_forces, then the Newton Hessian factor
  // contacts
  int ncon, nunit, nrow, nefc, solver_iter, iter_sum, sep_next, mpr_calls;   // iter_sum / mpr_calls: Newton iterations / MPR runs of this control step
  int njobs, job_head;     // convex jobs this env published for the block (collision()); job_head: head of the block's job queue
                           // (env 0 of the block only). NOTE: sizeof(EnvS) decides the envs per SM (CfgPyrRK4: 16592 B = 14)
  float con_dist[MAXCON], con_pos[MAXCON][3], con_frame[MAXCON][9], con_fri[MAXCON][5], con_imp[MAXCON], con_K[MAXCON],
      con_B[MAXCON], con_incl[MAXCON], con_mu[MAXCON];
  int con_dim[MAXCON], con_g1[MAXCON], con_g2[MAXCON], con_row[MAXCON];
  // Two phases share storage: (a) smooth dynamics scratch, dead once qfrc_smooth / qacc_smooth are known;
  // (b) the constraint phase: rows [0,nunit) unit rows (frictionloss, then joint limits), [nunit, nunit+nrow) contact
  //     rows, and the solver's vectors (alive from make_constraint to the integrator).
  union {
    struct {
      float xipos[NB][3], ximat[NB][9], xanchor[NV][3], xaxis[NV][3];
      float cinert[NB][10], crb[NB][10], cdof_dot[NV][6];
    };
    struct {
      float r_D[MAXEFC], r_aref[MAXEFC], r_jar[MAXEFC], r_Jv[MAXEFC], r_force[MAXEFC];
      float Ma[NV], grad[NV], Mgrad[NV], search[NV], Mv[NV], qfrc_constraint[NV];   // solver vectors
      float coneU[8], coneS[8];
      int r_ti[MAXEFC];                                      // type | id << 8 | k << 24  (k: row within contact / limit side)
      int d_lrow[NV][2];                                     // limit row of dof d (side 0/1) or -1
      unsigned char r_state[MAXEFC];
    };
  };
  int env;                           // row of this env in the applied-force buffers (c_applied[ms]);
                                     // sits in the alignment gap in front of J: sizeof(EnvS) is the same with and without it
  alignas(16) float J[MAXROW][JS];   // contact Jacobian rows, zero padded to a float4 multiple
#ifdef LS_EMULATE
  float Y[6][NV];
#endif
  // convex pairs: separating directions found by earlier evaluations of this control step (pair index, unit direction)
  int sep_pair[NSEP];
  float sep_dir[NSEP][3];
  // task
  float goal[4];
  float grf[3 * LS_MAX_GRF];   // use_foot_forces: per foot group, contact-frame force summed over the sub-steps
  const float* prm;        // this env's row of the parameter pool
  const int* pk_tab;       // table of the PRIMITIVE candidate pairs of the mid-phase: the model's (global) or the block's TMA-staged
                           // copy (shared): DevModel::pk_n packed pairs, directly followed by pk_n bounds (float)
};
#define PRM(field) (e.prm + m.po_##field)
#define ROW_TYPE(ti) ((ti) & 255)
#define ROW_ID(ti) (((ti) >> 8) & 0xffff)
#define ROW_K(ti) ((ti) >> 24)
#define ROW_PACK(type, id, k) ((type) | ((id) << 8) | ((k) << 24))

// ----------------------------------------------------------------------------------------------------------
// small math
// ----------------------------------------------------------------------------------------------------------
LS_DEV float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
LS_DEV void cross3(float* r, const float* a, const float* b) {
  float x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
LS_DEV float normalize3(float* a) {
  float n = sqrtf(dot3(a, a));
  if (n < LS_MINVAL) { a[0] = 1; a[1] = 0; a[2] = 0; }
  else { float inv = 1.0f / n; a[0] *= inv; a[1] *= inv; a[2] *= inv; }
  return n;
}
LS_DEV void mulmatvec3(float* r, const float* m, const float* v) {
  float x = m[0] * v[0] + m[1] * v[1] + m[2] * v[2], y = m[3] * v[0] + m[4] * v[1] + m[5] * v[2],
        z = m[6] * v[0] + m[7] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
LS_DEV void mulmatTvec3(float* r, const float* m, const float* v) {
  float x = m[0] * v[0] + m[3] * v[1] + m[6] * v[2], y = m[1] * v[0] + m[4] * v[1] + m[7] * v[2],
        z = m[2] * v[0] + m[5] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
LS_DEV void quat2mat(float* m, const float* q) {
  float q00 = q[0] * q[0], q01 = q[0] * q[1], q02 = q[0] * q[2], q03 = q[0] * q[3], q11 = q[1] * q[1], q12 = q[1] * q[2],
        q13 = q[1] * q[3], q22 = q[2] * q[2], q23 = q[2] * q[3], q33 = q[3] * q[3];
  m[0] = q00 + q11 - q22 - q33; m[4] = q00 - q11 + q22 - q33; m[8] = q00 - q11 - q22 + q33;
  m[1] = 2 * (q12 - q03); m[2] = 2 * (q13 + q02); m[3] = 2 * (q12 + q03);
  m[5] = 2 * (q23 - q01); m[6] = 2 * (q13 - q02); m[7] = 2 * (q23 + q01);
}
LS_DEV void mulquat(float* r, const float* a, const float* b) {
  float t0 = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], t1 = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
        t2 = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], t3 = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = t0; r[1] = t1; r[2] = t2; r[3] = t3;
}
LS_DEV void mulInertVec(float* res, const float* i, const float* v) {
  res[0] = i[0] * v[0] + i[3] * v[1] + i[4] * v[2] - i[8] * v[4] + i[7] * v[5];
  res[1] = i[3] * v[0] + i[1] * v[1] + i[5] * v[2] + i[8] * v[3] - i[6] * v[5];
  res[2] = i[4] * v[0] + i[5] * v[1] + i[2] * v[2] - i[7] * v[3] + i[6] * v[4];
  res[3] = i[8] * v[1] - i[7] * v[2] + i[9] * v[3];
  res[4] = i[6] * v[2] - i[8] * v[0] + i[9] * v[4];
  res[5] = i[7] * v[0] - i[6] * v[1] + i[9] * v[5];
}
LS_DEV void crossMotion(float* res, const float* vel, const float* v) {
  float a[3], b[3];
  cross3(res, vel, v);
  cross3(a, vel, v + 3);
  cross3(b, vel + 3, v);
  res[3] = a[0] + b[0]; res[4] = a[1] + b[1]; res[5] = a[2] + b[2];
}
LS_DEV void crossForce(float* res, const float* vel, const float* f) {
  float a[3], b[3];
  cross3(a, vel, f);
  cross3(b, vel + 3, f + 3);
  res[0] = a[0] + b[0]; res[1] = a[1] + b[1]; res[2] = a[2] + b[2];
  cross3(res + 3, vel, f + 3);
}

// ---- constraint impedance helpers (mj_makeImpedance) ----
LS_DEV float ls_pow(float x, float p) {
  // x in (0,1); p >= 1. power 2 (MuJoCo's default) is exact, other powers go through exp2/log2
  return p == 2.0f ? x * x : (p == 1.0f ? x : exp2f(p * log2f(x)));
}
LS_DEV void get_impedance(const float* solimp_in, float pos, float margin, float* imp) {
  float s0 = fminf(LS_MAXIMP, fmaxf(LS_MINIMP, solimp_in[0])), s1 = fminf(LS_MAXIMP, fmaxf(LS_MINIMP, solimp_in[1]));
  float s2 = fmaxf(0.0f, solimp_in[2]), s3 = fminf(LS_MAXIMP, fmaxf(LS_MINIMP, solimp_in[3])), s4 = fmaxf(1.0f, solimp_in[4]);
  if (s0 == s1 || s2 <= LS_MINVAL) { *imp = 0.5f * (s0 + s1); return; }
  float x = fabsf((pos - margin) / s2);
  if (x >= 1 || x <= 0) { *imp = (x >= 1 ? s1 : s0); return; }
  float y;
  if (s4 == 1) y = x;
  else if (x <= s3) y = ls_pow(x, s4) / ls_pow(s3, s4 - 1);
  else y = 1 - ls_pow(1 - x, s4) / ls_pow(1 - s3, s4 - 1);
  *imp = s0 + y * (s1 - s0);
}

LS_FN void impedance_KB(const float* solref, const float* solimp, float pos, float margin, float timestep, float* imp,
                         float* K, float* B) {
  float sr0 = solref[0], sr1 = solref[1];
  if (sr0 > 0) sr0 = fmaxf(sr0, 2 * timestep);
  get_impedance(solimp, pos, margin, imp);
  float dmax = fminf(LS_MAXIMP, fmaxf(LS_MINIMP, solimp[1]));
  if (sr0 > 0) { *K = 1 / fmaxf(LS_MINVAL, dmax * dmax * sr0 * sr0 * sr1 * sr1); *B = 2 / fmaxf(LS_MINVAL, dmax * sr0); }
  else { *K = -sr0 / fmaxf(LS_MINVAL, dmax * dmax); *B = -sr1 / fmaxf(LS_MINVAL, dmax); }
}

// ----------------------------------------------------------------------------------------------------------
// kinematics (mj_kinematics): level-synchronous over the tree, then geom centres
// ----------------------------------------------------------------------------------------------------------
// once per kernel (and per emulated env): the parts of the workspace that no phase rewrites
template <class C>
LS_FN void init_workspace(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  PAR_FOR(idx, EnvS<C>::NV * EnvS<C>::NVP) {
    int i = idx / EnvS<C>::NVP, j = idx - i * EnvS<C>::NVP;
    (&e.M[0][0])[idx] = (i == j && i >= m.nv) ? 1.0f : 0.0f;
  }
  PAR_FOR(k, EnvS<C>::NSEP) e.sep_pair[k] = -1;
  LANE0 { e.sep_next = 0; e.mpr_calls = 0; e.job_head = 0; e.njobs = 0; }
  // entries [nv, NV) of the solver vectors are never written by the phases (they loop to nv): keep them 0
  PAR_FOR(i, EnvS<C>::NV) {
    if (i >= m.nv) {
      e.qacc[i] = 0; e.qacc_ws[i] = 0; e.qacc_smooth[i] = 0;
      e.qfrc_smooth[i] = 0; e.qvel[i] = 0; e.qpos[i] = 0;
    }
  }
  SYNC();
}

// v rotated by the unit quaternion q:  v + 2 w (u x v) + 2 u x (u x v)
LS_DEV void rotvec(float* r, const float* q, const float* v) {
  float t[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  t[0] += t[0]; t[1] += t[1]; t[2] += t[2];
  float x = v[0] + q[0] * t[0] + (q[2] * t[2] - q[3] * t[1]), y = v[1] + q[0] * t[1] + (q[3] * t[0] - q[1] * t[2]),
        z = v[2] + q[0] * t[2] + (q[1] * t[1] - q[2] * t[0]);
  r[0] = x; r[1] = y; r[2] = z;
}

// mj_kinematics in three phases: (1) all joints in parallel: the joint's own quaternion / translation;
// (2) the kinematic chain, level by level, in quaternion algebra only (the only serial part: per joint one vector
// rotation and one quaternion product when the joint anchor is the body origin, which it is for almost every joint of
// the in-scope robots); (3) all bodies in parallel: rotation matrices, inertial frames; then geoms.
// one body of the kinematic chain; its joints' local data was staged in shared memory by phase 1 of kinematics():
// xanchor[j] = jnt_pos (body frame), xaxis[j] = jnt_axis (body frame), cdof_dot[j] = {joint quaternion | slide q, .., type,
// anchor-at-origin flag}; both are overwritten here with the world-frame anchor / axis.
template <class C>
LS_DEV void kin_body(EnvS<C>& e, const int b, const int p, const float* bpos, const float* bquat, const int jn,
                     const int ja) {
  float pos[3], quat[4], tmp[3];
  rotvec(tmp, e.xquat[p], bpos);
  for (int k = 0; k < 3; k++) pos[k] = e.xpos[p][k] + tmp[k];
  mulquat(quat, e.xquat[p], bquat);
  NOUNROLL for (int k = 0; k < jn; k++) {
    const int j = ja + k;
    const float* o = e.cdof_dot[j];
    const float jp[3] = {e.xanchor[j][0], e.xanchor[j][1], e.xanchor[j][2]};
    const float ja_[3] = {e.xaxis[j][0], e.xaxis[j][1], e.xaxis[j][2]};
    const bool at_origin = o[5] != 0.0f;
    float anchor[3] = {pos[0], pos[1], pos[2]}, axis[3];
    if (!at_origin) { rotvec(tmp, quat, jp); anchor[0] += tmp[0]; anchor[1] += tmp[1]; anchor[2] += tmp[2]; }
    rotvec(axis, quat, ja_);
    for (int c = 0; c < 3; c++) { e.xanchor[j][c] = anchor[c]; e.xaxis[j][c] = axis[c]; }
    if (o[4] != 0.0f) {                       // slide
      for (int c = 0; c < 3; c++) pos[c] += axis[c] * o[0];
    } else {
      mulquat(quat, quat, o);
      if (!at_origin) { rotvec(tmp, quat, jp); for (int c = 0; c < 3; c++) pos[c] = anchor[c] - tmp[c]; }
    }
  }
  const float inv = rsqrtf(quat[0] * quat[0] + quat[1] * quat[1] + quat[2] * quat[2] + quat[3] * quat[3]);
  for (int c = 0; c < 3; c++) e.xpos[b][c] = pos[c];
  for (int c = 0; c < 4; c++) e.xquat[b][c] = quat[c] * inv;
}

template <class C>
LS_FN void kinematics(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  LANE0 {
    e.xpos[0][0] = e.xpos[0][1] = e.xpos[0][2] = 0;
    e.xquat[0][0] = 1; e.xquat[0][1] = e.xquat[0][2] = e.xquat[0][3] = 0;
  }
  PAR_FOR(j, m.nv) {          // joint-local data -> shared-memory scratch (cdof_dot is free until smooth_forces)
    const float q = e.qpos[j] - m.qpos0[j];
    float* o = e.cdof_dot[j];
    const float ax = m.jnt_axis[3 * j], ay = m.jnt_axis[3 * j + 1], az = m.jnt_axis[3 * j + 2];
    const float px = m.jnt_pos[3 * j], py = m.jnt_pos[3 * j + 1], pz = m.jnt_pos[3 * j + 2];
    e.xaxis[j][0] = ax; e.xaxis[j][1] = ay; e.xaxis[j][2] = az;
    e.xanchor[j][0] = px; e.xanchor[j][1] = py; e.xanchor[j][2] = pz;
    o[5] = ((px == 0.0f) & (py == 0.0f) & (pz == 0.0f)) ? 1.0f : 0.0f;
    if (m.jnt_type[j] == LS_JNT_SLIDE) { o[0] = q; o[4] = 1.0f; }
    else {
      float sn, cs;
      sincosf(0.5f * q, &sn, &cs);
      o[0] = cs; o[1] = ax * sn; o[2] = ay * sn; o[3] = az * sn; o[4] = 0.0f;
    }
  }
  SYNC();
#ifdef LS_EMULATE
  for (int lev = 1; lev < m.nlevel; lev++)
    for (int b = 1; b < m.nb; b++)
      if (m.body_level[b] == lev)
        kin_body(e, b, m.body_parentid[b], m.body_pos + 3 * b, m.body_quat + 4 * b, m.body_jntnum[b], m.body_jntadr[b]);
#else
  {
    static_assert(C::NB <= 32, "lane b owns body b");
    // lane b owns body b (nb <= 32): its constants are loaded once, ahead of the serial level sweep, so that the sweep
    // itself touches registers and shared memory only
    const int b = LS_LANE;
    const bool has = b > 0 && b < m.nb;
    const int lev_b = has ? m.body_level[b] : -1, par = has ? m.body_parentid[b] : 0;
    const int jn = has ? m.body_jntnum[b] : 0, ja = has ? m.body_jntadr[b] : 0;
    float bpos[3] = {0, 0, 0}, bquat[4] = {1, 0, 0, 0};
    if (has) {
      for (int c = 0; c < 3; c++) bpos[c] = m.body_pos[3 * b + c];
      for (int c = 0; c < 4; c++) bquat[c] = m.body_quat[4 * b + c];
    }
    for (int lev = 1; lev < m.nlevel; lev++) {
      if (lev_b == lev) kin_body(e, b, par, bpos, bquat, jn, ja);
      SYNC();
    }
  }
#endif
  PAR_FOR(b, m.nb) {
    float mat[9], tmp[3], iq[4];
    quat2mat(mat, e.xquat[b]);
    for (int c = 0; c < 9; c++) e.xmat[b][c] = mat[c];
    mulmatvec3(tmp, mat, PRM(body_ipos) + 3 * b);
    for (int c = 0; c < 3; c++) e.xipos[b][c] = e.xpos[b][c] + tmp[c];
    mulquat(iq, e.xquat[b], PRM(body_iquat) + 4 * b);
    quat2mat(mat, iq);
    for (int c = 0; c < 9; c++) e.ximat[b][c] = mat[c];
  }
  SYNC();
  PAR_FOR(g, m.ng) {
    int b = m.geom_bodyid[g];
    float tmp[3];
    mulmatvec3(tmp, e.xmat[b], m.geom_pos + 3 * g);
    for (int c = 0; c < 3; c++) e.gxpos[g][c] = e.xpos[b][c] + tmp[c];
  }
  SYNC();
}

template <class C>
LS_DEV void geom_mat(const int ms, const EnvS<C>& e, int g, float* mat) {
  const DevModel& m = c_models[ms];
  float gq[4];
  mulquat(gq, e.xquat[m.geom_bodyid[g]], m.geom_quat + 4 * g);
  quat2mat(mat, gq);
}

// ----------------------------------------------------------------------------------------------------------
// mj_comPos (single kinematic tree: every body's root is body 1, its subtree CoM is the whole-robot CoM)
// ----------------------------------------------------------------------------------------------------------
template <class C>
LS_FN void com_pos(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  float sx = 0, sy = 0, sz = 0, sm = 0;
  PAR_FOR(b, m.nb) {
    float ms = PRM(body_mass)[b];
    sx += ms * e.xipos[b][0]; sy += ms * e.xipos[b][1]; sz += ms * e.xipos[b][2]; sm += ms;
  }
  sx = WARP_SUM(sx); sy = WARP_SUM(sy); sz = WARP_SUM(sz); sm = WARP_SUM(sm);
  float inv = 1.0f / sm;
  float com[3] = {sx * inv, sy * inv, sz * inv};
  LANE0 { e.com[0] = com[0]; e.com[1] = com[1]; e.com[2] = com[2]; }
  PAR_FOR(b, m.nb) {
    float* ci = e.cinert[b];
    if (b == 0) { for (int k = 0; k < 10; k++) ci[k] = 0; continue; }
    float dif[3] = {e.xipos[b][0] - com[0], e.xipos[b][1] - com[1], e.xipos[b][2] - com[2]};
    const float* R = e.ximat[b];
    const float* I = PRM(body_inertia) + 3 * b;
    float mass = PRM(body_mass)[b];
    float t[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) t[3 * r + c] = R[3 * r + c] * I[c];
    float r00 = t[0] * R[0] + t[1] * R[1] + t[2] * R[2], r11 = t[3] * R[3] + t[4] * R[4] + t[5] * R[5],
          r22 = t[6] * R[6] + t[7] * R[7] + t[8] * R[8], r01 = t[0] * R[3] + t[1] * R[4] + t[2] * R[5],
          r02 = t[0] * R[6] + t[1] * R[7] + t[2] * R[8], r12 = t[3] * R[6] + t[4] * R[7] + t[5] * R[8];
    ci[0] = r00 + mass * (dif[1] * dif[1] + dif[2] * dif[2]);
    ci[1] = r11 + mass * (dif[0] * dif[0] + dif[2] * dif[2]);
    ci[2] = r22 + mass * (dif[0] * dif[0] + dif[1] * dif[1]);
    ci[3] = r01 - mass * dif[0] * dif[1];
    ci[4] = r02 - mass * dif[0] * dif[2];
    ci[5] = r12 - mass * dif[1] * dif[2];
    ci[6] = mass * dif[0]; ci[7] = mass * dif[1]; ci[8] = mass * dif[2]; ci[9] = mass;
  }
  PAR_FOR(j, m.nv) {
    float* cd = e.cdof[j];
    if (m.jnt_type[j] == LS_JNT_SLIDE) {
      cd[0] = cd[1] = cd[2] = 0;
      cd[3] = e.xaxis[j][0]; cd[4] = e.xaxis[j][1]; cd[5] = e.xaxis[j][2];
    } else {
      float off[3] = {com[0] - e.xanchor[j][0], com[1] - e.xanchor[j][1], com[2] - e.xanchor[j][2]};
      cd[0] = e.xaxis[j][0]; cd[1] = e.xaxis[j][1]; cd[2] = e.xaxis[j][2];
      cross3(cd + 3, e.xaxis[j], off);
    }
  }
  SYNC();
}

// ----------------------------------------------------------------------------------------------------------
// dense SPD solves on identity-padded NV x NV matrices in shared memory (row stride NVP = NV + 1).
// Factor layout (chosen so that the triangular solves need no lane predicates): A[i][j] = L_ij for j < i,
// A[i][j] = 0 for NV > j >= i, and the padding column holds the inverse diagonal, A[i][NV] = 1 / L_ii.
// ----------------------------------------------------------------------------------------------------------
template <int NV, int NVP>
LS_FN void chol_factor(const int ms, float (*A)[NVP]) {
#ifdef LS_EMULATE
  for (int j = 0; j < NV; j++) {
    const float inv = rsqrtf(fmaxf(A[j][j], 1e-12f));
    A[j][NV] = inv;
    for (int i = j + 1; i < NV; i++) A[i][j] *= inv;
    for (int i = j + 1; i < NV; i++)
      for (int k = j + 1; k <= i; k++) A[i][k] = fmaf(-A[i][j], A[k][j], A[i][k]);
  }
  for (int i = 0; i < NV; i++) for (int j = i; j < NV; j++) A[i][j] = 0.0f;
  (void)ms;
#else
  // Lane i keeps row i in registers; column j of the factor is broadcast lane-to-lane with shuffles
  // (right-looking, ~2 instructions per updated entry, no shared-memory round trips inside the loop).
  // One __noinline__ copy per NV serves M, the Newton Hessian and the implicit-damping matrix.
  const int lane = LS_LANE, li = lane < NV ? lane : NV - 1;
  float a[NV], inv = 1.0f;
#pragma unroll
  for (int j = 0; j < NV; j++) a[j] = A[li][j];
#pragma unroll
  for (int j = 0; j < NV; j++) {
    const float r = rsqrtf(fmaxf(__shfl_sync(0xffffffffu, a[j], j), 1e-12f));
    if (lane == j) inv = r;
    a[j] *= r;
#pragma unroll
    for (int k = j + 1; k < NV; k++) a[k] = fmaf(-a[j], __shfl_sync(0xffffffffu, a[j], k), a[k]);
  }
  __syncwarp();
  if (lane < NV) {
#pragma unroll
    for (int j = 0; j < NV; j++) A[lane][j] = (j < lane) ? a[j] : 0.0f;
    A[lane][NV] = inv;
  }
  __syncwarp();
  (void)ms;
#endif
}
// solve L L^T x = b in place (x: shared memory vector of length >= NV, padded entries finite)
template <int NV, int NVP>
LS_FN void chol_solve(float (*L)[NVP], float* xs) {
#ifdef LS_EMULATE
  for (int i = 0; i < NV; i++) {
    float v = xs[i];
    for (int k = 0; k < i; k++) v -= L[i][k] * xs[k];
    xs[i] = v * L[i][NV];
  }
  for (int i = NV - 1; i >= 0; i--) {
    float v = xs[i];
    for (int k = i + 1; k < NV; k++) v -= L[k][i] * xs[k];
    xs[i] = v * L[i][NV];
  }
#else
  // lane i carries x_i; thanks to the zeros on and above the diagonal every lane executes the same FFMA
  const int lane = LS_LANE, li = lane < NV ? lane : NV - 1;
  float x = lane < NV ? xs[lane] : 0.0f;
  const float inv = L[li][NV];
#pragma unroll
  for (int j = 0; j < NV - 1; j++) x = fmaf(-L[li][j], __shfl_sync(0xffffffffu, x * inv, j), x);   // y_j = x_j / L_jj
  x *= inv;                                                                                          // x = y (L y = b)
#pragma unroll
  for (int j = NV - 1; j > 0; j--) x = fmaf(-L[j][li], __shfl_sync(0xffffffffu, x * inv, j), x);    // z_j = x_j / L_jj
  x *= inv;
  if (lane < NV) xs[lane] = x;
  __syncwarp();
#endif
}

// ----------------------------------------------------------------------------------------------------------
// mj_crb + factor: composite inertias up the tree, joint-space inertia M, L = chol(M)
// ----------------------------------------------------------------------------------------------------------
template <class C>
LS_FN void crb_factor(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  // composite inertia of body b = sum of cinert over its subtree = the bodies whose dof chain contains b's last dof
  // (all in one frame, so a plain sum; no level recursion)
  PAR_FOR(b, m.nb) {
    float acc[10];
    for (int k = 0; k < 10; k++) acc[k] = e.cinert[b][k];
    if (b > 0) {
      const int ld = 31 - LS_CLZ(m.body_dofmask[b]);
      NOUNROLL for (int c = b + 1; c < m.nb; c++) {
        if (!((m.body_dofmask[c] >> ld) & 1)) continue;
        for (int k = 0; k < 10; k++) acc[k] += e.cinert[c][k];
      }
    }
    for (int k = 0; k < 10; k++) e.crb[b][k] = acc[k];
  }
  SYNC();
  // (entries of M outside the dof chains stay 0 and the identity padding stays 1: init_workspace)
  PAR_FOR(i, m.nv) {
    float buf[6];
    mulInertVec(buf, e.crb[m.jnt_bodyid[i]], e.cdof[i]);
    NOUNROLL for (int j = i; j >= 0; j = m.dof_parentid[j]) {
      float v = 0;
      for (int k = 0; k < 6; k++) v += e.cdof[j][k] * buf[k];
      if (j == i) v += PRM(dof_armature)[i];
      e.M[i][j] = v;
      e.M[j][i] = v;
    }
  }
  SYNC();
  PAR_FOR(idx, EnvS<C>::NV * EnvS<C>::NVP) (&e.H[0][0])[idx] = (&e.M[0][0])[idx];
  SYNC();
  chol_factor<EnvS<C>::NV, EnvS<C>::NVP>(ms, e.H);
}

// ----------------------------------------------------------------------------------------------------------
// narrow phase (one lane per candidate pair). Raw contacts: dist, pos, frame(normal [+tangent hint])
// ----------------------------------------------------------------------------------------------------------
struct RawCon { float dist, pos[3], frame[6]; };

LS_FN int plane_sphere(RawCon* c, float margin, const float* pos1, const float* n, const float* pos2, float r) {
  float tmp[3] = {pos2[0] - pos1[0], pos2[1] - pos1[1], pos2[2] - pos1[2]};
  float cdist = dot3(tmp, n);
  if (cdist > margin + r) return 0;
  c->dist = cdist - r;
  for (int k = 0; k < 3; k++) { c->frame[k] = n[k]; c->frame[3 + k] = 0; c->pos[k] = pos2[k] + n[k] * (-c->dist * 0.5f - r); }
  return 1;
}
LS_FN int plane_capsule(RawCon* c, float margin, const float* pos1, const float* n, const float* pos2, const float* mat2,
                         const float* size2) {
  float axis[3] = {mat2[2], mat2[5], mat2[8]};
  float seg[3] = {axis[0] * size2[1], axis[1] * size2[1], axis[2] * size2[1]};
  float p[3] = {pos2[0] + seg[0], pos2[1] + seg[1], pos2[2] + seg[2]};
  int n1 = plane_sphere(c, margin, pos1, n, p, size2[0]);
  if (n1) for (int k = 0; k < 3; k++) c->frame[3 + k] = axis[k];
  p[0] = pos2[0] - seg[0]; p[1] = pos2[1] - seg[1]; p[2] = pos2[2] - seg[2];
  int n2 = plane_sphere(c + n1, margin, pos1, n, p, size2[0]);
  if (n2) for (int k = 0; k < 3; k++) c[n1].frame[3 + k] = axis[k];
  return n1 + n2;
}
LS_FN int plane_cylinder(RawCon* c, float margin, const float* pos1, const float* normal, const float* pos2,
                          const float* mat2, const float* size2) {
  float axis[3] = {mat2[2], mat2[5], mat2[8]};
  float d[3] = {pos2[0] - pos1[0], pos2[1] - pos1[1], pos2[2] - pos1[2]};
  float dist0 = dot3(d, normal);
  float prjaxis = dot3(normal, axis);
  if (prjaxis > 0) { axis[0] = -axis[0]; axis[1] = -axis[1]; axis[2] = -axis[2]; prjaxis = -prjaxis; }
  float vec[3] = {axis[0] * prjaxis - normal[0], axis[1] * prjaxis - normal[1], axis[2] * prjaxis - normal[2]};
  float len_sqr = dot3(vec, vec);
  if (len_sqr >= 1e-12f) {
    float scl = size2[0] * rsqrtf(len_sqr);
    vec[0] *= scl; vec[1] *= scl; vec[2] *= scl;
  } else {
    vec[0] = mat2[0] * size2[0]; vec[1] = mat2[3] * size2[0]; vec[2] = mat2[6] * size2[0];
  }
  float prjvec = dot3(vec, normal);
  axis[0] *= size2[1]; axis[1] *= size2[1]; axis[2] *= size2[1];
  prjaxis *= size2[1];
  int cnt = 0;
  if (dist0 + prjaxis + prjvec <= margin) {
    c[cnt].dist = dist0 + prjaxis + prjvec;
    for (int k = 0; k < 3; k++) {
      c[cnt].pos[k] = pos2[k] + vec[k] + axis[k] - normal[k] * c[cnt].dist * 0.5f;
      c[cnt].frame[k] = normal[k]; c[cnt].frame[3 + k] = 0;
    }
    cnt++;
  } else return 0;
  if (dist0 - prjaxis + prjvec <= margin) {
    c[cnt].dist = dist0 - prjaxis + prjvec;
    for (int k = 0; k < 3; k++) {
      c[cnt].pos[k] = pos2[k] + vec[k] - axis[k] - normal[k] * c[cnt].dist * 0.5f;
      c[cnt].frame[k] = normal[k]; c[cnt].frame[3 + k] = 0;
    }
    cnt++;
  }
  float prjvec1 = -prjvec * 0.5f;
  if (dist0 + prjaxis + prjvec1 <= margin) {
    float vec1[3];
    cross3(vec1, vec, axis);
    normalize3(vec1);
    float sc = size2[0] * 0.8660254037844386f;
    vec1[0] *= sc; vec1[1] *= sc; vec1[2] *= sc;
    for (int sgn = 1; sgn >= -1; sgn -= 2) {
      c[cnt].dist = dist0 + prjaxis + prjvec1;
      for (int k = 0; k < 3; k++) {
        c[cnt].pos[k] = pos2[k] + sgn * vec1[k] + axis[k] - vec[k] * 0.5f - normal[k] * c[cnt].dist * 0.5f;
        c[cnt].frame[k] = normal[k]; c[cnt].frame[3 + k] = 0;
      }
      cnt++;
    }
  }
  return cnt;
}
LS_FN int plane_box(RawCon* c, float margin, const float* pos1, const float* norm, const float* pos2, const float* mat2,
                     const float* size2) {
  float d[3] = {pos2[0] - pos1[0], pos2[1] - pos1[1], pos2[2] - pos1[2]};
  float dist = dot3(d, norm);
  int cnt = 0;
  for (int i = 0; i < 8; i++) {
    float vec[3] = {(i & 1 ? size2[0] : -size2[0]), (i & 2 ? size2[1] : -size2[1]), (i & 4 ? size2[2] : -size2[2])};
    float corner[3];
    mulmatvec3(corner, mat2, vec);
    float ldist = dot3(norm, corner);
    if (dist + ldist > margin || ldist > 0) continue;
    c[cnt].dist = dist + ldist;
    for (int k = 0; k < 3; k++) {
      c[cnt].pos[k] = pos2[k] + corner[k] - norm[k] * c[cnt].dist * 0.5f;
      c[cnt].frame[k] = norm[k]; c[cnt].frame[3 + k] = 0;
    }
    if (++cnt >= 4) break;
  }
  return cnt;
}
LS_FN int plane_mesh(RawCon* c, float margin, const float* pos1, const float* norm, const float* pos2, const float* mat2,
                      const float* verts, int nvert, float rbound) {
  float nl[3];
  mulmatTvec3(nl, mat2, norm);
  float d[3] = {pos2[0] - pos1[0], pos2[1] - pos1[1], pos2[2] - pos1[2]};
  float dist0 = dot3(d, norm);
  int cnt = 0;
  int taken[3];
  float mind2 = (0.3f * rbound) * (0.3f * rbound);
  // support vertex first, then the next-deepest vertices at least 0.3 rbound away from the FIRST contact only, 3 contacts at
  // most (oracle/locosim_ref.c plane_mesh: the rule the UnitreeH1.walk / .carry goldens pin)
  for (int pass = 0; pass < 3; pass++) {
    int best = -1; float bd = 1e30f;
    for (int i = 0; i < nvert; i++) {
      const float* v = verts + 3 * i;
      float dd = dist0 + dot3(nl, v);
      if (dd > margin || dd >= bd) continue;
      if (cnt > 0) {
        if (i == taken[0] || (cnt > 1 && i == taken[1])) continue;
        const float* w = verts + 3 * taken[0];
        float ex = v[0] - w[0], ey = v[1] - w[1], ez = v[2] - w[2];
        if (ex * ex + ey * ey + ez * ez < mind2) continue;
      }
      best = i; bd = dd;
    }
    if (best < 0) break;
    float vg[3];
    mulmatvec3(vg, mat2, verts + 3 * best);
    c[cnt].dist = bd;
    for (int k = 0; k < 3; k++) {
      c[cnt].pos[k] = pos2[k] + vg[k] - norm[k] * bd * 0.5f;
      c[cnt].frame[k] = norm[k]; c[cnt].frame[3 + k] = 0;
    }
    taken[cnt++] = best;
  }
  return cnt;
}
LS_FN int sphere_sphere_raw(RawCon* c, float margin, const float* pos1, float r1, const float* pos2, float r2) {
  float dif[3] = {pos2[0] - pos1[0], pos2[1] - pos1[1], pos2[2] - pos1[2]};
  float cdist = sqrtf(dot3(dif, dif));
  if (cdist > margin + r1 + r2) return 0;
  c->dist = cdist - r1 - r2;
  if (cdist < 1e-12f) { c->frame[0] = 1; c->frame[1] = 0; c->frame[2] = 0; }
  else { float inv = 1.0f / cdist; c->frame[0] = dif[0] * inv; c->frame[1] = dif[1] * inv; c->frame[2] = dif[2] * inv; }
  for (int k = 0; k < 3; k++) { c->frame[3 + k] = 0; c->pos[k] = pos1[k] + c->frame[k] * (r1 + 0.5f * c->dist); }
  return 1;
}
LS_FN int sphere_capsule(RawCon* c, float margin, const float* pos1, float r1, const float* pos2, const float* mat2,
                          const float* size2) {
  float axis[3] = {mat2[2], mat2[5], mat2[8]};
  float vec[3] = {pos1[0] - pos2[0], pos1[1] - pos2[1], pos1[2] - pos2[2]};
  float x = fminf(size2[1], fmaxf(-size2[1], dot3(axis, vec)));
  float p[3] = {pos2[0] + axis[0] * x, pos2[1] + axis[1] * x, pos2[2] + axis[2] * x};
  return sphere_sphere_raw(c, margin, pos1, r1, p, size2[0]);
}
// mjc_SphereBox: sphere g1 against box g2 (restated in oracle/locosim_ref.c sphere_box)
LS_FN int sphere_box(RawCon* c, float margin, const float* pos1, float r, const float* pos2, const float* mat2,
                     const float* size2) {
  const float tmp[3] = {pos1[0] - pos2[0], pos1[1] - pos2[1], pos1[2] - pos2[2]};
  float cen[3], cl[3], d[3], nb[3] = {0, 0, 0}, pl[3];
  mulmatTvec3(cen, mat2, tmp);
  for (int k = 0; k < 3; k++) { cl[k] = fmaxf(-size2[k], fminf(size2[k], cen[k])); d[k] = cen[k] - cl[k]; }
  const float dist = sqrtf(dot3(d, d));
  if (dist - r > margin) return 0;
  if (dist <= LS_MINVAL) {
    float closest = 2 * (size2[0] + size2[1] + size2[2]);
    int kk = 0;
    for (int i = 0; i < 6; i++) {
      const float f = fabsf(((i & 1) ? 1.0f : -1.0f) * size2[i >> 1] - cen[i >> 1]);
      if (closest > f) { closest = f; kk = i; }
    }
    for (int k = 0; k < 3; k++) nb[k] = (k == (kk >> 1)) ? ((kk & 1) ? 1.0f : -1.0f) : 0.0f;
    for (int k = 0; k < 3; k++) pl[k] = cen[k] + nb[k] * 0.5f * (closest - r);
    c->dist = -closest - r;
  } else {
    const float inv = 1.0f / dist;
    for (int k = 0; k < 3; k++) { nb[k] = d[k] * inv; pl[k] = cl[k] + nb[k] * 0.5f * (dist - r); }
    c->dist = dist - r;
  }
  float nw[3], pw[3];
  mulmatvec3(nw, mat2, nb);
  mulmatvec3(pw, mat2, pl);
  for (int k = 0; k < 3; k++) { c->frame[k] = -nw[k]; c->frame[3 + k] = 0; c->pos[k] = pos2[k] + pw[k]; }
  return 1;
}

LS_FN int capsule_capsule(RawCon* c, float margin, const float* pos1, const float* mat1, const float* size1,
                           const float* pos2, const float* mat2, const float* size2) {
  float a1[3] = {mat1[2], mat1[5], mat1[8]}, a2[3] = {mat2[2], mat2[5], mat2[8]};
  float dif[3] = {pos1[0] - pos2[0], pos1[1] - pos2[1], pos1[2] - pos2[2]};
  float ma = dot3(a1, a1), mb = -dot3(a1, a2), mc = dot3(a2, a2), u = -dot3(a1, dif), v = dot3(a2, dif);
  float det = ma * mc - mb * mb;
  float len1 = size1[1], len2 = size2[1];
  if (fabsf(det) >= 1e-10f) {
    float x1 = (mc * u - mb * v) / det, x2 = (ma * v - mb * u) / det;
    if (x1 > len1) { x1 = len1; x2 = (v - mb * len1) / mc; }
    else if (x1 < -len1) { x1 = -len1; x2 = (v + mb * len1) / mc; }
    if (x2 > len2) { x2 = len2; x1 = fminf(len1, fmaxf(-len1, (u - mb * len2) / ma)); }
    else if (x2 < -len2) { x2 = -len2; x1 = fminf(len1, fmaxf(-len1, (u + mb * len2) / ma)); }
    float p1[3] = {pos1[0] + a1[0] * x1, pos1[1] + a1[1] * x1, pos1[2] + a1[2] * x1};
    float p2[3] = {pos2[0] + a2[0] * x2, pos2[1] + a2[1] * x2, pos2[2] + a2[2] * x2};
    return sphere_sphere_raw(c, margin, p1, size1[0], p2, size2[0]);
  }
  int n = 0;
  for (int s = -1; s <= 1 && n < 2; s += 2) {
    float p1[3] = {pos1[0] + a1[0] * len1 * s, pos1[1] + a1[1] * len1 * s, pos1[2] + a1[2] * len1 * s};
    float vec[3] = {p1[0] - pos2[0], p1[1] - pos2[1], p1[2] - pos2[2]};
    float x2 = dot3(a2, vec);
    if (x2 > len2 || x2 < -len2) continue;
    float p2[3] = {pos2[0] + a2[0] * x2, pos2[1] + a2[1] * x2, pos2[2] + a2[2] * x2};
    n += sphere_sphere_raw(c + n, margin, p1, size1[0], p2, size2[0]);
  }
  for (int s = -1; s <= 1 && n < 2; s += 2) {
    float p2[3] = {pos2[0] + a2[0] * len2 * s, pos2[1] + a2[1] * len2 * s, pos2[2] + a2[2] * len2 * s};
    float vec[3] = {p2[0] - pos1[0], p2[1] - pos1[1], p2[2] - pos1[2]};
    float x1 = dot3(a1, vec);
    if (x1 >= len1 || x1 <= -len1) continue;
    float p1[3] = {pos1[0] + a1[0] * x1, pos1[1] + a1[1] * x1, pos1[2] + a1[2] * x1};
    n += sphere_sphere_raw(c + n, margin, p1, size1[0], p2, size2[0]);
  }
  return n;
}


// ----------------------------------------------------------------------------------------------------------
// General convex pairs (sphere | capsule | cylinder | box | mesh against cylinder | box | mesh): mjc_Convex = libccd's Minkowski Portal Refinement, restated in
// oracle/locosim_ref.c (ccd_mpr_penetration) where it is pinned by the reference goldens. Here: fp32, ONE pair at a
// time by the whole warp -- the control flow is warp-uniform, the mesh support function (argmax of dir . vertex over
// the hull vertices) is the parallel part: lanes stride over the vertices, then a warp argmax.
// fp32: CCD_EPS -> FLT_EPSILON for the sign tests, relative tests where libccd compares areas with an absolute epsilon;
// mpr_tolerance stays 1e-6 (the dot products it compares carry ~1e-8 of fp32 noise at these sizes).
// ----------------------------------------------------------------------------------------------------------
#define MPR_EPS 1.1920929e-7f
#define MPR_TOL 1e-6f
#define MPR_MAXIT 50
#if defined(LS_EMULATE)
static long g_mpr_supports = 0, g_mpr_calls = 0, g_mpr_candidates = 0, g_forward_evals = 0, g_sep_found = 0, g_sep_ok = 0, g_mpr_nohit = 0, g_obb_pass = 0;
#endif
struct MprSup { float v[3], v1[3], v2[3]; };
// world = 1: `verts` are WORLD-space points (pos + mat * vertex; the 8 corners of a box count as a mesh) staged in shared
// memory by convex_job, so a support call is a plain argmax of dir . vertex without any frame change; world = 0: analytic
// smooth geoms (sphere / capsule / cylinder) and meshes too large to stage (scanned in their own frame from global memory).
struct MprGeom { int type, vnum, world; const float* verts; float pos[3], mat[9], size[3], margin; };
LS_DEV bool mpr_is_zero(float x) { return fabsf(x) < MPR_EPS; }
LS_DEV bool mpr_eq(float a, float b) {
  float ab = fabsf(a - b);
  if (ab < MPR_EPS) return true;
  a = fabsf(a); b = fabsf(b);
  return b > a ? ab < MPR_EPS * b : ab < MPR_EPS * a;
}
LS_DEV void mpr_normalize(float* d) { const float inv = rsqrtf(dot3(d, d)); d[0] *= inv; d[1] *= inv; d[2] *= inv; }

// Per-warp MPR scratch in shared memory (it lives in the contact-Jacobian storage, free until make_constraint): the two
// geoms. The portal and every support point stay in registers; mpr_support is inlined into its callers (a lone warp's MPR
// call is pure latency: its lock-step block waits for it).
struct MprScratch { MprGeom g[2]; };

// mjccd_support of geom g (inflated by margin) in the unit world direction d, computed by the lanes [l0, l0 + nl) of the
// warp (GPU: one half-warp per geom, both geoms at once; emulation: one serial lane). All participating lanes return the
// same point. The first maximum of the vertex scan wins ties, like a serial scan.
LS_DEV void mpr_support_geom(const MprGeom& g, const float* d, float* res, int l0, int nl, unsigned mask) {
  float r[3] = {0, 0, 0};
  if (g.type == LS_GEOM_MESH || g.world) {
    float q[3] = {d[0], d[1], d[2]};
    if (!g.world) mulmatTvec3(q, g.mat, d);
    const float* v = g.verts;
    float mx = -3.0e38f;
    int best = 0x7fffffff;
#ifdef LS_EMULATE
    for (int i = 0; i < g.vnum; i++) {
      const float t = q[0] * v[3 * i] + q[1] * v[3 * i + 1] + q[2] * v[3 * i + 2];
      if (t > mx) { mx = t; best = i; }
    }
#else
    const int n = g.vnum;
    if (g.world) {                             // shared memory
#pragma unroll 2
      for (int i = LS_LANE - l0; i < n; i += nl) {
        const float t = q[0] * v[3 * i] + q[1] * v[3 * i + 1] + q[2] * v[3 * i + 2];
        if (t > mx) { mx = t; best = i; }
      }
    } else {                                   // global memory (L2): many loads in flight, the scan is pure latency
#pragma unroll 8
      for (int i = LS_LANE - l0; i < n; i += nl) {
        const float t = q[0] * __ldg(v + 3 * i) + q[1] * __ldg(v + 3 * i + 1) + q[2] * __ldg(v + 3 * i + 2);
        if (t > mx) { mx = t; best = i; }
      }
    }
    // argmax in two redux instructions: max of the order-preserving integer image of the dot product, then the smallest
    // index among the lanes that hold it. mx + 0.0f turns -0.0 into +0.0: the integer image orders -0.0 below +0.0, the
    // serial scan treats them as equal, and a maximum of 0 reached as -0.0 in one lane and +0.0 in a later one must
    // still go to the smaller index (tests/test_gpu_stages.py, check H)
    unsigned key = __float_as_uint(mx + 0.0f);
    key = (key & 0x80000000u) ? ~key : (key | 0x80000000u);
    const unsigned kmax = __reduce_max_sync(mask, key);
    best = (int)__reduce_min_sync(mask, key == kmax ? (unsigned)best : 0x7fffffffu);
#endif
    r[0] = v[3 * best]; r[1] = v[3 * best + 1]; r[2] = v[3 * best + 2];
    if (g.world) { for (int k = 0; k < 3; k++) res[k] = r[k] + d[k] * g.margin; return; }
  } else {
    float ld[3];
    mulmatTvec3(ld, g.mat, d);
    if (g.type == LS_GEOM_BOX) {
      for (int k = 0; k < 3; k++) r[k] = ld[k] >= 0 ? g.size[k] : -g.size[k];
    } else if (g.type == LS_GEOM_SPHERE) {
      for (int k = 0; k < 3; k++) r[k] = ld[k] * g.size[0];
    } else if (g.type == LS_GEOM_CAPSULE) {
      for (int k = 0; k < 3; k++) r[k] = ld[k] * g.size[0];
      r[2] += ld[2] >= 0 ? g.size[1] : -g.size[1];
    } else if (g.type == LS_GEOM_CYLINDER) {
      const float t = sqrtf(ld[0] * ld[0] + ld[1] * ld[1]);
      if (t > LS_MINVAL) { const float inv = g.size[0] / t; r[0] = ld[0] * inv; r[1] = ld[1] * inv; }
      r[2] = ld[2] >= 0 ? g.size[1] : -g.size[1];
    }
  }
  mulmatvec3(res, g.mat, r);
  for (int k = 0; k < 3; k++) res[k] += g.pos[k] + d[k] * g.margin;
}
// support point of the Minkowski difference in direction dir: v = v1 - v2
LS_DEV void mpr_support(const MprScratch* sc, const float* dir, MprSup& sp) {
#ifdef LS_EMULATE
  const float nd[3] = {-dir[0], -dir[1], -dir[2]};
  mpr_support_geom(sc->g[0], dir, sp.v1, 0, 1, 0u);
  mpr_support_geom(sc->g[1], nd, sp.v2, 0, 1, 0u);
  g_mpr_supports++;
#if defined(LS_TRACE)
  printf("    [f32] dir %.6f %.6f %.6f -> v %.7f %.7f %.7f\n", dir[0], dir[1], dir[2], sp.v1[0] - sp.v2[0], sp.v1[1] - sp.v2[1], sp.v1[2] - sp.v2[2]);
#endif
#else
  // lanes 0-15: geom 1 along +dir, lanes 16-31: geom 2 along -dir, at the same time; one shuffle round exchanges the points
  const int half = LS_LANE >> 4;
  const float sg = half ? -1.0f : 1.0f;
  const float d[3] = {sg * dir[0], sg * dir[1], sg * dir[2]};
  float r[3];
  mpr_support_geom(sc->g[half], d, r, half << 4, 16, half ? 0xffff0000u : 0x0000ffffu);
  for (int k = 0; k < 3; k++) {
    sp.v1[k] = __shfl_sync(0xffffffffu, r[k], 0);
    sp.v2[k] = __shfl_sync(0xffffffffu, r[k], 16);
  }
  if ((c_debug & 8) && LS_LANE == 0) atomicAdd(&g_dbg[1], 1ULL);
#endif
  for (int k = 0; k < 3; k++) sp.v[k] = sp.v1[k] - sp.v2[k];
}
LS_DEV void mpr_portal_dir(const MprSup* p, float* dir) {
  float a[3], b[3];
  for (int k = 0; k < 3; k++) { a[k] = p[2].v[k] - p[1].v[k]; b[k] = p[3].v[k] - p[1].v[k]; }
  cross3(dir, a, b);
  mpr_normalize(dir);
}
LS_DEV bool mpr_reach_tolerance(const MprSup* p, const MprSup& v4, const float* dir) {
  const float dv4 = dot3(v4.v, dir);
  const float d1 = fminf(fminf(dv4 - dot3(p[1].v, dir), dv4 - dot3(p[2].v, dir)), dv4 - dot3(p[3].v, dir));
  return mpr_eq(d1, MPR_TOL) || d1 < MPR_TOL;
}
LS_DEV void mpr_expand_portal(MprSup* p, const MprSup& v4) {
  float v4v0[3];
  cross3(v4v0, v4.v, p[0].v);
  if (dot3(p[1].v, v4v0) > 0) {
    if (dot3(p[2].v, v4v0) > 0) p[1] = v4; else p[3] = v4;
  } else {
    if (dot3(p[3].v, v4v0) > 0) p[2] = v4; else p[1] = v4;
  }
}
// Distance of the origin from the final portal triangle (ccdVec3PointTriDist2), once per MPR call, in DOUBLE precision on
// the fp32 portal points: the refined portal of a curved geom (cylinder rim) or of a finely tessellated hull is often a
// sliver (corner angle < 0.1 deg); wv - r^2 then cancels below fp32 resolution, the triangle would be classified as
// degenerate and the closest point taken on an edge instead of the face: penetration normals up to tens of degrees off
// (measured against the fp64 oracle on UnitreeH1's hip cylinder / mesh pairs). With the fp64 evaluation the classification
// is libccd's own (same epsilons as oracle/locosim_ref.c).
#define MPR_DEPS 2.220446049250313e-16
LS_DEV bool mprd_is_zero(double x) { return fabs(x) < MPR_DEPS; }
LS_DEV bool mprd_eq(double a, double b) {
  double ab = fabs(a - b);
  if (ab < MPR_DEPS) return true;
  a = fabs(a); b = fabs(b);
  return b > a ? ab < MPR_DEPS * b : ab < MPR_DEPS * a;
}
LS_DEV double mprd_point_seg_dist2(const double* x0, const double* b, double* wit) {      // distance of the origin
  const double d[3] = {b[0] - x0[0], b[1] - x0[1], b[2] - x0[2]};
  const double t = -(x0[0] * d[0] + x0[1] * d[1] + x0[2] * d[2]) / (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  if (t < 0 || mprd_is_zero(t)) { wit[0] = x0[0]; wit[1] = x0[1]; wit[2] = x0[2]; }
  else if (t > 1 || mprd_eq(t, 1.0)) { wit[0] = b[0]; wit[1] = b[1]; wit[2] = b[2]; }
  else for (int k = 0; k < 3; k++) wit[k] = d[k] * t + x0[k];
  return wit[0] * wit[0] + wit[1] * wit[1] + wit[2] * wit[2];
}
LS_DEV float mpr_point_tri_dist2(const float* x0f, const float* Bf, const float* Cf, float* witf) {
  double x0[3], B[3], C[3], d1[3], d2[3], wit[3];
  for (int k = 0; k < 3; k++) { x0[k] = x0f[k]; B[k] = Bf[k]; C[k] = Cf[k]; d1[k] = B[k] - x0[k]; d2[k] = C[k] - x0[k]; }
  const double v = d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2], w = d2[0] * d2[0] + d2[1] * d2[1] + d2[2] * d2[2];
  const double pp = x0[0] * d1[0] + x0[1] * d1[1] + x0[2] * d1[2], q = x0[0] * d2[0] + x0[1] * d2[1] + x0[2] * d2[2];
  const double r = d1[0] * d2[0] + d1[1] * d2[1] + d1[2] * d2[2];
  const double d = w * v - r * r;
  double s, t, dist;
  if (mprd_is_zero(d)) s = t = -1.0;
  else { s = (q * r - w * pp) / d; t = (-s * r - q) / w; }
  if ((mprd_is_zero(s) || s > 0) && (mprd_eq(s, 1.0) || s < 1) && (mprd_is_zero(t) || t > 0) && (mprd_eq(t, 1.0) || t < 1) &&
      (mprd_eq(t + s, 1.0) || t + s < 1)) {
    for (int k = 0; k < 3; k++) wit[k] = x0[k] + d1[k] * s + d2[k] * t;
    dist = wit[0] * wit[0] + wit[1] * wit[1] + wit[2] * wit[2];
  } else {
    double w2[3], dist2;
    dist = mprd_point_seg_dist2(x0, B, wit);
    dist2 = mprd_point_seg_dist2(x0, C, w2);
    if (dist2 < dist) { dist = dist2; wit[0] = w2[0]; wit[1] = w2[1]; wit[2] = w2[2]; }
    dist2 = mprd_point_seg_dist2(B, C, w2);
    if (dist2 < dist) { dist = dist2; wit[0] = w2[0]; wit[1] = w2[1]; wit[2] = w2[2]; }
  }
  // the direction is normalised in double as well (|wit| can be 1e-5: keep its relative precision), the depth returned as is
  const double n = sqrt(dist);
  if (n > 0) { witf[0] = (float)(wit[0] / n); witf[1] = (float)(wit[1] / n); witf[2] = (float)(wit[2] / n); }
  else { witf[0] = witf[1] = witf[2] = 0.0f; }
  return (float)dist;
}
LS_DEV void mpr_find_pos(const MprSup* p, float* pos) {
  float dir[3], vec[3], b[4], sum;
  mpr_portal_dir(p, dir);
  cross3(vec, p[1].v, p[2].v); b[0] = dot3(vec, p[3].v);
  cross3(vec, p[3].v, p[2].v); b[1] = dot3(vec, p[0].v);
  cross3(vec, p[0].v, p[1].v); b[2] = dot3(vec, p[3].v);
  cross3(vec, p[2].v, p[1].v); b[3] = dot3(vec, p[0].v);
  sum = b[0] + b[1] + b[2] + b[3];
  if (mpr_is_zero(sum) || sum < 0) {
    b[0] = 0;
    cross3(vec, p[2].v, p[3].v); b[1] = dot3(vec, dir);
    cross3(vec, p[3].v, p[1].v); b[2] = dot3(vec, dir);
    cross3(vec, p[1].v, p[2].v); b[3] = dot3(vec, dir);
    sum = b[1] + b[2] + b[3];
  }
  const float inv = 1.0f / sum;
  float p1[3] = {0, 0, 0}, p2[3] = {0, 0, 0};
  for (int i = 0; i < 4; i++) for (int k = 0; k < 3; k++) { p1[k] += p[i].v1[k] * b[i]; p2[k] += p[i].v2[k] * b[i]; }
  for (int k = 0; k < 3; k++) pos[k] = (p1[k] * inv + p2[k] * inv) * 0.5f;
}
// ccdMPRPenetration: true and (depth, dir, pos) if the inflated geoms intersect.
// (Tried and rejected: the same algorithm as ONE loop around ONE inlined support call, to shrink the code a lone warp has to
//  fetch - the library got 4 % smaller and every robot slower, Atlas.walk, which never calls this function, by 16 %: with
//  ~220 KB of SASS against 32 KB of instruction cache the LAYOUT of the hot functions matters more than their size.)
// returns false if the geoms do not intersect; `sep` then holds the last direction tested (a separating direction whenever
// the search stopped because a support point did not reach past the origin)
LS_FN bool mpr_penetration(const MprScratch* sc, float* depth, float* pdir, float* pos, float* sep) {
  const MprGeom& o1 = sc->g[0];
  const MprGeom& o2 = sc->g[1];
  MprSup p[4], v4;
  float dir[3], va[3], vb[3], dot;
  // ---- discoverPortal ----
  for (int k = 0; k < 3; k++) { p[0].v1[k] = o1.pos[k]; p[0].v2[k] = o2.pos[k]; p[0].v[k] = o1.pos[k] - o2.pos[k]; }
  if (mpr_eq(p[0].v[0], 0.0f) && mpr_eq(p[0].v[1], 0.0f) && mpr_eq(p[0].v[2], 0.0f)) p[0].v[0] += MPR_EPS * 10.0f;
  for (int k = 0; k < 3; k++) dir[k] = -p[0].v[k];
  mpr_normalize(dir);
  mpr_support(sc, dir, p[1]);
  dot = dot3(p[1].v, dir);
  sep[0] = dir[0]; sep[1] = dir[1]; sep[2] = dir[2];
  if (mpr_is_zero(dot) || dot < 0) return false;
  cross3(dir, p[0].v, p[1].v);
  if (!(dot3(dir, dir) > 1e-10f * dot3(p[0].v, p[0].v) * dot3(p[1].v, p[1].v))) {      // origin on the segment v0-v1 (relative test)
    for (int k = 0; k < 3; k++) { pos[k] = 0.5f * (p[1].v1[k] + p[1].v2[k]); pdir[k] = p[1].v[k]; }
    *depth = sqrtf(dot3(pdir, pdir));
    if (mpr_is_zero(*depth)) { pdir[0] = pdir[1] = pdir[2] = 0; *depth = 0; }      // touching contact: no normal
    else mpr_normalize(pdir);
    return true;
  }
  mpr_normalize(dir);
  mpr_support(sc, dir, p[2]);
  dot = dot3(p[2].v, dir);
  sep[0] = dir[0]; sep[1] = dir[1]; sep[2] = dir[2];
  if (mpr_is_zero(dot) || dot < 0) return false;
  for (int k = 0; k < 3; k++) { va[k] = p[1].v[k] - p[0].v[k]; vb[k] = p[2].v[k] - p[0].v[k]; }
  cross3(dir, va, vb);
  mpr_normalize(dir);
  if (dot3(dir, p[0].v) > 0) {
    const MprSup t = p[1]; p[1] = p[2]; p[2] = t;
    for (int k = 0; k < 3; k++) dir[k] = -dir[k];
  }
  NOUNROLL for (int guard = 0; guard < 4 * MPR_MAXIT; guard++) {
    mpr_support(sc, dir, p[3]);
    dot = dot3(p[3].v, dir);
    sep[0] = dir[0]; sep[1] = dir[1]; sep[2] = dir[2];
    if (mpr_is_zero(dot) || dot < 0) return false;
    bool cont = false;
    cross3(va, p[1].v, p[3].v);
    dot = dot3(va, p[0].v);
    if (dot < 0 && !mpr_is_zero(dot)) { p[2] = p[3]; cont = true; }
    if (!cont) {
      cross3(va, p[3].v, p[2].v);
      dot = dot3(va, p[0].v);
      if (dot < 0 && !mpr_is_zero(dot)) { p[1] = p[3]; cont = true; }
    }
    if (!cont) break;
    for (int k = 0; k < 3; k++) { va[k] = p[1].v[k] - p[0].v[k]; vb[k] = p[2].v[k] - p[0].v[k]; }
    cross3(dir, va, vb);
    mpr_normalize(dir);
  }
  // ---- refinePortal ----
  NOUNROLL for (int guard = 0;; guard++) {
    mpr_portal_dir(p, dir);
    dot = dot3(dir, p[1].v);
    if (mpr_is_zero(dot) || dot > 0) break;
    mpr_support(sc, dir, v4);
    dot = dot3(v4.v, dir);
    sep[0] = dir[0]; sep[1] = dir[1]; sep[2] = dir[2];
    if (!(mpr_is_zero(dot) || dot > 0) || mpr_reach_tolerance(p, v4, dir) || guard > 4 * MPR_MAXIT) return false;
    mpr_expand_portal(p, v4);
  }
  // ---- findPenetr ----
  NOUNROLL for (int it = 0;; it++) {
    mpr_portal_dir(p, dir);
    mpr_support(sc, dir, v4);
#if !defined(LS_EMULATE)
    if ((c_debug & 8) && LS_LANE == 0 && it > MPR_MAXIT) atomicAdd(&g_dbg[3], 1ULL);
    if ((c_debug & 8) && LS_LANE == 0 && !(dir[0] == dir[0])) atomicAdd(&g_dbg[4], 1ULL);
#endif
    if (mpr_reach_tolerance(p, v4, dir) || it > MPR_MAXIT) {
      *depth = sqrtf(mpr_point_tri_dist2(p[1].v, p[2].v, p[3].v, pdir));      // (pdir comes back normalised)
      if (mpr_is_zero(*depth)) pdir[0] = pdir[1] = pdir[2] = 0;
      mpr_find_pos(p, pos);
      return true;
    }
    mpr_expand_portal(p, v4);
  }
}

// mid-phase test for one candidate pair (see oracle/locosim_ref.c collision(): no margin in the filter); pk = pair_packed[p]
template <class C>
LS_DEV bool pair_filter(const int ms, const EnvS<C>& e, int p, int pk) {
  const DevModel& m = c_models[ms];
  const int g1 = pk & 0xfff, g2 = (pk >> 12) & 0xfff;
  const float d[3] = {e.gxpos[g2][0] - e.gxpos[g1][0], e.gxpos[g2][1] - e.gxpos[g1][1], e.gxpos[g2][2] - e.gxpos[g1][2]};
  const float bound = reinterpret_cast<const float*>(e.pk_tab + m.pk_n)[p];
  if (pk & (1 << 24)) {
    float mat1[9];
    geom_mat(ms, e, g1, mat1);
    const float n[3] = {mat1[2], mat1[5], mat1[8]};
    return dot3(d, n) <= bound;
  }
  return dot3(d, d) <= bound * bound;
}

// half extents of the geom's oriented bounding box in its own frame, inflated by mg (box / mesh: geom_size; sphere:
// r; capsule: (r, r, r + half length); cylinder: (r, r, half length))
LS_DEV void geom_halfext(int type, const float* size, float mg, float* h) {
  if (type == LS_GEOM_SPHERE) { h[0] = h[1] = h[2] = size[0] + mg; }
  else if (type == LS_GEOM_CAPSULE) { h[0] = h[1] = size[0] + mg; h[2] = size[0] + size[1] + mg; }
  else if (type == LS_GEOM_CYLINDER) { h[0] = h[1] = size[0] + mg; h[2] = size[1] + mg; }
  else { h[0] = size[0] + mg; h[1] = size[1] + mg; h[2] = size[2] + mg; }
}

// Capsule-hull test of a sphere | capsule | cylinder pair (d = pos2 - pos1; m1, m2: geom frames; s1, s2: geom_size): true
// if the geoms, each inflated by margin / 2, cannot touch. Each lies in the capsule around its axis segment (pos +- size[1]
// along the frame's z axis; a sphere's segment is its centre) of radius size[0] (a cylinder's rim is on that capsule), so
// axis segments further apart than the two radii plus the margin mean disjoint geoms, and MPR would report no contact.
// The segment distance is bounded from below in fp32 without an ill-conditioned solve: the closest points are either an
// endpoint of one segment and a point of the other (four point-segment distances: clamped projections, well conditioned),
// or interior to both, and then the distance is that of the two lines, |w . (u x v)| / |u x v|. The line distance is used
// whenever the closest points of the lines may be interior (1 mm of tolerance on their parameters). Within ~0.6 degrees
// of parallel, where fp32 cannot resolve the lines' distance, the endpoint distance less what sliding along both segments
// can gain bounds it instead. The fp32 error of every term is below 3e-6 m at these sizes; the 1e-5 m of slack is ten
// times MPR's tolerance.
LS_DEV float point_seg_dist2(const float* p, const float* u, float h) {
  const float uu = dot3(u, u), t = fminf(fmaxf(dot3(p, u) / uu, -h), h);
  const float q[3] = {p[0] - t * u[0], p[1] - t * u[1], p[2] - t * u[2]};
  return dot3(q, q);
}
LS_DEV bool capsule_hulls_apart(const float* d, const float* m1, int t1, const float* s1, const float* m2, int t2,
                                const float* s2, float margin) {
  const float h1 = t1 == LS_GEOM_SPHERE ? 0.0f : s1[1], h2 = t2 == LS_GEOM_SPHERE ? 0.0f : s2[1];
  const float u[3] = {m1[2], m1[5], m1[8]}, v[3] = {m2[2], m2[5], m2[8]};
  // endpoints of each segment against the other (relative to the other segment's centre)
  float p[3] = {-d[0] + h1 * u[0], -d[1] + h1 * u[1], -d[2] + h1 * u[2]};       // pos1 + h1 u - pos2
  float dist2 = point_seg_dist2(p, v, h2);
  for (int k = 0; k < 3; k++) p[k] = -d[k] - h1 * u[k];
  dist2 = fminf(dist2, point_seg_dist2(p, v, h2));
  for (int k = 0; k < 3; k++) p[k] = d[k] + h2 * v[k];                            // pos2 + h2 v - pos1
  dist2 = fminf(dist2, point_seg_dist2(p, u, h1));
  for (int k = 0; k < 3; k++) p[k] = d[k] - h2 * v[k];
  dist2 = fminf(dist2, point_seg_dist2(p, u, h1));
  if (h1 > 0 && h2 > 0) {
    // closest points of the lines pos1 + s u, pos2 + t v; w = pos1 - pos2
    const float a = dot3(u, u), e = dot3(v, v), b = dot3(u, v), c = -dot3(u, d), f = -dot3(v, d);
    float n[3];
    cross3(n, u, v);
    const float nn = dot3(n, n);
    if (nn < 1e-4f * a * e) {
      // nearly parallel: from interior closest points, slide both parameters alike (t against s if the axes are
      // antiparallel) until one reaches an endpoint: the distance grows by at most that slide times |u -+ v|
      const float sg = b >= 0 ? 1.0f : -1.0f, w[3] = {u[0] - sg * v[0], u[1] - sg * v[1], u[2] - sg * v[2]};
      const float lb = fmaxf(sqrtf(dist2) - 2.0f * fmaxf(h1, h2) * sqrtf(dot3(w, w)), 0.0f);
      dist2 = lb * lb;
    } else {
      const float den = a * e - b * b, s = (b * f - c * e) / den, t = (a * f - b * c) / den;
      if (fabsf(s) <= h1 + 1e-3f && fabsf(t) <= h2 + 1e-3f) {
        const float wn = dot3(d, n);
        dist2 = fminf(dist2, wn * wn / nn);
      }
    }
  }
  const float rr = s1[0] + s2[0] + margin + 1e-5f;
  return dist2 > rr * rr;
}

// second filter of a general convex pair that passed the bounding spheres
template <class C>
LS_FN bool convex_obb_filter(const int ms, const EnvS<C>& e, int p) {
  const DevModel& m = c_models[ms];
  const int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1];
  const float d[3] = {e.gxpos[g2][0] - e.gxpos[g1][0], e.gxpos[g2][1] - e.gxpos[g1][1], e.gxpos[g2][2] - e.gxpos[g1][2]};
#if defined(LS_EMULATE)
  g_mpr_candidates++;
#endif
  // Convex pair (box | mesh vs mesh): MPR reports a contact only if the (margin-inflated) geoms intersect. Their oriented
  // boxes (geom_size = the mesh's AABB in its own principal frame) contain them, so disjoint boxes mean no contact:
  // 15-axis separating-axis test of the two boxes (conservative prefilter: it never rejects an intersecting pair;
  // measured on the humanoid: of ~60 bone pairs per evaluation that pass the bounding spheres, 1.2 survive).
  float RA[9], RB[9];
  geom_mat(ms, e, g1, RA);
  geom_mat(ms, e, g2, RB);
  const float mg = 0.5f * fmaxf(m.geom_margin[g1], m.geom_margin[g2]) + 1e-6f;
  float a[3], b[3];
  geom_halfext(m.geom_type[g1], m.geom_size + 3 * g1, mg, a);
  geom_halfext(m.geom_type[g2], m.geom_size + 3 * g2, mg, b);
  float R[3][3], AR[3][3], t[3];
  for (int i = 0; i < 3; i++) {
    t[i] = RA[i] * d[0] + RA[3 + i] * d[1] + RA[6 + i] * d[2];                     // d in A's frame
    for (int j = 0; j < 3; j++) {
      R[i][j] = RA[i] * RB[j] + RA[3 + i] * RB[3 + j] + RA[6 + i] * RB[6 + j];     // A_i . B_j
      AR[i][j] = fabsf(R[i][j]) + 1e-6f;
    }
  }
  for (int i = 0; i < 3; i++)
    if (fabsf(t[i]) > a[i] + b[0] * AR[i][0] + b[1] * AR[i][1] + b[2] * AR[i][2]) return false;
  for (int j = 0; j < 3; j++)
    if (fabsf(t[0] * R[0][j] + t[1] * R[1][j] + t[2] * R[2][j]) > b[j] + a[0] * AR[0][j] + a[1] * AR[1][j] + a[2] * AR[2][j])
      return false;
  for (int i = 0; i < 3; i++) {
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;
    for (int j = 0; j < 3; j++) {
      const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      const float ra = a[i1] * AR[i2][j] + a[i2] * AR[i1][j], rb = b[j1] * AR[i][j2] + b[j2] * AR[i][j1];
      if (fabsf(t[i2] * R[i1][j] - t[i1] * R[i2][j]) > ra + rb) return false;
    }
  }
  return true;
}

// Third filter of a box-test survivor with pair flag 4 (sphere | capsule | cylinder vs cylinder, locosim_host.h): a box
// bounds a thin cylinder poorly next to a slanted capsule, and without this test such near misses each cost a job
// (UnitreeA1: the front hips' cylinders against the front legs). Rejecting a pair only skips MPR, which would not have
// reported a contact for it; its separating-direction cache entry (which, too, only ever skips MPR) is not refreshed.
// A stage of its own, called only for flagged pairs: models without them run the box test's code as before.
template <class C>
LS_FN bool convex_hull_filter(const int ms, const EnvS<C>& e, int p) {
  const DevModel& m = c_models[ms];
  const int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1];
  const float d[3] = {e.gxpos[g2][0] - e.gxpos[g1][0], e.gxpos[g2][1] - e.gxpos[g1][1], e.gxpos[g2][2] - e.gxpos[g1][2]};
  float RA[9], RB[9];
  geom_mat(ms, e, g1, RA);
  geom_mat(ms, e, g2, RB);
  return !capsule_hulls_apart(d, RA, m.geom_type[g1], m.geom_size + 3 * g1, RB, m.geom_type[g2], m.geom_size + 3 * g2,
                              fmaxf(m.geom_margin[g1], m.geom_margin[g2]));
}

// contact parameters (mj_contactParam), frame completion (mju_makeFrame) and storage of one raw contact
// inclusion distance of a contact of the pair (margin - gap): raw contacts with dist >= incl never enter the constraint set
LS_DEV float pair_incl(const DevModel& m, int g1, int g2, float margin) {
  return margin - fmaxf(m.geom_gap[g1], m.geom_gap[g2]);
}

// fill contact slot ci from a raw narrow-phase result: parameter mixing (mj_contactParam), impedance, frame
template <class C>
LS_FN void fill_contact(const int ms, EnvS<C>& e, const int ci, int g1, int g2, float incl, const RawCon* raw) {
  const DevModel& m = c_models[ms];
  {
    // contact parameters (mj_contactParam)
    int p1 = m.geom_priority[g1], p2 = m.geom_priority[g2];
    float fri[3], solref[2], solimp[5];
    if (p1 != p2) {
      int g = p1 > p2 ? g1 : g2;
      e.con_dim[ci] = m.geom_condim[g];
      for (int c = 0; c < 2; c++) solref[c] = m.geom_solref[2 * g + c];
      for (int c = 0; c < 5; c++) solimp[c] = m.geom_solimp[5 * g + c];
      for (int c = 0; c < 3; c++) fri[c] = PRM(geom_friction)[3 * g + c];
    } else {
      e.con_dim[ci] = m.geom_condim[g1] > m.geom_condim[g2] ? m.geom_condim[g1] : m.geom_condim[g2];
      float s1 = m.geom_solmix[g1], s2 = m.geom_solmix[g2], mix;
      if (s1 >= LS_MINVAL && s2 >= LS_MINVAL) mix = s1 / (s1 + s2);
      else if (s1 < LS_MINVAL && s2 < LS_MINVAL) mix = 0.5f;
      else if (s1 < LS_MINVAL) mix = 0.0f;
      else mix = 1.0f;
      const float *r1 = m.geom_solref + 2 * g1, *r2 = m.geom_solref + 2 * g2;
      if (r1[0] > 0 && r2[0] > 0) for (int c = 0; c < 2; c++) solref[c] = mix * r1[c] + (1 - mix) * r2[c];
      else for (int c = 0; c < 2; c++) solref[c] = fminf(r1[c], r2[c]);
      for (int c = 0; c < 5; c++) solimp[c] = mix * m.geom_solimp[5 * g1 + c] + (1 - mix) * m.geom_solimp[5 * g2 + c];
      for (int c = 0; c < 3; c++) fri[c] = fmaxf(PRM(geom_friction)[3 * g1 + c], PRM(geom_friction)[3 * g2 + c]);
    }
    impedance_KB(solref, solimp, raw->dist, incl, m.timestep, &e.con_imp[ci], &e.con_K[ci], &e.con_B[ci]);
    e.con_fri[ci][0] = fri[0]; e.con_fri[ci][1] = fri[0]; e.con_fri[ci][2] = fri[1]; e.con_fri[ci][3] = fri[2];
    e.con_fri[ci][4] = fri[2];
    e.con_incl[ci] = incl;
    e.con_dist[ci] = raw->dist;
    e.con_g1[ci] = g1; e.con_g2[ci] = g2;
    for (int c = 0; c < 3; c++) e.con_pos[ci][c] = raw->pos[c];
    // mju_makeFrame
    float f[9];
    for (int c = 0; c < 6; c++) f[c] = raw->frame[c];
    normalize3(f);
    if (dot3(f + 3, f + 3) < 0.25f) {
      f[3] = f[4] = f[5] = 0;
      if (f[1] < 0.5f && f[1] > -0.5f) f[4] = 1; else f[5] = 1;
    }
    float t = dot3(f, f + 3);
    for (int c = 0; c < 3; c++) f[3 + c] -= t * f[c];
    normalize3(f + 3);
    cross3(f + 6, f, f + 3);
    for (int c = 0; c < 9; c++) e.con_frame[ci][c] = f[c];
  }
}

// mjc_BoxBox, edge-edge branch (restated and pinned in oracle/locosim_ref.c box_box_edge: the reference golden
// HumanoidTorque4Ages.run.all): when the separating axis of least overlap is the cross product of an edge of each box, the
// contact is the midpoint of the closest points of those two edges. Returns 1 (contact in r[0..6]: dist, pos, normal),
// 0 (separated by more than the margin) or -1 (a face axis separates best, or a vertex is involved: caller falls back to MPR).
// Every lane computes the same thing (a few hundred flops, box-box pairs are rare: the humanoids' two feet).
LS_DEV int box_box_edge(float margin, const float* p1, const float* m1, const float* s1, const float* p2, const float* m2,
                        const float* s2, float* r) {
  float A[3][3], B[3][3];
  const float d[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  for (int i = 0; i < 3; i++) for (int k = 0; k < 3; k++) { A[i][k] = m1[3 * k + i]; B[i][k] = m2[3 * k + i]; }
  float best = -3.0e38f, bn[3] = {0, 0, 0};
  int bi = -1, bj = -1;
  for (int f = 0; f < 6; f++) {
    const float* ax = f < 3 ? A[f] : B[f - 3];
    float ra = 0, rb = 0;
    for (int i = 0; i < 3; i++) { ra += s1[i] * fabsf(dot3(A[i], ax)); rb += s2[i] * fabsf(dot3(B[i], ax)); }
    const float sep = fabsf(dot3(d, ax)) - ra - rb;
    if (sep > best) { best = sep; bi = -1; bj = f; }
  }
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    float ax[3];
    cross3(ax, A[i], B[j]);
    const float l2 = dot3(ax, ax);
    if (l2 < 1e-12f) continue;
    const float il = rsqrtf(l2);
    for (int k = 0; k < 3; k++) ax[k] *= il;
    float ra = 0, rb = 0;
    for (int k = 0; k < 3; k++) { ra += s1[k] * fabsf(dot3(A[k], ax)); rb += s2[k] * fabsf(dot3(B[k], ax)); }
    const float sd = dot3(d, ax), sep = fabsf(sd) - ra - rb;
    if (sep > best + 1e-7f) { best = sep; bi = i; bj = j; for (int k = 0; k < 3; k++) bn[k] = sd >= 0 ? ax[k] : -ax[k]; }
  }
  if (bi < 0) return -1;
  if (best > margin) return 0;
  float e1[3] = {p1[0], p1[1], p1[2]}, e2[3] = {p2[0], p2[1], p2[2]};
  for (int i = 0; i < 3; i++) if (i != bi) { const float sg = dot3(A[i], bn) >= 0 ? s1[i] : -s1[i]; for (int k = 0; k < 3; k++) e1[k] += sg * A[i][k]; }
  for (int j = 0; j < 3; j++) if (j != bj) { const float sg = dot3(B[j], bn) >= 0 ? -s2[j] : s2[j]; for (int k = 0; k < 3; k++) e2[k] += sg * B[j][k]; }
  const float rr[3] = {e1[0] - e2[0], e1[1] - e2[1], e1[2] - e2[2]};
  const float b = dot3(A[bi], B[bj]), cc = dot3(A[bi], rr), f = dot3(B[bj], rr), den = 1.0f - b * b;
  const float t = (b * f - cc) / den, u = (f - b * cc) / den;
  if (fabsf(t) > s1[bi] || fabsf(u) > s2[bj]) return -1;
  r[0] = best;
  for (int k = 0; k < 3; k++) { r[1 + k] = 0.5f * ((e1[k] + t * A[bi][k]) + (e2[k] + u * B[bj][k])); r[4 + k] = bn[k]; }
  return 1;
}

// warp-cooperative narrow phase of one convex pair (mjc_Convex): at most one contact.
// The pair belongs to env `o` (geom frames, separating-direction cache: read only); the executing warp's own env `e` only
// lends its contact-Jacobian storage as scratch. On the GPU the warps of a block SHARE these jobs (collision()): a lone
// warp running several MPR calls while its lock-step block waits was the largest cost of the bone-bone pairs.
// Result record res[8]: res[7] = 0 nothing to do (the cached direction still separates the pair, no MPR run),
//                                1 contact: res[0] dist, res[1..3] position, res[4..6] normal,
//                                2 MPR ran, no contact; res[1..3] = the last direction tested (refreshes o's cache),
//                                3 MPR ran, touching contact without a normal (ignored).
#define LS_MAXJOB 32
#define LS_MAXCONPAIR 50     // mjMAXCONPAIR: contacts of one pair (the terrain pass; every other routine returns at most 4)
#define LS_CAND_HULL(pk) (((pk) >> 11) & 0x8000)     // pair flag 4 (bit 26 of pair_packed) as bit 15 of a candidate entry
template <class C>
LS_FN void convex_job(const int ms, const EnvS<C>& o, EnvS<C>& e, int p, float* res) {
  const DevModel& m = c_models[ms];
  const int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1];
  const float margin = fmaxf(m.geom_margin[g1], m.geom_margin[g2]);
  // scratch + staged vertices live in the contact-Jacobian storage (nobody uses it before make_constraint)
  constexpr int SCR = (int)((sizeof(MprScratch) + 15) / 16 * 4);                  // floats taken by the scratch block
  MprScratch* sc = reinterpret_cast<MprScratch*>(&e.J[0][0]);
  float* buf = &e.J[0][0] + SCR;
  const int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
  // vertex sets: a mesh's hull vertices, a box's 8 corners (corner 0 = (+,+,+): ties resolve like sign(0) = +)
  const int n1 = t1 == LS_GEOM_MESH ? m.geom_meshnum[g1] : (t1 == LS_GEOM_BOX ? 8 : 0);
  const int n2 = t2 == LS_GEOM_MESH ? m.geom_meshnum[g2] : (t2 == LS_GEOM_BOX ? 8 : 0);
  const float* s1 = m.mesh_vert + 3 * m.geom_meshadr[g1];
  const float* s2 = m.mesh_vert + 3 * m.geom_meshadr[g2];
  // An MPR call scans the two vertex sets ~10 times each: whenever they fit (~400 vertices) the vertices of both geoms are
  // written ONCE, already in world coordinates, into shared memory (all loads in flight, parallel over the vertices), so
  // the support calls on the serial critical path are a bare argmax; larger pairs scan global memory in the mesh frame.
  const bool staged = 3 * (n1 + n2) <= EnvS<C>::MAXROW * EnvS<C>::JS - SCR;
  float m1[9], m2[9];
  geom_mat(ms, o, g1, m1);
  geom_mat(ms, o, g2, m2);
  LANE0 {                                      // descriptors first WITHOUT staged vertices (frame-local supports)
    MprGeom& a = sc->g[0];
    MprGeom& b = sc->g[1];
    a.type = t1; a.vnum = n1; a.margin = 0.5f * margin; a.world = 0; a.verts = s1;
    b.type = t2; b.vnum = n2; b.margin = 0.5f * margin; b.world = 0; b.verts = s2;
    for (int k = 0; k < 3; k++) {
      a.pos[k] = o.gxpos[g1][k]; b.pos[k] = o.gxpos[g2][k];
      a.size[k] = m.geom_size[3 * g1 + k]; b.size[k] = m.geom_size[3 * g2 + k];
    }
    for (int k = 0; k < 9; k++) { a.mat[k] = m1[k]; b.mat[k] = m2[k]; }
  }
  SYNC();
  if (C::BOXBOX && t1 == LS_GEOM_BOX && t2 == LS_GEOM_BOX) {        // mjc_BoxBox: the edge-edge branch is exact, the rest falls through to MPR
    float rb[7] = {0, 0, 0, 0, 0, 0, 0};
    const int nb = box_box_edge(margin, o.gxpos[g1], m1, m.geom_size + 3 * g1, o.gxpos[g2], m2, m.geom_size + 3 * g2, rb);
    if (nb >= 0) {
      LANE0 { for (int k = 0; k < 7; k++) res[k] = rb[k]; res[7] = nb > 0 ? 1.0f : 3.0f; }      // (3: nothing to record)
      return;
    }
  }
  float depth, dir[3], pos[3], sep[3] = {0, 0, 0};
  // A direction that separated this pair in an earlier evaluation of the control step is tried first (ONE support pair,
  // straight from the model's vertex arrays: nothing is staged for it; strict separation of the inflated geoms along it
  // means MPR would not report a contact either); if it fails the full MPR runs and its last test direction refreshes the
  // cache (applied by the owner, in job order).
  int slot = -1;
  for (int k = 0; k < EnvS<C>::NSEP; k++) if (o.sep_pair[k] == p) slot = k;
  float code = 0.0f, r[7] = {0, 0, 0, 0, 0, 0, 0};
  bool run = true;
  if (slot >= 0 && !(c_debug & 16)) {
    MprSup sp;
    const float cd[3] = {o.sep_dir[slot][0], o.sep_dir[slot][1], o.sep_dir[slot][2]};
    mpr_support(sc, cd, sp);
    if (dot3(sp.v, cd) < -1e-7f) run = false;
  }
  SYNC();                                      // (every lane is done reading the descriptors before lane 0 rewrites them)
  if (run && staged) {
    PAR_FOR4(i, n1 + n2) {
      const bool second = i >= n1;
      const int j = second ? i - n1 : i;
      const int ty = second ? t2 : t1;
      const float* mm = second ? m2 : m1;
      const float* gp = second ? o.gxpos[g2] : o.gxpos[g1];
      float v[3];
      if (ty == LS_GEOM_MESH) { const float* sv = (second ? s2 : s1) + 3 * j; v[0] = sv[0]; v[1] = sv[1]; v[2] = sv[2]; }
      else {
        const float* sz = m.geom_size + 3 * (second ? g2 : g1);
        v[0] = (j & 1) ? -sz[0] : sz[0]; v[1] = (j & 2) ? -sz[1] : sz[1]; v[2] = (j & 4) ? -sz[2] : sz[2];
      }
      float w[3];
      mulmatvec3(w, mm, v);
      buf[3 * i] = w[0] + gp[0]; buf[3 * i + 1] = w[1] + gp[1]; buf[3 * i + 2] = w[2] + gp[2];
    }
    LANE0 {
      if (n1 > 0) { sc->g[0].world = 1; sc->g[0].verts = buf; }
      if (n2 > 0) { sc->g[1].world = 1; sc->g[1].verts = buf + 3 * n1; }
    }
    SYNC();
  }
  if (run) {
#if defined(LS_EMULATE)
    g_mpr_calls++;
    const long sup0_ = g_mpr_supports;
#else
    if ((c_debug & 8) && LS_LANE == 0) atomicAdd(&g_dbg[0], 1ULL);
#endif
    const bool hit_ = mpr_penetration(sc, &depth, dir, pos, sep);
#if defined(LS_EMULATE) && defined(LS_MPRLOG)
    printf("MPR %d %d %d %d %ld %d\n", g1, g2, n1 / 3, n2 / 3, g_mpr_supports - sup0_, (int)hit_);
#endif
    if (!hit_) { code = 2.0f; r[1] = sep[0]; r[2] = sep[1]; r[3] = sep[2]; }
    else if (dir[0] == 0.0f && dir[1] == 0.0f && dir[2] == 0.0f) code = 3.0f;      // contact found but normal undefined
    else {
      code = 1.0f; r[0] = margin - depth;
      for (int k = 0; k < 3; k++) { r[1 + k] = pos[k]; r[4 + k] = dir[k]; }
    }
  }
  SYNC();                                      // (the scratch is free for the next job of this warp)
  LANE0 { for (int k = 0; k < 7; k++) res[k] = r[k]; res[7] = code; }
}

// owner side of a finished convex job: contact into the list, or the separating direction into the cache
template <class C>
LS_FN void convex_consume(const int ms, EnvS<C>& e, int p, const float* res) {
  const DevModel& m = c_models[ms];
  const int code = (int)res[7];
  if (code == 0) return;
  LANE0 { e.mpr_calls += 1; }
  if (code == 2) {
    int slot = -1;
    for (int k = 0; k < EnvS<C>::NSEP; k++) if (e.sep_pair[k] == p) slot = k;
    if (slot < 0) slot = e.sep_next & (EnvS<C>::NSEP - 1);
    SYNC();
    LANE0 {
      if (e.sep_pair[slot] != p) e.sep_next = e.sep_next + 1;
      e.sep_pair[slot] = p; e.sep_dir[slot][0] = res[1]; e.sep_dir[slot][1] = res[2]; e.sep_dir[slot][2] = res[3];
    }
    SYNC();
    return;
  }
  if (code != 1) return;
  const int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1];
  const float incl = pair_incl(m, g1, g2, fmaxf(m.geom_margin[g1], m.geom_margin[g2]));
  const int ci = e.ncon;
  if (res[0] < incl && ci < EnvS<C>::MAXCON) {
    LANE0 {
      RawCon rc;
      rc.dist = res[0];
      for (int k = 0; k < 3; k++) { rc.pos[k] = res[1 + k]; rc.frame[k] = res[4 + k]; rc.frame[3 + k] = 0; }
      fill_contact(ms, e, ci, g1, g2, incl, &rc);
      e.ncon = ci + 1;
    }
    SYNC();
  }
}

// narrow phase of pair p: up to 4 raw contacts (one lane per pair)
template <class C>
LS_FN int pair_narrow(const int ms, EnvS<C>& e, int p, RawCon* raw, int* g1_out, int* g2_out, float* margin_out) {
  const DevModel& m = c_models[ms];
  int g1 = m.pair_geom[2 * p], g2 = m.pair_geom[2 * p + 1];
  int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
  float margin = fmaxf(m.geom_margin[g1], m.geom_margin[g2]);
  const float *pos1 = e.gxpos[g1], *pos2 = e.gxpos[g2];
  const float *size1 = m.geom_size + 3 * g1, *size2 = m.geom_size + 3 * g2;
  float mat1[9], mat2[9];
  geom_mat(ms, e, g1, mat1);
  geom_mat(ms, e, g2, mat2);
  int n = 0;
  if (t1 == LS_GEOM_PLANE) {
    float nrm[3] = {mat1[2], mat1[5], mat1[8]};
    if (t2 == LS_GEOM_SPHERE) n = plane_sphere(raw, margin, pos1, nrm, pos2, size2[0]);
    else if (t2 == LS_GEOM_CAPSULE) n = plane_capsule(raw, margin, pos1, nrm, pos2, mat2, size2);
    else if (t2 == LS_GEOM_CYLINDER) n = plane_cylinder(raw, margin, pos1, nrm, pos2, mat2, size2);
    else if (t2 == LS_GEOM_BOX) n = plane_box(raw, margin, pos1, nrm, pos2, mat2, size2);
    else if (t2 == LS_GEOM_MESH)
      n = plane_mesh(raw, margin, pos1, nrm, pos2, mat2, m.mesh_vert + 3 * m.geom_meshadr[g2], m.geom_meshnum[g2],
                     m.geom_rbound[g2]);
  } else if (t1 == LS_GEOM_SPHERE && t2 == LS_GEOM_SPHERE) {
    n = sphere_sphere_raw(raw, margin, pos1, size1[0], pos2, size2[0]);
  } else if (t1 == LS_GEOM_SPHERE && t2 == LS_GEOM_CAPSULE) {
    n = sphere_capsule(raw, margin, pos1, size1[0], pos2, mat2, size2);
  } else if (t1 == LS_GEOM_CAPSULE && t2 == LS_GEOM_CAPSULE) {
    n = capsule_capsule(raw, margin, pos1, mat1, size1, pos2, mat2, size2);
  } else if (t1 == LS_GEOM_SPHERE && t2 == LS_GEOM_BOX) {
    n = sphere_box(raw, margin, pos1, size1[0], pos2, mat2, size2);
  }
  *g1_out = g1; *g2_out = g2; *margin_out = margin;
  return n;
}

#ifdef LOCOSIM_TERRAIN
// ---- mjc_ConvexHField: the pairs (terrain, g), after every other pair (include/locosim.h states the semantics) ----
// Prism k of a cell range with nc columns: row r = k / (2 nc), column c, triangle tri = k % 2 (row, column, triangle order).
// Its vertices (the strip order of MuJoCo's prism builder): triangle 0 = grid points (c, r), (c, r+1), (c+1, r); triangle
// 1 = (c, r+1), (c+1, r), (c+1, r+1); the diagonal runs from (c+1, r) to (c, r+1). Vertex order: the three bottom points
// (z = -base) first, then the three top points, each in that order (the support scan's first maximum wins: the same
// vertex order in tests/csrc/terrain_ref.c).
LS_DEV void terrain_prism(const DevTerrain& t, const int r, const int c, const int tri, float (*v)[3]) {
  const int rr[3] = {tri ? r + 1 : r, tri ? r : r + 1, tri ? r + 1 : r};
  const int c0[3] = {c, tri ? c + 1 : c, c + 1};
  const float dx = 2.0f * t.size[0] / (float)(t.ncol - 1), dy = 2.0f * t.size[1] / (float)(t.nrow - 1);
  for (int i = 0; i < 3; i++) {
    const float x = dx * (float)c0[i] - t.size[0], y = dy * (float)rr[i] - t.size[1];
    v[i][0] = v[3 + i][0] = x;
    v[i][1] = v[3 + i][1] = y;
    v[i][2] = -t.size[3];
    v[3 + i][2] = LS_LDG(t.data + rr[i] * t.ncol + c0[i]) * t.size[2];
  }
}
// half extent of a geom's support along the unit axis k of its frame's parent (closed form for sphere / capsule / cylinder
// / box, all symmetric about their centre)
LS_DEV float terrain_extent(const int type, const float* mat, const float* size, const int k) {
  const float a = fabsf(mat[3 * k + 2]);
  if (type == LS_GEOM_SPHERE) return size[0];
  if (type == LS_GEOM_CAPSULE) return size[0] + size[1] * a;
  if (type == LS_GEOM_CYLINDER) return size[0] * sqrtf(fmaxf(1.0f - a * a, 0.0f)) + size[1] * a;
  return fabsf(mat[3 * k]) * size[0] + fabsf(mat[3 * k + 1]) * size[1] + a * size[2];
}
template <class C>
LS_FN void terrain_pass(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  const DevTerrain& t = c_terrain[ms];
  constexpr int SCR = (int)((sizeof(MprScratch) + 15) / 16 * 4);
  MprScratch* sc = reinterpret_cast<MprScratch*>(&e.J[0][0]);      // (convex_job's scratch: free until make_constraint)
  float* buf = &e.J[0][0] + SCR;
  // the field's frame in the world: its geom position moved by -origin[env]
  float f[3] = {t.pos[0], t.pos[1], t.pos[2]};
  // (e.env < 0: a dataset row of locosim_create_dataset_inverse, which is not an env: the zero origin)
  if (t.origin && e.env >= 0) { f[0] -= LS_LDG(t.origin + 2 * e.env); f[1] -= LS_LDG(t.origin + 2 * e.env + 1); }
  const float dx = 2.0f * t.size[0] / (float)(t.ncol - 1), dy = 2.0f * t.size[1] / (float)(t.nrow - 1);
  NOUNROLL for (int q = 0; q < t.npair; q++) {
    if (e.ncon >= EnvS<C>::MAXCON) break;
    const int g1 = t.geom, g2 = m.pair_geom[2 * (t.p0 + q) + 1];
    const int t2 = m.geom_type[g2];
    const float margin = fmaxf(m.geom_margin[g1], m.geom_margin[g2]);
    float mat[9];
    geom_mat(ms, e, g2, mat);
    const float* sz = m.geom_size + 3 * g2;
    const float p[3] = {e.gxpos[g2][0] - f[0], e.gxpos[g2][1] - f[1], e.gxpos[g2][2] - f[2]};
    if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) continue;      // (no cell range for a non-finite pose)
    const float hx = terrain_extent(t2, mat, sz, 0), hy = terrain_extent(t2, mat, sz, 1), hz = terrain_extent(t2, mat, sz, 2);
    const float zmin = p[2] - hz;
    if (p[0] - hx - margin > t.size[0] || p[0] + hx + margin < -t.size[0] || p[1] - hy - margin > t.size[1] ||
        p[1] + hy + margin < -t.size[1] || zmin - margin > t.size[2] || p[2] + hz + margin < -t.size[3])
      continue;
    // cell range of the box (floor / ceil of the grid coordinates, clamped to the grid)
    int cmin = (int)floorf((p[0] - hx - margin + t.size[0]) / dx), cmax = (int)ceilf((p[0] + hx + margin + t.size[0]) / dx);
    int rmin = (int)floorf((p[1] - hy - margin + t.size[1]) / dy), rmax = (int)ceilf((p[1] + hy + margin + t.size[1]) / dy);
    cmin = cmin < 0 ? 0 : cmin; rmin = rmin < 0 ? 0 : rmin;
    cmax = cmax > t.ncol - 1 ? t.ncol - 1 : cmax; rmax = rmax > t.nrow - 1 ? t.nrow - 1 : rmax;
    const int nc = cmax - cmin, nprism = 2 * nc * (rmax - rmin);
    const float incl = pair_incl(m, g1, g2, margin);
    int cnt = 0;
    NOUNROLL for (int base = 0; base < nprism && cnt < LS_MAXCONPAIR; base += 32) {
      // the lanes test 32 prisms at once (all three top points below the geom's lowest point: skipped), the warp then runs
      // MPR on the rest in order
#ifdef LS_EMULATE
      unsigned live = 0;
      for (int l = 0; l < 32 && base + l < nprism; l++) {
        const int k = base + l, r = rmin + k / (2 * nc), c = cmin + (k % (2 * nc)) / 2;
        float v[6][3];
        terrain_prism(t, r, c, k & 1, v);
        if (!(v[3][2] < zmin - margin && v[4][2] < zmin - margin && v[5][2] < zmin - margin)) live |= 1u << l;
      }
#else
      bool ok = false;
      {
        const int k = base + LS_LANE;
        if (k < nprism) {
          const int r = rmin + k / (2 * nc), c = cmin + (k % (2 * nc)) / 2;
          float v[6][3];
          terrain_prism(t, r, c, k & 1, v);
          ok = !(v[3][2] < zmin - margin && v[4][2] < zmin - margin && v[5][2] < zmin - margin);
        }
      }
      unsigned live = __ballot_sync(0xffffffffu, ok);
#endif
      while (live && cnt < LS_MAXCONPAIR && e.ncon < EnvS<C>::MAXCON) {
        const int l = LS_FFS(live) - 1;
        live &= live - 1;
        const int k = base + l, r = rmin + k / (2 * nc), c = cmin + (k % (2 * nc)) / 2;
        LANE0 {
          float v[6][3], cen[3] = {0, 0, 0};
          terrain_prism(t, r, c, k & 1, v);
          for (int i = 0; i < 6; i++)
            for (int j = 0; j < 3; j++) { buf[3 * i + j] = v[i][j] + f[j]; cen[j] += v[i][j]; }
          MprGeom& a = sc->g[0];
          MprGeom& b = sc->g[1];
          a.type = LS_GEOM_MESH; a.vnum = 6; a.world = 1; a.verts = buf; a.margin = 0.5f * margin;
          b.type = t2; b.vnum = 0; b.world = 0; b.verts = nullptr; b.margin = 0.5f * margin;
          for (int j = 0; j < 3; j++) {
            a.pos[j] = cen[j] * (1.0f / 6.0f) + f[j];
            b.pos[j] = e.gxpos[g2][j];
            b.size[j] = sz[j];
          }
          for (int j = 0; j < 9; j++) b.mat[j] = mat[j];
        }
        SYNC();
        float depth, dir[3], pos[3], sep[3];
        const bool hit = mpr_penetration(sc, &depth, dir, pos, sep);
        SYNC();
        LANE0 { e.mpr_calls += 1; }
#if defined(LS_EMULATE)
        g_mpr_calls++;
#endif
        if (hit && !(dir[0] == 0.0f && dir[1] == 0.0f && dir[2] == 0.0f)) {
          cnt++;
          const float dist = margin - depth;
          if (dist < incl) {
            LANE0 {
              RawCon rc;
              rc.dist = dist;
              for (int j = 0; j < 3; j++) { rc.pos[j] = pos[j]; rc.frame[j] = dir[j]; rc.frame[3 + j] = 0; }
              fill_contact(ms, e, e.ncon, g1, g2, incl, &rc);
              e.ncon = e.ncon + 1;
            }
            SYNC();
          }
        }
      }
    }
  }
}
#endif

template <class C>
LS_FN void collision(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  LANE0 { e.ncon = 0; }
  SYNC();
  // Convex pairs (box | mesh vs mesh, mjc_Convex) that pass the bounding spheres are only COLLECTED in the pair loop
  // (compacted list in the constraint-row storage, which is free until make_constraint) and handled afterwards: the
  // oriented-box test runs on the compacted list (full lanes instead of a few lanes in every round of 32 pairs), the
  // survivors become JOBS (one warp-cooperative MPR each) that the warps of the block share, and every env then consumes
  // the results of its own jobs in pair order. Their contacts therefore FOLLOW the primitive contacts in the list (ordered
  // by pair among themselves); the order of constraint rows has no influence on the solution.
  // Layout of the 5 * MAXEFC floats: [results: LS_MAXJOB x 8 floats][candidate / job list: unsigned short ...].
  float* jobres = e.r_D;
  // (C::HULL: candidate entries carry pair flag 4 in bit 15 until the box test; job entries are plain pair indices)
  unsigned short* cand = reinterpret_cast<unsigned short*>(e.r_D + 8 * LS_MAXJOB);
  const int cand_max = (int)((5 * EnvS<C>::MAXEFC - 8 * LS_MAXJOB) * sizeof(float) / sizeof(unsigned short));
  static_assert(5 * EnvS<C>::MAXEFC - 8 * LS_MAXJOB >= 128, "room for the candidate list");
  int ncand = 0;
#ifdef LS_EMULATE
  for (int p = 0; p < m.np; p++) {
    const int pk = e.pk_tab[p];
    if (!pair_filter(ms, e, p, pk)) continue;
    if (pk & (2 << 24)) { if (ncand < cand_max) cand[ncand++] = (unsigned short)(p | (C::HULL ? LS_CAND_HULL(pk) : 0)); continue; }
    RawCon raw[4];
    int g1, g2; float margin;
    const int n = pair_narrow(ms, e, p, raw, &g1, &g2, &margin);
    const float incl = pair_incl(m, g1, g2, margin);
    for (int k = 0; k < n; k++)
      if (raw[k].dist < incl && e.ncon < EnvS<C>::MAXCON) fill_contact(ms, e, e.ncon++, g1, g2, incl, raw + k);
  }
  {
    int nsurv = 0;
    for (int k = 0; k < ncand; k++) {
      const int p = cand[k] & 0x7fff;
      if (convex_obb_filter(ms, e, p) && (!C::HULL || !(cand[k] & 0x8000) || (c_debug & 32) || convex_hull_filter(ms, e, p)))
        cand[nsurv++] = (unsigned short)p;
    }
    g_obb_pass += nsurv;                       // (the jobs of this evaluation)
    float tmp[8];
    for (int base = 0; base < nsurv; base += LS_MAXJOB) {
      const int nj = nsurv - base < LS_MAXJOB ? nsurv - base : LS_MAXJOB;
      for (int j = 0; j < nj; j++) convex_job(ms, e, e, cand[base + j], jobres + 8 * j);
      for (int j = 0; j < nj; j++) { for (int k = 0; k < 8; k++) tmp[k] = jobres[8 * j + k]; convex_consume(ms, e, cand[base + j], tmp); }
    }
  }
#else
  const int lane = LS_LANE;
  // The pair table holds the primitive pairs first (ModelPack order: modelpack.pack partitions it), then the general convex
  // pairs: the latter only need the bounding-sphere test and a compaction, a lean loop (2 rounds of 32 per iteration).
  const int np_prim = m.np_prim;
  PH_T0(tc);
  // C::PRIMLEAN: the primitive pairs get the same kind of lean loop (64 pairs per trip, both loads of a lane issued before
  // either test), their hits are compacted in pair order into the candidate area (which the convex loop below only
  // overwrites after the narrow sets have read it), and the narrow phase runs once per 32 hits (A1: its floor pairs in
  // contact, one set). Otherwise, and with LOCOSIM_DEBUG bit 64: rounds of 32 pairs, the narrow phase after every round
  // with a hit. Both give the same contact list. (`C::PRIMLEAN && lean` below, though `lean` implies it: so spelled, the
  // lean code is gone before code generation in the other configurations, whose kernels keep the code they had.)
  const bool lean = C::PRIMLEAN && !(c_debug & 64) && np_prim <= cand_max;
  int nprim = 0;
  if (C::PRIMLEAN && lean) {
    NOUNROLL for (int base = 0; base < np_prim; base += 64) {
      const int pa = base + lane, pb = pa + 32;
      const int ka = pa < np_prim ? e.pk_tab[pa] : 0, kb = pb < np_prim ? e.pk_tab[pb] : 0;
      const bool ha = pa < np_prim && pair_filter(ms, e, pa, ka);
      const bool hb = pb < np_prim && pair_filter(ms, e, pb, kb);
      const unsigned ma = __ballot_sync(0xffffffffu, ha), mb = __ballot_sync(0xffffffffu, hb);
      if (ma | mb) {
        const unsigned lt = (1u << lane) - 1u;
        if (ha) cand[nprim + __popc(ma & lt)] = (unsigned short)pa;
        if (hb) cand[nprim + __popc(ma) + __popc(mb & lt)] = (unsigned short)pb;
        nprim += __popc(ma) + __popc(mb);
      }
    }
    __syncwarp();
    PH_LAP(PH_COL_PRIM_FILTER, tc);
    PH_CNT(PH_COL_NPRIM, nprim);
  }
  // every set of 32: the lanes that hit run the narrow phase in parallel, an exclusive scan over the lanes' contact
  // counts assigns the slots, i.e. the list order is pair order, contact order within the pair: the same order as the
  // serial loop (and as the oracle)
  for (int base = 0; base < (C::PRIMLEAN && lean ? nprim : np_prim); base += 32) {
    PH_LAP(PH_COL_PRIM_NARROW, tc);                     // (the previous round's narrow phase)
    int p;
    bool hit;
    if (C::PRIMLEAN && lean) {
      hit = base + lane < nprim;
      p = hit ? (int)cand[base + lane] : 0;
    } else {
      p = base + lane;
      const int pk = p < np_prim ? e.pk_tab[p] : 0;
      hit = (p < np_prim) && pair_filter(ms, e, p, pk);
      const bool any = __any_sync(0xffffffffu, hit);
      PH_LAP(PH_COL_PRIM_FILTER, tc);
      if (!any) continue;                               // (most rounds of 32 pairs have no candidate at all)
      PH_CNT(PH_COL_NPRIM, __popc(__ballot_sync(0xffffffffu, hit)));
    }
    PH_CNT(PH_COL_PRIM_SETS, 1);
    RawCon raw[4];
    int g1 = 0, g2 = 0, n = 0, nact = 0;
    float margin = 0, incl = 0;
    if (hit) {
      n = pair_narrow(ms, e, p, raw, &g1, &g2, &margin);
      incl = pair_incl(m, g1, g2, margin);
      for (int k = 0; k < 4; k++) if (k < n && raw[k].dist < incl) nact++;
    }
    int incl_sum = nact;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl_sum, d);
      if (lane >= d) incl_sum += t;
    }
    const int total = __shfl_sync(0xffffffffu, incl_sum, 31);
    if (total == 0) continue;
    const int first = e.ncon + incl_sum - nact;
    if (nact > 0) {
      int w = 0;
      for (int k = 0; k < 4; k++) {
        if (k < n && raw[k].dist < incl) {
          const int ci = first + w++;
          if (ci < EnvS<C>::MAXCON) fill_contact(ms, e, ci, g1, g2, incl, raw + k);
        }
      }
    }
    __syncwarp();
    LANE0 { const int nc = e.ncon + total; e.ncon = nc < EnvS<C>::MAXCON ? nc : EnvS<C>::MAXCON; }
    __syncwarp();
  }
  PH_LAP(PH_COL_PRIM_NARROW, tc);
  if (C::CONVEX && !(c_debug & 4)) {
    const int npt = m.np;
    NOUNROLL for (int base = np_prim; base < npt; base += 64) {
      const int pa = base + lane, pb = pa + 32;
      const int ka = pa < npt ? m.pair_packed[pa] : 0, kb = pb < npt ? m.pair_packed[pb] : 0;      // (model table: global / L2)
      const float ba = pa < npt ? m.pair_bound[pa] : -1.0f, bb = pb < npt ? m.pair_bound[pb] : -1.0f;
      const float* xa1 = e.gxpos[ka & 0xfff];
      const float* xa2 = e.gxpos[(ka >> 12) & 0xfff];
      const float* xb1 = e.gxpos[kb & 0xfff];
      const float* xb2 = e.gxpos[(kb >> 12) & 0xfff];
      const float ax = xa2[0] - xa1[0], ay = xa2[1] - xa1[1], az = xa2[2] - xa1[2];
      const float bx = xb2[0] - xb1[0], by = xb2[1] - xb1[1], bz = xb2[2] - xb1[2];
      const bool ha = pa < npt && ax * ax + ay * ay + az * az <= ba * ba;
      const bool hb = pb < npt && bx * bx + by * by + bz * bz <= bb * bb;
      const unsigned ma = __ballot_sync(0xffffffffu, ha), mb = __ballot_sync(0xffffffffu, hb);
      if (ma | mb) {
        const unsigned lt = (1u << lane) - 1u;
        const int sa = ncand + __popc(ma & lt), sb = ncand + __popc(ma) + __popc(mb & lt);
        if (ha && sa < cand_max) cand[sa] = (unsigned short)(pa | (C::HULL ? LS_CAND_HULL(ka) : 0));
        if (hb && sb < cand_max) cand[sb] = (unsigned short)(pb | (C::HULL ? LS_CAND_HULL(kb) : 0));
        ncand += __popc(ma) + __popc(mb);
      }
    }
  }
  PH_LAP(PH_COL_SPHERES, tc);
  if (C::CONVEX) {
    if (ncand > cand_max) ncand = cand_max;
    __syncwarp();
    // (1) oriented-box test on the compacted candidates; the survivors are compacted in place (pair order is kept)
    int nsurv = 0;
    NOUNROLL for (int base = 0; base < ncand; base += 32) {
      const int c = base + lane < ncand ? (int)cand[base + lane] : -1, p = C::HULL ? c & 0x7fff : c;
      bool pass = c >= 0 && ((c_debug & 2) || convex_obb_filter(ms, e, p));
      if (C::HULL && pass && (c & 0x8000) && !(c_debug & 32)) pass = convex_hull_filter(ms, e, p);
      const unsigned pm = __ballot_sync(0xffffffffu, pass);
      __syncwarp();                              // (all 32 entries are read before the in-place compaction overwrites any)
      if (pass) cand[nsurv + __popc(pm & ((1u << lane) - 1u))] = (unsigned short)p;      // (slot <= base + lane: in place is safe)
      nsurv += __popc(pm);
      __syncwarp();
    }
    PH_LAP(PH_COL_OBB, tc);
    PH_CNT(PH_COL_NOBB, nsurv);
    if (c_debug & 1) nsurv = 0;
    // (2) the block's warps share the jobs: every env publishes its first LS_MAXJOB survivors, all warps drain the queue
    //     (dynamic: one shared-memory atomic per job), results land in the OWNER's record list. Block barriers: every
    //     warp of the block runs collision() the same number of times (ghost warps included). C::HULL: the first barrier
    //     tells every warp whether any env of the block has a job: if none has, that barrier is the only one, and nobody
    //     reads the counts (a warp that runs ahead to its next evaluation may overwrite its count at once).
    EnvS<C>* blk = &e - (threadIdx.x >> 5);
    const int nw = (int)(blockDim.x >> 5);
    const int nj = nsurv < LS_MAXJOB ? nsurv : LS_MAXJOB;
    PH_CNT(PH_COL_NJOBS, nj);
    LANE0 { e.njobs = nj; }
    PH_T0(t);
    bool any_jobs = true;
    if (C::HULL) any_jobs = __syncthreads_or(nj > 0);
    else __syncthreads();
    PH_LAP(PH_COL_QWAIT, tc);
    if (any_jobs) {
      int incl = lane < nw ? blk[lane].njobs : 0;
      __syncthreads();      // (everybody has read the counts: a warp that runs ahead may publish its next evaluation's count)
      const int mine = incl;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
      }
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      if (total > 0) {      // (C::HULL: always true here, but without it ptxas saves more registers around forward()'s calls)
        for (;;) {
          int g = 0;
          if (lane == 0) g = atomicAdd(&blk[0].job_head, 1);
          g = __shfl_sync(0xffffffffu, g, 0);
          if (g >= total) break;
          const int owner = __popc(__ballot_sync(0xffffffffu, incl <= g));         // first lane whose inclusive prefix exceeds g
          const int first = __shfl_sync(0xffffffffu, incl - mine, owner);
          EnvS<C>& o = blk[owner];
          const unsigned short* ocand = reinterpret_cast<const unsigned short*>(o.r_D + 8 * LS_MAXJOB);
          convex_job(ms, o, e, (int)ocand[g - first], o.r_D + 8 * (g - first));
        }
        PH_LAP(PH_COL_JOBS, tc);
        __syncthreads();
        PH_LAP(PH_CONVEX_QUEUE, t);
        PH_LAP(PH_COL_JOBS_WAIT, tc);
        if (threadIdx.x == 0) blk[0].job_head = 0;       // (next use is behind the next evaluation's first barrier)
        // (3) owners consume their records in pair order
        NOUNROLL for (int j = 0; j < nj; j++) {
          float rec[8];
          for (int k = 0; k < 8; k++) rec[k] = jobres[8 * j + k];
          __syncwarp();
          convex_consume(ms, e, (int)cand[j], rec);
        }
      }
    }
    // (4) overflow (more than LS_MAXJOB survivors in one evaluation: not seen in the in-scope models): the owner alone
    NOUNROLL for (int j = LS_MAXJOB; j < nsurv; j++) {
      float rec[8];
      convex_job(ms, e, e, (int)cand[j], jobres);
      __syncwarp();
      for (int k = 0; k < 8; k++) rec[k] = jobres[k];
      __syncwarp();
      convex_consume(ms, e, (int)cand[j], rec);
    }
    PH_LAP(PH_COL_CONSUME, tc);
  }
#endif
#ifdef LOCOSIM_TERRAIN
  if constexpr (C::TERRAIN) { SYNC(); terrain_pass(ms, e); }
#endif
  SYNC();
}

// ----------------------------------------------------------------------------------------------------------
// constraint assembly (mj_makeConstraint + mj_makeImpedance + mj_referenceConstraint)
// ----------------------------------------------------------------------------------------------------------
template <class C>
LS_FN void make_constraint(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  typedef EnvS<C> E;
  const int nv = m.nv;
  // ---- unit rows: frictionloss (static row slots) ----
  PAR_FOR(d, nv) {
    int r = m.dof_frow[d];
    if (r >= 0) e.r_ti[r] = ROW_PACK(ROW_FRICTION, d, 0);
    e.d_lrow[d][0] = -1; e.d_lrow[d][1] = -1;
  }
  SYNC();
  // ---- unit rows: joint limits (dynamic; deterministic order dof-major, lower side first) ----
  int nunit = m.nfric;
#ifdef LS_EMULATE
  for (int d = 0; d < nv; d++) {
    if (!m.jnt_limited[d]) continue;
    for (int side = 0; side < 2; side++) {
      float dist = side == 0 ? e.qpos[d] - m.jnt_range[2 * d] : m.jnt_range[2 * d + 1] - e.qpos[d];
      if (dist < m.jnt_margin[d]) {
        int r = nunit++;
        e.r_ti[r] = ROW_PACK(ROW_LIMIT, d, side);
        e.d_lrow[d][side] = r;
      }
    }
  }
#else
  {
    const int lane = LS_LANE;
    NOUNROLL for (int base = 0; base < 2 * nv; base += 32) {
      int idx = base + lane;
      int d = idx >> 1, side = idx & 1;
      bool act = false;
      if (idx < 2 * nv && m.jnt_limited[d]) {
        float dist = side == 0 ? e.qpos[d] - m.jnt_range[2 * d] : m.jnt_range[2 * d + 1] - e.qpos[d];
        act = dist < m.jnt_margin[d];
      }
      unsigned mask = __ballot_sync(0xffffffffu, act);
      if (act) {
        int r = nunit + __popc(mask & ((1u << lane) - 1));
        e.r_ti[r] = ROW_PACK(ROW_LIMIT, d, side);
        e.d_lrow[d][side] = r;
      }
      nunit += __popc(mask);
    }
  }
#endif
  // ---- contact rows: row offsets (serial, tiny) ----
  LANE0 {
    int nrow = 0, ncon = e.ncon;
    NOUNROLL for (int ci = 0; ci < ncon; ci++) {
      int dim = e.con_dim[ci];
      int nr = (dim == 1) ? 1 : (C::CONE == 1 ? dim : 2 * (dim - 1));
      if (nrow + nr > E::MAXROW) { ncon = ci; break; }
      e.con_row[ci] = nrow;
      nrow += nr;
    }
    e.ncon = ncon; e.nrow = nrow; e.nunit = nunit; e.nefc = nunit + nrow;
  }
  SYNC();
  const int ncon = e.ncon;
  // ---- contact Jacobian rows: one work item per (contact, dof) ----
  PAR_FOR(item, ncon * E::JS) {
    int ci = item / E::JS, d = item - ci * E::JS;      // d >= nv: zero padding columns
    int b1 = m.geom_bodyid[e.con_g1[ci]], b2 = m.geom_bodyid[e.con_g2[ci]];
    float s = 0;
    if (d < nv) {
      if ((m.body_dofmask[b2] >> d) & 1) s += 1.0f;
      if ((m.body_dofmask[b1] >> d) & 1) s -= 1.0f;
    }
    int dim = e.con_dim[ci], row0 = e.con_row[ci];
    int nr = (dim == 1) ? 1 : (C::CONE == 1 ? dim : 2 * (dim - 1));
    if (s == 0) { NOUNROLL for (int r = 0; r < nr; r++) e.J[row0 + r][d] = 0; continue; }
    float off[3] = {e.con_pos[ci][0] - e.com[0], e.con_pos[ci][1] - e.com[1], e.con_pos[ci][2] - e.com[2]};
    const float* cd = e.cdof[d];
    float jp[3], t[3];
    cross3(t, cd, off);
    for (int k = 0; k < 3; k++) jp[k] = s * (cd[3 + k] + t[k]);
    float jr[3] = {s * cd[0], s * cd[1], s * cd[2]};
    const float* f = e.con_frame[ci];
    float jd[6];
    for (int r = 0; r < 3; r++) { jd[r] = dot3(f + 3 * r, jp); jd[3 + r] = dot3(f + 3 * r, jr); }
    if (dim == 1) e.J[row0][d] = jd[0];
    else if (C::CONE == 1) {
#pragma unroll
      for (int r = 0; r < 6; r++) if (r < dim) e.J[row0 + r][d] = jd[r];
    } else {
#pragma unroll
      for (int r = 1; r < 6; r++) {
        if (r < dim) {
          float fr = e.con_fri[ci][r - 1];
          e.J[row0 + 2 * (r - 1)][d] = jd[0] + fr * jd[r];
          e.J[row0 + 2 * (r - 1) + 1][d] = jd[0] - fr * jd[r];
        }
      }
    }
  }
  // ---- contact row headers ----
  PAR_FOR(ci, ncon) {
    int dim = e.con_dim[ci], row0 = nunit + e.con_row[ci];
    int nr = (dim == 1) ? 1 : (C::CONE == 1 ? dim : 2 * (dim - 1));
    int tp = (dim == 1) ? ROW_CON_FRICTIONLESS : (C::CONE == 1 ? ROW_CON_ELLIPTIC : ROW_CON_PYRAMIDAL);
    NOUNROLL for (int r = 0; r < nr; r++) e.r_ti[row0 + r] = ROW_PACK(tp, ci, r);
  }
  SYNC();
  // ---- impedance -> D = 1/R, reference acceleration (mj_makeImpedance + mj_referenceConstraint) ----
  const int nefc = e.nefc;
  PAR_FOR(r, nefc) {
    const int ti = e.r_ti[r];
    const int tp = ROW_TYPE(ti), id = ROW_ID(ti), k = ROW_K(ti);
    float pos, margin, diag, vel, imp, K, B;
    if (tp == ROW_FRICTION) {
      pos = 0; margin = 0; diag = PRM(dof_invweight0)[id]; vel = e.qvel[id];
      impedance_KB(m.dof_solref + 2 * id, m.dof_solimp + 5 * id, pos, margin, m.timestep, &imp, &K, &B);
    } else if (tp == ROW_LIMIT) {
      pos = k == 0 ? e.qpos[id] - m.jnt_range[2 * id] : m.jnt_range[2 * id + 1] - e.qpos[id];
      margin = m.jnt_margin[id]; diag = PRM(dof_invweight0)[id]; vel = k == 0 ? e.qvel[id] : -e.qvel[id];
      impedance_KB(m.jnt_solref + 2 * id, m.jnt_solimp + 5 * id, pos, margin, m.timestep, &imp, &K, &B);
    } else {
      pos = e.con_dist[id]; margin = e.con_incl[id];
      imp = e.con_imp[id]; K = e.con_K[id]; B = e.con_B[id];
      const int g1 = e.con_g1[id], g2 = e.con_g2[id];
      float tran = PRM(geom_invweight0)[2 * g1] + PRM(geom_invweight0)[2 * g2];
      if (tp == ROW_CON_PYRAMIDAL) diag = tran + e.con_fri[id][0] * e.con_fri[id][0] * tran;
      else diag = k < 3 ? tran : PRM(geom_invweight0)[2 * g1 + 1] + PRM(geom_invweight0)[2 * g2 + 1];
      const float* Jr = e.J[r - nunit];
      vel = 0;
#pragma unroll 4
      for (int d = 0; d < nv; d++) vel = fmaf(Jr[d], e.qvel[d], vel);
    }
    float R = fmaxf(LS_MINVAL, (1 - imp) * diag / imp);
    if (tp == ROW_FRICTION || (tp == ROW_CON_ELLIPTIC && k > 0)) K = 0;
    e.r_aref[r] = -B * vel - K * imp * (pos - margin);
    e.r_D[r] = 1.0f / R;
  }
  SYNC();
  // ---- frictional contacts: regularised cone mu and the D of the friction dimensions ----
  PAR_FOR(ci, ncon) {
    int dim = e.con_dim[ci];
    if (dim == 1) continue;
    int i = nunit + e.con_row[ci];
    float f0 = e.con_fri[ci][0];
    if (C::CONE == 0) {
      float mu = f0 * rsqrtf(fmaxf(LS_MINVAL, m.impratio));
      e.con_mu[ci] = mu;
      float Dpy = e.r_D[i] / (2 * mu * mu);
      NOUNROLL for (int j = 0; j < 2 * (dim - 1); j++) e.r_D[i + j] = Dpy;
    } else {
      float D0 = e.r_D[i];
      float ir = fmaxf(LS_MINVAL, m.impratio);
      float D1 = D0 * ir;                          // R1 = R0 / impratio
      e.r_D[i + 1] = D1;
      e.con_mu[ci] = f0 * rsqrtf(ir);              // mu = friction[0] * sqrt(R1 / R0)
      NOUNROLL for (int j = 1; j < dim - 1; j++) {
        float fj = e.con_fri[ci][j];
        e.r_D[i + j + 1] = D1 * fj * fj / (f0 * f0);   // R[j+1] = R1 * f0^2 / fj^2
      }
    }
  }
  SYNC();
}

// ----------------------------------------------------------------------------------------------------------
// velocity-dependent smooth terms: comVel, RNE bias, passive, actuation -> qfrc_smooth, qacc_smooth
// ----------------------------------------------------------------------------------------------------------
// the force of actuator i at the env's state and e.ctrl, before the gear: ctrl clamped to its range, gain and bias, the
// force clamped to its range. smooth_forces and forward_outputs' dof row both take it from here, so the dof outputs and
// forward_dynamics' dof row agree bit for bit.
template <class C>
LS_DEV float actuator_force(const DevModel& m, const EnvS<C>& e, const int i) {
  float c = e.ctrl[i];
  if (m.actuator_ctrllimited[i]) c = fminf(m.actuator_ctrlrange[2 * i + 1], fmaxf(m.actuator_ctrlrange[2 * i], c));
  const int d = m.actuator_dof[i];
  float f = m.actuator_gain[i] * c + m.actuator_bias[3 * i] + m.actuator_bias[3 * i + 1] * e.qpos[d] +
            m.actuator_bias[3 * i + 2] * e.qvel[d];
  if (m.actuator_forcelimited[i]) f = fminf(m.actuator_forcerange[2 * i + 1], fmaxf(m.actuator_forcerange[2 * i], f));
  return f;
}

// mj_comVel + mj_rne (bias forces) without tree recursion: all spatial vectors live in one frame (world-aligned, at the
// CoM), so the velocity / bias acceleration of a body is a plain SUM over the dofs of its chain (bit mask
// body_dofmask) and the force a dof feels is a plain sum over the bodies of its subtree. Three fully parallel passes.
template <class C>
LS_FN void smooth_forces(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv;
  // (A) cdof_dot_j = cvel(just above dof j) x cdof_j
  PAR_FOR(j, nv) {
    unsigned mask = (unsigned)m.body_dofmask[m.jnt_bodyid[j]] & ((1u << j) - 1u);
    float v[6] = {0, 0, 0, 0, 0, 0};
    while (mask) {
      const int i = LS_FFS(mask) - 1;
      mask &= mask - 1;
      const float qv = e.qvel[i];
      for (int c = 0; c < 6; c++) v[c] = fmaf(e.cdof[i][c], qv, v[c]);
    }
    float cdd[6];
    crossMotion(cdd, v, e.cdof[j]);
    for (int c = 0; c < 6; c++) e.cdof_dot[j][c] = cdd[c];
  }
  SYNC();
  // (B) per body: cvel, cacc (gravity enters as the world's upward acceleration), f = I cacc + cvel x* (I cvel)
  //     -> crb[b][0..5] (the composite inertias are dead once M is assembled); minus the applied wrench, moved from the
  //     body's CoM to the frame's origin e.com (mj_xfrcAccumulate: pass (C) turns it into J^T wrench in qfrc_smooth)
  const float* __restrict__ xfrc = c_applied[ms].xfrc;
  PAR_FOR(b, m.nb) {
    float* f = e.crb[b];
    if (b == 0) { for (int k = 0; k < 6; k++) f[k] = 0; continue; }
    unsigned mask = (unsigned)m.body_dofmask[b];
    float cvel[6] = {0, 0, 0, 0, 0, 0}, cacc[6] = {0, 0, 0, -m.gravity[0], -m.gravity[1], -m.gravity[2]};
    while (mask) {
      const int i = LS_FFS(mask) - 1;
      mask &= mask - 1;
      const float qv = e.qvel[i];
      for (int c = 0; c < 6; c++) { cvel[c] = fmaf(e.cdof[i][c], qv, cvel[c]); cacc[c] = fmaf(e.cdof_dot[i][c], qv, cacc[c]); }
    }
    float t1[6], t2[6], t3[6];
    mulInertVec(t1, e.cinert[b], cacc);
    mulInertVec(t2, e.cinert[b], cvel);
    crossForce(t3, cvel, t2);
    for (int k = 0; k < 6; k++) f[k] = t1[k] + t3[k];
    if (xfrc) {
      const float* w = xfrc + ((size_t)e.env * m.nb + b) * 6;
      const float F[3] = {LS_LDG(w), LS_LDG(w + 1), LS_LDG(w + 2)};
      const float r[3] = {e.xipos[b][0] - e.com[0], e.xipos[b][1] - e.com[1], e.xipos[b][2] - e.com[2]};
      float rxF[3];
      cross3(rxF, r, F);
      for (int k = 0; k < 3; k++) { f[k] -= LS_LDG(w + 3 + k) + rxF[k]; f[3 + k] -= F[k]; }
    }
  }
  SYNC();
  // (C) bias force of dof j = cdof_j . (sum of f over the bodies below j);  qfrc_smooth = passive - bias + applied + actuator
  const float* __restrict__ qfrc = c_applied[ms].qfrc;
  PAR_FOR(j, nv) {
    float F[6] = {0, 0, 0, 0, 0, 0};
    NOUNROLL for (int b = 1; b < m.nb; b++) {
      if (!((m.body_dofmask[b] >> j) & 1)) continue;
      for (int c = 0; c < 6; c++) F[c] += e.crb[b][c];
    }
    float bias = 0;
    for (int c = 0; c < 6; c++) bias += e.cdof[j][c] * F[c];
    float passive = -PRM(jnt_stiffness)[j] * (e.qpos[j] - m.qpos_spring[j]) - PRM(dof_damping)[j] * e.qvel[j];
    e.qfrc_smooth[j] = qfrc ? passive - bias + LS_LDG(qfrc + (size_t)e.env * nv + j) : passive - bias;
  }
  SYNC();
  PAR_FOR(i, m.nu) {
    const float f = actuator_force(m, e, i);     // (before the dof load: in the other order the step kernels' code changes)
    const int d = m.actuator_dof[i];
    // one actuator per dof in all in-scope models -> no write conflict
    e.qfrc_smooth[d] += m.actuator_gear[i] * f;
    // dof outputs: the force of this evaluation, for dof_outputs after the integrator (not from a warp that shadows
    // another env: it may be a sub-step ahead of the env's own warp). The force, not gear * force: a second use of that
    // product would cost the sum above its fused multiply-add, and change qfrc_smooth whether or not anything is registered.
    float* const act = c_dof_act[ms];
    if (act && e.substep >= 0) act[(size_t)e.env * m.nu + i] = f;
  }
  SYNC();
  PAR_FOR(j, EnvS<C>::NV) e.qacc_smooth[j] = j < nv ? e.qfrc_smooth[j] : 0.0f;
  SYNC();
  chol_solve<EnvS<C>::NV, EnvS<C>::NVP>(e.H, e.qacc_smooth);
}

// ----------------------------------------------------------------------------------------------------------
// Newton solver (mj_solNewton), warp-parallel over rows / matrix entries
// ----------------------------------------------------------------------------------------------------------
template <class C>
LS_FN void mulM(const int ms, const EnvS<C>& e, float* res, const float* v) {
  const DevModel& m = c_models[ms];
  PAR_FOR(i, m.nv) {
    float a = 0;
    for (int j = 0; j < m.nv; j++) a += e.M[i][j] * v[j];
    res[i] = a;
  }
}
// res[r] = (J v)[r] for all rows
template <class C>
LS_FN void mulJ(const int ms, const EnvS<C>& e, float* res, const float* v) {
  const DevModel& m = c_models[ms];
  const int nunit = e.nunit, nefc = e.nefc, nv = m.nv;
  PAR_FOR(r, nefc) {
    if (r < nunit) { const int ti = e.r_ti[r]; float vv = v[ROW_ID(ti)]; res[r] = ROW_K(ti) == 1 ? -vv : vv; }
    else {
      // v is one of the NV-long solver vectors (entries >= nv are kept at 0, init_workspace), J rows are zero padded
      const float4* Jr = reinterpret_cast<const float4*>(e.J[r - nunit]);
      float a = 0;
#pragma unroll
      for (int q = 0; q < EnvS<C>::JS / 4; q++) {
        const float4 j4 = Jr[q];
        a = fmaf(j4.x, v[4 * q], a);
        if (4 * q + 1 < EnvS<C>::NV) a = fmaf(j4.y, v[4 * q + 1], a);
        if (4 * q + 2 < EnvS<C>::NV) a = fmaf(j4.z, v[4 * q + 2], a);
        if (4 * q + 3 < EnvS<C>::NV) a = fmaf(j4.w, v[4 * q + 3], a);
      }
      res[r] = a;
    }
  }
}

// states, forces, cost from jar (= e.r_jar). Returns the constraint cost (all lanes).
template <class C>
LS_FN float constraint_update(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  const int nefc = e.nefc, nunit = e.nunit;
  float cost = 0;
  PAR_FOR(r, nefc) {
    const int ti = e.r_ti[r];
    const int tp = ROW_TYPE(ti);
    float jar = e.r_jar[r], D = e.r_D[r];
    if (tp == ROW_FRICTION) {
      float f = PRM(dof_frictionloss)[ROW_ID(ti)], Rf = f / D;
      if (jar <= -Rf) { e.r_state[r] = ST_LINEARNEG; e.r_force[r] = f; cost += -0.5f * Rf * f - f * jar; }
      else if (jar >= Rf) { e.r_state[r] = ST_LINEARPOS; e.r_force[r] = -f; cost += -0.5f * Rf * f + f * jar; }
      else { e.r_state[r] = ST_QUADRATIC; e.r_force[r] = -D * jar; cost += 0.5f * D * jar * jar; }
    } else if (tp == ROW_CON_ELLIPTIC) {
      if (ROW_K(ti) != 0) continue;   // handled by the contact's first row
      int ci = ROW_ID(ti), dim = e.con_dim[ci];
      float mu = e.con_mu[ci];
      float U[6];
      U[0] = jar * mu;
      float TT = 0;
      NOUNROLL for (int j = 1; j < dim; j++) { U[j] = e.r_jar[r + j] * e.con_fri[ci][j - 1]; TT += U[j] * U[j]; }
      float N = U[0], T = sqrtf(TT);
      if (T < 1e-12f) T = 0.0f;   // fp32: 1/T^3 in the cone Hessian would overflow
      if (N >= mu * T || (T <= 0 && N >= 0)) {
        NOUNROLL for (int j = 0; j < dim; j++) { e.r_force[r + j] = 0; e.r_state[r + j] = ST_SATISFIED; }
      } else if (mu * N + T <= 0 || (T <= 0 && N < 0)) {
        NOUNROLL for (int j = 0; j < dim; j++) {
          float jj = e.r_jar[r + j], Dj = e.r_D[r + j];
          e.r_force[r + j] = -Dj * jj; e.r_state[r + j] = ST_QUADRATIC; cost += 0.5f * Dj * jj * jj;
        }
      } else {
        float Dm = D / fmaxf(LS_MINVAL, mu * mu * (1 + mu * mu));
        float NmT = N - mu * T;
        cost += 0.5f * Dm * NmT * NmT;
        float f0 = -Dm * NmT * mu;
        e.r_force[r] = f0; e.r_state[r] = ST_CONE;
        NOUNROLL for (int j = 1; j < dim; j++) { e.r_force[r + j] = -f0 / T * U[j] * e.con_fri[ci][j - 1]; e.r_state[r + j] = ST_CONE; }
      }
    } else {
      if (jar < 0) { e.r_state[r] = ST_QUADRATIC; e.r_force[r] = -D * jar; cost += 0.5f * D * jar * jar; }
      else { e.r_state[r] = ST_SATISFIED; e.r_force[r] = 0; }
    }
  }
  (void)nunit;
  cost = WARP_SUM(cost);
  SYNC();
  return cost;
}

// qfrc_constraint = J^T force ; returns total cost incl. Gauss term
// second half of mj_constraintUpdate: qfrc_constraint = J^T force; returns the Gauss term of the cost
template <class C>
LS_FN float finish_constraint(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nrow = e.nrow, nunit = e.nunit;
  float g = 0;
  PAR_FOR(d, nv) {
    float a = 0;
    int fr = m.dof_frow[d];
    if (fr >= 0) a += e.r_force[fr];
    int l0 = e.d_lrow[d][0], l1 = e.d_lrow[d][1];
    if (l0 >= 0) a += e.r_force[l0];
    if (l1 >= 0) a -= e.r_force[l1];
#pragma unroll 4
    for (int r = 0; r < nrow; r++) a = fmaf(e.J[r][d], e.r_force[nunit + r], a);
    e.qfrc_constraint[d] = a;
    g += 0.5f * (e.Ma[d] - e.qfrc_smooth[d]) * (e.qacc[d] - e.qacc_smooth[d]);
  }
  g = WARP_SUM(g);
  SYNC();
  return g;
}
template <class C>
LS_FN float update_constraint(const int ms, EnvS<C>& e, float* gauss_out) {
  const float cost = constraint_update(ms, e);
  const float g = finish_constraint(ms, e);
  *gauss_out = g;
  return cost + g;
}

#ifndef LS_EMULATE
// CUDA build, nv <= 20: H = M + J^T diag(w) J (+ cone blocks) accumulated in registers by 24 lanes. Lanes 0..NV-1 own
// row `lane`, columns 0..11 (chunks 0-2 of four); for rows >= 12, whose lower triangle reaches beyond column 11, helper
// lanes NV.. own columns 8..19 (chunks 2-4). Every lane therefore runs 3 float4 chunks per active constraint row instead
// of 5. The factorisation (chol_factor) only reads the lower triangle.
template <class C>
LS_FN void make_hessian_split(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  typedef EnvS<C> E;
  constexpr int NV = E::NV, JS = E::JS;
  static_assert(JS == 20 && NV >= 12 && NV + (NV - 12) <= 32, "split layout: 5 chunks, helpers for rows 12..NV-1");
  const int nv = m.nv, nrow = e.nrow, nunit = e.nunit;
  const int lane = LS_LANE;
  const bool owner = lane < NV, helper = lane >= NV && lane < NV + (NV - 12);
  const int row = owner ? lane : (helper ? 12 + (lane - NV) : NV - 1);
  const int q0 = helper ? 2 : 0;                       // first of this lane's three chunks
  const int c0 = 4 * q0;
  PAR_FOR(r, e.nefc) e.r_Jv[r] = (e.r_state[r] == ST_QUADRATIC) ? e.r_D[r] : 0.0f;
  float h[12];
#pragma unroll
  for (int k = 0; k < 12; k++) h[k] = (c0 + k < NV) ? e.M[row][c0 + k] : 0.0f;
  __syncwarp();
  const float* w = e.r_Jv + nunit;
  // The rows with w != 0 (quadratic zone; satisfied / linear / cone rows have w = 0), as a warp-uniform bit list in row
  // order. The loop loads the next listed row's weight, column entry and chunks before the current row's FFMAs, so a row
  // costs its FFMAs instead of a weight load, a branch and the row's loads in series. Same rows, same order, same fmaf
  // chain per h[k] as a plain scan.
  static_assert(E::MAXROW <= 64, "row list: two ballots");
  unsigned long long rest =
      (unsigned long long)__ballot_sync(0xffffffffu, lane < nrow && !(w[lane] == 0.0f)) |
      (unsigned long long)__ballot_sync(0xffffffffu, lane + 32 < nrow && !(w[lane + 32] == 0.0f)) << 32;
  if (rest) {
    int r = __ffsll((long long)rest) - 1;
    rest &= rest - 1;
    float wr = w[r], jr = e.J[r][row];
    const float4* rp = reinterpret_cast<const float4*>(e.J[r]) + q0;
    float4 v[3] = {rp[0], rp[1], rp[2]};
    for (;;) {
      const bool more = rest != 0;
      r = more ? __ffsll((long long)rest) - 1 : r;   // (after the last row: a harmless reload of it)
      rest &= rest - 1;
      const float wn = w[r], jn = e.J[r][row];
      const float4* rn = reinterpret_cast<const float4*>(e.J[r]) + q0;
      const float4 vn[3] = {rn[0], rn[1], rn[2]};
      const float t = wr * jr;
#pragma unroll
      for (int q = 0; q < 3; q++) {
        h[4 * q] = fmaf(t, v[q].x, h[4 * q]); h[4 * q + 1] = fmaf(t, v[q].y, h[4 * q + 1]);
        h[4 * q + 2] = fmaf(t, v[q].z, h[4 * q + 2]); h[4 * q + 3] = fmaf(t, v[q].w, h[4 * q + 3]);
      }
      if (!more) break;
      wr = wn; jr = jn;
#pragma unroll
      for (int q = 0; q < 3; q++) v[q] = vn[q];
    }
  }
  // unit rows (frictionloss / joint limits) only touch the diagonal
  if ((owner || helper) && row < nv) {
    float dsum = 0;
    const int fr = m.dof_frow[row];
    if (fr >= 0) dsum += e.r_Jv[fr];
    const int l0 = e.d_lrow[row][0], l1 = e.d_lrow[row][1];
    if (l0 >= 0) dsum += e.r_Jv[l0];
    if (l1 >= 0) dsum += e.r_Jv[l1];
#pragma unroll
    for (int k = 0; k < 12; k++) if (c0 + k == row) h[k] += dsum;
  }
  if (C::CONE == 1) {
    // The contacts in the cone zone as a warp-uniform bit list in contact order (lane ci tests contact ci). A contact's
    // rows (dim <= 6) are read into registers by fully unrolled, predicated loads that the compiler issues together, so
    // the contact costs its arithmetic instead of one shared-memory round trip per row and loop. The expressions are
    // those of make_hessian_wide with coneS[a] = sc[a], coneU[a] = cu[a].
    static_assert(E::MAXCON <= 32, "cone list: one ballot");
    unsigned cones = __ballot_sync(0xffffffffu, lane < e.ncon && e.r_state[nunit + e.con_row[lane]] == ST_CONE);
    while (cones) {
      const int ci = __ffs((int)cones) - 1;
      cones &= cones - 1;
      const int r0 = nunit + e.con_row[ci];
      const int dim = e.con_dim[ci], jr0 = r0 - nunit;
      const float mu = e.con_mu[ci];
      float jar[6], sc[6], jc[6];
#pragma unroll
      for (int a = 0; a < 6; a++) {
        jar[a] = a < dim ? e.r_jar[r0 + a] : 0.0f;
        sc[a] = a == 0 ? mu : (a < dim ? e.con_fri[ci][a - 1] : 0.0f);
        jc[a] = a < dim ? e.J[jr0 + a][row] : 0.0f;
      }
      float TT = 0;
#pragma unroll
      for (int j = 1; j < 6; j++) if (j < dim) { float u = jar[j] * sc[j]; TT += u * u; }
      const float N = jar[0] * mu, T = sqrtf(TT), invT = 1.0f / T;
      float cu[6];                                                             // unit tangential direction U / T
#pragma unroll
      for (int a = 0; a < 6; a++) cu[a] = jar[a] * sc[a] * invT;
      const float Dm = e.r_D[r0] / fmaxf(LS_MINVAL, mu * mu * (1 + mu * mu));
      const float kk = mu * N * invT, c2 = mu * mu - kk;
      // Hc (jar space) = Dm S [ e0 e0^T - mu (e0 u^T + u e0^T) + (mu N / T) u u^T + c2 I_t ] S  with u = U / T (unit,
      // tangential only; no 1/T^3 factor, which overflows in fp32 for a vanishing tangential velocity), I_t tangential:
      // v = Hc p for this lane's column p_a = J[a][row] in O(dim), then H[row][:] += sum_b v_b J[b][:]
      const float p0 = sc[0] * jc[0];
      float pU = 0;
#pragma unroll
      for (int a = 1; a < 6; a++) if (a < dim) pU = fmaf(cu[a], sc[a] * jc[a], pU);
#pragma unroll
      for (int b2 = 0; b2 < 6; b2++) {
        if (b2 >= dim) break;
        float vb;
        if (b2 == 0) vb = p0 - mu * pU;
        else vb = cu[b2] * (kk * pU - mu * p0) + c2 * sc[b2] * jc[b2];
        vb *= Dm * sc[b2];
        const float4* rp = reinterpret_cast<const float4*>(e.J[jr0 + b2]) + q0;
#pragma unroll
        for (int q = 0; q < 3; q++) {
          const float4 v = rp[q];
          h[4 * q] = fmaf(vb, v.x, h[4 * q]); h[4 * q + 1] = fmaf(vb, v.y, h[4 * q + 1]);
          h[4 * q + 2] = fmaf(vb, v.z, h[4 * q + 2]); h[4 * q + 3] = fmaf(vb, v.w, h[4 * q + 3]);
        }
      }
    }
  }
  // owners publish columns 0..11, helpers 12..NV-1 (their columns 8..11 duplicate the owner's values)
  if (owner) {
#pragma unroll
    for (int k = 0; k < 12; k++) e.H[row][k] = h[k];
  } else if (helper) {
#pragma unroll
    for (int k = 4; k < 12; k++) if (c0 + k < NV) e.H[row][c0 + k] = h[k];
  }
  __syncwarp();
  PH_T0(t);
  chol_factor<NV, E::NVP>(ms, e.H);
  PH_LAP(PH_CHOL_FACTOR, t);
}

// CUDA build, any nv <= 32: lane i accumulates the whole row i of H in registers
template <class C>
LS_FN void make_hessian_wide(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  typedef EnvS<C> E;
  constexpr int NV = E::NV, JS = E::JS;
  const int nv = m.nv, nrow = e.nrow, nunit = e.nunit;
  const int lane = LS_LANE, li = lane < NV ? lane : NV - 1;
  PAR_FOR(r, e.nefc) e.r_Jv[r] = (e.r_state[r] == ST_QUADRATIC) ? e.r_D[r] : 0.0f;
  float h[JS];
#pragma unroll
  for (int j = 0; j < NV; j++) h[j] = e.M[li][j];
#pragma unroll
  for (int j = NV; j < JS; j++) h[j] = 0.0f;
  __syncwarp();
  const float* w = e.r_Jv + nunit;
  NOUNROLL for (int r = 0; r < nrow; r++) {
    const float wr = w[r];
    if (wr == 0.0f) continue;                       // warp-uniform: satisfied / linear / cone rows
    const float t = wr * e.J[r][li];
    const float4* row = reinterpret_cast<const float4*>(e.J[r]);
#pragma unroll
    for (int q = 0; q < JS / 4; q++) {
      float4 v = row[q];
      h[4 * q] = fmaf(t, v.x, h[4 * q]); h[4 * q + 1] = fmaf(t, v.y, h[4 * q + 1]);
      h[4 * q + 2] = fmaf(t, v.z, h[4 * q + 2]); h[4 * q + 3] = fmaf(t, v.w, h[4 * q + 3]);
    }
  }
  // unit rows (frictionloss / joint limits) only touch the diagonal
  if (lane < nv) {
    float dsum = 0;
    int fr = m.dof_frow[lane];
    if (fr >= 0) dsum += e.r_Jv[fr];
    int l0 = e.d_lrow[lane][0], l1 = e.d_lrow[lane][1];
    if (l0 >= 0) dsum += e.r_Jv[l0];
    if (l1 >= 0) dsum += e.r_Jv[l1];
#pragma unroll
    for (int j = 0; j < NV; j++) if (j == lane) h[j] += dsum;
  }
  if (C::CONE == 1) {
    NOUNROLL for (int ci = 0; ci < e.ncon; ci++) {
      const int r0 = nunit + e.con_row[ci];
      if (e.r_state[r0] != ST_CONE) continue;
      const int dim = e.con_dim[ci], jr0 = r0 - nunit;
      const float mu = e.con_mu[ci];
      float TT = 0;
      NOUNROLL for (int j = 1; j < dim; j++) { float u = e.r_jar[r0 + j] * e.con_fri[ci][j - 1]; TT += u * u; }
      const float N = e.r_jar[r0] * mu, T = sqrtf(TT), invT = 1.0f / T;
      if (lane < dim) {
        float sc = lane == 0 ? mu : e.con_fri[ci][lane - 1];
        e.coneS[lane] = sc; e.coneU[lane] = e.r_jar[r0 + lane] * sc * invT;     // unit tangential direction U / T
      }
      __syncwarp();
      const float Dm = e.r_D[r0] / fmaxf(LS_MINVAL, mu * mu * (1 + mu * mu));
      const float kk = mu * N * invT, c2 = mu * mu - kk;
      // Hc (jar space) = Dm S [ e0 e0^T - mu (e0 u^T + u e0^T) + (mu N / T) u u^T + c2 I_t ] S  with u = U / T, I_t tangential.
      // v = Hc p for this lane's column p_a = J[a][lane] in O(dim), then H[lane][:] += sum_b v_b J[b][:]
      float p0 = e.coneS[0] * e.J[jr0][li], pU = 0;
      NOUNROLL for (int a = 1; a < dim; a++) pU = fmaf(e.coneU[a], e.coneS[a] * e.J[jr0 + a][li], pU);
      NOUNROLL for (int b = 0; b < dim; b++) {
        float vb;
        if (b == 0) vb = p0 - mu * pU;
        else vb = e.coneU[b] * (kk * pU - mu * p0) + c2 * e.coneS[b] * e.J[jr0 + b][li];
        vb *= Dm * e.coneS[b];
        const float4* row = reinterpret_cast<const float4*>(e.J[jr0 + b]);
#pragma unroll
        for (int q = 0; q < JS / 4; q++) {
          float4 v = row[q];
          h[4 * q] = fmaf(vb, v.x, h[4 * q]); h[4 * q + 1] = fmaf(vb, v.y, h[4 * q + 1]);
          h[4 * q + 2] = fmaf(vb, v.z, h[4 * q + 2]); h[4 * q + 3] = fmaf(vb, v.w, h[4 * q + 3]);
        }
      }
      __syncwarp();
    }
  }
  if (lane < NV) {
#pragma unroll
    for (int j = 0; j < NV; j++) e.H[lane][j] = h[j];
  }
  __syncwarp();
  PH_T0(t);
  chol_factor<NV, E::NVP>(ms, e.H);
  PH_LAP(PH_CHOL_FACTOR, t);
}
template <class C>
LS_DEV void make_hessian(const int ms, EnvS<C>& e) {
  if constexpr (EnvS<C>::JS == 20) make_hessian_split(ms, e);
  else make_hessian_wide(ms, e);
}
#else
template <class C>
LS_FN void make_hessian(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  typedef EnvS<C> E;
  const int nv = m.nv, nrow = e.nrow, nunit = e.nunit;
  const int ntri = nv * (nv + 1) / 2;
  // per-row weights: D for rows in the quadratic zone, 0 otherwise (r_Jv is free between line searches)
  PAR_FOR(r, e.nefc) e.r_Jv[r] = (e.r_state[r] == ST_QUADRATIC) ? e.r_D[r] : 0.0f;
  SYNC();
  const float* w = e.r_Jv + nunit;
  // H = M + J^T diag(w) J  over the lower triangle (index table: m.tri_ij packs (i << 8) | j)
  PAR_FOR(idx, ntri) {
    const int ij = m.tri_ij[idx];
    const int i = ij >> 8, j = ij & 255;
    float h = e.M[i][j];
#pragma unroll 4
    for (int r = 0; r < nrow; r++) h += w[r] * e.J[r][i] * e.J[r][j];
    if (i == j) {
      int fr = m.dof_frow[i];
      if (fr >= 0) h += e.r_Jv[fr];
      int l0 = e.d_lrow[i][0], l1 = e.d_lrow[i][1];
      if (l0 >= 0) h += e.r_Jv[l0];
      if (l1 >= 0) h += e.r_Jv[l1];
    }
    e.H[i][j] = h;
  }
  // identity padding (rows nv..NV-1 still hold the previous factor, whose diagonal is stored as 0), as the CUDA variants
  // seed it from M: the padding column then holds 1, not rsqrt(1e-12)
  PAR_FOR(i, E::NV) if (i >= nv) e.H[i][i] = 1.0f;
  SYNC();
  // cone contacts (elliptic, middle zone): H += Jc^T Hc Jc, one contact at a time
  if (C::CONE == 1) {
    NOUNROLL for (int ci = 0; ci < e.ncon; ci++) {
      int r0 = nunit + e.con_row[ci];
      if (e.r_state[r0] != ST_CONE) continue;
      int dim = e.con_dim[ci];
      float mu = e.con_mu[ci];
      float* U = e.coneU;
      float* scl = e.coneS;
      float TT = 0;
      NOUNROLL for (int j = 1; j < dim; j++) { float u = e.r_jar[r0 + j] * e.con_fri[ci][j - 1]; TT += u * u; }
      float N = e.r_jar[r0] * mu, T = sqrtf(TT), invT = 1.0f / T;
      PAR_FOR(j, dim) {
        float sc = j == 0 ? mu : e.con_fri[ci][j - 1];
        scl[j] = sc; U[j] = e.r_jar[r0 + j] * sc * invT;      // unit tangential direction (see the CUDA variants)
      }
      SYNC();
      float Dm = e.r_D[r0] / fmaxf(LS_MINVAL, mu * mu * (1 + mu * mu));
      float kk = mu * N * invT, c2 = mu * mu - kk;
      // Y[a][d] = sum_b Hc[a][b] J[b][d]
      PAR_FOR(item, dim * nv) {
        int a = item / nv, d = item - a * nv;
        float y = 0;
        NOUNROLL for (int b = 0; b < dim; b++) {
          float h;
          if (a == 0 && b == 0) h = 1;
          else if (a == 0) h = -mu * U[b];
          else if (b == 0) h = -mu * U[a];
          else h = kk * U[a] * U[b] + (a == b ? c2 : 0.0f);
          y += Dm * h * scl[a] * scl[b] * e.J[r0 - nunit + b][d];
        }
        e.Y[a][d] = y;
      }
      SYNC();
      PAR_FOR(idx, ntri) {
        const int ij = m.tri_ij[idx];
        const int i = ij >> 8, j = ij & 255;
        float h = 0;
        NOUNROLL for (int a = 0; a < dim; a++) h += e.J[r0 - nunit + a][i] * e.Y[a][j];
        e.H[i][j] += h;
      }
      SYNC();
    }
  }
  chol_factor<E::NV, E::NVP>(ms, e.H);
}

#endif

struct LSPoint { float alpha, cost, d1, d2; };

// Per line search: for every elliptic contact the alpha-independent sums of the cone coordinates
// (UU, UV, VV -> r_aref[r..r+2]) and the coefficients of its bottom-zone quadratic qc(alpha) = c0 + c1 alpha + c2 alpha^2
// (-> r_force[r..r+2]).  r_aref is dead once jar has been formed and r_force is rewritten by the update_constraint that
// follows every line search (elliptic contacts have dim >= 3 rows, so the three slots per array exist).
template <class C>
LS_FN void ls_prepare(const int ms, EnvS<C>& e) {
  const int nefc = e.nefc;
  PAR_FOR(r, nefc) {
    const int ti = e.r_ti[r];
    if (ROW_TYPE(ti) != ROW_CON_ELLIPTIC || ROW_K(ti) != 0) continue;
    const int ci = ROW_ID(ti), dim = e.con_dim[ci];
    float ja = e.r_jar[r], jv = e.r_Jv[r], D = e.r_D[r];
    float UU = 0, UV = 0, VV = 0, c0 = 0.5f * D * ja * ja, c1 = D * ja * jv, c2 = 0.5f * D * jv * jv;
    NOUNROLL for (int j = 1; j < dim; j++) {
      const float fr = e.con_fri[ci][j - 1];
      const float aj = e.r_jar[r + j], vj = e.r_Jv[r + j], Dj = e.r_D[r + j];
      const float u = aj * fr, v = vj * fr;
      UU += u * u; UV += u * v; VV += v * v;
      c0 += 0.5f * Dj * aj * aj; c1 += Dj * aj * vj; c2 += 0.5f * Dj * vj * vj;
    }
    e.r_aref[r] = UU; e.r_aref[r + 1] = UV; e.r_aref[r + 2] = VV;
    e.r_force[r] = c0; e.r_force[r + 1] = c1; e.r_force[r + 2] = c2;
  }
  SYNC();
}

#if defined(LS_EMULATE)
static long g_ls_evals = 0, g_ls_searches = 0;
#endif
template <class C>
LS_FN LSPoint ls_eval(const int ms, const EnvS<C>& e, const float* qg, float alpha) {
#if defined(LS_EMULATE)
  g_ls_evals++;
#endif
  PH_T0(t);
  const DevModel& m = c_models[ms];
  const int nefc = e.nefc;
  float c = 0, d1 = 0, d2 = 0;
  PAR_FOR(r, nefc) {
    const int ti = e.r_ti[r];
    const int tp = ROW_TYPE(ti);
    float ja = e.r_jar[r], jv = e.r_Jv[r], D = e.r_D[r];
    float x = ja + alpha * jv;
    if (tp == ROW_FRICTION) {
      float f = PRM(dof_frictionloss)[ROW_ID(ti)], Rf = f / D;
      if (x <= -Rf) { c += f * (-0.5f * Rf - x); d1 += -f * jv; }
      else if (x >= Rf) { c += f * (-0.5f * Rf + x); d1 += f * jv; }
      else { c += 0.5f * D * x * x; d1 += D * x * jv; d2 += D * jv * jv; }
    } else if (tp == ROW_CON_ELLIPTIC) {
      if (ROW_K(ti) != 0) continue;
      // alpha-independent sums over the contact's rows were prepared once per line search (ls_prepare)
      const int ci = ROW_ID(ti);
      const float mu = e.con_mu[ci];
      const float U0 = ja * mu, V0 = jv * mu, UU = e.r_aref[r], UV = e.r_aref[r + 1], VV = e.r_aref[r + 2];
      const float c1 = e.r_force[r + 1], c2 = e.r_force[r + 2];
      const float qc = e.r_force[r] + alpha * (c1 + alpha * c2), q1 = c1 + 2 * alpha * c2, q2 = 2 * c2;
      float N = U0 + alpha * V0;
      float Tsqr = UU + alpha * (2 * UV + alpha * VV);
      if (Tsqr <= 0) {
        if (N < 0) { c += qc; d1 += q1; d2 += q2; }
      } else {
        float T = sqrtf(Tsqr);
        if (T < 1e-12f) { if (N < 0) { c += qc; d1 += q1; d2 += q2; } }
        else if (N >= mu * T) {
        } else if (mu * N + T <= 0) { c += qc; d1 += q1; d2 += q2; }
        else {
          float Dm = D / fmaxf(LS_MINVAL, mu * mu * (1 + mu * mu));
          // T'' = (VV T^2 - W^2) / T^3 >= 0 (Cauchy-Schwarz). In fp32 the difference of the two quotients VV/T - W^2/T^3
          // cancels catastrophically where the tangential velocity passes through ~0 on the search line and came out
          // hugely negative: d2 <= 0 -> "curvature" LS_MINVAL -> alpha ~ 1e18 -> non-finite state. Clamped numerator.
          const float W = UV + alpha * VV;
          float N1 = V0, T1 = W / T, T2 = fmaxf(0.0f, VV * Tsqr - W * W) / (T * Tsqr);
          float NmT = N - mu * T, s = N1 - mu * T1;
          c += 0.5f * Dm * NmT * NmT;
          d1 += Dm * NmT * s;
          d2 += Dm * (s * s + NmT * (-mu * T2));
        }
      }
    } else {
      if (x < 0) { c += 0.5f * D * x * x; d1 += D * x * jv; d2 += D * jv * jv; }
    }
  }
  c = WARP_SUM(c); d1 = WARP_SUM(d1); d2 = WARP_SUM(d2);
  c += alpha * alpha * qg[2] + alpha * qg[1] + qg[0];
  d1 += 2 * alpha * qg[2] + qg[1];
  d2 += 2 * qg[2];
  if (d2 <= 0) d2 = LS_MINVAL;
  LSPoint p = {alpha, c, d1, d2};
  PH_LAP(PH_LS_EVAL, t);
  PH_CNT(PH_LS_EVALS, 1);
#if defined(LS_EMULATE) && defined(LS_TRACE)
  printf("    ls_eval alpha %.6e cost %.9e d1 %.6e d2 %.6e (qg %.4e %.4e %.4e)\n", alpha, c, d1, d2, qg[0], qg[1], qg[2]);
#endif
  return p;
}

template <class C>
LS_FN float line_search(const int ms, EnvS<C>& e, const SolverOpts so, float gauss, float scale, float cost0) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv;
  float sn = 0, q1 = 0, q2 = 0, gs = 0;
  mulM(ms, e, e.Mv, e.search);
  mulJ(ms, e, e.r_Jv, e.search);
  SYNC();
  PAR_FOR(i, nv) {
    float s = e.search[i];
    sn += s * s;
    q1 += s * (e.Ma[i] - e.qfrc_smooth[i]);
    q2 += 0.5f * s * e.Mv[i];
    gs += s * e.grad[i];
  }
  sn = WARP_SUM(sn); q1 = WARP_SUM(q1); q2 = WARP_SUM(q2); gs = WARP_SUM(gs);
  float snorm = sqrtf(sn);
  if (snorm < LS_MINVAL) return 0;
  float gtol = so.tolerance * so.ls_tolerance * snorm / scale;
  float qg[3] = {gauss, q1, q2};
#if defined(LS_EMULATE)
  g_ls_searches++;
#endif
  if (C::CONE == 1) ls_prepare(ms, e);
  // The point alpha = 0 needs no evaluation: its cost is the current cost, its slope is grad . search and, because
  // search = -H^-1 grad with the exact Hessian of this point, its curvature search^T H search equals -slope.
  // (gs >= 0 -- the fp32 factorisation lost positive definiteness and `search` is not a descent direction -- is rare:
  //  then the point is evaluated honestly, so that its curvature is the true, positive one.)
  LSPoint p0 = {0.0f, cost0, gs, -gs};
  if (!(gs < 0)) p0 = ls_eval(ms, e, qg, 0.0f);
  LSPoint p1 = ls_eval(ms, e, qg, p0.alpha - p0.d1 / p0.d2);
  if (!(p1.cost <= p0.cost)) p1 = p0;               // (also catches a non-finite evaluation)
  if (fabsf(p1.d1) < gtol) return p1.alpha;
  int iter = 0;
  float dir = p1.d1 < 0 ? 1.0f : -1.0f;
  LSPoint p2 = p1;
  while (p1.d1 * dir <= -gtol && iter < so.ls_iter) {
    p2 = p1;
    p1 = ls_eval(ms, e, qg, p1.alpha - p1.d1 / p1.d2);
    iter++;
    if (fabsf(p1.d1) < gtol) return p1.alpha;
  }
  if (iter >= so.ls_iter) return p1.alpha;
  LSPoint lo = p2, hi = p1;
  LSPoint best = (p1.cost < p2.cost) ? p1 : p2;
  while (iter < so.ls_iter) {
    float amin = fminf(lo.alpha, hi.alpha), amax = fmaxf(lo.alpha, hi.alpha);
    // Newton from the better end if it stays inside the bracket, else bisect
    float a = best.alpha - best.d1 / best.d2;
    if (!(a > amin && a < amax)) a = 0.5f * (lo.alpha + hi.alpha);
    if (!(a > amin && a < amax)) break;
    LSPoint pm = ls_eval(ms, e, qg, a);
    iter++;
    if (pm.cost < best.cost) best = pm;
    if (fabsf(pm.d1) < gtol) return pm.alpha;
    if (pm.d1 * dir < 0) lo = pm; else hi = pm;
    best = (lo.cost < hi.cost) ? lo : hi;
  }
  return best.alpha;
}

// gradient of the cost at qacc (mj_solNewton: grad = M qacc - qfrc_smooth - J^T force); returns |grad|^2
template <class C>
LS_FN float update_gradient(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  float gn = 0;
  PAR_FOR(i, EnvS<C>::NV) {
    float g = i < m.nv ? e.Ma[i] - e.qfrc_smooth[i] - e.qfrc_constraint[i] : 0.0f;
    e.grad[i] = g; e.Mgrad[i] = g;
    gn += g * g;
  }
  gn = WARP_SUM(gn);
  SYNC();
  return gn;
}

template <class C>
LS_FN void fwd_constraint(const int ms, EnvS<C>& e, const SolverOpts so) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nefc = e.nefc;
  const float scale = 1.0f / (PRM(meaninertia)[0] * (nv > 1 ? nv : 1));
  float gauss = 0, cost = 0, gn = 0;
  int iter = 0;
  PH_T0(t);
  if (nefc == 0) {
    PAR_FOR(i, nv) { e.qacc[i] = e.qacc_smooth[i]; e.qfrc_constraint[i] = 0; }
    SYNC();
  } else {
    // ---- warmstart choice (mj_solNewton start point): the cost at qacc_smooth is evaluated FIRST, so that the states
    //      and forces left behind belong to the warmstart, which wins almost always and then needs no re-evaluation ----
    mulJ(ms, e, e.r_jar, e.qacc_smooth);
    SYNC();
    PAR_FOR(r, nefc) e.r_jar[r] -= e.r_aref[r];
    SYNC();
    const float cs = constraint_update(ms, e);          // (Gauss term is 0 at qacc_smooth)
    PAR_FOR(i, nv) e.qacc[i] = e.qacc_ws[i];
    SYNC();
    mulM(ms, e, e.Ma, e.qacc);
    mulJ(ms, e, e.r_Jv, e.qacc);
    SYNC();
    // jar <- J qacc_ws - aref, the smooth point's jar is parked in r_Jv
    PAR_FOR(r, nefc) { float t = e.r_jar[r]; e.r_jar[r] = e.r_Jv[r] - e.r_aref[r]; e.r_Jv[r] = t; }
    SYNC();
    const float cwc = constraint_update(ms, e);
    gauss = finish_constraint(ms, e);
    cost = cwc + gauss;
    if (cost > cs) {                                    // rare: fall back to the unconstrained acceleration
      PAR_FOR(i, nv) e.qacc[i] = e.qacc_smooth[i];
      PAR_FOR(r, nefc) e.r_jar[r] = e.r_Jv[r];
      SYNC();
      mulM(ms, e, e.Ma, e.qacc);
      SYNC();
      cost = update_constraint(ms, e, &gauss);
    }
    gn = update_gradient(ms, e);
  }
  // ---- Newton iterations ----
  // Order differs from mj_solNewton in one respect: the convergence test comes BEFORE the Hessian of the new point is
  // assembled and factored, so the last iteration's factorisation (never used) is not computed.
  // fp32 termination: scaled gradient below tolerance, or a Newton step with exact line search that did not lower the
  // cost any more (the cost value has reached its fp32 resolution; further iterations only move noise).
  bool active = nefc > 0 && so.max_iter > 0 && scale * sqrtf(gn) >= so.tolerance;
  bool force_dirty = false;   // ls_prepare borrows r_force / r_aref of the elliptic rows
  PH_LAP(PH_WARMSTART, t);
  while (BLOCK_ANY(so.sync_iters, active)) {
    PH_LAP(PH_NEWTON_WAIT, t);
    PH_CNT(PH_NEWTON_TRIPS, 1);
    // (warps whose env has converged keep passing the same barriers until the whole block is done)
    if (active) make_hessian(ms, e);
    BLOCK_SYNC(so.sync_phases & 64);
    PH_LAP(PH_MAKE_HESSIAN, t);
    float alpha = 0;
    if (active) {
      chol_solve<EnvS<C>::NV, EnvS<C>::NVP>(e.H, e.Mgrad);
      PAR_FOR(i, EnvS<C>::NV) e.search[i] = i < nv ? -e.Mgrad[i] : 0.0f;   // (padding read by the unrolled J product)
      SYNC();
      PH_LAP(PH_CHOL_SOLVE, t);
      alpha = line_search(ms, e, so, gauss, scale, cost);
      if (!(fabsf(alpha) <= 1e30f)) alpha = 0;      // never step to a non-finite point
      if (alpha == 0) { active = false; force_dirty = (C::CONE == 1); }
    }
    BLOCK_SYNC(so.sync_phases & 128);
    PH_LAP(PH_LINE_SEARCH, t);
    if (active) {
      PAR_FOR(i, nv) { e.qacc[i] += alpha * e.search[i]; e.Ma[i] += alpha * e.Mv[i]; }
      PAR_FOR(r, nefc) e.r_jar[r] += alpha * e.r_Jv[r];
      SYNC();
      const float oldcost = cost;
      cost = update_constraint(ms, e, &gauss);
      PH_LAP(PH_UPDATE_CONSTRAINT, t);
      gn = update_gradient(ms, e);
      PH_LAP(PH_UPDATE_GRADIENT, t);
      iter++;
#if defined(LS_EMULATE) && defined(LS_TRACE)
      printf("  it %2d alpha %.3e cost %.9e impr %.3e grad %.3e nefc %d\n", iter, alpha, cost, scale * (oldcost - cost),
             scale * sqrtf(gn), nefc);
#endif
      active = iter < so.max_iter && scale * sqrtf(gn) >= so.tolerance && cost < oldcost;
    }
  }
  PH_LAP(PH_NEWTON_WAIT, t);                                  // (the barrier that ended the loop)
  if (force_dirty) cost = update_constraint(ms, e, &gauss);   // rare: restore efc_force for contact_forces()
  LANE0 { e.solver_iter = iter; e.iter_sum += iter; }
  PAR_FOR(i, nv) e.qacc_ws[i] = e.qacc[i];
  SYNC();
  PH_LAP(PH_NEWTON_TAIL, t);
  PH_CNT(PH_NEWTON_ITERS, iter);
}

// ----------------------------------------------------------------------------------------------------------
// forward dynamics + integrators
// ----------------------------------------------------------------------------------------------------------
template <class C>
LS_FN void forward(const int ms, EnvS<C>& e, const SolverOpts so) {
  const DevModel& m = c_models[ms];
  BLOCK_SYNC(so.sync_phases & 1);
#if defined(LS_EMULATE)
  g_forward_evals++;
#endif
  PH_T0(t);
  kinematics(ms, e);
  BLOCK_SYNC(so.sync_phases & 2);
  PH_LAP(PH_KINEMATICS, t);
  com_pos(ms, e);
  PH_LAP(PH_COM_POS, t);
  crb_factor(ms, e);
  BLOCK_SYNC(so.sync_phases & 4);
  PH_LAP(PH_CRB_FACTOR, t);
  smooth_forces(ms, e);        // last user of the smooth-dynamics scratch that the constraint rows overlay
  BLOCK_SYNC(so.sync_phases & 8);
  PH_LAP(PH_SMOOTH_FORCES, t);
  collision(ms, e);
  BLOCK_SYNC(so.sync_phases & 16);
  PH_LAP(PH_COLLISION, t);
  make_constraint(ms, e);
  BLOCK_SYNC(so.sync_phases & 32);
  PH_LAP(PH_MAKE_CONSTRAINT, t);
  fwd_constraint(ms, e, so);
}

// whether qpos or qvel is non-finite at any of the env's nv dofs, or `bad` (a caller's test of further entries, per lane)
// is set on any lane: the same answer on every lane of the warp
template <class C>
LS_DEV bool nonfinite_state(const EnvS<C>& e, const int nv, bool bad = false) {
  PAR_FOR(i, nv) bad |= !(isfinite(e.qpos[i]) && isfinite(e.qvel[i]));
#ifndef LS_EMULATE
  bad = __any_sync(0xffffffffu, bad);
#endif
  return bad;
}

// ----------------------------------------------------------------------------------------------------------
// inverse dynamics (locosim_inverse): MuJoCo 2.3.7's continuous-time mj_inverse
// ----------------------------------------------------------------------------------------------------------
// qfrc_smooth = passive - bias: passes (A) - (C) of smooth_forces without the applied and actuator forces, which mj_inverse
// does not subtract. Kept apart from smooth_forces, whose code the step kernels must keep unchanged; qfrc_smooth lies
// outside the storage that collision() and make_constraint() overwrite.
template <class C>
LS_FN void passive_bias(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv;
  PAR_FOR(j, nv) {
    unsigned mask = (unsigned)m.body_dofmask[m.jnt_bodyid[j]] & ((1u << j) - 1u);
    float v[6] = {0, 0, 0, 0, 0, 0};
    while (mask) {
      const int i = LS_FFS(mask) - 1;
      mask &= mask - 1;
      const float qv = e.qvel[i];
      for (int c = 0; c < 6; c++) v[c] = fmaf(e.cdof[i][c], qv, v[c]);
    }
    float cdd[6];
    crossMotion(cdd, v, e.cdof[j]);
    for (int c = 0; c < 6; c++) e.cdof_dot[j][c] = cdd[c];
  }
  SYNC();
  PAR_FOR(b, m.nb) {
    float* f = e.crb[b];
    if (b == 0) { for (int k = 0; k < 6; k++) f[k] = 0; continue; }
    unsigned mask = (unsigned)m.body_dofmask[b];
    float cvel[6] = {0, 0, 0, 0, 0, 0}, cacc[6] = {0, 0, 0, -m.gravity[0], -m.gravity[1], -m.gravity[2]};
    while (mask) {
      const int i = LS_FFS(mask) - 1;
      mask &= mask - 1;
      const float qv = e.qvel[i];
      for (int c = 0; c < 6; c++) { cvel[c] = fmaf(e.cdof[i][c], qv, cvel[c]); cacc[c] = fmaf(e.cdof_dot[i][c], qv, cacc[c]); }
    }
    float t1[6], t2[6], t3[6];
    mulInertVec(t1, e.cinert[b], cacc);
    mulInertVec(t2, e.cinert[b], cvel);
    crossForce(t3, cvel, t2);
    for (int k = 0; k < 6; k++) f[k] = t1[k] + t3[k];
  }
  SYNC();
  PAR_FOR(j, nv) {
    float F[6] = {0, 0, 0, 0, 0, 0};
    NOUNROLL for (int b = 1; b < m.nb; b++) {
      if (!((m.body_dofmask[b] >> j) & 1)) continue;
      for (int c = 0; c < 6; c++) F[c] += e.crb[b][c];
    }
    float bias = 0;
    for (int c = 0; c < 6; c++) bias += e.cdof[j][c] * F[c];
    float passive = -PRM(jnt_stiffness)[j] * (e.qpos[j] - m.qpos_spring[j]) - PRM(dof_damping)[j] * e.qvel[j];
    e.qfrc_smooth[j] = passive - bias;
  }
  SYNC();
}

// qfrc_inverse = M qacc + bias - passive - J^T efc_force into out[0, nv), for the state e.qpos / e.qvel, the acceleration
// e.qacc and the parameters e.prm (the caller has run init_workspace; entries >= nv of e.qacc are 0). efc_force is the
// solver's soft-constraint map (constraint_update) of jar = J qacc - aref over the rows the state gives: the contact set
// of collision() and the row cap of make_constraint(), as in forward(). A non-finite qpos, qvel or qacc gives a row of
// zeros before anything reaches collision(). A whole-warp call; it writes nothing but out and the env's working set.
template <class C>
LS_FN void inverse_dynamics(const int ms, EnvS<C>& e, float* out) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv;
  bool bad = false;
  PAR_FOR(i, nv) bad |= !isfinite(e.qacc[i]);
  if (nonfinite_state(e, nv, bad)) {
    PAR_FOR(i, nv) out[i] = 0.0f;
    SYNC();
    return;
  }
  kinematics(ms, e);
  com_pos(ms, e);
  crb_factor(ms, e);
  passive_bias(ms, e);         // (before collision: the constraint rows overlay the scratch it reads)
  collision(ms, e);
  make_constraint(ms, e);
  const int nefc = e.nefc, nunit = e.nunit, nrow = e.nrow;
  mulJ(ms, e, e.r_jar, e.qacc);
  SYNC();
  PAR_FOR(r, nefc) e.r_jar[r] -= e.r_aref[r];
  SYNC();
  constraint_update(ms, e);
  mulM(ms, e, e.Ma, e.qacc);
  SYNC();
  // J^T efc_force in finish_constraint's order (its Gauss term reads qacc_smooth, which this path does not compute)
  PAR_FOR(d, nv) {
    float a = 0;
    const int fr = m.dof_frow[d];
    if (fr >= 0) a += e.r_force[fr];
    const int l0 = e.d_lrow[d][0], l1 = e.d_lrow[d][1];
    if (l0 >= 0) a += e.r_force[l0];
    if (l1 >= 0) a -= e.r_force[l1];
    for (int r = 0; r < nrow; r++) a = fmaf(e.J[r][d], e.r_force[nunit + r], a);
    out[d] = e.Ma[d] - e.qfrc_smooth[d] - a;
  }
  SYNC();
}

// ----------------------------------------------------------------------------------------------------------
// dynamics terms (locosim_dynamics_terms): M, qfrc_bias, qfrc_passive, the whole-robot CoM and mass, mj_jacBody at xpos of
// every body and mj_jacSubtreeCom of the robot
// ----------------------------------------------------------------------------------------------------------
// one env's rows of the outputs (each may be NULL): M [nv, nv], bias [nv], passive [nv], com [LS_COM_DIM], jac [nb, 6, nv],
// jac_com [3, nv]
struct DynOut {
  float *M, *bias, *passive, *com, *jac, *jac_com;
};

// The terms for the state e.qpos / e.qvel and the parameters e.prm (the caller has run init_workspace). A non-finite qpos
// or qvel gives zero rows. Each output is written with nv innermost, one lane per entry.
//   M:        crb_factor's e.M (dof_armature included).
//   com:      com_pos's e.com, then the total mass summed as com_pos sums it.
//   jac:      column d of body b, for d on b's chain: cdof[d] = (w, v) at e.com moved to xpos_b, (w, v + w x (xpos_b - com)),
//             as body_outputs moves the velocity; 0 elsewhere.
//   jac_com:  column d = (m_sub v + w x h_sub) / m_total, m_sub and h_sub the mass and first moment about e.com of the
//             subtree of d's body, which crb_factor's composite inertia crb holds (entries 9 and 6-8).
//   bias / passive: passive_bias's passes (A) and (B) (RNE at qacc = 0 with gravity; the body forces are left in e.crb), then
//             its pass (C) here with the two terms kept apart. passive_bias itself is called unchanged, so inverse_kernel
//             keeps its code; it overwrites crb, so the Jacobians are written first.
// A whole-warp call; it writes nothing but the outputs and the env's working set.
template <class C>
LS_FN void dynamics_terms(const int ms, EnvS<C>& e, const DynOut o) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nb = m.nb;
  if (nonfinite_state(e, nv)) {
    if (o.M) PAR_FOR(k, nv * nv) o.M[k] = 0.0f;
    if (o.bias) PAR_FOR(k, nv) o.bias[k] = 0.0f;
    if (o.passive) PAR_FOR(k, nv) o.passive[k] = 0.0f;
    if (o.com) PAR_FOR(k, LS_COM_DIM) o.com[k] = 0.0f;
    if (o.jac) PAR_FOR(k, nb * 6 * nv) o.jac[k] = 0.0f;
    if (o.jac_com) PAR_FOR(k, 3 * nv) o.jac_com[k] = 0.0f;
    SYNC();
    return;
  }
  kinematics(ms, e);
  com_pos(ms, e);
  if (o.M || o.jac_com) crb_factor(ms, e);
  float mass = 0;
  PAR_FOR(b, nb) mass += PRM(body_mass)[b];
  mass = WARP_SUM(mass);
  if (o.M) PAR_FOR(k, nv * nv) {
    const int i = k / nv;
    o.M[k] = e.M[i][k - i * nv];
  }
  if (o.com) PAR_FOR(k, LS_COM_DIM) o.com[k] = k < 3 ? e.com[k] : mass;
  if (o.jac) PAR_FOR(k, nb * 6 * nv) {
    const int br = k / nv, d = k - br * nv, b = br / 6, r = br - 6 * b;
    float x = 0.0f;
    if (b > 0 && ((m.body_dofmask[b] >> d) & 1)) {
      const float* cd = e.cdof[d];
      if (r < 3) {
        x = cd[r];
      } else {
        const int c = r - 3, c1 = c == 2 ? 0 : c + 1, c2 = c == 0 ? 2 : c - 1;
        const float p1 = e.xpos[b][c1] - e.com[c1], p2 = e.xpos[b][c2] - e.com[c2];
        x = cd[r] + (cd[c1] * p2 - cd[c2] * p1);
      }
    }
    o.jac[k] = x;
  }
  if (o.jac_com) {
    const float inv = 1.0f / mass;
    PAR_FOR(k, 3 * nv) {
      const int c = k / nv, d = k - c * nv, c1 = c == 2 ? 0 : c + 1, c2 = c == 0 ? 2 : c - 1;
      const float* cd = e.cdof[d];
      const float* h = e.crb[m.jnt_bodyid[d]];
      o.jac_com[k] = (h[9] * cd[3 + c] + (cd[c1] * h[6 + c2] - cd[c2] * h[6 + c1])) * inv;
    }
  }
  SYNC();
  if (o.bias || o.passive) {
    passive_bias(ms, e);
    PAR_FOR(j, nv) {
      float F[6] = {0, 0, 0, 0, 0, 0};
      NOUNROLL for (int b = 1; b < nb; b++) {
        if (!((m.body_dofmask[b] >> j) & 1)) continue;
        for (int c = 0; c < 6; c++) F[c] += e.crb[b][c];
      }
      float bias = 0;
      for (int c = 0; c < 6; c++) bias += e.cdof[j][c] * F[c];
      if (o.bias) o.bias[j] = bias;
      if (o.passive) o.passive[j] = -PRM(jnt_stiffness)[j] * (e.qpos[j] - m.qpos_spring[j]) - PRM(dof_damping)[j] * e.qvel[j];
    }
    SYNC();
  }
}

template <class C>
LS_FN void euler_step(const int ms, EnvS<C>& e) {
  const DevModel& m = c_models[ms];
  typedef EnvS<C> E;
  const int nv = m.nv;
  const float h = m.timestep;
  if (m.has_damping) {
    // (M + h*diag(damping)) qacc = qfrc_smooth + qfrc_constraint   (mj_Euler, implicit in joint damping)
    PAR_FOR(idx, E::NV * E::NVP) (&e.H[0][0])[idx] = (&e.M[0][0])[idx];
    SYNC();
    PAR_FOR(i, E::NV) {
      if (i < nv) { e.H[i][i] += h * PRM(dof_damping)[i]; e.Mgrad[i] = e.qfrc_smooth[i] + e.qfrc_constraint[i]; }
      else e.Mgrad[i] = 0.0f;
    }
    SYNC();
    chol_factor<E::NV, E::NVP>(ms, e.H);
    chol_solve<E::NV, E::NVP>(e.H, e.Mgrad);
    PAR_FOR(i, nv) { float v = e.qvel[i] + h * e.Mgrad[i]; e.qvel[i] = v; e.qpos[i] += h * v; }
  } else {
    PAR_FOR(i, nv) { float v = e.qvel[i] + h * e.qacc[i]; e.qvel[i] = v; e.qpos[i] += h * v; }
  }
  SYNC();
}

template <class C>
LS_FN void rk4_step(const int ms, EnvS<C>& e, const SolverOpts so) {
  const DevModel& m = c_models[ms];
  // classic RK4 (mj_RungeKutta N=4); forward() for stage 0 has already been evaluated by the caller
  const int nv = m.nv;
  const float h = m.timestep;
  PAR_FOR(i, nv) {
    e.x0q[i] = e.qpos[i]; e.x0v[i] = e.qvel[i];
    e.accq[i] = e.qvel[i] * (1.0f / 6); e.accv[i] = e.qacc[i] * (1.0f / 6);
  }
  SYNC();
  const float A[3] = {0.5f, 0.5f, 1.0f};
  const float B[3] = {1.0f / 3, 1.0f / 3, 1.0f / 6};
  for (int s = 0; s < 3; s++) {
    PAR_FOR(i, nv) {
      float fv = e.qvel[i], fa = e.qacc[i];   // F[s] = (qvel, qacc) of the previous stage
      e.qpos[i] = e.x0q[i] + h * A[s] * fv;
      e.qvel[i] = e.x0v[i] + h * A[s] * fa;
    }
    SYNC();
    forward(ms, e, so);
    PAR_FOR(i, nv) { e.accq[i] += B[s] * e.qvel[i]; e.accv[i] += B[s] * e.qacc[i]; }
    SYNC();
  }
  PAR_FOR(i, nv) { e.qvel[i] = e.x0v[i] + h * e.accv[i]; e.qpos[i] = e.x0q[i] + h * e.accq[i]; }
  SYNC();
}

// mj_contactForce: the contact-frame force of contact ci (normal, tangent 1, tangent 2, torsion, rolling 1, rolling 2; zeros
// past its dim) from the constraint forces of the last forward evaluation
template <class C>
LS_DEV void contact_frame_force(const EnvS<C>& e, const int ci, float* f) {
  const int r0 = e.nunit + e.con_row[ci], dim = e.con_dim[ci];
#pragma unroll
  for (int j = 0; j < 6; j++) f[j] = 0;
  if (dim == 1) f[0] = e.r_force[r0];
  else if (C::CONE == 1) {
#pragma unroll
    for (int j = 0; j < 6; j++) if (j < dim) f[j] = e.r_force[r0 + j];
  } else {
    // mju_decodePyramid: normal = sum of the edge forces, component i = (f_2(i-1) - f_2(i-1)+1) * mu_(i-1)
    const int ne = 2 * (dim - 1);
    NOUNROLL for (int j = 0; j < ne; j++) f[0] += e.r_force[r0 + j];
#pragma unroll
    for (int j = 1; j < 6; j++)
      if (j < dim) f[j] = (e.r_force[r0 + 2 * (j - 1)] - e.r_force[r0 + 2 * (j - 1) + 1]) * e.con_fri[ci][j - 1];
  }
}

// contact outputs (locosim_set_contact_outputs): per body the wrench its contacts of this sub-step's last forward evaluation
// exert on it (force, and torque about xpos, world frame), accumulated into the env's row of the caller's buffer as the mean
// over the control step's n_sub sub-steps: global sub-step k = 0 writes, later ones add, k = n_sub - 1 scales by 1 / n_sub.
// The buffer is the only carry, so the sub-step and persistent kernels need no field of their own. One lane per body, each
// scanning the contact list in list order: the same summation order in every kernel, and no atomics. The row is read past L1
// (the persistent kernel: another SM may have written it in an earlier chunk of the step).
// After the last sub-step the row of a non-finite env is zeroed, as its observation is (the epilogue's test on the same
// state; made here rather than in the epilogue, where it costs every step kernel spills whether or not anything is
// registered). The sub-step index lives in EnvS::substep, not in an argument: a value live across the sub-step changes
// the step kernels' register allocation and stack frames whether or not anything is registered.
template <class C>
LS_FN void contact_wrench(const int ms, EnvS<C>& e) {
  static_assert(C::NB <= 32, "contact_wrench: one lane per body");
  const int k = e.substep;
  if (k < 0) return;
  const DevModel& m = c_models[ms];
  const int n_sub = c_contact[ms].n_substeps;
  float* row = c_contact[ms].wrench + (size_t)e.env * m.nb * LS_CONTACT_DIM;
  const int ncon = e.ncon;
  bool bad = false;
  if (k == n_sub - 1) {
    PAR_FOR(i, m.nv) bad |= !(isfinite(e.qpos[i]) && isfinite(e.qvel[i]));
#ifndef LS_EMULATE
    bad = __any_sync(0xffffffffu, bad);
#endif
  }
  PAR_FOR(b, m.nb) {
    float w[6] = {0, 0, 0, 0, 0, 0};
    if (b > 0) {                                   // (the world row stays exact zeros)
      NOUNROLL for (int ci = 0; ci < ncon; ci++) {
        const int b1 = m.geom_bodyid[e.con_g1[ci]], b2 = m.geom_bodyid[e.con_g2[ci]];
        if (b != b1 && b != b2) continue;
        float f[6];
        contact_frame_force(e, ci, f);
        const float* fr = e.con_frame[ci];
        float F[3], T[3], rxF[3];
        for (int c = 0; c < 3; c++) {
          F[c] = f[0] * fr[c] + f[1] * fr[3 + c] + f[2] * fr[6 + c];
          T[c] = f[3] * fr[c] + f[4] * fr[3 + c] + f[5] * fr[6 + c];
        }
        const float r[3] = {e.con_pos[ci][0] - e.xpos[b][0], e.con_pos[ci][1] - e.xpos[b][1], e.con_pos[ci][2] - e.xpos[b][2]};
        cross3(rxF, r, F);
        // the frame normal points from geom1 to geom2: +wrench on geom2's body, - on geom1's (mj_rnePostConstraint)
        const float s = b == b2 ? 1.0f : -1.0f;
        for (int c = 0; c < 3; c++) { w[c] += s * F[c]; w[3 + c] += s * (rxF[c] + T[c]); }
      }
    }
    float* dst = row + b * LS_CONTACT_DIM;
    for (int c = 0; c < LS_CONTACT_DIM; c++) {
      float v = k == 0 ? w[c] : LS_LDCG(dst + c) + w[c];
      if (k == n_sub - 1) v = bad ? 0.0f : v * (1.0f / (float)n_sub);
      dst[c] = v;
    }
  }
  SYNC();
  LANE0 e.substep = k + 1;
  SYNC();
}

// dof outputs (locosim_set_dof_outputs): per dof qfrc_actuator (summed over the dof's actuators in actuator order from the
// scratch smooth_forces wrote), qfrc_constraint and qacc of this sub-step's last forward evaluation, accumulated into the
// env's row of the caller's buffer as the contact outputs are: global sub-step k = 0 writes, later ones add, k = n_sub - 1
// scales by 1 / n_sub and zeroes a non-finite env. One lane per dof, the same order in every kernel, no atomics; rows and
// scratch are read past L1 (the persistent kernel: another SM may have written the row in an earlier chunk of the step).
// Runs before contact_wrench and advances EnvS::substep only when contact_wrench will not.
template <class C>
LS_FN void dof_outputs(const int ms, EnvS<C>& e) {
  const int k = e.substep;
  if (k < 0) return;
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nu = m.nu, n_sub = c_dof[ms].n_substeps;
  float* row = c_dof[ms].out + (size_t)e.env * nv * LS_DOF_DIM;
  const float* act = c_dof_act[ms] + (size_t)e.env * nu;
  bool bad = false;
  if (k == n_sub - 1) {
    PAR_FOR(i, nv) bad |= !(isfinite(e.qpos[i]) && isfinite(e.qvel[i]));
#ifndef LS_EMULATE
    bad = __any_sync(0xffffffffu, bad);
#endif
  }
  PAR_FOR(j, nv) {
    float fa = 0;
    NOUNROLL for (int i = 0; i < nu; i++) if (m.actuator_dof[i] == j) fa += m.actuator_gear[i] * LS_LDCG(act + i);
    const float w[LS_DOF_DIM] = {fa, e.qfrc_constraint[j], e.qacc[j]};
    float* dst = row + j * LS_DOF_DIM;
    for (int c = 0; c < LS_DOF_DIM; c++) {
      float v = k == 0 ? w[c] : LS_LDCG(dst + c) + w[c];
      if (k == n_sub - 1) v = bad ? 0.0f : v * (1.0f / (float)n_sub);
      dst[c] = v;
    }
  }
  SYNC();
  if (!c_contact[ms].wrench) {
    LANE0 e.substep = k + 1;
    SYNC();
  }
}

// contact list (locosim_set_contact_list_outputs): at the control step's last sub-step (k == n_sub - 1) the contact list of
// its last forward evaluation, in list order, into the env's rows of the caller's buffers: lane ci writes row ci, contacts
// below ncon from EnvS (the frame, position and dist of fill_contact; f of contact_frame_force, as mj_contactForce), every
// other row zeros and ids -1; a non-finite env (the epilogue's test on the same state) gets ncon = 0. Earlier sub-steps
// write nothing. Runs before dof_outputs and contact_wrench and advances EnvS::substep only when neither will.
template <class C>
LS_FN void contact_list(const int ms, EnvS<C>& e) {
  static_assert(C::MAXCON <= 32, "contact_list: one lane per contact");
  const int k = e.substep;
  if (k < 0) return;
  const DevConList& cl = c_conlist[ms];
  if (k == cl.n_substeps - 1) {
    const DevModel& m = c_models[ms];
    bool bad = false;
    PAR_FOR(i, m.nv) bad |= !(isfinite(e.qpos[i]) && isfinite(e.qvel[i]));
#ifndef LS_EMULATE
    bad = __any_sync(0xffffffffu, bad);
#endif
    const int ncon = bad ? 0 : e.ncon;
    float* rows = c_conrows[ms].con + (size_t)e.env * C::MAXCON * LS_CONLIST_DIM;
    int* ids = c_conrows[ms].id + (size_t)e.env * C::MAXCON * LS_CONLIST_ID_DIM;
    PAR_FOR(ci, C::MAXCON) {
      float* r = rows + ci * LS_CONLIST_DIM;
      int* d = ids + ci * LS_CONLIST_ID_DIM;
      if (ci < ncon) {
        float f[6];
        contact_frame_force(e, ci, f);
        const int g1 = e.con_g1[ci], g2 = e.con_g2[ci];
        r[LS_CONLIST_DIST] = e.con_dist[ci];
        for (int c = 0; c < 3; c++) r[LS_CONLIST_POS + c] = e.con_pos[ci][c];
        for (int c = 0; c < 9; c++) r[LS_CONLIST_FRAME + c] = e.con_frame[ci][c];
        for (int c = 0; c < 6; c++) r[LS_CONLIST_FORCE + c] = f[c];
        d[LS_CONLIST_GEOM1] = g1; d[LS_CONLIST_GEOM2] = g2;
        d[LS_CONLIST_BODY1] = m.geom_bodyid[g1]; d[LS_CONLIST_BODY2] = m.geom_bodyid[g2];
        d[LS_CONLIST_CONDIM] = e.con_dim[ci];
      } else {
        for (int c = 0; c < LS_CONLIST_DIM; c++) r[c] = 0.0f;
        for (int c = 0; c < LS_CONLIST_ID_DIM; c++) d[c] = -1;
      }
    }
    LANE0 cl.ncon[e.env] = ncon;
    SYNC();
  }
  if (!c_dof[ms].out && !c_contact[ms].wrench) {
    LANE0 e.substep = k + 1;
    SYNC();
  }
}

// use_foot_forces (base.py:623-631,656-679 -> mushroom _get_collision_force -> mj_contactForce): per foot group the
// contact-frame force (normal, tangent 1, tangent 2) of the FIRST contact between the floor and a geom of the group, in
// contact-list order, from the constraint forces of the sub-step's (last) forward evaluation; summed over sub-steps. Then
// the contact list, the dof outputs and the contact outputs of the sub-step, each while registered.
template <class C>
LS_FN void contact_forces(const int ms, EnvS<C>& e, const int* grf_group, int n_grf) {
  const int nunit = e.nunit, ncon = e.ncon;
  // lane ci looks at contact ci (ncon <= MAXCON <= 32); the first match of every group is a warp-wide minimum.
  // (A scalar "scan the list until the first match" loop was miscompiled by nvcc 12.9 for the pyramidal
  //  instantiations: the membership test read contact ci+1 while the forces were taken from contact ci.)
  int ga = -1, gb = -1;
  const int lane = LS_LANE;
#ifdef LS_EMULATE
  for (int k = 0; k < n_grf; k++) {
    int first = ncon;
    for (int ci = ncon - 1; ci >= 0; ci--) {
      ga = grf_group[e.con_g1[ci]]; gb = grf_group[e.con_g2[ci]];
      if ((ga == LS_GRF_FLOOR && gb == k) || (gb == LS_GRF_FLOOR && ga == k)) first = ci;
    }
#else
  if (n_grf > 0 && lane < ncon) { ga = grf_group[e.con_g1[lane]]; gb = grf_group[e.con_g2[lane]]; }
  for (int k = 0; k < n_grf; k++) {
    const bool hit = (ga == LS_GRF_FLOOR && gb == k) || (gb == LS_GRF_FLOOR && ga == k);
    const unsigned mask = __ballot_sync(0xffffffffu, hit);
    const int first = mask ? __ffs(mask) - 1 : ncon;
#endif
    if (first >= ncon) continue;
    LANE0 {
      float f[6];
      contact_frame_force(e, first, f);
      e.grf[3 * k] += f[0]; e.grf[3 * k + 1] += f[1]; e.grf[3 * k + 2] += f[2];
    }
  }
  SYNC();
  if (c_conlist[ms].ncon) contact_list(ms, e);
  if (c_dof[ms].out) dof_outputs(ms, e);
  if (c_contact[ms].wrench) contact_wrench(ms, e);
}

template <class C>
LS_FN void physics_substeps(const int ms, EnvS<C>& e, const SolverOpts so, int nsub, const int* grf_group, int n_grf) {
  const DevModel& m = c_models[ms];
  for (int k = 0; k < nsub; k++) {
    PH_T0(t_sub);
    forward(ms, e, so);
    PH_T0(t);
    if constexpr (C::RK4 == 1) rk4_step(ms, e, so); else euler_step(ms, e);
    // (the contact and dof outputs and the contact list are written from contact_forces' call rather than calls of their own:
    //  another call site here changes the step kernels' register allocation and spills whether or not anything is registered)
    if (n_grf > 0 || c_contact[ms].wrench || c_dof[ms].out || c_conlist[ms].ncon) contact_forces(ms, e, grf_group, n_grf);
    PH_LAP(PH_INTEGRATOR, t);
    PH_LAP(PH_SUBSTEP, t_sub);
    PH_CNT(PH_SUBSTEPS, 1);
  }
}

// ----------------------------------------------------------------------------------------------------------
// forward dynamics outputs (locosim_forward): one mj_forward, then mj_rnePostConstraint's body accelerations and forces
// ----------------------------------------------------------------------------------------------------------
// one env's rows of the outputs (each may be NULL): dof [nv, LS_DOF_DIM], body_acc [nb, LS_BODY_ACC_DIM], cfrc_int and
// cfrc_ext [nb, LS_CONTACT_DIM]
struct FwdOut {
  float *dof, *body_acc, *cfrc_int, *cfrc_ext;
};

// The outputs of the forward evaluation forward() has just made (the caller ran it at e.qpos / e.qvel / e.ctrl). In order:
//   (1) the dof row: per dof the sum of gear * actuator_force over its actuators in actuator order, qfrc_constraint and
//       qacc, read before anything below overwrites the storage they share with cinert / cdof_dot;
//   (2) cfrc_ext from the contacts, one lane per body, as contact_wrench sums them (force, torque about xpos, world);
//   (3) kinematics and com_pos again (xipos, ximat, cinert and the joint frames lie under the constraint rows; both are
//       deterministic functions of qpos, so xpos, com and cdof come out with the same bits), cdof_dot as passive_bias
//       builds it, and the applied wrench xfrc_applied[b], moved from xipos to xpos, added to cfrc_ext;
//   (4) per body cvel and cacc = -g + sum over its chain of (cdof qacc + cdof_dot qvel) (spatial, about com); body_acc is
//       mj_objectAcceleration at xpos: (alpha, a + alpha x r + w x (v + w x r)), r = xpos - com; the body force
//       f = cinert cacc + cvel x* (cinert cvel) - cfrc_ext (about com);
//   (5) cfrc_int[b] = the sum of f over b's subtree (b and its descendants, in body order), moved to xpos.
// cfrc_ext and f are kept in e.H (the Newton Hessian's factor, dead after the solve). Row 0 of body_acc is (0, -g), of
// cfrc_int and cfrc_ext zeros. A whole-warp call; it writes nothing but the outputs and the env's working set.
template <class C>
LS_FN void forward_outputs(const int ms, EnvS<C>& e, const FwdOut o) {
  typedef EnvS<C> E;
  static_assert(C::NB <= 32, "forward_outputs: one lane per body");
  static_assert(2 * E::NB * 6 <= E::NV * E::NVP, "forward_outputs: cfrc_ext and the body forces fit in H");
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nb = m.nb, nu = m.nu;
  if (o.dof) PAR_FOR(j, nv) {
    float fa = 0;
    NOUNROLL for (int i = 0; i < nu; i++) if (m.actuator_dof[i] == j) fa += m.actuator_gear[i] * actuator_force(m, e, i);
    float* dst = o.dof + j * LS_DOF_DIM;
    dst[0] = fa; dst[1] = e.qfrc_constraint[j]; dst[2] = e.qacc[j];
  }
  SYNC();
  if (!o.body_acc && !o.cfrc_int && !o.cfrc_ext) return;
  float (*ext)[6] = reinterpret_cast<float (*)[6]>(&e.H[0][0]);
  float (*frc)[6] = ext + E::NB;
  const bool need_ext = o.cfrc_ext || o.cfrc_int;
  if (need_ext) {
    const int ncon = e.ncon;
    PAR_FOR(b, nb) {
      float w[6] = {0, 0, 0, 0, 0, 0};
      if (b > 0) {
        NOUNROLL for (int ci = 0; ci < ncon; ci++) {
          const int b1 = m.geom_bodyid[e.con_g1[ci]], b2 = m.geom_bodyid[e.con_g2[ci]];
          if (b != b1 && b != b2) continue;
          float f[6];
          contact_frame_force(e, ci, f);
          const float* fr = e.con_frame[ci];
          float F[3], T[3], rxF[3];
          for (int c = 0; c < 3; c++) {
            F[c] = f[0] * fr[c] + f[1] * fr[3 + c] + f[2] * fr[6 + c];
            T[c] = f[3] * fr[c] + f[4] * fr[3 + c] + f[5] * fr[6 + c];
          }
          const float r[3] = {e.con_pos[ci][0] - e.xpos[b][0], e.con_pos[ci][1] - e.xpos[b][1], e.con_pos[ci][2] - e.xpos[b][2]};
          cross3(rxF, r, F);
          const float s = b == b2 ? 1.0f : -1.0f;    // (the frame normal points from geom1 to geom2)
          for (int c = 0; c < 3; c++) { w[c] += s * F[c]; w[3 + c] += s * (rxF[c] + T[c]); }
        }
      }
      for (int c = 0; c < 6; c++) ext[b][c] = w[c];
    }
    SYNC();
  }
  kinematics(ms, e);
  com_pos(ms, e);
  PAR_FOR(j, nv) {
    unsigned mask = (unsigned)m.body_dofmask[m.jnt_bodyid[j]] & ((1u << j) - 1u);
    float v[6] = {0, 0, 0, 0, 0, 0};
    while (mask) {
      const int i = LS_FFS(mask) - 1;
      mask &= mask - 1;
      const float qv = e.qvel[i];
      for (int c = 0; c < 6; c++) v[c] = fmaf(e.cdof[i][c], qv, v[c]);
    }
    float cdd[6];
    crossMotion(cdd, v, e.cdof[j]);
    for (int c = 0; c < 6; c++) e.cdof_dot[j][c] = cdd[c];
  }
  const float* __restrict__ xfrc = c_applied[ms].xfrc;
  if (need_ext && xfrc) PAR_FOR(b, nb) {
    if (b == 0) continue;
    const float* w = xfrc + ((size_t)e.env * nb + b) * 6;
    const float F[3] = {LS_LDG(w), LS_LDG(w + 1), LS_LDG(w + 2)};
    const float r[3] = {e.xipos[b][0] - e.xpos[b][0], e.xipos[b][1] - e.xpos[b][1], e.xipos[b][2] - e.xpos[b][2]};
    float rxF[3];
    cross3(rxF, r, F);
    for (int c = 0; c < 3; c++) { ext[b][c] += F[c]; ext[b][3 + c] += rxF[c] + LS_LDG(w + 3 + c); }
  }
  SYNC();
  if (o.cfrc_ext) PAR_FOR(k, nb * LS_CONTACT_DIM) o.cfrc_ext[k] = ext[k / 6][k % 6];
  PAR_FOR(b, nb) {
    unsigned mask = b > 0 ? (unsigned)m.body_dofmask[b] : 0u;
    float cvel[6] = {0, 0, 0, 0, 0, 0}, cacc[6] = {0, 0, 0, -m.gravity[0], -m.gravity[1], -m.gravity[2]};
    while (mask) {
      const int i = LS_FFS(mask) - 1;
      mask &= mask - 1;
      const float qv = e.qvel[i], qa = e.qacc[i];
      for (int c = 0; c < 6; c++) {
        cvel[c] = fmaf(e.cdof[i][c], qv, cvel[c]);
        cacc[c] = fmaf(e.cdof_dot[i][c], qv, fmaf(e.cdof[i][c], qa, cacc[c]));
      }
    }
    const float r[3] = {e.xpos[b][0] - e.com[0], e.xpos[b][1] - e.com[1], e.xpos[b][2] - e.com[2]};
    if (o.body_acc) {
      float wr[3], ar[3], vp[3], wv[3];
      cross3(wr, cvel, r);
      cross3(ar, cacc, r);
      for (int c = 0; c < 3; c++) vp[c] = cvel[3 + c] + wr[c];
      cross3(wv, cvel, vp);
      float* dst = o.body_acc + b * LS_BODY_ACC_DIM;
      for (int c = 0; c < 3; c++) { dst[c] = cacc[c]; dst[3 + c] = cacc[3 + c] + ar[c] + wv[c]; }
    }
    if (o.cfrc_int) {
      float* f = frc[b];
      if (b == 0) { for (int c = 0; c < 6; c++) f[c] = 0; continue; }
      float t1[6], t2[6], t3[6], rxF[3];
      mulInertVec(t1, e.cinert[b], cacc);
      mulInertVec(t2, e.cinert[b], cvel);
      crossForce(t3, cvel, t2);
      // cfrc_ext about com: torque + (xpos - com) x force
      cross3(rxF, r, ext[b]);
      for (int c = 0; c < 3; c++) { f[c] = t1[c] + t3[c] - (ext[b][3 + c] + rxF[c]); f[3 + c] = t1[3 + c] + t3[3 + c] - ext[b][c]; }
    }
  }
  SYNC();
  if (o.cfrc_int) PAR_FOR(b, nb) {
    float F[6] = {0, 0, 0, 0, 0, 0};
    if (b > 0) {
      for (int c = 0; c < 6; c++) F[c] = frc[b][c];
      NOUNROLL for (int k = b + 1; k < nb; k++) {
        int a = m.body_parentid[k];
        while (a > b) a = m.body_parentid[a];
        if (a != b) continue;
        for (int c = 0; c < 6; c++) F[c] += frc[k][c];
      }
    }
    // about xpos: torque + (com - xpos) x force
    const float r[3] = {e.com[0] - e.xpos[b][0], e.com[1] - e.xpos[b][1], e.com[2] - e.xpos[b][2]};
    float rxF[3];
    cross3(rxF, r, F + 3);
    float* dst = o.cfrc_int + b * LS_CONTACT_DIM;
    for (int c = 0; c < 3; c++) { dst[c] = b > 0 ? F[3 + c] : 0.0f; dst[3 + c] = b > 0 ? F[c] + rxF[c] : 0.0f; }
  }
  SYNC();
}

// locosim_forward's evaluation of one env: forward() at e.qpos / e.qvel / e.ctrl (the caller ran init_workspace and loaded
// the warm start), then forward_outputs. A non-finite qpos, qvel or ctrl gives zero rows before anything is evaluated.
template <class C>
LS_FN void forward_dynamics(const int ms, EnvS<C>& e, const SolverOpts so, const FwdOut o) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nb = m.nb, nu = m.nu;
  bool bad = false;
  PAR_FOR(i, nu) bad |= !isfinite(e.ctrl[i]);
  if (nonfinite_state(e, nv, bad)) {
    if (o.dof) PAR_FOR(k, nv * LS_DOF_DIM) o.dof[k] = 0.0f;
    if (o.body_acc) PAR_FOR(k, nb * LS_BODY_ACC_DIM) o.body_acc[k] = 0.0f;
    if (o.cfrc_int) PAR_FOR(k, nb * LS_CONTACT_DIM) o.cfrc_int[k] = 0.0f;
    if (o.cfrc_ext) PAR_FOR(k, nb * LS_CONTACT_DIM) o.cfrc_ext[k] = 0.0f;
    SYNC();
    return;
  }
  forward(ms, e, so);
  forward_outputs(ms, e, o);
}

// ----------------------------------------------------------------------------------------------------------
// task layer: observation gather, termination, reward, reset from the trajectory table
// ----------------------------------------------------------------------------------------------------------
template <class C>
LS_DEV float obs_value(const DevTask& t, const EnvS<C>& e, int k) {
  int idx = t.obs_src_idx[k];
  int ty = t.obs_src_type[k];
  if (ty == LS_OBS_GRF) return e.grf[idx] * (1.0f / (1000.0f * (float)t.n_substeps));
  if (ty == LS_OBS_PARAM) return e.prm[t.po_user + idx];
  return ty == LS_OBS_QPOS ? e.qpos[idx] : (ty == LS_OBS_QVEL ? e.qvel[idx] : e.goal[idx]);
}

// value `kind` (LS_OBS_QPOS / LS_OBS_QVEL) number idx of a reset row: recentred root x / y, and -- setup_random_rot,
// unitreeA1.py:270-285 -> utils/math.py rotate_obs -- yaw + angle wrapped to [-pi, pi), root (vx, vy) rotated by angle
LS_DEV float reset_value(const DevTask& t, const float* row, int nv, int kind, int idx, float angle) {
  if (kind == LS_OBS_QPOS) {
    if (idx == t.recenter0 || idx == t.recenter1) return 0.0f;
    float q = row[idx];
    if (idx == t.rot[0]) {
      const float two_pi = 6.283185307179586f;
      q = q + angle + 3.14159265358979f;
      q = q - two_pi * floorf(q / two_pi) - 3.14159265358979f;
    }
    return q;
  }
  float v = row[nv + idx];
  if (t.rot[0] >= 0 && (idx == t.rot[1] || idx == t.rot[2])) {
    float sn, cs;
    sincosf(angle, &sn, &cs);
    const float vx = row[nv + t.rot[1]], vy = row[nv + t.rot[2]];
    v = idx == t.rot[1] ? cs * vx - sn * vy : sn * vx + cs * vy;
  }
  return v;
}

// every reset of an env zeroes its rows of the applied-force buffers (mj_resetData); a whole-warp call
LS_DEV void zero_applied(const int ms, const int env) {
  const DevModel& m = c_models[ms];
  const DevApplied& ap = c_applied[ms];
  if (ap.xfrc) PAR_FOR(k, 6 * m.nb) ap.xfrc[(size_t)env * 6 * m.nb + k] = 0.0f;
  if (ap.qfrc) PAR_FOR(k, m.nv) ap.qfrc[(size_t)env * m.nv + k] = 0.0f;
}

// ----------------------------------------------------------------------------------------------------------
// body outputs (locosim_set_body_outputs): mj_kinematics + mj_comPos + mj_comVel on the env's current qpos / qvel, then per
// body xpos, xquat and the velocity of the body-frame origin (mj_objectVelocity, mjOBJ_XBODY, world frame: angular, linear)
// ----------------------------------------------------------------------------------------------------------
// A whole-warp call. It rewrites the kinematics (xpos, xquat, xmat, gxpos, com, cdof) and the smooth-dynamics scratch of the
// union; every forward() recomputes all of them before reading them, and nothing a sub-step launch carries to the next one
// (SplitState / PersistQueue carry record: counters, separating directions, foot forces) lives there. LS_BODY_DIM floats
// per body go to dst and to dst2 (either may be NULL).
template <class C>
LS_FN void body_outputs(const int ms, EnvS<C>& e, float* dst, float* dst2) {
  const DevModel& m = c_models[ms];
  kinematics(ms, e);
  com_pos(ms, e);
  PAR_FOR(b, m.nb) {
    // spatial velocity at e.com (mj_comVel): sum of cdof_d qvel_d over the dofs on the path root..b
    float v[6] = {0, 0, 0, 0, 0, 0};
    unsigned mask = (unsigned)m.body_dofmask[b];
    while (mask) {
      const int d = LS_FFS(mask) - 1;
      mask &= mask - 1u;
      const float qd = e.qvel[d];
      for (int c = 0; c < 6; c++) v[c] += e.cdof[d][c] * qd;
    }
    // linear part moved from e.com to xpos: v + w x (xpos - com)
    const float r[3] = {e.xpos[b][0] - e.com[0], e.xpos[b][1] - e.com[1], e.xpos[b][2] - e.com[2]};
    float wr[3];
    cross3(wr, v, r);
    float o[LS_BODY_DIM] = {e.xpos[b][0], e.xpos[b][1], e.xpos[b][2], e.xquat[b][0], e.xquat[b][1], e.xquat[b][2],
                            e.xquat[b][3], v[0], v[1], v[2], v[3] + wr[0], v[4] + wr[1], v[5] + wr[2]};
    if (b == 0) for (int k = 7; k < LS_BODY_DIM; k++) o[k] = 0.0f;      // (the world: exact zeros, not 0 * x)
    if (dst) for (int k = 0; k < LS_BODY_DIM; k++) dst[b * LS_BODY_DIM + k] = o[k];
    if (dst2) for (int k = 0; k < LS_BODY_DIM; k++) dst2[b * LS_BODY_DIM + k] = o[k];
  }
  SYNC();
}

// d_body rows of an env the step kernel is about to reset (whole warp, from reset_env): its returned state exists only until
// reset_env overwrites it. Zeros for a non-finite env (the epilogue's test; such an env is always reset). The env is marked,
// and body_kernel, which writes every other row from the stored state after the step, leaves these rows alone.
template <class C>
LS_DEV void body_rows_terminal(const int ms, EnvS<C>& e, const int env) {
  const DevBodyOut bo = c_bodyout[ms];
  if (!bo.body) return;
  const DevModel& m = c_models[ms];
  bool bad = false;
  PAR_FOR(i, m.nv) bad |= !(isfinite(e.qpos[i]) && isfinite(e.qvel[i]));
#ifndef LS_EMULATE
  bad = __any_sync(0xffffffffu, bad);
#endif
  float* body = bo.body + (size_t)env * m.nb * LS_BODY_DIM;
  if (bad) PAR_FOR(k, m.nb * LS_BODY_DIM) body[k] = 0.0f;
  else body_outputs(ms, e, body, (float*)nullptr);
  LANE0 bo.reset_mark[env] = 1;
}

// reference rows (locosim_set_reference_outputs): the body outputs of the state that a reset onto table row `row` under
// rotation `angle` gives (reset_value: root x / y zeroed, setup_random_rot's yaw and root (vx, vy) turned), with the
// parameters e.prm. A whole-warp call; it overwrites e.qpos / e.qvel and what body_outputs rewrites. LS_BODY_DIM floats per
// body go to dst and to dst2 (either may be NULL).
template <class C>
LS_DEV void reference_outputs(const int ms, const DevTask& t, EnvS<C>& e, const float* row, float angle, float* dst,
                              float* dst2) {
  const int nv = c_models[ms].nv;
  PAR_FOR(i, nv) {
    e.qpos[i] = reset_value(t, row, nv, LS_OBS_QPOS, i, angle);
    e.qvel[i] = reset_value(t, row, nv, LS_OBS_QVEL, i, angle);
  }
  SYNC();
  body_outputs(ms, e, dst, dst2);
}

template <class C>
LS_FN void reset_env(const int ms, const DevTask& t, EnvS<C>& e, int traj_no, int step_no, float angle) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv, ncol = 2 * nv + t.n_goal;
  const float* row = t.table + ((size_t)traj_no * t.traj_len + step_no) * ncol;
  body_rows_terminal(ms, e, e.env);            // d_body of the terminal state, before it is overwritten
  PAR_FOR(i, nv) {
    e.qpos[i] = reset_value(t, row, nv, LS_OBS_QPOS, i, angle);
    e.qvel[i] = reset_value(t, row, nv, LS_OBS_QVEL, i, angle);
    e.qacc_ws[i] = 0; e.qacc[i] = 0;
  }
  PAR_FOR(k, t.n_goal) e.goal[k] = row[2 * nv + k];
  PAR_FOR(k, 3 * LS_MAX_GRF) e.grf[k] = 0;     // mean_grf is reset with the episode (reset observation: zeros)
  zero_applied(ms, e.env);
  SYNC();
}

// ----------------------------------------------------------------------------------------------------------
// ray casting (locosim_ray): MuJoCo 2.3.7's mj_ray / engine_ray.c for the primitives, a GJK ray cast on the convex hull of
// a mesh geom's vertices. One thread per ray; every routine works in the geom's frame (lp, lv: the ray's point and
// direction there) and returns the distance in units of |lv| (-1: no hit) and an outward normal `ln` (not unit length).
// ----------------------------------------------------------------------------------------------------------
// one geom as the rays of one env see it: its world frame after kinematics() and what the routines read of the model
struct RayGeom {
  float pos[3], mat[9], size[3], rbound;
  int type, body, vnum, sel;       // sel: LS_RAY_STATIC (no dof on the path to the world: MuJoCo's body_weldid 0) or LS_RAY_DYNAMIC
  const float* verts;              // mesh: the hull vertices in the geom frame (mesh_vert)
};

template <class C>
LS_DEV void ray_stage_geom(const int ms, const EnvS<C>& e, const int g, RayGeom& r) {
  const DevModel& m = c_models[ms];
  for (int k = 0; k < 3; k++) { r.pos[k] = e.gxpos[g][k]; r.size[k] = m.geom_size[3 * g + k]; }
  geom_mat(ms, e, g, r.mat);
  r.rbound = m.geom_rbound[g];
  r.type = m.geom_type[g];
  r.body = m.geom_bodyid[g];
  r.sel = m.body_dofmask[r.body] == 0 ? LS_RAY_STATIC : LS_RAY_DYNAMIC;
  r.vnum = r.type == LS_GEOM_MESH ? m.geom_meshnum[g] : 0;
  r.verts = r.type == LS_GEOM_MESH ? m.mesh_vert + 3 * m.geom_meshadr[g] : nullptr;
}

// the ray of a query frame (LS_RAY_WORLD / BODY / HEADING / TRACK of body fb) in world coordinates
template <class C>
LS_DEV void ray_to_world(const EnvS<C>& e, const int frame, const int fb, const float* pnt, const float* vec, float* p,
                         float* v) {
  if (frame == LS_RAY_WORLD) {
    for (int k = 0; k < 3; k++) { p[k] = pnt[k]; v[k] = vec[k]; }
  } else if (frame == LS_RAY_BODY) {
    rotvec(p, e.xquat[fb], pnt);
    rotvec(v, e.xquat[fb], vec);
    for (int k = 0; k < 3; k++) p[k] += e.xpos[fb][k];
  } else if (frame == LS_RAY_HEADING) {
    // yaw of the body's x axis; a vertical x axis has no heading: the world's then
    const float* q = e.xquat[fb];
    const float fx = 1 - 2 * (q[2] * q[2] + q[3] * q[3]), fy = 2 * (q[1] * q[2] + q[0] * q[3]);
    const float h = sqrtf(fx * fx + fy * fy);
    const float c = h > 1e-6f ? fx / h : 1.0f, s = h > 1e-6f ? fy / h : 0.0f;
    p[0] = c * pnt[0] - s * pnt[1] + e.xpos[fb][0]; p[1] = s * pnt[0] + c * pnt[1] + e.xpos[fb][1]; p[2] = pnt[2] + e.xpos[fb][2];
    v[0] = c * vec[0] - s * vec[1]; v[1] = s * vec[0] + c * vec[1]; v[2] = vec[2];
  } else {
    for (int k = 0; k < 3; k++) { p[k] = pnt[k] + e.xpos[fb][k]; v[k] = vec[k]; }
  }
}

// roots x[0] <= x[1] of |p + x v|^2 = r2 over the first n coordinates, taken about the ray's point closest to the centre
// (fp32 keeps its accuracy far from the geom there); returns the smaller non-negative root or -1 (MuJoCo's ray_quad)
LS_DEV float ray_quad(const float* p, const float* v, const int n, const float r2, float* x) {
  float a = 0, b = 0, q2 = 0;
  for (int k = 0; k < n; k++) { a += v[k] * v[k]; b += p[k] * v[k]; }
  x[0] = x[1] = -1;
  if (a < LS_MINVAL) return -1;
  const float t0 = -b / a;
  for (int k = 0; k < n; k++) { const float q = p[k] + t0 * v[k]; q2 += q * q; }
  if (q2 > r2) return -1;
  const float d = sqrtf((r2 - q2) / a);
  x[0] = t0 - d; x[1] = t0 + d;
  return x[0] >= 0 ? x[0] : (x[1] >= 0 ? x[1] : -1);
}

// one-sided plane: hit from its +z side only, within size[0:2] where those are non-zero
LS_DEV float ray_plane(const float* s, const float* lp, const float* lv, float* ln) {
  if (lv[2] > -LS_MINVAL) return -1;
  const float x = -lp[2] / lv[2];
  if (x < 0) return -1;
  const float p0 = lp[0] + x * lv[0], p1 = lp[1] + x * lv[1];
  if ((s[0] > 0 && fabsf(p0) > s[0]) || (s[1] > 0 && fabsf(p1) > s[1])) return -1;
  ln[0] = 0; ln[1] = 0; ln[2] = 1;
  return x;
}

LS_DEV float ray_sphere(const float* s, const float* lp, const float* lv, float* ln) {
  float xx[2];
  const float x = ray_quad(lp, lv, 3, s[0] * s[0], xx);
  for (int k = 0; k < 3; k++) ln[k] = lp[k] + x * lv[k];
  return x;
}

LS_DEV float ray_ellipsoid(const float* s, const float* lp, const float* lv, float* ln) {
  const float sp[3] = {lp[0] / s[0], lp[1] / s[1], lp[2] / s[2]}, sv[3] = {lv[0] / s[0], lv[1] / s[1], lv[2] / s[2]};
  float xx[2];
  const float x = ray_quad(sp, sv, 3, 1.0f, xx);
  for (int k = 0; k < 3; k++) ln[k] = (lp[k] + x * lv[k]) / (s[k] * s[k]);
  return x;
}

// the round side of a capsule or cylinder (radius s[0], half length s[1]): the first root within the flat ends
LS_DEV void ray_round_side(const float* s, const float* lp, const float* lv, float& x, float* ln) {
  float xx[2];
  const float sol = ray_quad(lp, lv, 2, s[0] * s[0], xx);
  if (sol >= 0 && fabsf(lp[2] + sol * lv[2]) <= s[1] && (x < 0 || sol < x)) {
    x = sol;
    ln[0] = lp[0] + sol * lv[0]; ln[1] = lp[1] + sol * lv[1]; ln[2] = 0;
  }
}

LS_DEV float ray_capsule(const float* s, const float* lp, const float* lv, float* ln) {
  float x = -1;
  ray_round_side(s, lp, lv, x, ln);
  for (int side = -1; side <= 1; side += 2) {           // hemispheres beyond the ends
    const float dp[3] = {lp[0], lp[1], lp[2] - side * s[1]};
    float xx[2];
    ray_quad(dp, lv, 3, s[0] * s[0], xx);
    for (int j = 0; j < 2; j++) {
      if (xx[j] >= 0 && side * (lp[2] + xx[j] * lv[2]) >= s[1] && (x < 0 || xx[j] < x)) {
        x = xx[j];
        for (int k = 0; k < 3; k++) ln[k] = dp[k] + x * lv[k];
      }
    }
  }
  return x;
}

LS_DEV float ray_cylinder(const float* s, const float* lp, const float* lv, float* ln) {
  float x = -1;
  if (fabsf(lv[2]) > LS_MINVAL) {
    for (int side = -1; side <= 1; side += 2) {
      const float sol = (side * s[1] - lp[2]) / lv[2];
      const float p0 = lp[0] + sol * lv[0], p1 = lp[1] + sol * lv[1];
      if (sol >= 0 && p0 * p0 + p1 * p1 <= s[0] * s[0] && (x < 0 || sol < x)) {
        x = sol; ln[0] = 0; ln[1] = 0; ln[2] = (float)side;
      }
    }
  }
  ray_round_side(s, lp, lv, x, ln);
  return x;
}

LS_DEV float ray_box(const float* s, const float* lp, const float* lv, float* ln) {
  float x = -1;
  for (int i = 0; i < 3; i++) {
    if (fabsf(lv[i]) <= LS_MINVAL) continue;
    const int j = i == 0 ? 1 : 0, k = i == 2 ? 1 : 2;
    for (int side = -1; side <= 1; side += 2) {
      const float sol = (side * s[i] - lp[i]) / lv[i];
      if (sol >= 0 && fabsf(lp[j] + sol * lv[j]) <= s[j] && fabsf(lp[k] + sol * lv[k]) <= s[k] && (x < 0 || sol < x)) {
        x = sol; ln[0] = ln[1] = ln[2] = 0; ln[i] = (float)side;
      }
    }
  }
  return x;
}

// the hull cast runs in fp64: GJK's simplex steps lose fp32 accuracy near the hull's edges
LS_DEV double dot3d(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
LS_DEV void cross3d(double* r, const double* a, const double* b) {
  r[0] = a[1] * b[2] - a[2] * b[1]; r[1] = a[2] * b[0] - a[0] * b[2]; r[2] = a[0] * b[1] - a[1] * b[0];
}
// closest point to the origin of the triangle (a, b, c) (Ericson, Real-Time Collision Detection 5.1.5); `keep` gets the
// vertices it is a combination of (bits 0-2)
LS_DEV void hull_closest_tri(const double* a, const double* b, const double* c, double* cp, int& keep) {
  double ab[3], ac[3];
  for (int k = 0; k < 3; k++) { ab[k] = b[k] - a[k]; ac[k] = c[k] - a[k]; }
  const double d1 = -dot3d(ab, a), d2 = -dot3d(ac, a);
  if (d1 <= 0 && d2 <= 0) { for (int k = 0; k < 3; k++) cp[k] = a[k]; keep = 1; return; }
  const double d3 = -dot3d(ab, b), d4 = -dot3d(ac, b);
  if (d3 >= 0 && d4 <= d3) { for (int k = 0; k < 3; k++) cp[k] = b[k]; keep = 2; return; }
  const double vc = d1 * d4 - d3 * d2;
  if (vc <= 0 && d1 >= 0 && d3 <= 0) {
    const double t = d1 / (d1 - d3);
    for (int k = 0; k < 3; k++) cp[k] = a[k] + t * ab[k];
    keep = 3; return;
  }
  const double d5 = -dot3d(ab, c), d6 = -dot3d(ac, c);
  if (d6 >= 0 && d5 <= d6) { for (int k = 0; k < 3; k++) cp[k] = c[k]; keep = 4; return; }
  const double vb = d5 * d2 - d1 * d6;
  if (vb <= 0 && d2 >= 0 && d6 <= 0) {
    const double t = d2 / (d2 - d6);
    for (int k = 0; k < 3; k++) cp[k] = a[k] + t * ac[k];
    keep = 5; return;
  }
  const double va = d3 * d6 - d5 * d4;
  if (va <= 0 && d4 - d3 >= 0 && d5 - d6 >= 0) {
    const double t = (d4 - d3) / ((d4 - d3) + (d5 - d6));
    for (int k = 0; k < 3; k++) cp[k] = b[k] + t * (c[k] - b[k]);
    keep = 6; return;
  }
  const double den = 1.0 / (va + vb + vc), v = vb * den, w = vc * den;
  for (int k = 0; k < 3; k++) cp[k] = a[k] + v * ab[k] + w * ac[k];
  keep = 7;
}

// v = the origin minus its closest point in conv(y[0..n)), n <= 4; y is reduced to the points that closest point needs
LS_DEV void hull_closest(double (*y)[3], int& n, double* v) {
  double cp[3];
  int keep = 1;
  if (n == 1) {
    for (int k = 0; k < 3; k++) cp[k] = y[0][k];
  } else if (n == 2) {
    double d[3];
    for (int k = 0; k < 3; k++) d[k] = y[1][k] - y[0][k];
    const double dd = dot3d(d, d), t = dd > 0 ? -dot3d(y[0], d) / dd : 0.0f;
    if (t <= 0) { keep = 1; for (int k = 0; k < 3; k++) cp[k] = y[0][k]; }
    else if (t >= 1) { keep = 2; for (int k = 0; k < 3; k++) cp[k] = y[1][k]; }
    else { keep = 3; for (int k = 0; k < 3; k++) cp[k] = y[0][k] + t * d[k]; }
  } else if (n == 3) {
    hull_closest_tri(y[0], y[1], y[2], cp, keep);
  } else {
    // tetrahedron: the closest of the faces whose plane separates the origin from the opposite vertex; none: inside
    const int face[4][4] = {{0, 1, 2, 3}, {0, 2, 3, 1}, {0, 3, 1, 2}, {1, 3, 2, 0}};
    double best = 3.0e38;
    keep = 15;
    cp[0] = cp[1] = cp[2] = 0;
    for (int f = 0; f < 4; f++) {
      const double *a = y[face[f][0]], *b = y[face[f][1]], *c = y[face[f][2]], *d = y[face[f][3]];
      double ab[3], ac[3], nn[3];
      for (int k = 0; k < 3; k++) { ab[k] = b[k] - a[k]; ac[k] = c[k] - a[k]; }
      cross3d(nn, ab, ac);
      double ad[3];
      for (int k = 0; k < 3; k++) ad[k] = d[k] - a[k];
      const double so = -dot3d(nn, a), sd = dot3d(nn, ad);
      if (so * sd > 0) continue;                        // the origin is on the inner side of this face
      double q[3];
      int kf;
      hull_closest_tri(a, b, c, q, kf);
      const double dq = dot3d(q, q);
      if (dq < best) {
        best = dq;
        for (int k = 0; k < 3; k++) cp[k] = q[k];
        keep = 0;
        for (int j = 0; j < 3; j++) if (kf & (1 << j)) keep |= 1 << face[f][j];
      }
    }
  }
  int m = 0;
  for (int i = 0; i < n; i++)
    if (keep & (1 << i)) { if (m != i) for (int k = 0; k < 3; k++) y[m][k] = y[i][k]; m++; }
  n = m;
  for (int k = 0; k < 3; k++) v[k] = -cp[k];
}

// index of the hull vertex farthest along d (the first of equals, like mpr_support_geom's scan)
LS_DEV int hull_support(const float* vt, const int nv, const double* d) {
  double mx = -3.0e38;
  int best = 0;
  for (int i = 0; i < nv; i++) {
    const double t = d[0] * vt[3 * i] + d[1] * vt[3 * i + 1] + d[2] * vt[3 * i + 2];
    if (t > mx) { mx = t; best = i; }
  }
  return best;
}

// GJK ray cast (van den Bergen, "Ray casting against general convex objects with application to continuous collision
// detection", 2004) of s + x r against the hull of vt[0..nv) (bounding radius rb): the smallest x >= 0 on or in the hull, and
// the outward normal of the support plane it stops at (zero when s itself is in the hull: x = 0). -1: a miss. tol: the
// distance at which the point counts as on the hull.
LS_DEV double hull_cast(const float* vt, const int nv, const double rb, const double* s, const double* r, const double tol,
                        double* ln) {
  double lam = 0, x[3] = {s[0], s[1], s[2]}, v[3], P[4][3], y[4][3];
  int np = 0;
  for (int k = 0; k < 3; k++) { v[k] = x[k] - vt[k]; ln[k] = 0; }
  for (int it = 0; it < 64; it++) {
    if (dot3d(v, v) <= tol * tol) break;
    const float* pf = vt + 3 * hull_support(vt, nv, v);
    const double p[3] = {pf[0], pf[1], pf[2]};
    const double w[3] = {x[0] - p[0], x[1] - p[1], x[2] - p[2]};
    const double vw = dot3d(v, w);
    bool dup = false;
    for (int i = 0; i < np; i++) dup |= P[i][0] == p[0] && P[i][1] == p[1] && P[i][2] == p[2];
    if (vw > 0) {
      const double vr = dot3d(v, r);
      if (vr >= 0) return -1;
      lam -= vw / vr;
      for (int k = 0; k < 3; k++) { x[k] = s[k] + lam * r[k]; ln[k] = v[k]; }
    } else if (dup) {
      break;                                            // no support point left that moves x or v: x is on the hull
    }
    if (!dup) { for (int k = 0; k < 3; k++) P[np][k] = p[k]; np++; }
    for (int i = 0; i < np; i++) for (int k = 0; k < 3; k++) y[i][k] = P[i][k] - x[k];
    hull_closest(y, np, v);
    for (int i = 0; i < np; i++) for (int k = 0; k < 3; k++) P[i][k] = y[i][k] + x[k];
  }
  // GJK reaches a face only linearly in fp32: where x stopped on three support points that span a face of the hull (no
  // vertex beyond their plane), take the ray's crossing of that plane, and its normal, when it lies within the distance
  // GJK left
  // GJK reaches a face only linearly: where x stopped on three support points that span a face of the hull (no vertex
  // beyond their plane), take the ray's crossing of that plane, and its normal, when it lies within the distance GJK left.
  // np = 4: x ended in a tetrahedron of support points; of its faces that qualify, the ray enters the hull through the one
  // it crosses last (at an edge, the other face's plane is crossed earlier)
  const double rl = sqrt(dot3d(r, r)), left = 4 * sqrt(dot3d(v, v)) + tol, lam0 = lam;
  bool refined = false;
  for (int f = 0; f < (np == 4 ? 4 : (np == 3 ? 1 : 0)) && dot3d(ln, ln) > 0; f++) {
    const double *a = P[f == 3 ? 1 : 0], *b = P[f == 2 ? 3 : (f == 3 ? 2 : 1)], *c = P[f == 1 ? 3 : (f == 3 ? 3 : 2)];
    double e1[3], e2[3], n[3], d[3];
    for (int k = 0; k < 3; k++) { e1[k] = b[k] - a[k]; e2[k] = c[k] - a[k]; d[k] = a[k] - s[k]; }
    cross3d(n, e1, e2);
    const double nr = dot3d(n, r), nn = sqrt(dot3d(n, n));
    if (!(fabs(nr) > 1e-4 * nn * rl)) continue;
    if (nr > 0) for (int k = 0; k < 3; k++) n[k] = -n[k];
    const float* far = vt + 3 * hull_support(vt, nv, n);
    if (n[0] * (far[0] - a[0]) + n[1] * (far[1] - a[1]) + n[2] * (far[2] - a[2]) > 1e-5 * nn * rb) continue;
    const double l2 = dot3d(n, d) / dot3d(n, r);
    if (fabs(l2 - lam0) * rl <= left && (!refined || l2 > lam)) {
      lam = l2;
      refined = true;
      for (int k = 0; k < 3; k++) ln[k] = n[k];
    }
  }
  return lam;
}

// a mesh geom: its hull. A ray that starts in the hull leaves it where the reversed ray, cast from beyond the bounding
// sphere, enters it.
LS_DEV float ray_mesh(const RayGeom& g, const float* lpf, const float* lvf, float* lnf) {
  const double lp[3] = {lpf[0], lpf[1], lpf[2]}, lv[3] = {lvf[0], lvf[1], lvf[2]};
  const double pl = sqrt(dot3d(lp, lp)), vl = sqrt(dot3d(lv, lv));
  double ln[3];
  double x = hull_cast(g.verts, g.vnum, g.rbound, lp, lv, 1e-9 * (pl + g.rbound), ln);
  if (x == 0) {
    const double T = (pl + 2 * g.rbound + 1e-3) / vl;
    const double s2[3] = {lp[0] + T * lv[0], lp[1] + T * lv[1], lp[2] + T * lv[2]}, r2[3] = {-lv[0], -lv[1], -lv[2]};
    const double back = hull_cast(g.verts, g.vnum, g.rbound, s2, r2, 1e-9 * (T * vl + g.rbound), ln);
    x = back < 0 ? 0.0 : fmax(T - back, 0.0);
  }
  for (int k = 0; k < 3; k++) lnf[k] = (float)ln[k];
  return (float)x;
}

// the world ray p + x v against the geoms G[0..ng) that `sel` (LS_RAY_STATIC | LS_RAY_DYNAMIC) selects, except those of body
// `exclude`: the smallest x >= 0 (MuJoCo's mj_ray), its geom (-1 and x = -1: nothing is hit) and the unit outward normal
// there, world frame (zeros for a miss). Bounding spheres (geom_rbound) reject most geoms first, as ray_eliminate does.
LS_DEV float ray_geoms(const RayGeom* G, const int ng, const float* p, const float* v, const int exclude, const int sel,
                       int* geom, float* nrm) {
  float best = -1, bn[3] = {0, 0, 0};
  int bg = -1;
  const float vv = dot3(v, v);
  if (vv > 0) {
    for (int g = 0; g < ng; g++) {
      const RayGeom& r = G[g];
      if (!(r.sel & sel) || r.body == exclude) continue;
      const float d[3] = {p[0] - r.pos[0], p[1] - r.pos[1], p[2] - r.pos[2]};
      if (r.type != LS_GEOM_PLANE) {
        const float rb = r.rbound * 1.0001f + 1e-6f, b = dot3(d, v), dd = dot3(d, d);
        if (dd > rb * rb) {
          if (b >= 0) continue;                         // outside, moving away
          const float t0 = -b / vv, q[3] = {d[0] + t0 * v[0], d[1] + t0 * v[1], d[2] + t0 * v[2]};
          if (dot3(q, q) > rb * rb) continue;
          if (best >= 0 && t0 - rb / sqrtf(vv) > best) continue;   // the sphere lies beyond the nearest hit
        }
      }
      float lp[3], lv[3], ln[3] = {0, 0, 0};
      mulmatTvec3(lp, r.mat, d);
      mulmatTvec3(lv, r.mat, v);
      float x;
      switch (r.type) {
        case LS_GEOM_PLANE: x = ray_plane(r.size, lp, lv, ln); break;
        case LS_GEOM_SPHERE: x = ray_sphere(r.size, lp, lv, ln); break;
        case LS_GEOM_CAPSULE: x = ray_capsule(r.size, lp, lv, ln); break;
        case LS_GEOM_ELLIPSOID: x = ray_ellipsoid(r.size, lp, lv, ln); break;
        case LS_GEOM_CYLINDER: x = ray_cylinder(r.size, lp, lv, ln); break;
        case LS_GEOM_BOX: x = ray_box(r.size, lp, lv, ln); break;
        case LS_GEOM_MESH: x = ray_mesh(r, lp, lv, ln); break;
        default: x = -1;
      }
      if (x >= 0 && (best < 0 || x < best)) {
        best = x; bg = g;
        mulmatvec3(bn, r.mat, ln);
      }
    }
  }
  const float nl = dot3(bn, bn);
  const float inv = nl > 0 ? rsqrtf(nl) : 0.0f;
  for (int k = 0; k < 3; k++) nrm[k] = bn[k] * inv;
  *geom = bg;
  return best;
}

#ifdef LOCOSIM_TERRAIN
// ---- mj_rayHfield: a ray against the terrain solid of env `env` (include/locosim.h: the top surface's triangles with the
// collision's diagonal, the four sides and the base at -base). In the field's frame (unrotated: a translation by the
// field's position moved by -origin[env]); returns the first hit in units of |v| (-1: none) and the outward unit normal.
// The top surface is walked cell by cell along the ray (2D DDA between the ray's entry into and exit from the field's
// box); the triangles are intersected two-sided (Moeller-Trumbore), the sides and the base as bounded planes.
LS_DEV float ray_tri(const float* o, const float* v, const float* a, const float* b, const float* c, float* n) {
  const float e1[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, e2[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
  float h[3], q[3];
  cross3(h, v, e2);
  const float det = dot3(e1, h);
  if (fabsf(det) < 1e-20f) return -1;
  const float inv = 1.0f / det, s[3] = {o[0] - a[0], o[1] - a[1], o[2] - a[2]};
  const float u = inv * dot3(s, h);
  if (u < 0 || u > 1) return -1;
  cross3(q, s, e1);
  const float w = inv * dot3(v, q);
  if (w < 0 || u + w > 1) return -1;
  const float x = inv * dot3(e2, q);
  if (x < 0) return -1;
  cross3(n, e1, e2);
  if (n[2] < 0) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
  return x;
}
LS_DEV float ray_hfield(const DevTerrain& t, const float* lp, const float* v, float* n) {
  const float rx = t.size[0], ry = t.size[1], el = t.size[2], bs = t.size[3];
  const float lo[3] = {-rx, -ry, -bs}, hi[3] = {rx, ry, el};
  float tin = 0.0f, tout = 3.0e38f;
  for (int k = 0; k < 3; k++) {
    if (fabsf(v[k]) < LS_MINVAL) { if (lp[k] < lo[k] || lp[k] > hi[k]) return -1; continue; }
    const float a = (lo[k] - lp[k]) / v[k], b = (hi[k] - lp[k]) / v[k];
    tin = fmaxf(tin, fminf(a, b)); tout = fminf(tout, fmaxf(a, b));
  }
  if (tin > tout) return -1;
  const int nr = t.nrow, nc = t.ncol;
  const float dx = 2.0f * rx / (float)(nc - 1), dy = 2.0f * ry / (float)(nr - 1);
  float best = -1;
  auto clampi = [](int x, int a, int b) { return x < a ? a : (x > b ? b : x); };
  auto take = [&](float x, const float* nn) {
    if (x >= 0 && (best < 0 || x < best)) { best = x; n[0] = nn[0]; n[1] = nn[1]; n[2] = nn[2]; }
  };
  // sides (x = -+rx: column 0 / ncol - 1; y = -+ry: row 0 / nrow - 1) up to the surface height along the edge, and the base
  for (int sd = 0; sd < 4; sd++) {
    const int ax = sd >> 1, oth = 1 - ax;
    const float plane = (sd & 1) ? hi[ax] : lo[ax];
    if (fabsf(v[ax]) < LS_MINVAL) continue;
    const float x = (plane - lp[ax]) / v[ax];
    if (x < 0) continue;
    const float w = lp[oth] + x * v[oth], z = lp[2] + x * v[2];
    if (w < lo[oth] || w > hi[oth] || z < -bs) continue;
    const int ns = ax ? nc : nr;                           // samples along the edge
    const float ds = ax ? dx : dy, g = (w - lo[oth]) / ds;
    const int i = clampi((int)floorf(g), 0, ns - 2);
    const int fixed = (sd & 1) ? (ax ? nr - 1 : nc - 1) : 0;
    const int i0 = ax ? fixed * nc + i : i * nc + fixed, i1 = ax ? i0 + 1 : i0 + nc;
    const float f = g - (float)i, hz = (LS_LDG(t.data + i0) * (1.0f - f) + LS_LDG(t.data + i1) * f) * el;
    if (z > hz) continue;
    float nn[3] = {0, 0, 0};
    nn[ax] = (sd & 1) ? 1.0f : -1.0f;
    take(x, nn);
  }
  if (fabsf(v[2]) >= LS_MINVAL) {
    const float x = (-bs - lp[2]) / v[2], px = lp[0] + x * v[0], py = lp[1] + x * v[1];
    const float nn[3] = {0, 0, -1};
    if (x >= 0 && px >= -rx && px <= rx && py >= -ry && py <= ry) take(x, nn);
  }
  // the top surface, cell by cell from the ray's entry into the box
  const float x0 = lp[0] + tin * v[0], y0 = lp[1] + tin * v[1];
  int c = clampi((int)floorf((x0 + rx) / dx), 0, nc - 2), r = clampi((int)floorf((y0 + ry) / dy), 0, nr - 2);
  const int sc = v[0] > 0 ? 1 : -1, sr = v[1] > 0 ? 1 : -1;
  const float tdx = fabsf(v[0]) > LS_MINVAL ? dx / fabsf(v[0]) : 3.0e38f, tdy = fabsf(v[1]) > LS_MINVAL ? dy / fabsf(v[1]) : 3.0e38f;
  float tnx = fabsf(v[0]) > LS_MINVAL ? ((float)(c + (sc > 0)) * dx - rx - lp[0]) / v[0] : 3.0e38f;
  float tny = fabsf(v[1]) > LS_MINVAL ? ((float)(r + (sr > 0)) * dy - ry - lp[1]) / v[1] : 3.0e38f;
  for (int guard = 0; guard < nr + nc; guard++) {
    for (int tri = 0; tri < 2; tri++) {
      const int rr[3] = {tri ? r + 1 : r, tri ? r : r + 1, tri ? r + 1 : r};
      const int cc[3] = {c, tri ? c + 1 : c, c + 1};
      float P[3][3], nn[3];
      for (int i = 0; i < 3; i++) {
        P[i][0] = dx * (float)cc[i] - rx; P[i][1] = dy * (float)rr[i] - ry;
        P[i][2] = LS_LDG(t.data + rr[i] * nc + cc[i]) * el;
      }
      const float x = ray_tri(lp, v, P[0], P[1], P[2], nn);
      if (x >= 0) { const float il = rsqrtf(dot3(nn, nn)); nn[0] *= il; nn[1] *= il; nn[2] *= il; take(x, nn); }
    }
    const float tnext = fminf(tnx, tny);
    if ((best >= 0 && best <= tnext) || tnext > tout) break;     // (a later cell's hits lie beyond this cell's exit)
    if (tnx < tny) { c += sc; tnx += tdx; } else { r += sr; tny += tdy; }
    if (c < 0 || c > nc - 2 || r < 0 || r > nr - 2) break;
  }
  return best;
}
// the terrain's hit of a ray of env `env` (world frame), merged into the nearest hit of the other geoms (dist / geom / nrm,
// as ray_geoms returns them): the terrain is welded to the world (LS_RAY_STATIC, body 0)
LS_DEV void ray_terrain(const int ms, const int env, const float* p, const float* v, const int exclude, const int sel,
                        float* dist, int* geom, float* nrm) {
  const DevTerrain& t = c_terrain[ms];
  if (!(sel & LS_RAY_STATIC) || exclude == 0 || !(dot3(v, v) > 0)) return;
  float f[3] = {t.pos[0], t.pos[1], t.pos[2]};
  if (t.origin) { f[0] -= LS_LDG(t.origin + 2 * env); f[1] -= LS_LDG(t.origin + 2 * env + 1); }
  const float lp[3] = {p[0] - f[0], p[1] - f[1], p[2] - f[2]};
  float n[3];
  const float x = ray_hfield(t, lp, v, n);
  if (x >= 0 && (*dist < 0 || x < *dist)) {
    *dist = x; *geom = t.geom;
    for (int k = 0; k < 3; k++) nrm[k] = n[k];
  }
}
#endif
