// Host-side helpers shared by the CUDA engine (locosim.cu) and the serial emulation build (locosim_emu.cpp):
// parse the ModelPack / TaskSpec wire blobs (include/*.h), convert reals to fp32, derive the engine-only tables,
// and bind DevModel / DevTask pointer views onto a (host or device) base address.
#pragma once
#include <cstring>
#include <string>
#include <vector>

#include "locosim_config.h"
#include "locosim_core.cuh"

struct HostModel {
  std::vector<int> ints;      // all int fields in wire order, then body_level, body_dofmask, dof_frow
  std::vector<float> reals;   // all real fields in wire order (fp32)
  int nb, nv, ng, nu, np, nm, integrator, cone, iterations, nlevel, nfric, has_damping;
  float timestep, gravity[3], impratio, tolerance, meaninertia;
  int max_condim;
  int np_prim;                 // leading primitive pairs of the candidate-pair table (the general convex pairs follow)
  int nterr = 0;               // trailing pairs (terrain, g) of the table; the mid-phase tables cover the np - nterr others
  int hf_nrow = 0, hf_ncol = 0, hf_geom = -1;   // height field (terrain) grid and geom; hf_nrow = 0: no terrain
  float hf_size[4] = {0, 0, 0, 0};              // (rx, ry, elevation, base)
  float hf_pos[3] = {0, 0, 0};                  // the terrain geom's position (its frame's origin in the world)
  size_t hf_off = 0;           // offset of hfield_data[nrow * ncol] in `reals` (after the wire fields)
  int po[13], pool_P;          // parameter pool row layout (float offsets), see domain_randomization.py POOL_FIELDS
  std::vector<float> default_row;   // the model's own parameters as one pool row
};

static inline std::string parse_model(HostModel& h, const int* ints, int n_ints, const double* reals, int n_reals) {
  if (n_ints < MPI_HEADER_LEN || ints[MPI_MAGIC] != LOCOSIM_MP_MAGIC) return "bad ModelPack magic";
  if (ints[MPI_VERSION] != LOCOSIM_MP_VERSION) return "ModelPack version mismatch";
  int nb = h.nb = ints[MPI_NBODY], nv = h.nv = ints[MPI_NV], ng = h.ng = ints[MPI_NGEOM], nu = h.nu = ints[MPI_NU],
      np = h.np = ints[MPI_NPAIR], nm = h.nm = ints[MPI_NMESHVERT];
  h.integrator = ints[MPI_INTEGRATOR]; h.cone = ints[MPI_CONE]; h.iterations = ints[MPI_ITERATIONS];
  h.timestep = (float)reals[MPR_TIMESTEP];
  for (int k = 0; k < 3; k++) h.gravity[k] = (float)reals[MPR_GRAV_X + k];
  h.impratio = (float)reals[MPR_IMPRATIO]; h.tolerance = (float)reals[MPR_TOLERANCE];
  h.meaninertia = (float)reals[MPR_MEANINERTIA];
  if (nv > 31) return "nv > 31 not supported by the dof bitmask";
  size_t ni = 0, nr = 0;
#define X(name, cnt) ni += (size_t)(cnt);
  LOCOSIM_MP_INT_FIELDS(X)
#undef X
#define X(name, cnt) nr += (size_t)(cnt);
  LOCOSIM_MP_REAL_FIELDS(X)
#undef X
  h.hf_nrow = ints[MPI_HF_NROW]; h.hf_ncol = ints[MPI_HF_NCOL];
  if (h.hf_nrow < 0 || h.hf_ncol < 0 || (h.hf_nrow > 0) != (h.hf_ncol > 0) || (h.hf_nrow > 0 && (h.hf_nrow < 2 || h.hf_ncol < 2)))
    return "bad height field grid (nrow, ncol >= 2, or both 0)";
  if ((size_t)h.hf_nrow * (size_t)h.hf_ncol > (1u << 24)) return "height field larger than 2^24 samples";
  const size_t nhf = (size_t)h.hf_nrow * (size_t)h.hf_ncol;
  for (int k = 0; k < 4; k++) h.hf_size[k] = (float)reals[MPR_HF_SIZE + k];
  if ((size_t)n_ints != MPI_HEADER_LEN + ni || (size_t)n_reals != MPR_HEADER_LEN + nr + nhf) return "ModelPack size mismatch";
  h.ints.assign(ints + MPI_HEADER_LEN, ints + n_ints);
  h.reals.resize(nr + nhf);
  for (size_t i = 0; i < nr + nhf; i++) h.reals[i] = (float)reals[MPR_HEADER_LEN + i];
  h.hf_off = nr;
  // locate the arrays we need for the derived tables
  const int* ip = h.ints.data();
  const int *body_parentid = 0, *body_lastdof = 0, *dof_parentid = 0, *geom_condim = 0, *pair_geom = 0, *geom_type = 0;
#define X(name, cnt) if (std::string(#name) == "body_parentid") body_parentid = ip; \
                     if (std::string(#name) == "body_lastdof") body_lastdof = ip;   \
                     if (std::string(#name) == "dof_parentid") dof_parentid = ip;   \
                     if (std::string(#name) == "geom_condim") geom_condim = ip;     \
                     if (std::string(#name) == "pair_geom") pair_geom = ip;         \
                     if (std::string(#name) == "geom_type") geom_type = ip;         \
                     ip += (cnt);
  LOCOSIM_MP_INT_FIELDS(X)
#undef X
  const float* rp = h.reals.data();
  const float *dof_frictionloss = 0, *dof_damping = 0, *geom_rbound = 0, *geom_quat = 0, *geom_pos = 0;
#define X(name, cnt) if (std::string(#name) == "dof_frictionloss") dof_frictionloss = rp; \
                     if (std::string(#name) == "dof_damping") dof_damping = rp;           \
                     if (std::string(#name) == "geom_rbound") geom_rbound = rp;           \
                     if (std::string(#name) == "geom_quat") geom_quat = rp;               \
                     if (std::string(#name) == "geom_pos") geom_pos = rp;                 \
                     rp += (cnt);
  LOCOSIM_MP_REAL_FIELDS(X)
#undef X
  std::vector<int> level(nb, 0), mask(nb, 0), frow(nv, -1);
  int nlevel = 1;
  for (int b = 1; b < nb; b++) {
    level[b] = level[body_parentid[b]] + 1;
    if (level[b] + 1 > nlevel) nlevel = level[b] + 1;
    int msk = 0;
    for (int d = body_lastdof[b]; d >= 0; d = dof_parentid[d]) msk |= (1 << d);
    mask[b] = msk;
    if (b > 1 && body_parentid[b] == 0) return "more than one kinematic tree (root body) is not supported";
  }
  int nfric = 0;
  h.has_damping = 0;
  for (int d = 0; d < nv; d++) {
    if (dof_frictionloss[d] > 0) frow[d] = nfric++;
    if (dof_damping[d] > 0) h.has_damping = 1;
  }
  h.max_condim = 1;
  for (int g = 0; g < ng; g++) if (geom_condim[g] > h.max_condim) h.max_condim = geom_condim[g];
  h.nlevel = nlevel; h.nfric = nfric;
  h.ints.insert(h.ints.end(), level.begin(), level.end());
  h.ints.insert(h.ints.end(), mask.begin(), mask.end());
  h.ints.insert(h.ints.end(), frow.begin(), frow.end());
  for (int i = 0; i < 32; i++) for (int j = 0; j <= i; j++) h.ints.push_back((i << 8) | j);   // row-major lower triangle, n <= 32
  // packed candidate-pair table of the mid-phase: g1 | g2 << 12 | flags << 24 (1: g1 is a plane, 2: general convex
  // pair, 4: capsule-hull test) and, as float bits, the bound of the bounding-sphere test (rbound[g2] for planes, else
  // rbound[g1] + rbound[g2])
  if (ng >= 4096) return "more than 4095 geoms";
  if (np >= 32768) return "more than 32767 candidate pairs";         // (15-bit pair index in collision()'s candidate list)
  // the terrain: the last geom, on the world body, unrotated; its pairs (terrain, g) close the pair table
  {
    int nhfg = 0;
    for (int g = 0; g < ng; g++) if (geom_type[g] == LS_GEOM_HFIELD) nhfg++;
    if (nhfg != (h.hf_nrow > 0 ? 1 : 0) || (nhfg && geom_type[ng - 1] != LS_GEOM_HFIELD))
      return "a height field needs its grid, and is the model's last geom (one per model)";
    if (nhfg) {
      h.hf_geom = ng - 1;
      const float* q = geom_quat + 4 * (ng - 1);
      if (!(q[0] == 1.0f && q[1] == 0.0f && q[2] == 0.0f && q[3] == 0.0f)) return "a rotated height field is not supported";
      if (!(h.hf_size[0] > 0 && h.hf_size[1] > 0 && h.hf_size[2] >= 0 && h.hf_size[3] > 0)) return "bad height field size";
      for (int k = 0; k < 3; k++) h.hf_pos[k] = geom_pos[3 * (ng - 1) + k];
    }
    int nt = 0;
    while (nt < np && geom_type[pair_geom[2 * (np - 1 - nt)]] == LS_GEOM_HFIELD) nt++;
    for (int p = 0; p < np - nt; p++)
      if (geom_type[pair_geom[2 * p]] == LS_GEOM_HFIELD) return "terrain pairs not last in the candidate-pair table (modelpack.pack)";
    h.nterr = nt;
    np -= nt;                                    // (the mid-phase tables below cover the other pairs)
  }
  h.np_prim = np;
  bool seen_convex = false;
  for (int p = 0; p < np; p++) {
    const int g1 = pair_geom[2 * p], g2 = pair_geom[2 * p + 1];
    int flags = 0;
    if (geom_type[g1] == LS_GEOM_PLANE) flags |= 1;
    else {
      // dedicated primitive routines: sphere-sphere, sphere-capsule, capsule-capsule, sphere-box; everything else is a
      // general convex pair (mjc_Convex / MPR)  [same rule as modelpack.py convex_pair_mask]
      const int t1 = geom_type[g1], t2 = geom_type[g2];
      const bool prim = (t1 == LS_GEOM_SPHERE && (t2 == LS_GEOM_SPHERE || t2 == LS_GEOM_CAPSULE || t2 == LS_GEOM_BOX)) ||
                        (t1 == LS_GEOM_CAPSULE && t2 == LS_GEOM_CAPSULE);
      if (!prim) flags |= 2;
      // 4: a general convex pair of axial geoms (sphere | capsule | cylinder vs cylinder): its box test is followed by the
      // exact capsule-hull test (locosim_core.cuh convex_hull_filter)
      auto axial = [](int t) { return t == LS_GEOM_SPHERE || t == LS_GEOM_CAPSULE || t == LS_GEOM_CYLINDER; };
      if (!prim && axial(t1) && axial(t2)) flags |= 4;
    }
    if (flags & 2) { if (!seen_convex) h.np_prim = p; seen_convex = true; }
    else if (seen_convex) return "candidate pairs not partitioned (primitive pairs first, general convex pairs last: modelpack.pack)";
    h.ints.push_back(g1 | (g2 << 12) | (flags << 24));
  }
  for (int p = 0; p < np; p++) {
    const int g1 = pair_geom[2 * p], g2 = pair_geom[2 * p + 1];
    const float b = geom_type[g1] == LS_GEOM_PLANE ? geom_rbound[g2] : geom_rbound[g1] + geom_rbound[g2];
    int bits;
    memcpy(&bits, &b, 4);
    h.ints.push_back(bits);
  }
  // ---- parameter pool layout: POOL_FIELDS of loco_mujoco_b200/domain_randomization.py, meaninertia, LS_POOL_USER user
  //      features, padded to 4
  {
    const char* names[11] = {"dof_damping", "dof_frictionloss", "dof_armature", "jnt_stiffness", "dof_invweight0", "body_mass",
                             "body_inertia", "body_ipos", "body_iquat", "geom_friction", "geom_invweight0"};
    int off = 0;
    for (int k = 0; k < 11; k++) {
      const float* src = nullptr; int cnt = 0;
      const float* q = h.reals.data();
#define X(name, c) if (std::string(#name) == names[k]) { src = q; cnt = (c); } q += (c);
      LOCOSIM_MP_REAL_FIELDS(X)
#undef X
      h.po[k] = off;
      h.default_row.insert(h.default_row.end(), src, src + cnt);
      off += cnt;
    }
    h.po[11] = off;
    h.default_row.push_back(h.meaninertia);
    off += 1;
    h.po[12] = off;                                    // user features (LS_OBS_PARAM)
    for (int k = 0; k < LS_POOL_USER; k++) h.default_row.push_back(0.0f);
    off += LS_POOL_USER;
    while (off % 4) { h.default_row.push_back(0.0f); off++; }
    h.pool_P = off;
  }
  (void)nu; (void)np; (void)nm;
  return "";
}

static inline void bind_model(DevModel& m, const HostModel& h, const int* ibase, const float* rbase) {
  m.nb = h.nb; m.nv = h.nv; m.ng = h.ng; m.nu = h.nu; m.np = h.np; m.nm = h.nm;
  m.integrator = h.integrator; m.cone = h.cone; m.iterations = h.iterations; m.nlevel = h.nlevel; m.nfric = h.nfric;
  m.timestep = h.timestep; m.gravity[0] = h.gravity[0]; m.gravity[1] = h.gravity[1]; m.gravity[2] = h.gravity[2];
  m.impratio = h.impratio; m.tolerance = h.tolerance; m.meaninertia = h.meaninertia; m.has_damping = h.has_damping;
  m.np_prim = h.np_prim; m.pk_n = h.np - h.nterr;
  m.np = h.np - h.nterr;           // (the terrain pairs are the terrain pass's: locosim_core.cuh terrain_pass)
  const int nb = h.nb, nv = h.nv, ng = h.ng, nu = h.nu, np = h.np, nm = h.nm;
  const int* ip = ibase;
  const float* rp = rbase;
#define X(name, cnt) m.name = ip; ip += (cnt);
  LOCOSIM_MP_INT_FIELDS(X)
#undef X
#define X(name, cnt) m.name = rp; rp += (cnt);
  LOCOSIM_MP_REAL_FIELDS(X)
#undef X
  m.body_level = ip; ip += nb;
  m.body_dofmask = ip; ip += nb;
  m.dof_frow = ip; ip += nv;
  m.tri_ij = ip; ip += 32 * 33 / 2;
  m.pair_packed = ip; ip += m.np;
  m.pair_bound = reinterpret_cast<const float*>(ip); ip += m.np;
  m.po_dof_damping = h.po[0]; m.po_dof_frictionloss = h.po[1]; m.po_dof_armature = h.po[2]; m.po_jnt_stiffness = h.po[3];
  m.po_dof_invweight0 = h.po[4]; m.po_body_mass = h.po[5]; m.po_body_inertia = h.po[6]; m.po_body_ipos = h.po[7];
  m.po_body_iquat = h.po[8]; m.po_geom_friction = h.po[9]; m.po_geom_invweight0 = h.po[10]; m.po_meaninertia = h.po[11]; m.po_user = h.po[12];
  m.pool_P = h.pool_P;
  (void)nu; (void)nm; (void)ng;
}

// ---- which compiled configuration (locosim_config.h) runs a model: one rule for the CUDA engine and the emulation build ----
static inline bool has_convex_pairs(const HostModel& hm) {
  DevModel v;
  bind_model(v, hm, hm.ints.data(), hm.reals.data());
  for (int p = 0; p < v.np; p++)
    if (v.pair_packed[p] & (2 << 24)) return true;
  return false;
}
static inline bool has_boxbox_pairs(const HostModel& hm) {
  DevModel v;
  bind_model(v, hm, hm.ints.data(), hm.reals.data());
  for (int p = 0; p < v.np; p++)
    if (v.geom_type[v.pair_geom[2 * p]] == LS_GEOM_BOX && v.geom_type[v.pair_geom[2 * p + 1]] == LS_GEOM_BOX) return true;
  return false;
}
template <class C>
static inline bool cfg_fits(const HostModel& hm, int obs_dim) {
  if (!C::CONVEX && has_convex_pairs(hm)) return false;
  if (!C::BOXBOX && has_boxbox_pairs(hm)) return false;
  if ((int)C::TERRAIN != (hm.hf_nrow > 0 ? 1 : 0)) return false;
  return hm.nv <= C::NV && hm.nb <= C::NB && hm.ng <= C::NG && obs_dim <= C::MAXOBS && hm.cone == (int)C::CONE &&
         hm.integrator == (int)C::RK4;
}
// 0 CfgEllEuler, 1 CfgPyrEuler, 2 CfgPyrRK4, 3 CfgPyrEuler29, 4 CfgPyrRK4_31, 5 CfgPyrEuler31, 6 CfgEllEulerTerrain, -1 none
// fits (the first that fits wins, so a model keeps the smallest configuration it fits; a model with a terrain fits
// CfgEllEulerTerrain only)
static inline int select_cfg(const HostModel& hm, int obs_dim) {
  if (hm.hf_nrow > 0) return cfg_fits<CfgEllEulerTerrain>(hm, obs_dim) ? 6 : -1;
  if (cfg_fits<CfgEllEuler>(hm, obs_dim)) return 0;
  if (cfg_fits<CfgPyrEuler>(hm, obs_dim)) return 1;
  if (cfg_fits<CfgPyrRK4>(hm, obs_dim)) return 2;
  if (cfg_fits<CfgPyrEuler29>(hm, obs_dim)) return 3;
  if (cfg_fits<CfgPyrRK4_31>(hm, obs_dim)) return 4;
  if (cfg_fits<CfgPyrEuler31>(hm, obs_dim)) return 5;
  return -1;
}

struct HostTask {
  std::vector<int> ints;
  std::vector<float> reals;
  int obs_dim, n_done, reward_type, n_substeps, n_traj, traj_len, n_goal, recenter0, recenter1, ri[4], use_absorbing;
  int n_grf = 0, n_grf_geom = 0;
  int rot[3] = {-1, -1, -1};
  float rp[2];
  float track[4] = {0, 0, 0, 0};
};

static inline std::string parse_task(HostTask& t, int nu, int nv, int ng, const int* ti, int nti, const double* tr, int ntr) {
  if (nti < TKI_HEADER_LEN || ti[TKI_MAGIC] != LOCOSIM_TASK_MAGIC) return "bad TaskSpec magic";
  if (ti[TKI_VERSION] != LOCOSIM_TASK_VERSION) return "TaskSpec version mismatch";
  t.obs_dim = ti[TKI_OBS_DIM]; t.n_done = ti[TKI_N_DONE]; t.reward_type = ti[TKI_REWARD_TYPE];
  t.n_substeps = ti[TKI_N_SUBSTEPS]; t.n_traj = ti[TKI_N_TRAJ]; t.traj_len = ti[TKI_TRAJ_LEN]; t.n_goal = ti[TKI_N_GOAL];
  t.recenter0 = ti[TKI_RECENTER0]; t.recenter1 = ti[TKI_RECENTER1];
  for (int k = 0; k < 4; k++) t.ri[k] = ti[TKI_REWARD_I0 + k];
  t.use_absorbing = ti[TKI_USE_ABSORBING];
  t.n_grf = ti[TKI_N_GRF]; t.n_grf_geom = ti[TKI_N_GRF_GEOM];
  if (t.n_grf < 0 || t.n_grf > LS_MAX_GRF) return "n_grf out of range";
  t.rp[0] = (float)tr[TKR_REWARD_P0]; t.rp[1] = (float)tr[TKR_REWARD_P1];
  for (int k = 0; k < 3; k++) t.rot[k] = ti[TKI_ROT_Q + k];
  for (int k = 0; k < 4; k++) t.track[k] = (float)tr[TKR_TRACK_WP + k];
  if (t.rot[0] >= nv || t.rot[1] >= nv || t.rot[2] >= nv) return "random-rotation index out of range";
  size_t ni = 2 * (size_t)t.obs_dim + t.n_done + (size_t)nu + (size_t)t.n_grf_geom;
  size_t nr = 2 * (size_t)nu + 2 * (size_t)t.n_done + (size_t)t.n_traj * t.traj_len * (2 * nv + t.n_goal);
  if ((size_t)nti != TKI_HEADER_LEN + ni || (size_t)ntr != TKR_HEADER_LEN + nr) return "TaskSpec size mismatch";
  if (t.n_goal > 4) return "n_goal > 4";
  if (t.n_grf > 0 && t.n_grf_geom != ng) return "grf_group length != ngeom";
  t.ints.assign(ti + TKI_HEADER_LEN, ti + nti);
  t.reals.resize(nr);
  for (size_t i = 0; i < nr; i++) t.reals[i] = (float)tr[TKR_HEADER_LEN + i];
  return "";
}

static inline void bind_task(DevTask& d, const HostTask& t, int nu, const int* ibase, const float* rbase) {
  d.obs_dim = t.obs_dim; d.n_done = t.n_done; d.reward_type = t.reward_type; d.n_substeps = t.n_substeps;
  d.n_traj = t.n_traj; d.traj_len = t.traj_len; d.n_goal = t.n_goal; d.recenter0 = t.recenter0; d.recenter1 = t.recenter1;
  for (int k = 0; k < 4; k++) d.ri[k] = t.ri[k];
  d.use_absorbing = t.use_absorbing; d.rp[0] = t.rp[0]; d.rp[1] = t.rp[1]; d.n_grf = t.n_grf;
  for (int k = 0; k < 3; k++) d.rot[k] = t.rot[k];
  for (int k = 0; k < 4; k++) d.track[k] = t.track[k];
  const int* ip = ibase;
  d.obs_src_type = ip; ip += t.obs_dim; d.obs_src_idx = ip; ip += t.obs_dim; d.done_obs_idx = ip; ip += t.n_done; d.act_idx = ip; ip += nu;
  d.grf_group = ip;
  const float* rp = rbase;
  d.act_mean = rp; rp += nu; d.act_delta = rp; rp += nu; d.done_lo = rp; rp += t.n_done; d.done_hi = rp; rp += t.n_done;
  d.table = rp;
}
