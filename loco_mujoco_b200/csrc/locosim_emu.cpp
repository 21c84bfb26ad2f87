// Serial CPU emulation of the warp-cooperative engine core (development aid only; see locosim_core.cuh).
// Built by tools/build_emu.sh into scratch/; NOT shipped, NOT loaded by the product path.
#define LS_EMULATE 1
#define LOCOSIM_TERRAIN 1      // (the terrain configuration's collision pass: see locosim_terrain.cu)
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "locosim_config.h"
#include "locosim_host.h"

struct EmuBase {
  HostModel hm;
  DevModel m;
  DevApplied ap = {nullptr, nullptr};
  DevContact cw = {nullptr, 1};
  DevDof dof = {nullptr, 1};
  DevConList cl = {nullptr, 1};
  DevConRows cr = {nullptr, nullptr};
  DevTerrain terr = {};              // the terrain configuration's height field; origin: row 0 of the engine's [N, 2]
  std::vector<float> act;            // the dof outputs' actuator-force scratch (row 0 of the engine's [N, nu])
  SolverOpts so;
  std::vector<int> grf_group; int n_grf = 0;
  virtual ~EmuBase() {}
  virtual void reset(const double* q, const double* v) = 0;
  virtual void step(const double* ctrl, int nsub) = 0;
  virtual void fwd(const double* ctrl) = 0;
  virtual void get(double* q, double* v, double* qacc, double* ws) = 0;
  virtual void set_ws(const double* w) = 0;
  virtual int info(int k) = 0;
  virtual void bind_prm() = 0;
  virtual void contact(int k, double* o) = 0;
  virtual void grf(double* o, int clear) = 0;
  virtual void frames(double* gx, double* bx) = 0;
  virtual void poison() = 0;
  virtual void body(float* out) = 0;
  virtual void ref(const DevTask& t, const float* row, float angle, float* out) = 0;
  virtual void inv(const double* qacc, float* out) = 0;
  virtual void dyn(const DynOut& o) = 0;
  virtual void fwd_out(const double* ctrl, const FwdOut& o) = 0;
  virtual int max_contacts() = 0;
  virtual void ray(const float* pnt, const float* vec, int n_rays, int frame, int fb, int exclude, int flags, float* dist,
                   int* geom, float* normal) = 0;
};
template <class C>
struct EmuT : EmuBase {
  EnvS<C> e;
  EmuT() { memset(&e, 0, sizeof(e)); }
  void reset(const double* q, const double* v) override {
    for (int i = 0; i < m.nv; i++) { e.qpos[i] = (float)q[i]; e.qvel[i] = (float)v[i]; e.qacc_ws[i] = 0; e.qacc[i] = 0; }
  }
  void step(const double* ctrl, int nsub) override {
    for (int i = 0; i < m.nu; i++) e.ctrl[i] = (float)ctrl[i];
    c_models[0] = m; c_terrain[0] = terr; c_applied[0] = ap; c_contact[0] = cw; c_contact[0].n_substeps = nsub;
    c_dof[0] = dof; c_dof[0].n_substeps = nsub; c_dof_act[0] = dof.out ? act.data() : nullptr;
    c_conlist[0] = cl; c_conlist[0].n_substeps = nsub; c_conrows[0] = cr;
    e.substep = 0;
    physics_substeps(0, e, so, nsub, grf_group.data(), n_grf);
  }
  void fwd(const double* ctrl) override {
    for (int i = 0; i < m.nu; i++) e.ctrl[i] = (float)ctrl[i];
    c_models[0] = m; c_terrain[0] = terr; c_applied[0] = ap; c_dof[0] = dof; c_dof_act[0] = dof.out ? act.data() : nullptr;
    forward(0, e, so);
  }
  void get(double* q, double* v, double* qacc, double* ws) override {
    for (int i = 0; i < m.nv; i++) {
      if (q) q[i] = e.qpos[i];
      if (v) v[i] = e.qvel[i];
      if (qacc) qacc[i] = e.qacc[i];
      if (ws) ws[i] = e.qacc_ws[i];
    }
  }
  void set_ws(const double* w) override { for (int i = 0; i < m.nv; i++) e.qacc_ws[i] = (float)w[i]; }
  int info(int k) override { return k == 0 ? e.ncon : (k == 1 ? e.nefc : e.solver_iter); }
  void contact(int k, double* o) override {
    o[0] = e.con_g1[k]; o[1] = e.con_g2[k]; o[2] = e.con_dim[k]; o[3] = e.con_dist[k];
    int r0 = e.nunit + e.con_row[k], dim = e.con_dim[k];
    for (int j = 0; j < 8; j++) o[4 + j] = (j < (C::CONE == 1 || dim == 1 ? dim : 2 * (dim - 1))) ? e.r_force[r0 + j] : 0.0;
    for (int j = 0; j < 3; j++) { o[12 + j] = e.con_frame[k][j]; o[15 + j] = e.con_pos[k][j]; }
  }
  void grf(double* o, int clear) override { for (int k = 0; k < 3 * LS_MAX_GRF; k++) { o[k] = e.grf[k]; if (clear) e.grf[k] = 0; } }
  void frames(double* gx, double* bx) override {
    for (int g = 0; g < m.ng; g++) for (int k = 0; k < 3; k++) gx[3 * g + k] = e.gxpos[g][k];
    for (int b = 0; b < m.nb; b++) { for (int k = 0; k < 3; k++) bx[7 * b + k] = e.xpos[b][k]; for (int k = 0; k < 4; k++) bx[7 * b + 3 + k] = e.xquat[b][k]; }
  }
  // What a sub-step launch of the CUDA engine (substep_kernel) starts from: the working set is lost except the fields it
  // carries in HBM between launches (state, warm start, control, goal, the step's counters, the separating-direction cache,
  // the summed foot forces); everything else is poisoned, then rebuilt the way the kernel rebuilds it.
  void poison() override {
    EnvS<C>* keep = new EnvS<C>(e);
    memset((void*)&e, 0xff, sizeof(e));
    for (int i = 0; i < m.nv; i++) { e.qpos[i] = keep->qpos[i]; e.qvel[i] = keep->qvel[i]; e.qacc_ws[i] = keep->qacc_ws[i]; e.qacc[i] = 0; }
    for (int i = 0; i < m.nu; i++) e.ctrl[i] = keep->ctrl[i];
    for (int k = 0; k < 4; k++) e.goal[k] = keep->goal[k];
    e.prm = keep->prm; e.pk_tab = keep->pk_tab; e.env = keep->env;
    init_workspace(0, e);
    e.iter_sum = keep->iter_sum; e.mpr_calls = keep->mpr_calls; e.sep_next = keep->sep_next;
    for (int k = 0; k < EnvS<C>::NSEP; k++) {
      e.sep_pair[k] = keep->sep_pair[k];
      for (int j = 0; j < 3; j++) e.sep_dir[k][j] = keep->sep_dir[k][j];
    }
    for (int k = 0; k < 3 * LS_MAX_GRF; k++) e.grf[k] = keep->grf[k];
    delete keep;
  }
  void body(float* out) override { c_models[0] = m; c_terrain[0] = terr; body_outputs(0, e, out, (float*)nullptr); }
  void ref(const DevTask& t, const float* row, float angle, float* out) override {
    c_models[0] = m; c_terrain[0] = terr;
    reference_outputs(0, t, e, row, angle, out, (float*)nullptr);
  }
  void inv(const double* qacc, float* out) override {
    c_models[0] = m; c_terrain[0] = terr;
    e.substep = -1;
    for (int i = 0; i < m.nv; i++) e.qacc[i] = (float)qacc[i];
    inverse_dynamics(0, e, out);
  }
  void dyn(const DynOut& o) override {
    c_models[0] = m; c_terrain[0] = terr;
    e.substep = -1;
    dynamics_terms(0, e, o);
  }
  void fwd_out(const double* ctrl, const FwdOut& o) override {
    for (int i = 0; i < m.nu; i++) e.ctrl[i] = (float)ctrl[i];
    c_models[0] = m; c_terrain[0] = terr; c_applied[0] = ap;
    e.substep = -1;
    init_workspace(0, e);
    forward_dynamics(0, e, so, o);
  }
  int max_contacts() override { return C::MAXCON; }
  void ray(const float* pnt, const float* vec, int n_rays, int frame, int fb, int exclude, int flags, float* dist, int* geom,
           float* normal) override {
    c_models[0] = m; c_terrain[0] = terr;
    const bool bad = nonfinite_state(e, m.nv);
    std::vector<RayGeom> G(m.ng);
    if (!bad) {
      kinematics(0, e);
      for (int g = 0; g < m.ng; g++) ray_stage_geom(0, e, g, G[g]);
    }
    for (int k = 0; k < n_rays; k++) {
      float p[3], v[3], nrm[3] = {0, 0, 0};
      dist[k] = -1; geom[k] = -1;
      if (!bad) {
        ray_to_world(e, frame, fb, pnt + 3 * k, vec + 3 * k, p, v);
        dist[k] = ray_geoms(G.data(), m.ng, p, v, exclude, flags, geom + k, nrm);
        if (C::TERRAIN) ray_terrain(0, 0, p, v, exclude, flags, dist + k, geom + k, nrm);
      }
      if (normal) for (int c = 0; c < 3; c++) normal[3 * k + c] = nrm[c];
    }
  }
  void bind_prm() override { e.prm = hm.default_row.data(); e.pk_tab = m.pair_packed; c_models[0] = m; c_terrain[0] = terr; init_workspace(0, e); }
};

extern "C" {
// the configuration the CUDA engine would run the model with (select_cfg; observation sizes fit every configuration)
int emu_select_cfg(const int* ints, int n_ints, const double* reals, int n_reals) {
  HostModel hm;
  if (!parse_model(hm, ints, n_ints, reals, n_reals).empty()) return -1;
  return select_cfg(hm, 0);
}
EmuBase* emu_create(const int* ints, int n_ints, const double* reals, int n_reals) {
  HostModel hm;
  std::string err = parse_model(hm, ints, n_ints, reals, n_reals);
  if (!err.empty()) { fprintf(stderr, "emu: %s\n", err.c_str()); return nullptr; }
  EmuBase* s;
  switch (select_cfg(hm, 0)) {
    case 0: s = new EmuT<CfgEllEuler>(); break;
    case 1: s = new EmuT<CfgPyrEuler>(); break;
    case 2: s = new EmuT<CfgPyrRK4>(); break;
    case 3: s = new EmuT<CfgPyrEuler29>(); break;
    case 4: s = new EmuT<CfgPyrRK4_31>(); break;
    case 5: s = new EmuT<CfgPyrEuler31>(); break;
    case 6: s = new EmuT<CfgEllEulerTerrain>(); break;
    default: fprintf(stderr, "emu: no compiled configuration fits this model\n"); return nullptr;
  }
  s->hm = hm;
  bind_model(s->m, s->hm, s->hm.ints.data(), s->hm.reals.data());
  if (s->hm.hf_nrow > 0) {
    DevTerrain& t = s->terr;
    t.data = s->hm.reals.data() + s->hm.hf_off; t.origin = nullptr;
    t.nrow = s->hm.hf_nrow; t.ncol = s->hm.hf_ncol; t.geom = s->hm.hf_geom; t.p0 = s->hm.np - s->hm.nterr; t.npair = s->hm.nterr;
    for (int k = 0; k < 4; k++) t.size[k] = s->hm.hf_size[k];
    for (int k = 0; k < 3; k++) t.pos[k] = s->hm.hf_pos[k];
  }
  s->bind_prm();
  s->so.tolerance = 1e-5f; s->so.ls_tolerance = 0.1f; s->so.max_iter = 20; s->so.ls_iter = 16;
  return s;
}
void emu_destroy(EmuBase* s) { delete s; }
void emu_set_opts(EmuBase* s, float tol, float ls_tol, int max_iter, int ls_iter) {
  s->so.tolerance = tol; s->so.ls_tolerance = ls_tol; s->so.max_iter = max_iter; s->so.ls_iter = ls_iter;
}
void emu_reset(EmuBase* s, const double* qpos, const double* qvel) { s->reset(qpos, qvel); }
void emu_step(EmuBase* s, const double* ctrl, int nsub) { s->step(ctrl, nsub); }
void emu_forward(EmuBase* s, const double* ctrl) { s->fwd(ctrl); }
void emu_get_state(EmuBase* s, double* qpos, double* qvel) { s->get(qpos, qvel, nullptr, nullptr); }
void emu_get_qacc(EmuBase* s, double* qacc) { s->get(nullptr, nullptr, qacc, nullptr); }
void emu_get_ws(EmuBase* s, double* w) { s->get(nullptr, nullptr, nullptr, w); }
void emu_set_ws(EmuBase* s, const double* w) { s->set_ws(w); }
// applied forces of the emulated env (row 0 of the engine's layout: xfrc fp32 [nb, 6], qfrc fp32 [nv]; either may be NULL),
// read by every later emu_step / emu_forward from the caller's memory
void emu_set_applied(EmuBase* s, float* xfrc, float* qfrc) { s->ap.xfrc = xfrc; s->ap.qfrc = qfrc; }
// body outputs of the emulated env's current state (locosim_set_body_outputs): fp32 [nb, LS_BODY_DIM] into `out`
void emu_body_outputs(EmuBase* s, float* out) { s->body(out); }
// reference row (locosim_set_reference_outputs) of one reset-table row `row` (fp32, qpos then qvel) under rotation `angle`,
// with the model's own parameters: fp32 [nb, LS_BODY_DIM] into `out`. recenter: the qpos indices of root x / y; rot: the
// qpos index of the yaw and the dof indices of root vx / vy under setup_random_rot, or NULL. Leaves the emulated env in that
// reset state.
void emu_reference_row(EmuBase* s, const float* row, const int* recenter, const int* rot, float angle, float* out) {
  DevTask t;
  memset(&t, 0, sizeof(t));
  t.recenter0 = recenter[0]; t.recenter1 = recenter[1];
  for (int k = 0; k < 3; k++) t.rot[k] = rot ? rot[k] : -1;
  s->ref(t, row, angle, out);
}
// inverse dynamics (locosim_inverse) of the emulated env's current state at the acceleration qacc [nv]: fp32 [nv] into `out`,
// with the model's own parameters. Overwrites the env's acceleration and constraint working set (not its state or warm
// start), as a forward evaluation would.
void emu_inverse(EmuBase* s, const double* qacc, float* out) { s->inv(qacc, out); }
// dynamics terms (locosim_dynamics_terms) of the emulated env's current state, with the model's own parameters: row 0 of
// each output's layout (M fp32 [nv, nv], bias / passive [nv], com [LS_COM_DIM], jac [nb, 6, nv], jac_com [3, nv]; each may
// be NULL). Overwrites the env's kinematics and smooth-dynamics working set (not its state or warm start).
void emu_dynamics_terms(EmuBase* s, float* M, float* bias, float* passive, float* com, float* jac, float* jac_com) {
  s->dyn(DynOut{M, bias, passive, com, jac, jac_com});
}
// forward dynamics (locosim_forward) of the emulated env's current state and warm start at ctrl [nu] (fp64; the engine's
// ctrl, not the action), with the applied forces of emu_set_applied and the model's own parameters: row 0 of each output's
// layout (dof fp32 [nv, LS_DOF_DIM], body_acc [nb, LS_BODY_ACC_DIM], cfrc_int / cfrc_ext [nb, LS_CONTACT_DIM]; each may be
// NULL). Leaves the state as it was; the warm start becomes this evaluation's qacc, as after emu_forward.
void emu_forward_outputs(EmuBase* s, const double* ctrl, float* dof, float* body_acc, float* cfrc_int, float* cfrc_ext) {
  s->fwd_out(ctrl, FwdOut{dof, body_acc, cfrc_int, cfrc_ext});
}
// contact outputs of the emulated env (locosim_set_contact_outputs; row 0 of the engine's layout: fp32 [nb, LS_CONTACT_DIM], or
// NULL): every later emu_step(ctrl, nsub) runs as one control step of nsub sub-steps and leaves their mean wrench there
void emu_set_contact(EmuBase* s, float* wrench) { s->cw.wrench = wrench; }
// dof outputs of the emulated env (locosim_set_dof_outputs; row 0 of the engine's layout: fp32 [nv, LS_DOF_DIM], or NULL):
// every later emu_step(ctrl, nsub) runs as one control step of nsub sub-steps and leaves their mean there
void emu_set_dof(EmuBase* s, float* out) {
  s->act.assign(s->m.nu > 0 ? s->m.nu : 1, 0.0f);
  s->dof.out = out;
}
// contact list of the emulated env (locosim_set_contact_list_outputs; row 0 of the engine's layout: int32 [1], fp32
// [MAXCON, LS_CONLIST_DIM], int32 [MAXCON, LS_CONLIST_ID_DIM], all three or all NULL): every later emu_step(ctrl, nsub) runs
// as one control step of nsub sub-steps and leaves the list of its last sub-step there
void emu_set_contact_list(EmuBase* s, int* ncon, float* con, int* id) {
  s->cl.ncon = ncon; s->cr.con = con; s->cr.id = id;
}
// ray casting (locosim_ray) of the emulated env's current state, with the model's own parameters: the rays pnt / vec fp32
// [n_rays, 3] in `frame` of body fb, one at a time through the kernels' routines; dist fp32 [n_rays], geom int32 [n_rays],
// normal fp32 [n_rays, 3] (may be NULL). No argument is checked here (locosim_ray checks them). Overwrites the env's
// kinematics (not its state or warm start).
void emu_ray(EmuBase* s, const float* pnt, const float* vec, int n_rays, int frame, int fb, int exclude, int flags,
             float* dist, int* geom, float* normal) {
  s->ray(pnt, vec, n_rays, frame, fb, exclude, flags, dist, geom, normal);
}
// terrain origin of the emulated env (locosim_set_terrain_origin; row 0 of the engine's layout: fp32 [2], or NULL = zeros),
// read by every later step and query from the caller's memory
void emu_set_terrain_origin(EmuBase* s, float* origin) { s->terr.origin = origin; }
// the configuration's per-env contact cap (locosim_max_contacts)
int emu_max_contacts(EmuBase* s) { return s->max_contacts(); }
long emu_mpr_stat(int k) { long v[8] = {g_forward_evals, g_mpr_candidates, g_mpr_calls, g_mpr_supports, g_sep_found, g_sep_ok, g_mpr_nohit, g_obb_pass}; return v[k]; }
// the diagnostic switches of the emulated engine (LOCOSIM_DEBUG; e.g. 32: no capsule-hull test)
void emu_set_debug(int v) { c_debug = v; }
// capsule_hulls_apart of two geoms (type, position, row-major frame, geom_size) with the pair's margin
int emu_capsule_hulls_apart(int t1, const float* pos1, const float* m1, const float* s1, int t2, const float* pos2,
                            const float* m2, const float* s2, float margin) {
  const float d[3] = {pos2[0] - pos1[0], pos2[1] - pos1[1], pos2[2] - pos1[2]};
  return capsule_hulls_apart(d, m1, t1, s1, m2, t2, s2, margin) ? 1 : 0;
}
long emu_ls_evals() { return g_ls_evals; }
long emu_ls_searches() { return g_ls_searches; }
int emu_ncon(EmuBase* s) { return s->info(0); }
void emu_contact(EmuBase* s, int k, double* o) { s->contact(k, o); }
void emu_set_grf(EmuBase* s, const int* group, int ng, int n_grf) { s->grf_group.assign(group, group + ng); s->n_grf = n_grf; }
void emu_get_grf(EmuBase* s, double* o, int clear) { s->grf(o, clear); }
void emu_frames(EmuBase* s, double* gx, double* bx) { s->frames(gx, bx); }
int emu_nefc(EmuBase* s) { return s->info(1); }
void emu_poison(EmuBase* s) { s->poison(); }
int emu_iter(EmuBase* s) { return s->info(2); }
int emu_sizeof_env(int which) {
  switch (which) {
    case 0: return (int)sizeof(EnvS<CfgEllEuler>);
    case 1: return (int)sizeof(EnvS<CfgPyrEuler>);
    case 3: return (int)sizeof(EnvS<CfgPyrEuler29>);
    case 4: return (int)sizeof(EnvS<CfgPyrRK4_31>);
    case 5: return (int)sizeof(EnvS<CfgPyrEuler31>);
    case 6: return (int)sizeof(EnvS<CfgEllEulerTerrain>);
    default: return (int)sizeof(EnvS<CfgPyrRK4>);
  }
}
}
