/*
 * Per-body contact wrenches (include/locosim.h locosim_set_contact_outputs) on top of the fp64 CPU oracle -- TEST
 * INFRASTRUCTURE.
 *
 * The oracle (oracle/locosim_ref.c) stays the fixed yardstick of the physics it already covers; this translation unit
 * compiles it in and restates the documented MuJoCo computation around it:
 *   mj_contactForce: the contact-frame force f of a contact (elliptic: its dim constraint forces; pyramidal: mju_decodePyramid),
 *                    which the oracle's ref_get_contact already decodes;
 *   world wrench:    F = f0 n + f1 t1 + f2 t2, T = f3 n + f4 t1 + f5 t2 (frame rows n, t1, t2; n points from geom1 to geom2);
 *   per body:        +F and (pos - xpos[b2]) x F + T on geom2's body, the negatives (about xpos[b1]) on geom1's body, the
 *                    signs of mj_rnePostConstraint; the world row stays zero;
 * and the window of the engine's output: the mean over a control step's sub-steps, each sub-step's contact list, xpos and
 * constraint forces taken after it (its last dynamics evaluation: Euler's only one, RK4's fourth stage).
 * Built by tests/contact_wrench_ref.py into tests/_build.
 */
#include "../../oracle/locosim_ref.c"

int refcw_nbody(const RefSim* s) { return s->m.nb; }

/* contact k of the last forward evaluation with its whole frame: out[0] = dist, out[1..3] = pos, out[4..12] = frame (rows n,
 * t1, t2), out[13] = geom1, out[14] = geom2, out[15] = dim, out[16..21] = the contact-frame force of mj_contactForce */
void refcw_get_contact(const RefSim* s, int k, double* out) {
  const Contact* c = &s->con[k];
  double o[16];
  ref_get_contact(s, k, o);
  out[0] = c->dist;
  for (int j = 0; j < 3; j++) out[1 + j] = c->pos[j];
  for (int j = 0; j < 9; j++) out[4 + j] = c->frame[j];
  out[13] = c->geom1; out[14] = c->geom2; out[15] = c->dim;
  for (int j = 0; j < 6; j++) out[16 + j] = o[10 + j];
}

/* per-body contact wrench [nb, 6] (force, torque about xpos; world frame) of the last forward evaluation, ADDED to out */
void refcw_add_wrench(const RefSim* s, double* out) {
  const Model* m = &s->m;
  for (int k = 0; k < s->ncon; k++) {
    const Contact* c = &s->con[k];
    double o[16], F[3], T[3];
    ref_get_contact(s, k, o);
    const double* f = o + 10;
    for (int j = 0; j < 3; j++) {
      F[j] = f[0] * c->frame[j] + f[1] * c->frame[3 + j] + f[2] * c->frame[6 + j];
      T[j] = f[3] * c->frame[j] + f[4] * c->frame[3 + j] + f[5] * c->frame[6 + j];
    }
    const int bs[2] = {m->geom_bodyid[c->geom1], m->geom_bodyid[c->geom2]};
    for (int side = 0; side < 2; side++) {
      const int b = bs[side];
      if (b == 0) continue;
      const double sg = side == 1 ? 1.0 : -1.0;
      double r[3] = {c->pos[0] - s->xpos[b][0], c->pos[1] - s->xpos[b][1], c->pos[2] - s->xpos[b][2]}, rxF[3];
      cross3(rxF, r, F);
      for (int j = 0; j < 3; j++) {
        out[6 * b + j] += sg * F[j];
        out[6 * b + 3 + j] += sg * (rxF[j] + T[j]);
      }
    }
  }
}

/* the physics of one control step of a RefEnv (action in [-1, 1] -> ctrl as refenv_step maps it, n_substeps sub-steps of
 * ref_step) and the mean per-body contact wrench over its sub-steps into wrench [nb, 6]; observation, reward and termination
 * are not evaluated: compare the state (ref_get_state) */
void refcw_env_step(RefEnv* e, const double* action, double* wrench) {
  const Task* t = &e->task;
  RefSim* s = e->sim;
  double ctrl[MAXNV];
  memset(ctrl, 0, sizeof(ctrl));
  for (int i = 0; i < s->m.nu; i++) ctrl[t->act_idx[i]] = action[i] * t->act_delta[i] + t->act_mean[i];
  memset(wrench, 0, sizeof(double) * 6 * s->m.nb);
  for (int k = 0; k < t->n_substeps; k++) {
    ref_step(s, ctrl, 1);
    refcw_add_wrench(s, wrench);
  }
  for (int j = 0; j < 6 * s->m.nb; j++) wrench[j] /= t->n_substeps;
}

/* the same for a bare RefSim: nsub sub-steps at ctrl */
void refcw_step(RefSim* s, const double* ctrl, int nsub, double* wrench) {
  memset(wrench, 0, sizeof(double) * 6 * s->m.nb);
  for (int k = 0; k < nsub; k++) {
    ref_step(s, ctrl, 1);
    refcw_add_wrench(s, wrench);
  }
  for (int j = 0; j < 6 * s->m.nb; j++) wrench[j] /= nsub;
}
