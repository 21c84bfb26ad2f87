/*
 * Height-field terrain (include/locosim.h locosim_set_terrain_origin: MuJoCo 2.3.7's hfield geom and mjc_ConvexHField as this
 * project defines them) on top of the fp64 CPU oracle -- TEST INFRASTRUCTURE.
 *
 * The oracle (oracle/locosim_ref.c) stays the fixed yardstick of the physics it already covers; this translation unit
 * compiles it in and adds the terrain around it:
 *   - a ModelPack with a terrain is loaded by the oracle without its trailing hfield_data and without the terrain pairs
 *     (they close the pair table, so the oracle's collision() sees the other pairs only);
 *   - hfield_pair: the cell range of a geom's bounding box, the prisms in (row, column, triangle) order, the skip test, and
 *     one MPR per prism through the oracle's own convex_pair (ccd_mpr_penetration). A prism is handed to it as a 6-vertex
 *     mesh geom of a scratch model (bottom vertices first, then the top ones, each in the triangle's order: the support
 *     scan's first maximum wins, as in the engine), centred on the vertices' mean;
 *   - reft_forward / reft_step: the oracle's mj_forward with the terrain contacts appended after the oracle's own ones
 *     (before make_constraint), and Euler sub-steps on it.
 * Built by tests/terrain_ref.py into tests/_build.
 */
#include "../../oracle/locosim_ref.c"

#define TERR_MAXCONPAIR 50

typedef struct {
  int nrow, ncol, geom, p0, npair;
  double size[4], pos[3], origin[2];
  double* data;
} Terrain;

typedef struct {
  RefSim* s;
  Terrain t;
} TSim;

/* one scratch model for the prism MPRs: geom 0 = the prism (mesh of 6 vertices), geom 1 = the robot geom */
static __thread RefSim* g_scr;
static __thread int g_scr_type[2], g_scr_adr[2] = {0, 0}, g_scr_num[2] = {6, 0};
static __thread double g_scr_size[6], g_scr_vert[18];

static void prism(const Terrain* t, int r, int c, int tri, double v[6][3]) {
  const int rr[3] = {tri ? r + 1 : r, tri ? r : r + 1, tri ? r + 1 : r};
  const int cc[3] = {c, tri ? c + 1 : c, c + 1};
  const double dx = 2 * t->size[0] / (t->ncol - 1), dy = 2 * t->size[1] / (t->nrow - 1);
  for (int i = 0; i < 3; i++) {
    v[i][0] = v[3 + i][0] = dx * cc[i] - t->size[0];
    v[i][1] = v[3 + i][1] = dy * rr[i] - t->size[1];
    v[i][2] = -t->size[3];
    v[3 + i][2] = t->data[rr[i] * t->ncol + cc[i]] * t->size[2];
  }
}

static double extent(int type, const double* mat, const double* size, int k) {
  double a = fabs(mat[3 * k + 2]);
  if (type == LS_GEOM_SPHERE) return size[0];
  if (type == LS_GEOM_CAPSULE) return size[0] + size[1] * a;
  if (type == LS_GEOM_CYLINDER) return size[0] * sqrt(fmax(1 - a * a, 0)) + size[1] * a;
  return fabs(mat[3 * k]) * size[0] + fabs(mat[3 * k + 1]) * size[1] + a * size[2];
}

/* mjc_ConvexHField of the terrain and a geom (type, world position, world frame, size): up to TERR_MAXCONPAIR raw contacts
 * (dist, world position, normal from the terrain into the geom); *nmpr counts the MPR runs */
static int hfield_pair(const Terrain* t, int type, const double* gpos, const double* gmat, const double* gsize, double margin,
                       RawCon* out, long* nmpr) {
  const double f[3] = {t->pos[0] - t->origin[0], t->pos[1] - t->origin[1], t->pos[2]};
  const double p[3] = {gpos[0] - f[0], gpos[1] - f[1], gpos[2] - f[2]};      /* the geom in the field's frame */
  if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) return 0;
  const double hx = extent(type, gmat, gsize, 0), hy = extent(type, gmat, gsize, 1), hz = extent(type, gmat, gsize, 2);
  const double zmin = p[2] - hz;
  if (p[0] - hx - margin > t->size[0] || p[0] + hx + margin < -t->size[0] || p[1] - hy - margin > t->size[1] ||
      p[1] + hy + margin < -t->size[1] || zmin - margin > t->size[2] || p[2] + hz + margin < -t->size[3])
    return 0;
  const double dx = 2 * t->size[0] / (t->ncol - 1), dy = 2 * t->size[1] / (t->nrow - 1);
  int cmin = (int)floor((p[0] - hx - margin + t->size[0]) / dx), cmax = (int)ceil((p[0] + hx + margin + t->size[0]) / dx);
  int rmin = (int)floor((p[1] - hy - margin + t->size[1]) / dy), rmax = (int)ceil((p[1] + hy + margin + t->size[1]) / dy);
  if (cmin < 0) cmin = 0;
  if (rmin < 0) rmin = 0;
  if (cmax > t->ncol - 1) cmax = t->ncol - 1;
  if (rmax > t->nrow - 1) rmax = t->nrow - 1;
  if (!g_scr) g_scr = (RefSim*)calloc(1, sizeof(RefSim));
  Model* m = &g_scr->m;
  m->geom_type = g_scr_type; m->geom_meshadr = g_scr_adr; m->geom_meshnum = g_scr_num;
  m->geom_size = g_scr_size; m->mesh_vert = g_scr_vert;
  g_scr_type[0] = LS_GEOM_MESH; g_scr_type[1] = type;
  for (int k = 0; k < 3; k++) { g_scr_size[3 + k] = gsize[k]; g_scr->gxpos[1][k] = p[k]; }
  for (int k = 0; k < 9; k++) { g_scr->gxmat[1][k] = gmat[k]; g_scr->gxmat[0][k] = (k % 4 == 0); }
  int cnt = 0;
  for (int r = rmin; r < rmax; r++)
    for (int c = cmin; c < cmax; c++)
      for (int tri = 0; tri < 2; tri++) {
        double v[6][3], cen[3] = {0, 0, 0};
        prism(t, r, c, tri, v);
        if (v[3][2] < zmin - margin && v[4][2] < zmin - margin && v[5][2] < zmin - margin) continue;
        for (int i = 0; i < 6; i++) for (int k = 0; k < 3; k++) cen[k] += v[i][k] / 6;
        for (int i = 0; i < 6; i++) for (int k = 0; k < 3; k++) g_scr_vert[3 * i + k] = v[i][k] - cen[k];
        for (int k = 0; k < 3; k++) g_scr->gxpos[0][k] = cen[k];
        if (nmpr) (*nmpr)++;
        RawCon rc;
        if (convex_pair(&rc, g_scr, 0, 1, margin) == 1) {
          for (int k = 0; k < 3; k++) rc.pos[k] += f[k];
          out[cnt++] = rc;
          if (cnt >= TERR_MAXCONPAIR) return cnt;
        }
      }
  return cnt;
}

/* ---- a sim with a terrain ---- */
TSim* reft_create(const int* ints, int n_ints, const double* reals, int n_reals) {
  const int nrow = ints[MPI_HF_NROW], ncol = ints[MPI_HF_NCOL];
  const int nhf = nrow * ncol;
  TSim* ts = (TSim*)calloc(1, sizeof(TSim));
  ts->s = ref_create(ints, n_ints, reals, n_reals - nhf);
  if (!ts->s) { free(ts); return NULL; }
  Model* m = &ts->s->m;
  Terrain* t = &ts->t;
  t->nrow = nrow; t->ncol = ncol; t->geom = -1;
  if (nhf > 0) {
    t->geom = m->ng - 1;
    for (int k = 0; k < 4; k++) t->size[k] = reals[MPR_HF_SIZE + k];
    for (int k = 0; k < 3; k++) t->pos[k] = m->geom_pos[3 * t->geom + k];
    t->data = (double*)malloc(sizeof(double) * nhf);
    memcpy(t->data, reals + n_reals - nhf, sizeof(double) * nhf);
    int nt = 0;
    while (nt < m->np && m->pair_geom[2 * (m->np - 1 - nt)] == t->geom) nt++;
    t->npair = nt;
    t->p0 = m->np - nt;
    m->np = t->p0;                   /* the oracle's collision() runs the other pairs */
  }
  return ts;
}
void reft_destroy(TSim* ts) { if (ts) { ref_destroy(ts->s); free(ts->t.data); free(ts); } }
RefSim* reft_sim(TSim* ts) { return ts->s; }
void reft_set_origin(TSim* ts, double ox, double oy) { ts->t.origin[0] = ox; ts->t.origin[1] = oy; }

static long g_terr_mpr = 0;
long reft_mpr_calls(void) { return g_terr_mpr; }

static void terrain_collision(TSim* ts) {
  RefSim* s = ts->s;
  const Model* m = &s->m;
  const Terrain* t = &ts->t;
  RawCon raw[TERR_MAXCONPAIR];
  for (int q = 0; q < t->npair; q++) {
    const int g1 = t->geom, g2 = m->pair_geom[2 * (t->p0 + q) + 1];
    const double margin = fmax(m->geom_margin[g1], m->geom_margin[g2]);
    const int n = hfield_pair(t, m->geom_type[g2], s->gxpos[g2], s->gxmat[g2], m->geom_size + 3 * g2, margin, raw, &g_terr_mpr);
    for (int k = 0; k < n && s->ncon < MAXCON; k++) {
      Contact* c = &s->con[s->ncon++];
      c->dist = raw[k].dist;
      memcpy(c->pos, raw[k].pos, sizeof(c->pos));
      memcpy(c->frame, raw[k].frame, sizeof(c->frame));
      make_frame(c->frame);
      c->geom1 = g1; c->geom2 = g2;
      contact_params(m, g1, g2, c);
      c->exclude = (c->dist >= c->includemargin);
      c->efc_address = -1;
      c->mu = 0;
    }
  }
}

/* the oracle's forward() with the terrain contacts after its own */
void reft_forward(TSim* ts, const double* ctrl) {
  RefSim* s = ts->s;
  const Model* m = &s->m;
  int nv = m->nv;
  if (ctrl) memcpy(s->ctrl, ctrl, sizeof(double) * m->nu);
  kinematics(s);
  comPos(s);
  crb(s);
  collision(s);
  terrain_collision(ts);
  make_constraint(s);
  comVel(s);
  passive(s);
  reference_constraint(s);
  rne_bias(s);
  actuation(s);
  for (int i = 0; i < nv; i++) {
    s->qfrc_smooth[i] = s->qfrc_passive[i] - s->qfrc_bias[i] + s->qfrc_actuator[i];
    s->qacc_smooth[i] = s->qfrc_smooth[i];
  }
  chol_solve(s->LM, nv, s->qacc_smooth);
  fwd_constraint(s);
}

/* nsub Euler sub-steps at ctrl (the terrain configuration is Euler only) */
void reft_step(TSim* ts, const double* ctrl, int nsub) {
  for (int k = 0; k < nsub; k++) {
    reft_forward(ts, ctrl);
    euler(ts->s);
  }
}

/* single geom against a terrain: type, world position, row-major world frame, size, margin; the field (nrow x ncol samples
 * `data`, size[4], geom position pos[3], origin[2]); out [TERR_MAXCONPAIR, 7] = dist, pos, normal; returns the count */
int reft_debug_geom(int nrow, int ncol, const double* data, const double* size, const double* pos, const double* origin,
                    int type, const double* gpos, const double* gmat, const double* gsize, double margin, double* out,
                    long* nmpr) {
  Terrain t;
  memset(&t, 0, sizeof(t));
  t.nrow = nrow; t.ncol = ncol; t.data = (double*)data;
  for (int k = 0; k < 4; k++) t.size[k] = size[k];
  for (int k = 0; k < 3; k++) t.pos[k] = pos[k];
  t.origin[0] = origin[0]; t.origin[1] = origin[1];
  RawCon raw[TERR_MAXCONPAIR];
  int n = hfield_pair(&t, type, gpos, gmat, gsize, margin, raw, nmpr);
  for (int i = 0; i < n; i++) {
    out[7 * i] = raw[i].dist;
    for (int k = 0; k < 3; k++) { out[7 * i + 1 + k] = raw[i].pos[k]; out[7 * i + 4 + k] = raw[i].frame[k]; }
  }
  return n;
}
