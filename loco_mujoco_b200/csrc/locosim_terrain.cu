// locosim_terrain.cu -- the kernels of the terrain configuration (locosim_config.h CfgEllEulerTerrain: UnitreeA1 on a height
// field), in a translation unit of their own that is linked into the engine library next to locosim.cu. It compiles the
// kernel templates of locosim.cu (step, sub-step and persistent kernels, launch and setup, body rows, the on-demand
// queries) for this configuration only, with LOCOSIM_TERRAIN defined: collision() then ends with the height-field pass
// (locosim_core.cuh terrain_pass). No other unit defines the macro, so their kernels keep their code. The handle, the
// C-ABI and the config-free kernels (reset, save / load state, regrouping) stay in locosim.cu, which calls the entry points
// below for configuration index 6.
//
// As in locosim_configs31.cu, the engine source is compiled inside a namespace of its own and this unit has its own
// __constant__ slots: the model's, every registered buffer's, and the terrain's (c_terrain: grid, size, heights and the
// registered origin buffer), all written by locosim_terrain_sync_model.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/locosim.h"
#include "../../include/locosim_modelpack.h"
#include "../../include/locosim_task.h"

#define LOCOSIM_EXTRA_CONFIGS_TU 1
#define LOCOSIM_TERRAIN 1
#define LS_DATASET_ENV(r) (-1 - (r))    // (dataset rows of locosim_create_dataset_inverse: no env, the zero terrain origin)
namespace locosimterrain {
#include "locosim.cu"

// the terrain pass adds no per-env shared memory: UnitreeA1 keeps its envs per SM
static_assert(sizeof(EnvS<CfgEllEulerTerrain>) == sizeof(EnvS<CfgEllEuler>), "the terrain configuration's EnvS is A1's");
}  // namespace locosimterrain

typedef locosimterrain::locosim_handle HandleTerrain;

extern "C" {

int locosim_terrain_sync_model(HandleTerrain* h) {
  using namespace locosimterrain;
  DevTerrain t;
  const HostModel& hm = h->hm;
  t.data = h->d_mreals + hm.hf_off;
  t.origin = h->terrain_origin;
  t.nrow = hm.hf_nrow; t.ncol = hm.hf_ncol; t.geom = hm.hf_geom; t.p0 = hm.np - hm.nterr; t.npair = hm.nterr;
  for (int k = 0; k < 4; k++) t.size[k] = hm.hf_size[k];
  for (int k = 0; k < 3; k++) t.pos[k] = hm.hf_pos[k];
  CK(cudaMemcpyToSymbol(c_terrain, &t, sizeof(DevTerrain), sizeof(DevTerrain) * h->slot));
  CK(cudaMemcpyToSymbol(c_models, &h->dm, sizeof(DevModel), sizeof(DevModel) * h->slot));
  CK(cudaMemcpyToSymbol(c_applied, &h->applied, sizeof(DevApplied), sizeof(DevApplied) * h->slot));
  CK(cudaMemcpyToSymbol(c_bodyout, &h->bodyout, sizeof(DevBodyOut), sizeof(DevBodyOut) * h->slot));
  CK(cudaMemcpyToSymbol(c_refout, &h->refout, sizeof(DevRefOut), sizeof(DevRefOut) * h->slot));
  CK(cudaMemcpyToSymbol(c_contact, &h->contact, sizeof(DevContact), sizeof(DevContact) * h->slot));
  CK(cudaMemcpyToSymbol(c_dof, &h->dof, sizeof(DevDof), sizeof(DevDof) * h->slot));
  CK(cudaMemcpyToSymbol(c_dof_act, &h->dof_act, sizeof(float*), sizeof(float*) * h->slot));
  CK(cudaMemcpyToSymbol(c_conrows, &h->conrows, sizeof(DevConRows), sizeof(DevConRows) * h->slot));
  CK(cudaMemcpyToSymbol(c_conlist, &h->conlist, sizeof(DevConList), sizeof(DevConList) * h->slot));
  return 0;
}

int locosim_terrain_setup(HandleTerrain* h) {
  using namespace locosimterrain;
  if (h->cfg != 6) { h->err = "not the terrain configuration"; return 1; }
  if (locosim_terrain_sync_model(h)) return 1;
  return setup_cfg<CfgEllEulerTerrain>(h);
}

int locosim_terrain_step(HandleTerrain* h, const float* a, float* o, float* r, uint8_t* d, float* no, int auto_reset,
                         cudaStream_t s) {
  using namespace locosimterrain;
  return launch_step<CfgEllEulerTerrain>(h, a, o, r, d, no, auto_reset, s);
}

int locosim_terrain_body(HandleTerrain* h, const uint8_t* mask, int parts, cudaStream_t s) {
  using namespace locosimterrain;
  return launch_body<CfgEllEulerTerrain>(h, mask, nullptr, 0, parts, s);
}

int locosim_terrain_dataset_bodies(HandleTerrain* h, float* body, float* next_body, cudaStream_t s) {
  using namespace locosimterrain;
  return launch_dataset_bodies<CfgEllEulerTerrain>(h, body, next_body, s);
}

int locosim_terrain_inverse(HandleTerrain* h, const float* qacc, float* qfrc, cudaStream_t s) {
  using namespace locosimterrain;
  return launch_inverse<CfgEllEulerTerrain>(h, qacc, qfrc, s);
}

int locosim_terrain_dynamics(HandleTerrain* h, const locosimterrain::DynOut* o, cudaStream_t s) {
  using namespace locosimterrain;
  return launch_dynamics<CfgEllEulerTerrain>(h, *o, s);
}

int locosim_terrain_forward(HandleTerrain* h, const float* action, const locosimterrain::FwdOut* o, cudaStream_t s) {
  using namespace locosimterrain;
  return launch_forward<CfgEllEulerTerrain>(h, action, *o, s);
}

int locosim_terrain_ray(HandleTerrain* h, const locosimterrain::RayArgs* a, cudaStream_t s) {
  using namespace locosimterrain;
  return launch_ray<CfgEllEulerTerrain>(h, *a, s);
}

int locosim_terrain_dataset_inverse(HandleTerrain* h, float* qfrc, cudaStream_t s) {
  using namespace locosimterrain;
  return launch_dataset_inverse<CfgEllEulerTerrain>(h, qfrc, s);
}

}
