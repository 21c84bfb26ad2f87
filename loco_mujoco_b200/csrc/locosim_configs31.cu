// locosim_configs31.cu -- the step kernels of the two 31-dof configurations (locosim_config.h: CfgPyrRK4_31 for Atlas with
// arms, CfgPyrEuler31 for Talos with arms), in a translation unit of their own that is linked into the engine library
// next to locosim.cu. It compiles the kernel templates of locosim.cu (step, sub-step and persistent kernels, launch and
// setup) for these two configurations only; the handle, the C-ABI and the reset / dataset / regrouping kernels stay in
// locosim.cu, which calls the entry points below for configuration indices 4 and 5.
//
// Each translation unit has its own __constant__ model slots (no relocatable device code): this unit's slot of a handle is
// written here at setup and after a parameter-pool upload, locosim.cu writes its own. The engine source is compiled inside
// namespace locosim31 so that its external device functions (the __noinline__ phases) do not collide with locosim.cu's at
// link time; the system and ABI headers are included first, outside it.
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
namespace locosim31 {
#include "locosim.cu"

// sizeof(EnvS) decides the envs resident per SM (see locosim.cu)
static_assert(sizeof(EnvS<CfgPyrRK4_31>) * 8 <= 232448, "Atlas with arms: 8 envs per SM");
static_assert(sizeof(EnvS<CfgPyrEuler31>) * 8 <= 232448, "Talos with arms: 8 envs per SM");
}  // namespace locosim31

// the handle is locosim.cu's (the same struct definition, compiled in both units)
typedef locosim31::locosim_handle Handle31;

extern "C" {

int locosim_configs31_sync_model(Handle31* h) {
  using namespace locosim31;
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

int locosim_configs31_setup(Handle31* h) {
  using namespace locosim31;
  if (locosim_configs31_sync_model(h)) return 1;
  switch (h->cfg) {
    case 4: return setup_cfg<CfgPyrRK4_31>(h);
    case 5: return setup_cfg<CfgPyrEuler31>(h);
    default: h->err = "not a 31-dof configuration"; return 1;
  }
}

int locosim_configs31_step(Handle31* h, const float* a, float* o, float* r, uint8_t* d, float* no, int auto_reset,
                           cudaStream_t s) {
  using namespace locosim31;
  switch (h->cfg) {
    case 4: return launch_step<CfgPyrRK4_31>(h, a, o, r, d, no, auto_reset, s);
    case 5: return launch_step<CfgPyrEuler31>(h, a, o, r, d, no, auto_reset, s);
    default: h->err = "not a 31-dof configuration"; return 1;
  }
}

int locosim_configs31_body(Handle31* h, const uint8_t* mask, int parts, cudaStream_t s) {
  using namespace locosim31;
  switch (h->cfg) {
    case 4: return launch_body<CfgPyrRK4_31>(h, mask, nullptr, 0, parts, s);
    case 5: return launch_body<CfgPyrEuler31>(h, mask, nullptr, 0, parts, s);
    default: h->err = "not a 31-dof configuration"; return 1;
  }
}

int locosim_configs31_dataset_bodies(Handle31* h, float* body, float* next_body, cudaStream_t s) {
  using namespace locosim31;
  switch (h->cfg) {
    case 4: return launch_dataset_bodies<CfgPyrRK4_31>(h, body, next_body, s);
    case 5: return launch_dataset_bodies<CfgPyrEuler31>(h, body, next_body, s);
    default: h->err = "not a 31-dof configuration"; return 1;
  }
}

int locosim_configs31_inverse(Handle31* h, const float* qacc, float* qfrc, cudaStream_t s) {
  using namespace locosim31;
  switch (h->cfg) {
    case 4: return launch_inverse<CfgPyrRK4_31>(h, qacc, qfrc, s);
    case 5: return launch_inverse<CfgPyrEuler31>(h, qacc, qfrc, s);
    default: h->err = "not a 31-dof configuration"; return 1;
  }
}

int locosim_configs31_dynamics(Handle31* h, const locosim31::DynOut* o, cudaStream_t s) {
  using namespace locosim31;
  switch (h->cfg) {
    case 4: return launch_dynamics<CfgPyrRK4_31>(h, *o, s);
    case 5: return launch_dynamics<CfgPyrEuler31>(h, *o, s);
    default: h->err = "not a 31-dof configuration"; return 1;
  }
}

int locosim_configs31_forward(Handle31* h, const float* action, const locosim31::FwdOut* o, cudaStream_t s) {
  using namespace locosim31;
  switch (h->cfg) {
    case 4: return launch_forward<CfgPyrRK4_31>(h, action, *o, s);
    case 5: return launch_forward<CfgPyrEuler31>(h, action, *o, s);
    default: h->err = "not a 31-dof configuration"; return 1;
  }
}

int locosim_configs31_dataset_inverse(Handle31* h, float* qfrc, cudaStream_t s) {
  using namespace locosim31;
  switch (h->cfg) {
    case 4: return launch_dataset_inverse<CfgPyrRK4_31>(h, qfrc, s);
    case 5: return launch_dataset_inverse<CfgPyrEuler31>(h, qfrc, s);
    default: h->err = "not a 31-dof configuration"; return 1;
  }
}

}
