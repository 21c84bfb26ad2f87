// locosim_ray.cu -- the ray kernels of locosim_ray (include/locosim.h) for all six configurations, in a translation unit of
// their own that is linked into the engine library next to locosim.cu and locosim_configs31.cu. It compiles locosim.cu's
// ray_kernel template (and the core stages it calls) only; the C-ABI, its checks and the handle stay in locosim.cu, which
// calls the entry points below. Keeping the query out of the step kernels' units leaves their compiled code as it is.
//
// As in locosim_configs31.cu, the engine source is compiled inside a namespace of its own (locosimray) and this unit has its
// own __constant__ model slots: locosim.cu writes a handle's slot here through locosim_ray_sync_model when the handle is
// created and after a parameter-pool upload.
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
namespace locosimray {
#include "locosim.cu"
}  // namespace locosimray

typedef locosimray::locosim_handle HandleRay;

extern "C" {

int locosim_ray_sync_model(HandleRay* h) {
  using namespace locosimray;
  CK(cudaMemcpyToSymbol(c_models, &h->dm, sizeof(DevModel), sizeof(DevModel) * h->slot));
  return 0;
}

int locosim_ray_launch(HandleRay* h, const locosimray::RayArgs* a, cudaStream_t s) {
  using namespace locosimray;
  switch (h->cfg) {
    case 0: return launch_ray<CfgEllEuler>(h, *a, s);
    case 1: return launch_ray<CfgPyrEuler>(h, *a, s);
    case 3: return launch_ray<CfgPyrEuler29>(h, *a, s);
    case 4: return launch_ray<CfgPyrRK4_31>(h, *a, s);
    case 5: return launch_ray<CfgPyrEuler31>(h, *a, s);
    default: return launch_ray<CfgPyrRK4>(h, *a, s);
  }
}

}
