// CUDA stage probe with the 31-dof configurations (test-only library, built by tests/full_body.py into tests/_build/ from
// this file and the engine's second translation unit, locosim_configs31.cu, with the product's nvcc flags). It is the probe
// of stage_probe.cu with its two dispatchers extended:
//   probe_forward_run: configurations 4 (CfgPyrRK4_31) and 5 (CfgPyrEuler31) as well;
//   probe_chol:        the register-resident Cholesky at NV = 31 as well.
// The handle is the product's (locosim_create sets up the 31-dof configurations in their own unit and copies the model
// descriptor, pair-table staging included, into this unit's __constant__ slots, where the probe kernel reads it).
#define probe_forward_run probe_forward_run_up_to_29
#define probe_chol probe_chol_up_to_29
#include "stage_probe.cu"
#undef probe_forward_run
#undef probe_chol

extern "C" {
int probe_forward_run(locosim_t* h, const float* q, const float* v, const float* w, const float* c, const int* perm, void* rec) {
  ProbeRec* r = reinterpret_cast<ProbeRec*>(rec);
  switch (h->cfg) {
    case 4: return probe_launch<CfgPyrRK4_31>(h, q, v, w, c, perm, r);
    case 5: return probe_launch<CfgPyrEuler31>(h, q, v, w, c, perm, r);
    default: return probe_forward_run_up_to_29(h, q, v, w, c, perm, rec);
  }
}

int probe_chol(int nv, const float* A, const float* b, float* L, float* x, int n) {
  if (nv != 31) return probe_chol_up_to_29(nv, A, b, L, x, n);
  probe_chol_kernel<31><<<n, 32>>>(A, b, L, x, n);
  return cudaDeviceSynchronize() != cudaSuccess;
}
}
