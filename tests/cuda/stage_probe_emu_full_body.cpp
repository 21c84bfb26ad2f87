// Serial stage probe with the 31-dof configurations (test-only): the serial probe of stage_probe_emu.cpp with its dispatch
// extended to configurations 4 (CfgPyrRK4_31) and 5 (CfgPyrEuler31). Same record layout as every probe (stage_probe.h).
#define probe_emu_forward probe_emu_forward_up_to_29
#include "stage_probe_emu.cpp"
#undef probe_emu_forward

extern "C" int probe_emu_forward(const int* ints, int n_ints, const double* reals, int n_reals, const double* q,
                                 const double* v, const double* w, const double* c, int n, void* rec) {
  HostModel hm;
  std::string err = parse_model(hm, ints, n_ints, reals, n_reals);
  if (!err.empty()) { fprintf(stderr, "probe_emu: %s\n", err.c_str()); return -1; }
  ProbeRec* r = reinterpret_cast<ProbeRec*>(rec);
  const int cfg = select_cfg(hm, 0);
  switch (cfg) {
    case 4: run<CfgPyrRK4_31>(hm, q, v, w, c, n, r); return cfg;
    case 5: run<CfgPyrEuler31>(hm, q, v, w, c, n, r); return cfg;
    default: return probe_emu_forward_up_to_29(ints, n_ints, reals, n_reals, q, v, w, c, n, rec);
  }
}
