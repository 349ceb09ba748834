// The extern "C" entry points of include/nero_b200.h that span kernel files; every other one is defined beside its kernels.
#include "common.cuh"

namespace nero {
// each of k_shade.cu, k_mcshade.cu and k_envmap.cu keeps its own __constant__ copy of the IDE table
int set_ide_table(const float* mat17x36_host);
int set_ide_table_mc(const float* mat17x36_host);
int set_ide_table_env(const float* mat17x36_host);
}  // namespace nero

extern "C" {

int nero_version(void) { return 100; }

int nero_set_ide_table(const float* mat17x36_host) {
  int rc = nero::set_ide_table(mat17x36_host);
  if (rc == NERO_OK) rc = nero::set_ide_table_mc(mat17x36_host);
  return rc != NERO_OK ? rc : nero::set_ide_table_env(mat17x36_host);
}

int nero_abi_sizeof(int which) {
  switch (which) {
    case 0: return int(sizeof(nero_chain_layer));
    case 1: return int(sizeof(nero_chain_params));
    case 2: return int(sizeof(nero_mc_params));
    case 3: return int(sizeof(nero_finish_job));
    case 4: return int(sizeof(nero_prep_job));
    case 5: return int(sizeof(nero_relight_params));
    case 6: return int(sizeof(nero_depth_params));
    default: return -1;
  }
}

}  // extern "C"
