// examples/repair_static_user_model.cu - examples/repair_model.cuh on the static tier: up to eight machines, the crew's pool
// and the bench in registers (cmb::StaticSim<8, 0>).  Trials with more machines, or whose machines exit holding crew, are
// re-run on the general engine from the same template.
//
//   python scripts/build_model.py examples/repair_static_user_model.cu
#include "../cimba_b200/csrc/cmb_launch.cuh"
#include "repair_model.cuh"

CMB_EXPORT_STATIC_MODEL(repair_example::RepairT, 8, 0, "repair")
