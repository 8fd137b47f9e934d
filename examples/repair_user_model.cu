// examples/repair_user_model.cu - examples/repair_model.cuh (a machine shop: a repair crew of `servers` units shared by
// params[0] machines, one inspection bench) as a loadable model library on the general engine.
//
//   python scripts/build_model.py examples/repair_user_model.cu
//   >>> mid = cimba_b200.load_model("cimba_b200/lib/models/librepair_user_model.so")
#include "../cimba_b200/csrc/cmb_launch.cuh"
#include "repair_model.cuh"

CMB_EXPORT_MODEL(repair_example::Repair, "machine shop: repair crew pool and inspection bench")
