// examples/clinic_static_user_model.cu - examples/clinic_model.cuh on the static tier: one arrival process, three desks and two
// queues (cmb::StaticSim<4, 2>).  Its sampled holds are drawn by the dispatcher, the ziggurats' rectangles first.
//
//   python scripts/build_model.py examples/clinic_static_user_model.cu
#include "../cimba_b200/csrc/cmb_launch.cuh"
#include "clinic_model.cuh"

CMB_EXPORT_STATIC_MODEL(clinic_example::ClinicT, 4, 2, "clinic")
