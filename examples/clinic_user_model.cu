// examples/clinic_user_model.cu - examples/clinic_model.cuh (a walk-in clinic drawing every cmb_random distribution, with
// cmb_datasummary / cmb_wtdsummary statistics) as a loadable model library on the general engine.
//
//   python scripts/build_model.py examples/clinic_user_model.cu
//   >>> mid = cimba_b200.load_model("cimba_b200/lib/models/libclinic_user_model.so")
#include "../cimba_b200/csrc/cmb_launch.cuh"
#include "clinic_model.cuh"

CMB_EXPORT_MODEL(clinic_example::Clinic, "walk-in clinic: every cmb_random distribution, alias routing, summaries")
