// examples/event_churn_static_user_model.cu - examples/event_model.cuh's EventChurnT on the static tier (cmb::StaticSim<3, 0, 10>
// in its second form): every query and pattern call it makes has one exact answer there, so no trial goes to the general engine.
//
//   python scripts/build_model.py examples/event_churn_static_user_model.cu
#include "../cimba_b200/csrc/cmb_launch.cuh"
#include "event_model.cuh"

CMB_EXPORT_STATIC_MODEL_EVENTS(event_example::EventChurnT, 3, 0, event_example::EVENT_CHURN_SLOTS, "event_churn")
