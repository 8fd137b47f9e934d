// examples/event_static_user_model.cu - examples/event_model.cuh's EventTestT on the static tier (cmb::StaticSim<1, 0, 10> in its
// second form, events by handle).  Its wildcard loop finds three events at once, whose order only the general engine's heap array
// decides, so every trial is flagged and re-run on the general engine from the same template.
//
//   python scripts/build_model.py examples/event_static_user_model.cu
#include "../cimba_b200/csrc/cmb_launch.cuh"
#include "event_model.cuh"

CMB_EXPORT_STATIC_MODEL_EVENTS(event_example::EventTest, 1, 0, event_example::EVENT_TEST_SLOTS, "event")
