// examples/event_user_model.cu - examples/event_model.cuh's EventTestT (the reference's test of its event queue, test/test_event.c)
// as a loadable model library on the general engine.
//
//   python scripts/build_model.py examples/event_user_model.cu
//   >>> mid = cimba_b200.load_model("cimba_b200/lib/models/libevent_user_model.so")
#include "../cimba_b200/csrc/cmb_launch.cuh"
#include "event_model.cuh"

CMB_EXPORT_MODEL(event_example::EventTest<cimba_b200::cmb::Sim>, "event queue test: queries, patterns, wildcards, clear")
