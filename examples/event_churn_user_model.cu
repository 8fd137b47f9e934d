// examples/event_churn_user_model.cu - examples/event_model.cuh's EventChurnT (processes holding exponential times, tickers that
// query the event list, find, reschedule and cancel by pattern) as a loadable model library on the general engine.
//
//   python scripts/build_model.py examples/event_churn_user_model.cu
#include "../cimba_b200/csrc/cmb_launch.cuh"
#include "event_model.cuh"

CMB_EXPORT_MODEL(event_example::EventChurnT<cimba_b200::cmb::Sim>, "event churn: queue queries and patterns at every event")
