// TEST-ONLY: the 32-lane fiber emulation (emu_lanes.cpp) with its HBM build compiled wide (-DDCU_WIDE=1 before the first inclusion of
// window_core.cuh): tier 1 of emu_lanes_run_batch runs the build the library runs as dcuw, under the lane schedules of emu_lanes.cpp.
// Built as libemu_wide_lanes.so by tests/test_deep_windows.py; never linked into the product library.
#define DCU_WIDE 1
#include "emu_lanes.cpp"
