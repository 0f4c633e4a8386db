// TEST-ONLY: the single-lane host emulation (emu.cpp) with its HBM build compiled wide (-DDCU_WIDE=1 before the first inclusion of
// window_core.cuh): namespace dcu is then the build the library runs as dcuw -- 32-bit slice offsets and k-mer counts -- and tier 1 of
// emu_run_batch has the capacities the library's wide pass gives it (the large-workspace capacities at the batch's own size).  The
// shared-memory and hybrid builds of this library are the ordinary ones (window_core.cuh drops DCU_WIDE after the first build).
// Built as libemu_wide.so by tests/test_deep_windows.py; never linked into the product library.
#define DCU_WIDE 1
#include "emu.cpp"
