/*
 * tests/hostsim/sizes.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here).
 * The sizes of the structs whose byte counts rt_table_create (csrc/b200rt.cu) compares with the
 * shared-memory budget, as the host compiler lays them out from the same headers.
 */
#define RT_HOSTSIM 1
#include "cuda_runtime.h"
#include "../../rayoptics_b200/csrc/rt_lean.cuh"

using namespace b200rt;

extern "C" int hostsim_struct_sizes(int64_t *out)
{
    out[0] = (int64_t)sizeof(rt_surface_desc);
    out[1] = (int64_t)sizeof(LeanSurf);
    out[2] = (int64_t)sizeof(LeanIdx);
    out[3] = (int64_t)sizeof(LeanPoly);
    return 0;
}
